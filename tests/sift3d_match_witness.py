"""A float64 witness of SIFT3D's monodirectional matching (reference src/oc_sift.cpp:1251-1418), independent of the float32 oracle
and of the kernels: the same decisions, taken on distances that carry no rounding a float32 sum could flip.

  - Distances (:1272-1281) are float64 squared Euclidean distances from chunked Gram products, |a|^2 + |b|^2 - 2 a.b, with each
    row's REFINE nearest recomputed as direct float64 sums of squared differences.  Identical
    descriptors are grouped first (by their bits), so that copies get the same distance exactly, and a reference row equal to a
    target row is at distance 0 exactly, as the float32 sum is.
  - The scan's top two (:1283-1294) keeps the first index of equal distances (strict '<' over ascending j): a group of identical
    target descriptors is represented by its first index, and ties the row exactly (d1 = d0) when it has two members or more.
  - The ratio test (:1298-1303) compares d0 < r^2 d1 with r^2 = ratio * ratio rounded to float, as the reference forms it.
  - Both sorts (:1307, :1325) are stable, the many-to-one runs (:1330-1389) are every maximal run of equal target index, the last
    one included (at :1335 the reference compares the last element with the stale one past the resized end, a row that failed
    the ratio test with tar_idx -1, so a run that ends the list is closed like the others), and a run keeps its nearest
    reference keypoint if that passes the ratio test against the run's second.  If every reference keypoint passes
    the ratio test, matched_amount stays 0 (:1309-1317) and nothing is returned.

match() also reports the rows whose decision float32 could take differently: a nearest distinct target within REL of the nearest
(relative gap), a ratio test within REL of its threshold, or membership in a run whose own test is that close.  Of those, the
near-copy rows are marginal only because the targets within REL of their nearest are near-copies of it (squared distance below
NEAR_COPY): which of them is nearest is a rounding choice, but a pair that differs must name one of them."""
import numpy as np

REL = 1e-4
NEAR_COPY = 1e-8  # squared distance below which two unit-norm target descriptors are near-copies (distinct ones: >= 1e-3)
REFINE = 8  # nearest distances per row recomputed as direct float64 sums
FLT_MAX = float(np.finfo(np.float32).max)


def _groups(d):
    """(first index of each group of bit-identical rows, ordered by it; group size; group of each row)"""
    if len(d) == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros(0, np.int64)
    _, first, inv, cnt = np.unique(np.ascontiguousarray(d, np.float32).view(np.uint32), axis=0, return_index=True, return_inverse=True,
                                   return_counts=True)
    order = np.argsort(first)
    rank = np.empty_like(order)
    rank[order] = np.arange(len(order))
    return first[order], cnt[order], rank[inv.ravel()]


def distances(d1, d2, chunk=512):
    """float64 squared distances [n1, n2] by chunked Gram products, exactly 0 between identical rows"""
    a, b = np.asarray(d1, np.float64), np.asarray(d2, np.float64)
    bb = (b * b).sum(1)
    out = np.empty((len(a), len(b)), np.float64)
    keys = {row.tobytes(): j for j, row in enumerate(np.ascontiguousarray(d2, np.float32))}
    for s in range(0, len(a), chunk):
        c = a[s:s + chunk]
        out[s:s + chunk] = np.maximum((c * c).sum(1)[:, None] + bb[None, :] - 2.0 * (c @ b.T), 0.0)
    # the Gram form loses about 1e-16 absolutely (|a|^2 is ~1): recompute each row's nearest few directly, so that small distances
    # keep their relative precision (rows near-identical to a target sit at 1e-12 and below)
    k = min(REFINE, len(b))
    if k:
        near = np.argpartition(out, k - 1, axis=1)[:, :k]
        for s in range(0, len(a), chunk):
            rows = np.arange(s, min(s + chunk, len(a)))
            diff = a[rows, None, :] - b[near[rows]]
            out[rows[:, None], near[rows]] = (diff * diff).sum(2)
    for i, row in enumerate(np.ascontiguousarray(d1, np.float32)):
        j = keys.get(row.tobytes())
        if j is not None:
            out[i, j] = 0.0
    return out


def match(desc1, desc2, ratio=0.85):
    """Returns (pairs [m, 2] int64 (reference, target) in output order, info): info holds d0, d1 (float64, FLT_MAX where the scan
    found nothing), index0 (-1 there) and marginal, a bool per reference row."""
    d1 = np.asarray(desc1, np.float32).reshape(-1, 768)
    d2 = np.asarray(desc2, np.float32).reshape(-1, 768)
    n1, n2 = len(d1), len(d2)
    r2 = float(np.float32(ratio) * np.float32(ratio))
    f1, _, g1 = _groups(d1)
    f2, c2, _ = _groups(d2)
    D = distances(d1[f1], d2[f2])[g1] if n1 and n2 else np.zeros((n1, 0))
    D[np.isnan(D)] = np.inf  # a NaN distance never enters the scan's top two
    d0 = np.full(n1, FLT_MAX)
    dd1 = np.full(n1, FLT_MAX)
    second = np.full(n1, np.inf)  # nearest distinct target group after the nearest
    idx0 = np.full(n1, -1, np.int64)
    if n2:
        g0 = np.argmin(D, axis=1)  # first minimum: the lowest first index among equal distances
        rows = np.arange(n1)
        d0 = D[rows, g0]
        idx0 = f2[g0]
        if D.shape[1] > 1:
            rest = D.copy()
            rest[rows, g0] = np.inf
            second = rest.min(axis=1)
        dd1 = np.where(c2[g0] > 1, d0, np.minimum(second, FLT_MAX))
        lost = np.isinf(d0)  # only NaN distances: the scan keeps nothing
        d0, dd1, idx0 = np.where(lost, FLT_MAX, d0), np.where(lost, FLT_MAX, dd1), np.where(lost, -1, idx0)
    with np.errstate(invalid="ignore", divide="ignore"):
        gap = np.where(d0 > 0, (second - d0) / d0, np.inf)
        # a d1 of FLT_MAX is the scan's initial value, not a sum: the test against it has no rounding to flip
        rmargin = np.where((dd1 > 0) & (dd1 < FLT_MAX), np.abs(d0 - r2 * dd1) / dd1, np.inf)
    by_gap = gap < REL
    marginal = by_gap | (rmargin < REL)
    passed = d0 < r2 * dd1
    # km: (ref_idx, tar_idx, dist) per row, -1 where the ratio test failed; first sort: descending ref_idx, stable
    ref = np.where(passed, np.arange(n1), -1)
    order = np.argsort(-ref, kind="stable")
    ref, tar, dist = ref[order], np.where(passed, idx0, -1)[order], np.where(passed, d0, 0.0)[order]
    none = np.nonzero(ref == -1)[0]
    matched = int(none[0]) if len(none) else 0
    pairs = []
    if matched > 1:
        ref, tar, dist = ref[:matched], tar[:matched], dist[:matched]
        order = np.argsort(-tar, kind="stable")
        ref, tar, dist = ref[order].copy(), tar[order], dist[order]
        s = 0
        while s < matched:
            e = s + 1
            while e < matched and tar[e] == tar[s]:
                e += 1
            if e - s > 1:
                ci, cd = [-1, -1], [FLT_MAX, FLT_MAX]
                for c in range(s, e):
                    if dist[c] < cd[0]:
                        ci[1], cd[1], ci[0], cd[0] = ci[0], cd[0], ref[c], dist[c]
                    elif dist[c] < cd[1]:
                        ci[1], cd[1] = ref[c], dist[c]
                members = ref[s:e].copy()
                ref[s:e] = -1
                if cd[0] < r2 * cd[1]:
                    ref[s] = ci[0]
                close = cd[1] > 0 and (abs(cd[0] - r2 * cd[1]) / cd[1] < REL or (cd[0] != cd[1] and (cd[1] - cd[0]) / max(cd[0], 1e-300) < REL))
                if close:
                    marginal[members] = True
                    by_gap[members] = False  # no longer explained by near-copies alone
            s = e
        pairs = [(int(r), int(t)) for r, t in zip(ref, tar) if r > -1]
    # near-copies: rows marginal only because their two nearest distinct targets are themselves nearly one descriptor, so either
    # may be the nearest; the pair must then name one of the two
    near_copy = np.zeros(n1, bool)
    alternatives = {}  # near-copy row -> first indices of the targets within REL of its nearest
    for r in np.nonzero(by_gap & ~(rmargin < REL))[0]:
        close = np.nonzero(D[r] <= d0[r] * (1 + REL))[0]
        t = d2[f2[close]].astype(np.float64)
        if (((t - t[np.searchsorted(close, g0[r])]) ** 2).sum(1) < NEAR_COPY).all():
            near_copy[r] = True
            alternatives[int(r)] = set(f2[close].tolist())
    return np.array(pairs, np.int64).reshape(-1, 2), dict(d0=d0, d1=dd1, index0=idx0, marginal=marginal, near_copy=near_copy,
                                                          alternatives=alternatives)


def compare(ref_xyz, tar_xyz, kp1, kp2, pairs, info):
    """Compare matched coordinates (float32 [m, 3] each, as ocb_sift3d returns them) with the witness pairs on keypoints kp1, kp2
    (float32 [n, 18], image coordinates in columns 3:6).  The GPU's coordinates are mapped back to keypoint indices (every index at
    that position); a pair either side has alone must belong to a marginal reference row or point at the nearest target of one.
    Returns (pairs only the GPU has, pairs only the witness has, marginal rows, the differing pairs that are not excused), the pairs
    as tuples of keypoint indices (a coordinate that names no keypoint stays a coordinate)."""
    def index(kp):
        m = {}
        for i, c in enumerate(np.ascontiguousarray(kp[:, 3:6], np.float32)):
            m.setdefault(c.tobytes(), []).append(i)
        return m

    i1, i2 = index(kp1), index(kp2)
    got = {}
    for a, b in zip(np.ascontiguousarray(ref_xyz, np.float32), np.ascontiguousarray(tar_xyz, np.float32)):
        key = (tuple(i1.get(a.tobytes(), [("?",) + tuple(a.tolist())])), tuple(i2.get(b.tobytes(), [("?",) + tuple(b.tolist())])))
        got[key] = got.get(key, 0) + 1
    want = {}
    for r, t in pairs:
        key = (tuple(i1[kp1[r, 3:6].tobytes()]), tuple(i2[kp2[t, 3:6].tobytes()]))
        want[key] = want.get(key, 0) + 1
    only_gpu = [k for k in got for _ in range(got[k] - want.get(k, 0))]
    only_wit = [k for k in want for _ in range(want[k] - got.get(k, 0))]
    marginal = np.nonzero(info["marginal"])[0]
    other = np.nonzero(info["marginal"] & ~info["near_copy"])[0]
    # a marginal row excuses its own pair and pairs on its nearest target; a near-copy row only pairs on one of its near-copies
    excused_ref = set(other.tolist())
    excused_tar = set(info["index0"][other].tolist()).union(*info["alternatives"].values())
    bad = [k for k in only_gpu + only_wit
           if not (set(k[0]) & excused_ref or set(k[1]) & excused_tar)]
    return only_gpu, only_wit, marginal, bad
