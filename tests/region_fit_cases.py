"""RegionFit witness and two-set cases (test infrastructure).

`witness` restates RegionFit2D / RegionFit3D setNeighbor(reliable) + compute(queue) (reference src/oc_region_fit.cpp) without a
grid, on strain_cases.py's rules with the neighbours taken from the reliable set:
- neighbours: every reliable POI with a finite position whose float32 squared distance (x then y (then z), one rounding per
  operation) to the queue POI is strictly below float32(radius * radius);
- fewer than k_min found: the min(k_min, finite reliable POIs) nearest, ordered by (float32 d^2, reliable index);
- no ZNCC filter; a queue POI with a non-finite position is left alone;
- at least k_min neighbours: the float64 least-squares plane [1, dx, dy(, dz)] over u, v (, w) with offsets float32(q - p),
  column-pivoted Householder QR, unknowns past the numerical rank set to 0 (strain_cases._pivoted, whose near-tie branches are
  all kept).  It writes u ux uy (uz) v .. as float32 and zncc = 0; nothing else changes.

Queue records start with garbage first-order fields and a ZNCC that no fit writes, so a POI whose ZNCC field still holds its
input bits was not fitted."""
import collections

import numpy as np
from scipy.spatial import cKDTree

import strain_cases as sc

F = np.float32
LAYOUT = {  # record floats -> dims, ZNCC field, the written first-order fields (u .. per displacement component)
    25: dict(d=2, zncc=16, fields=(2, 3, 4, 8, 9, 10)),
    31: dict(d=3, zncc=18, fields=tuple(range(3, 15))),
}
TOL = 2e-6  # FP64 normal equations (the kernel) against FP64 Householder QR (the witness), relative above 1

Witness = collections.namedtuple("Witness", "out computed alts fallback")
Case = collections.namedtuple("Case", "name rel q radius k_min")


def layout(q):
    return LAYOUT[q.shape[1]]


def neighbour_sets(rel, qpos, radius, k_min):
    """Per query position: (reliable indices of its neighbours, used the k-nearest fallback)."""
    D = qpos.shape[1]
    pos = rel[:, :D]
    fin = np.flatnonzero(np.isfinite(pos).all(1))
    P = pos[fin]
    with np.errstate(over="ignore"):
        r2 = F(F(radius) * F(radius))
    tree = cKDTree(P.astype(np.float64)) if len(fin) else None
    sets = [None] * len(qpos)
    if len(fin) and r2 > 0 and len(qpos):
        if np.isinf(r2):
            cand = [np.arange(len(fin))] * len(qpos)
        else:
            cand = tree.query_ball_point(qpos.astype(np.float64), float(np.sqrt(np.float64(r2))) * (1 + 1e-5) + 1e-30)
        for t, c in enumerate(cand):
            c = np.asarray(c, np.int64)
            sets[t] = np.sort(fin[c[sc.dist2(qpos[t], P[c]) < r2]])
    fallback = np.zeros(len(qpos), bool)
    k = min(k_min, len(fin))
    for t in range(len(qpos)):
        if sets[t] is not None and len(sets[t]) >= k_min:
            continue
        fallback[t] = True
        if k <= 0:
            sets[t] = np.zeros(0, np.int64)
            continue
        kk = min(len(fin), k + 16)
        dd, _ = tree.query(qpos[t].astype(np.float64), k=kk)
        bound = np.atleast_1d(dd)[-1]
        if kk < len(fin) and np.isfinite(bound):
            cand = np.asarray(tree.query_ball_point(qpos[t].astype(np.float64), bound * (1 + 1e-5) + 1e-30), np.int64)
        else:
            cand = np.arange(len(fin))
        with np.errstate(over="ignore"):
            d = sc.dist2(qpos[t], P[cand])
        idx = fin[cand]
        sets[t] = np.sort(idx[np.lexsort((idx, d))[:k]])
    return sets, fallback


def witness(rel, q, radius, k_min):
    """RegionFit on a copy of q (POI2D [n,25] or POI3D [n,31]) with the reliable records rel.  Returns Witness(out, computed,
    alts, fallback): alts maps a POI whose fit hangs on a near tie to every acceptable row of the written fields."""
    L = layout(q)
    D, fields = L["d"], list(L["fields"])
    C = D + 1
    out = q.copy()
    computed = np.zeros(len(q), bool)
    fallback = np.zeros(len(q), bool)
    alts = {}
    centres = np.flatnonzero(np.isfinite(q[:, :D]).all(1))
    if not len(centres):
        return Witness(out, computed, alts, fallback)
    sets, fb = neighbour_sets(rel, q[centres, :D], radius, k_min)
    fallback[centres] = fb
    disp = rel[:, list(fields[::C])].astype(np.float64)  # u, v (, w)
    for t, i in enumerate(centres):
        f = sets[t]
        if len(f) < k_min:
            continue
        computed[i] = True
        A = np.ones((len(f), C))
        with np.errstate(over="ignore", invalid="ignore"):
            A[:, 1:] = (rel[f, :D] - q[i, :D]).astype(F)
        B = disp[f]
        full = len(f) >= C and np.isfinite(A).all()
        if full:
            s = np.linalg.svd(A, compute_uv=False)
            full = s[-1] > 1e-3 * s[0]
        if full:
            sols = [np.linalg.lstsq(A, B, rcond=None)[0]]
        else:
            sols = sc._pivoted(A, B)
        rows = [X.T.reshape(-1).astype(F) for X in sols]  # [u ux uy (uz), v ..]
        out[i, fields] = rows[0]
        out[i, L["zncc"]] = 0
        if len(rows) > 1:
            alts[int(i)] = np.stack(rows)
    return Witness(out, computed, alts, fallback)


def compare(got, q, w, tol=TOL, name=""):
    """Hold a RegionFit result to the witness: the same POIs written, every field but the written ones and the ZNCC
    bit-identical to the input (every field of an unwritten POI), zncc = 0 and the written fields within tol (relative above 1;
    the nearest acceptable row for a near tie).  Returns (POIs written, largest difference)."""
    L = layout(q)
    fields = list(L["fields"])
    other = np.ones(q.shape[1], bool)
    other[fields] = False
    other[L["zncc"]] = False
    bad = np.flatnonzero((sc.bits(got[:, other]) != sc.bits(q[:, other])).any(1))
    assert len(bad) == 0, "%s: fields that are not written changed at POIs %s" % (name, bad[:8])
    written = sc.bits(got[:, L["zncc"]]) != sc.bits(q[:, L["zncc"]])
    wrong = np.flatnonzero(written != w.computed)
    assert len(wrong) == 0, "%s: %d POIs written differently, e.g. %s (got %s, witness %s, fallback %s)" % (
        name, len(wrong), wrong[:8], written[wrong[:8]], w.computed[wrong[:8]], w.fallback[wrong[:8]])
    untouched = np.flatnonzero(~written)
    assert np.array_equal(sc.bits(got[untouched]), sc.bits(q[untouched])), "%s: an unwritten POI changed" % name
    idx = np.flatnonzero(written)
    if not len(idx):
        return 0, 0.0
    assert np.all(got[idx, L["zncc"]] == 0), name
    a = got[idx][:, fields].astype(np.float64)
    b = w.out[idx][:, fields].astype(np.float64)
    d = (np.abs(a - b) / np.maximum(1.0, np.abs(b))).max(1)
    for t, i in enumerate(idx):
        if int(i) in w.alts:
            alt = w.alts[int(i)].astype(np.float64)
            d[t] = min(d[t], (np.abs(a[t] - alt) / np.maximum(1.0, np.abs(alt))).max(1).min())
    worst = int(np.argmax(d))
    assert d[worst] < tol, "%s: POI %d differs by %.3g (got %s, witness %s)" % (name, idx[worst], d[worst], a[worst], b[worst])
    return len(idx), float(d.max())


# ------------------------------------------------------------------------------------------------ case generators
def _kind(D):
    return 3 if D == 3 else 2


def reliable_set(pos, rng, noise=0.3):
    """POI records at pos with strain_cases' seeded affine displacement field plus noise (every neighbour moves the fit)."""
    pos = np.asarray(pos, F)
    return sc.queue(_kind(pos.shape[1]), pos, rng, noise=noise)


def queue_set(pos, rng):
    """Unreliable POI records at pos: garbage first-order fields, random second-order terms, a low ZNCC, the rest random too."""
    pos = np.asarray(pos, F)
    D = pos.shape[1]
    q = rng.uniform(-50, 50, (len(pos), 25 if D == 2 else 31)).astype(F)
    q[:, :D] = pos
    q[:, LAYOUT[q.shape[1]]["zncc"]] = rng.uniform(0.05, 0.6, len(pos))
    return q


def split(name, pos, rng, radius, k_min, frac=0.2):
    """Every position a reliable POI except a random fraction, which form the queue."""
    pos = np.asarray(pos)
    sel = rng.uniform(size=len(pos)) < frac
    return Case(name, reliable_set(pos[~sel], rng), queue_set(pos[sel], rng), radius, k_min)


def basic_cases(seed=0):
    rng = np.random.default_rng(seed)
    out = []
    for D in (2, 3):
        n, ext = (3000, 300.0) if D == 2 else (4000, 60.0)
        out.append(split("uniform_%d" % D, rng.uniform(0, ext, (n, D)), rng, 12.0 if D == 2 else 6.0, 9 if D == 2 else 12))
        out.append(split("uniform_sparse_%d" % D, rng.uniform(-ext, ext, (n // 4, D)), rng, 9.0, 6))  # many fall back
    # lattices: the reliable POIs on a 3 px lattice, queries at lattice holes and between them -- shells of equal distances
    for k in (6, 7, 9, 10, 13):
        pos, r = sc.lattice(2, 14, 3.0, seed + k)
        out.append(split("lattice2_k%d" % k, pos, r, 2.0, k, 0.15))
        out.append(split("lattice2_r3_k%d" % k, pos, r, 3.0, k, 0.15))  # d^2 = 9 = r^2: the first shell is out
    for k in (8, 20):
        pos, r = sc.lattice(3, 7, 3.0, seed + k)
        out.append(split("lattice3_k%d" % k, pos, r, 2.0, k, 0.15))
    g = np.stack(np.meshgrid(np.arange(20) * 3.0, np.arange(20) * 3.0, indexing="ij"), -1).reshape(-1, 2) + 100
    between = g[:150] + 1.5
    out.append(Case("lattice2_midpoints", reliable_set(g, rng), queue_set(between, rng), 2.2, 9))
    return out


def boundary_cases():
    """strain_cases' cell-boundary sets (centres on both sides of computed cell edges, neighbours at float32 d^2 = r^2 - 1 ulp
    and = r^2): every POI reliable and every POI queried."""
    out = []
    for kind in (2, 3):
        for r in (20.0, 7.5, 1.0):
            c, _ = sc.cell_boundary(kind, r)
            D = 3 if kind == 3 else 2
            rng = np.random.default_rng(int(r * 10) + kind)
            rel = reliable_set(c.q[:, :D], rng)
            out.append(Case("cell_boundary_%d_r%g" % (kind, r), rel, queue_set(c.q[:, :D], rng), r, 5))
    return out


def outside_cases(seed=0):
    """Queries outside the reliable bounding box, on every side: within one radius of it (their neighbours lie in the edge
    cells), just beyond one cell edge, and far away (the k-nearest fallback); also with a grown cell."""
    rng = np.random.default_rng(seed)
    out = []
    for D, r in ((2, 10.0), (3, 6.0), (2, 0.75)):
        ext = 20 * r if D == 2 else 8 * r
        rel_pos = rng.uniform(0, ext, (6000 if D == 2 else 5000, D))
        lo, hi = rel_pos.min(0), rel_pos.max(0)
        qs = []
        for axis in range(D):
            for side, edge in ((-1, lo[axis]), (1, hi[axis])):
                for off in (0.0, 0.2, 0.4, 0.6, 0.9, 0.999, 1.0, 1.001, 1.05, 1.5, 2.2, 3.5, 40.0):
                    p = rng.uniform(lo, hi, (8 if off < 0.8 else 3, D))
                    p[:, axis] = edge + side * off * r
                    qs.append(p)
        corners = np.stack(np.meshgrid(*[[lo[d] - 0.7 * r, hi[d] + 0.7 * r] for d in range(D)], indexing="ij"), -1).reshape(-1, D)
        q = np.concatenate(qs + [corners])
        rel = reliable_set(rel_pos, rng)
        # queries exactly on the radius shell of the extreme reliable POIs, from outside the box
        ext_pts = [int(np.argmin(rel[:, a])) for a in range(D)] + [int(np.argmax(rel[:, a])) for a in range(D)]
        shell = []
        for t, i in enumerate(ext_pts):
            u = np.zeros(D)
            u[t % D] = -1.0 if t < D else 1.0
            for inside in (True, False):
                s, _ = sc.shell_point(rel[i, :D], u, r, inside)
                shell.append(s)
        q = np.concatenate([q, np.array(shell, np.float64)])
        out.append(Case("outside_%d_r%g" % (D, r), rel, queue_set(q, rng), r, 3))
    # a reliable set whose extent grows the cell (65 537+ cells of the radius per axis), queries beyond both ends
    a = rng.uniform(0, 150, (600, 2))
    far = np.concatenate([a, a[:300] + 2e6])
    q = np.concatenate([a[::7] + [0, -160], a[::9] + 2e6 + [0, 155], np.array([[-30.0, -30.0], [2e6 + 200, 2e6 + 200]])])
    out.append(Case("outside_grown_2", reliable_set(far, rng), queue_set(q, rng), 20.0, 5))
    return out


def knn_cases(seed=0):
    """The k-nearest fallback with n_reliable below, at and above k_min, and a radius too small for anyone."""
    rng = np.random.default_rng(seed)
    out = []
    for D in (2, 3):
        k = 9 if D == 2 else 12
        for n_rel in (k - 3, k, k + 4):
            rel = reliable_set(rng.uniform(0, 50, (n_rel, D)), rng)
            out.append(Case("knn_%d_n%d_k%d" % (D, n_rel, k), rel, queue_set(rng.uniform(-10, 60, (40, D)), rng), 3.0, k))
        rel = reliable_set(rng.uniform(0, 400, (1500, D)), rng)
        out.append(Case("knn_fallback_%d" % D, rel, queue_set(rng.uniform(0, 400, (300, D)), rng), 4.0, k))
    return out


def rank_cases(seed=0):
    rng = np.random.default_rng(seed)
    out = []
    row = np.stack([np.arange(60) * 2.0, np.full(60, 5.0)], 1)
    out.append(Case("rank_row_2", reliable_set(row, rng), queue_set(np.stack([rng.uniform(0, 118, 30), rng.uniform(2, 8, 30)], 1), rng), 7.0, 3))
    t = rng.uniform(0, 100, 120)
    out.append(Case("rank_diagonal_2", reliable_set(np.stack([t, t], 1), rng), queue_set(np.stack([t[:40], t[:40]], 1) + 0.5, rng), 9.0, 3))
    t3 = rng.uniform(0, 100, 150)
    out.append(Case("rank_diagonal_3", reliable_set(np.stack([t3, t3, 0.5 * t3], 1), rng),
                    queue_set(np.stack([t3[:40], t3[:40], 0.5 * t3[:40]], 1), rng), 9.0, 3))
    a, b = rng.uniform(0, 60, (2, 600))
    plane = np.stack([a, b, 0.5 * a - 0.25 * b + 3], 1)
    out.append(Case("rank_coplanar_3", reliable_set(plane, rng), queue_set(plane[:80] + [0, 0, 0.5], rng), 9.0, 5))
    dup = np.repeat(rng.uniform(0, 60, (80, 2)), 3, 0)
    out.append(Case("rank_duplicates_2", reliable_set(dup, rng), queue_set(dup[::3][:40] + 0.25, rng), 8.0, 5))
    one = np.full((10, 3), 4.0)
    out.append(Case("rank_one_position_3", reliable_set(one, rng), queue_set(rng.uniform(0, 8, (12, 3)), rng), 20.0, 5))
    return out


def nonfinite_cases(seed=0):
    """NaN and +-inf coordinates in the reliable set (never a neighbour) and in the queue (left alone), first and last too."""
    rng = np.random.default_rng(seed)
    out = []
    vals = np.array([np.nan, np.inf, -np.inf], F)
    for D in (2, 3):
        ext = 200 if D == 2 else 60
        rel = reliable_set(rng.uniform(0, ext, (900, D)), rng)
        q = queue_set(rng.uniform(0, ext, (300, D)), rng)
        for arr in (rel, q):
            bad = np.r_[0, rng.choice(np.arange(1, len(arr) - 1), len(arr) // 10, replace=False), len(arr) - 1]
            for t, i in enumerate(bad):
                arr[i, t % D] = vals[t % 3]
        out.append(Case("nonfinite_%d" % D, rel, q, 15.0, 8))
        allbad = rel[:50].copy()
        allbad[:, 0] = np.nan
        for k in (5, 0):
            out.append(Case("reliable_all_nonfinite_%d_k%d" % (D, k), allbad, q[:60].copy(), 15.0, k))
    return out


def value_cases(seed=0):
    """Radius and k_min at their edges, and an empty reliable set."""
    rng = np.random.default_rng(seed)
    out = []
    for D in (2, 3):
        ext = 120 if D == 2 else 40
        rel = reliable_set(rng.uniform(0, ext, (600, D)), rng)
        q = queue_set(rng.uniform(-5, ext + 5, (150, D)), rng)
        for r in (-12.0, np.inf, -np.inf, np.nan, 0.0, 1e-30, 1e20):
            out.append(Case("radius_%d_%g" % (D, r), rel, q, r, 5))
        for k in (0, -3, 1):
            out.append(Case("kmin_%d_%d" % (D, k), rel, q, 10.0, k))
            out.append(Case("kmin_nan_radius_%d_%d" % (D, k), rel, q, np.nan, k))
        empty = np.zeros((0, 25 if D == 2 else 31), F)
        for k in (5, 0):
            out.append(Case("empty_reliable_%d_k%d" % (D, k), empty, q, 10.0, k))
    return out


def small_cases():
    return basic_cases() + boundary_cases() + outside_cases() + knn_cases() + rank_cases() + nonfinite_cases() + value_cases()
