"""Strain witness and case generators (test infrastructure).

`witness` restates Strain::compute(queue) (reference src/oc_strain.cpp:158-250, :252-371, :373-487) without a grid:
- neighbours: scipy cKDTree candidates over a slightly enlarged radius, each rechecked with the reference's rule (nanoflann
  L2_Simple_Adaptor, src/oc_nearest_neighbor.cpp:124-157): squared distance accumulated in float32, x then y (then z), one
  rounding per operation, kept when strictly below float32(radius * radius), over every POI with a finite position;
- fewer than k_min found: the k nearest, ordered by (float32 d^2, original index);
- the fit runs over the neighbours whose ZNCC fields all pass (>=, NaN fails) and needs at least k_min of them;
- the fit: float64 least squares [1, dx, dy(, dz)] g = u | v (| w) with offsets float32(q - p), column-pivoted Householder QR
  (largest remaining column norm first, the first of equals), unknowns past the numerical rank set to 0.  Where the pivot
  order or the rank hangs on a near tie the POI is non-decisive and every branch's solution is kept.

A queue's strain fields start at SENTINEL, which no fit here produces, so a POI whose strain fields still hold it was not
fitted."""
import collections

import numpy as np
from scipy.spatial import cKDTree

F = np.float32
SENTINEL = F(7.0)
RANK_TOL = 1e-12  # squared residual column norm over the largest squared column norm (the oracle and the kernel)
TIE = 1e-9        # relative gap of two column norms below which the pivot order is not decided by the data
LAYOUT = {  # record floats -> search dims, fit dims, first fit coordinate, ZNCC fields, strain fields, displacement fields
    25: dict(sd=2, fd=2, fc=0, zncc=(16,), strain=slice(20, 23), disp=(2, 8)),
    31: dict(sd=3, fd=3, fc=0, zncc=(18,), strain=slice(22, 28), disp=(3, 7, 11)),
    28: dict(sd=2, fd=3, fc=14, zncc=(5, 6, 7), strain=slice(20, 26), disp=(2, 3, 4)),
}

Witness = collections.namedtuple("Witness", "out computed checked alts fallback")


def layout(q):
    return LAYOUT[q.shape[1]]


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def dist2(p, q):
    """float32 squared distance of positions q [..., D] from p [..., D], x then y (then z), one rounding per operation."""
    p, q = np.asarray(p, F), np.asarray(q, F)
    d = q[..., 0] - p[..., 0]
    r = d * d
    for k in range(1, p.shape[-1]):
        d = q[..., k] - p[..., k]
        r = r + d * d
    return r


def good(q, thr):
    return np.all(q[:, list(layout(q)["zncc"])] >= F(thr), axis=1)


def neighbour_sets(q, centres, radius, k_min):
    """Per centre: (indices of its neighbours, used the k-nearest fallback)."""
    sd = layout(q)["sd"]
    pos = q[:, :sd]
    fin = np.flatnonzero(np.isfinite(pos).all(1))
    P = pos[fin]
    with np.errstate(over="ignore"):
        r2 = F(F(radius) * F(radius))  # overflows to inf from |radius| ~ 1.9e19 on, as in the reference
    tree = cKDTree(P.astype(np.float64)) if len(fin) else None
    centres = np.asarray(centres, np.int64)
    sets = [None] * len(centres)
    if len(fin) and r2 > 0:
        if np.isinf(r2):
            cand = [np.arange(len(fin))] * len(centres)
        else:
            cand = tree.query_ball_point(pos[centres].astype(np.float64), float(np.sqrt(np.float64(r2))) * (1 + 1e-5) + 1e-30)
        lens = np.array([len(c) for c in cand], np.int64)
        flat = np.concatenate([np.asarray(c, np.int64) for c in cand]) if lens.sum() else np.zeros(0, np.int64)
        owner = np.repeat(np.arange(len(centres)), lens)
        keep = dist2(pos[centres[owner]], P[flat]) < r2
        split = np.cumsum(lens)[:-1]
        for t, (f, k) in enumerate(zip(np.split(flat, split), np.split(keep, split))):
            sets[t] = np.sort(fin[f[k]])
    fallback = np.zeros(len(centres), bool)
    k = min(k_min, len(fin))
    for t, c in enumerate(centres):
        if sets[t] is not None and len(sets[t]) >= k_min:
            continue
        fallback[t] = True
        if k <= 0:
            sets[t] = np.zeros(0, np.int64)
            continue
        kk = min(len(fin), k + 16)
        dd, _ = tree.query(pos[c].astype(np.float64), k=kk)
        bound = np.atleast_1d(dd)[-1]
        if kk < len(fin) and np.isfinite(bound):
            cand = np.asarray(tree.query_ball_point(pos[c].astype(np.float64), bound * (1 + 1e-5) + 1e-30), np.int64)
        else:
            cand = np.arange(len(fin))
        d = dist2(pos[c], P[cand])
        idx = fin[cand]
        order = np.lexsort((idx, d))[:k]
        sets[t] = np.sort(idx[order])
    return sets, fallback


def _pivoted(A, B):
    """Basic solutions [C, NB] of min |A x - B| by column-pivoted Householder QR, one per branch of a near tie."""
    m, C = A.shape
    out = []

    def step(A, B, perm, k, first):
        norms = (A[k:, k:] ** 2).sum(0) if k < min(C, m) else np.zeros(0)
        if len(norms):
            if k == 0:
                first = norms.max()
            best = int(np.argmax(norms))
            nb = norms[best]
            if nb > first * RANK_TOL:
                choices = [best] + [j for j in range(len(norms)) if j != best and nb - norms[j] <= TIE * nb]
                for j in choices:
                    A2, B2, p2 = A.copy(), B.copy(), list(perm)
                    A2[:, [k, k + j]] = A2[:, [k + j, k]]
                    p2[k], p2[k + j] = p2[k + j], p2[k]
                    alpha = -np.sqrt(norms[j]) if A2[k, k] > 0 else np.sqrt(norms[j])
                    v = A2[k:, k].copy()
                    v[0] -= alpha
                    vn = v @ v
                    if vn > 0:
                        A2[k:, k:] -= np.outer(v, 2 * (v @ A2[k:, k:]) / vn)
                        B2[k:] -= np.outer(v, 2 * (v @ B2[k:]) / vn)
                    step(A2, B2, p2, k + 1, first)
                if nb > first * RANK_TOL * 100:
                    return
                # close to the rank threshold: rank k is a branch as well
        x = np.zeros((C, B.shape[1]))
        if k:
            y = np.linalg.solve(np.triu(A[:k, :k]), B[:k])
            x[perm[:k]] = y
        out.append(x)

    step(np.array(A, np.float64), np.array(B, np.float64), list(range(C)), 0, 0.0)
    return out


def _strain_rows(X, fd, approximation):
    """Strain fields (float32, as the reference rounds them) from gradients X [N, C, FD]."""
    g = X.astype(F)
    if fd == 2:
        ux, uy, vx, vy = g[:, 1, 0], g[:, 2, 0], g[:, 1, 1], g[:, 2, 1]
        if approximation == 2:
            return np.stack([ux + F(0.5) * (ux * ux + vx * vx), vy + F(0.5) * (uy * uy + vy * vy),
                             F(0.5) * (uy + vx + uy * ux + vy * vx)], 1)
        return np.stack([ux, vy, F(0.5) * (uy + vx)], 1)
    ux, uy, uz = g[:, 1, 0], g[:, 2, 0], g[:, 3, 0]
    vx, vy, vz = g[:, 1, 1], g[:, 2, 1], g[:, 3, 1]
    wx, wy, wz = g[:, 1, 2], g[:, 2, 2], g[:, 3, 2]
    if approximation == 2:
        return np.stack([ux + F(0.5) * (ux * ux + vx * vx + wx * wx), vy + F(0.5) * (uy * uy + vy * vy + wy * wy),
                         wz + F(0.5) * (uz * uz + vz * vz + wz * wz), F(0.5) * (uy + vx + uy * ux + vy * vx + wy * wx),
                         F(0.5) * (vz + wy + uz * uy + vz * vy + wz * wy), F(0.5) * (wx + uz + ux * uz + vx * vz + wx * wz)], 1)
    return np.stack([ux, vy, wz, F(0.5) * (uy + vx), F(0.5) * (vz + wy), F(0.5) * (wx + uz)], 1)


def witness(q, radius, k_min, thr=0.9, approximation=1, subset=None, only=None):
    """Strain::compute(queue) on a copy of q (POI2D [n,25], POI3D [n,31] or POI2DS [n,28]); only=i: Strain::compute(&q[i], queue).
    subset: evaluate only these POIs (checked marks them).  Returns Witness(out, computed, checked, alts, fallback): alts maps a
    non-decisive POI to every acceptable strain row."""
    L = layout(q)
    sd, fd, fc, sl = L["sd"], L["fd"], L["fc"], L["strain"]
    C = fd + 1
    n = len(q)
    out = q.copy()
    fin = np.isfinite(q[:, :sd]).all(1)
    ok = good(q, thr)
    if only is not None:
        checked = np.zeros(n, bool)
        checked[only] = True
        cand = fin & checked
    else:
        checked = np.ones(n, bool) if subset is None else np.isin(np.arange(n), subset)
        cand = fin & ok & checked
    centres = np.flatnonzero(cand)
    computed = np.zeros(n, bool)
    fallback = np.zeros(n, bool)
    alts = {}
    if approximation not in (1, 2) or not len(centres):
        return Witness(out, computed, checked, alts, fallback)
    sets, fb = neighbour_sets(q, centres, radius, k_min)
    fallback[centres] = fb
    fits = [s[ok[s]] for s in sets]
    m = np.array([len(f) for f in fits])
    use = m >= k_min
    fitc, fits, m = centres[use], [f for f, u in zip(fits, use) if u], m[use]
    computed[fitc] = True
    coords = q[:, fc:fc + fd]
    disp = q[:, list(L["disp"])].astype(np.float64)
    X = np.zeros((len(fitc), C, fd))
    slow = np.zeros(len(fitc), bool)
    # full-rank fits: zero rows leave a least-squares solution alone, so each bucket of similar m is one stacked QR
    bucket = np.maximum(C, 1 << np.ceil(np.log2(np.maximum(m, 1))).astype(int))
    for M in np.unique(bucket):
        sel = np.flatnonzero(bucket == M)
        A = np.zeros((len(sel), M, C))
        B = np.zeros((len(sel), M, fd))
        for r, t in enumerate(sel):
            f = fits[t]
            A[r, :len(f), 0] = 1
            A[r, :len(f), 1:] = (coords[f] - coords[fitc[t]]).astype(F)
            B[r, :len(f)] = disp[f]
        Qm, R = np.linalg.qr(A)
        s = np.linalg.svd(R, compute_uv=False)
        full = (m[sel] >= C) & (s[:, -1] > 1e-3 * s[:, 0])
        X[sel[full]] = np.linalg.solve(R[full], np.swapaxes(Qm[full], 1, 2) @ B[full])
        slow[sel[~full]] = True
    for t in np.flatnonzero(slow):
        f = fits[t]
        A = np.ones((len(f), C))
        A[:, 1:] = (coords[f] - coords[fitc[t]]).astype(F)
        sols = _pivoted(A, disp[f])
        X[t] = sols[0]
        if len(sols) > 1:
            rows = _strain_rows(np.stack(sols), fd, approximation)
            alts[int(fitc[t])] = rows
    out[fitc, sl] = _strain_rows(X, fd, approximation)
    return Witness(out, computed, checked, alts, fallback)


def compare(got, q, w, tol, name=""):
    """Hold a Strain result to the witness: the same fitted POIs among the checked ones, strains within tol (relative to the
    POI's largest strain where that exceeds 1; the nearest acceptable row for a non-decisive POI), every other field and every unfitted POI's strain bit-identical to the input.
    Returns (POIs fitted, largest difference)."""
    sl = layout(q)["strain"]
    other = np.ones(q.shape[1], bool)
    other[sl] = False
    bad = np.flatnonzero((bits(got[:, other]) != bits(q[:, other])).any(1))
    assert len(bad) == 0, "%s: fields outside the strain changed at POIs %s" % (name, bad[:8])
    changed = (bits(got[:, sl]) != bits(q[:, sl])).any(1)
    wrong = np.flatnonzero(w.checked & (changed != w.computed))
    assert len(wrong) == 0, "%s: %d POIs fitted differently, e.g. %s (kernel %s, witness %s, fallback %s)" % (
        name, len(wrong), wrong[:8], changed[wrong[:8]], w.computed[wrong[:8]], w.fallback[wrong[:8]])
    idx = np.flatnonzero(w.checked & w.computed)
    if not len(idx):
        return 0, 0.0
    # absolute below 1, relative above: a Green strain squares the gradients, and float32 rounds a strain of 100 to 8e-6
    scale = np.maximum(1.0, np.abs(w.out[idx, sl].astype(np.float64)).max(1))
    d = np.abs(got[idx, sl].astype(np.float64) - w.out[idx, sl]).max(1)
    for t, i in enumerate(idx):
        if int(i) in w.alts:
            d[t] = min(d[t], np.abs(got[i, sl].astype(np.float64) - w.alts[int(i)]).max(1).min())
    d = d / scale
    worst = int(np.argmax(d))
    assert d[worst] < tol, "%s: POI %d differs by %.3g (kernel %s, witness %s)" % (name, idx[worst], d[worst], got[idx[worst], sl],
                                                                                 w.out[idx[worst], sl])
    return len(idx), float(d.max())


# ------------------------------------------------------------------------------------------------ case generators
Case = collections.namedtuple("Case", "name q radius k_min thr")


def empty(kind, n):
    """n records of POI2D (kind 2), POI3D (3) or POI2DS (23) with the strain fields at SENTINEL."""
    q = np.zeros((n, {2: 25, 3: 31, 23: 28}[kind]), F)
    q[:, LAYOUT[q.shape[1]]["strain"]] = SENTINEL
    return q


def fill(q, rng, noise=0.3, bad=0.1, thr=0.9):
    """A seeded affine displacement field plus noise over the positions, ZNCC in [thr + 0.01, 1) with a fraction `bad` below thr.
    POI2DS: ref_coor on a curved surface over (x, y) so that the 3D plane fit is well posed.  The noise makes every neighbour
    count: adding or dropping one moves the fitted gradients far beyond the kernel's tolerance."""
    L = layout(q)
    n = len(q)
    pos = q[:, :L["sd"]].astype(np.float64)
    pos = np.where(np.isfinite(pos), pos, 0)
    if q.shape[1] == 28:
        x, y = pos[:, 0], pos[:, 1]
        q[:, 14] = x - 40
        q[:, 15] = y + 25
        q[:, 16] = 400 + 2 * np.sin(x / 9.0) * np.cos(y / 7.0) + rng.normal(0, 0.05, n)
        fit = q[:, 14:17].astype(np.float64)
    else:
        fit = pos
    fit = fit - np.nanmin(fit, 0)
    G = rng.normal(0, 0.01, (fit.shape[1], len(L["disp"])))
    c = rng.normal(0, 1, len(L["disp"]))
    d = fit @ G + c + rng.normal(0, noise, (n, len(L["disp"])))
    for k, col in enumerate(L["disp"]):
        q[:, col] = d[:, k]
    z = list(L["zncc"])
    q[:, z] = rng.uniform(thr + 0.01, 1.0, (n, len(z)))
    low = rng.uniform(size=n) < bad
    q[low, z[0]] = rng.uniform(0.3, thr - 0.01, low.sum())
    return q


def queue(kind, pos, rng, **kw):
    pos = np.asarray(pos, F)
    q = empty(kind, len(pos))
    q[:, :pos.shape[1]] = pos
    return fill(q, rng, **kw)


def host_grid(pos, radius):
    """The host side of the kernel's grid in numpy: lo = the float32 bbox minimum, cell = |radius|, inv = float32(1 / cell) * 0.999f,
    cell index floor(float32(float32(p - lo) * inv)) (before any growth)."""
    lo = np.min(pos, 0).astype(F)
    inv = F(F(1.0 / abs(float(radius))) * F(0.999))
    return lo, inv


def cell_edge(lo, inv, k):
    """Smallest float32 coordinate whose cell index is k."""
    x = F(lo + F(k / np.float64(inv)))
    cell = lambda v: np.floor(F(F(v - lo) * inv))
    while cell(x) >= k:
        x = np.nextafter(x, F(-np.inf))
    while cell(x) < k:
        x = np.nextafter(x, F(np.inf))
    return x


def shell_point(p, direction, radius, inside):
    """A float32 point near p + radius * direction whose float32 squared distance from p is r2 - 1 ulp (inside) or exactly r2
    (outside), r2 = float32(radius^2); when no such point lies within a few ulps, the closest one on the required side."""
    p = np.asarray(p, F)
    r2 = F(F(radius) * F(radius))
    target = np.nextafter(r2, F(0)) if inside else r2
    u = np.asarray(direction, np.float64)
    ideal = p.astype(np.float64) + radius * u / np.linalg.norm(u)
    D = len(p)
    steps = np.arange(-6, 7)
    grid = np.stack(np.meshgrid(*([steps] * D), indexing="ij"), -1).reshape(-1, D)
    base = ideal.astype(F)
    cand = base.copy()[None].repeat(len(grid), 0)
    for k in range(D):
        sp = np.spacing(np.abs(base[k])).astype(F)
        cand[:, k] = (base[k].astype(np.float64) + grid[:, k] * np.float64(sp)).astype(F)
    d = dist2(p[None], cand)
    hit = np.flatnonzero(d == target)
    if not len(hit):
        hit = np.flatnonzero(d < r2) if inside else np.flatnonzero(d >= r2)
        hit = hit[np.argsort(np.abs(d[hit].astype(np.float64) - np.float64(target)))[:1]]
    return cand[hit[0]], bool(d[hit[0]] == target)


def directions(D):
    g = np.stack(np.meshgrid(*([[-1, 0, 1]] * D), indexing="ij"), -1).reshape(-1, D)
    return g[np.abs(g).sum(1) > 0]


def cell_boundary(kind, radius, seed=0):
    """Centre POIs on both sides of computed cell edges (x, y and, in 3D, z), each with neighbours at float32 d^2 = r^2 - 1 ulp
    and = r^2 in all 8 / 26 directions.  Returns (case, fraction of shell points placed exactly)."""
    rng = np.random.default_rng(seed)
    D = 3 if kind == 3 else 2
    lo = np.array([13.25, -7.5, 2.0][:D], F)
    lo_, inv = host_grid(lo[None], radius)
    pts, exact = [lo], []
    spacing = 6  # cells between neighbouring centres
    for axis in range(D):
        for k in (3, 3 + spacing):
            e = cell_edge(lo[axis], inv, k)
            for x in (e, np.nextafter(e, F(-np.inf))):
                c = np.array([cell_edge(lo[a], inv, 3 + spacing * (2 + axis)) + F(0.25 * radius) for a in range(D)], F)
                c[axis] = x
                pts.append(c)
                for u in directions(D):
                    for inside in (True, False):
                        s, ex = shell_point(c, u, radius, inside)
                        pts.append(s)
                        exact.append(ex)
    pos = np.array(pts, F)
    pos = np.unique(pos, axis=0)
    pos = pos[rng.permutation(len(pos))]
    pos = np.concatenate([lo[None], pos[np.any(pos != lo, 1)]])  # the bbox minimum stays lo
    q = queue(kind, pos, rng, noise=0.5, bad=0.05)
    return Case("cell_boundary_%d_r%g" % (kind, radius), q, radius, 5, 0.9), float(np.mean(exact))


def uniform(kind, n, extent, radius, k_min=5, seed=0, lo=0.0, **kw):
    rng = np.random.default_rng(seed)
    D = 3 if kind == 3 else 2
    pos = rng.uniform(lo, lo + extent, (n, D))
    return Case("uniform_%d_n%d" % (kind, n), queue(kind, pos, rng, **kw), radius, k_min, 0.9)


def lattice(kind, side, spacing, seed=0):
    D = 3 if kind == 3 else 2
    g = np.stack(np.meshgrid(*([np.arange(side) * spacing] * D), indexing="ij"), -1).reshape(-1, D).astype(F) + F(100)
    rng = np.random.default_rng(seed)
    return g[rng.permutation(len(g))], rng


def coordinate_cases(seed=0):
    rng = np.random.default_rng(seed)
    out = []
    for kind in (2, 3, 23):
        D = 3 if kind == 3 else 2
        n = 400 if D == 2 else 1500
        out.append(Case("box_pm300_%d" % kind, queue(kind, rng.uniform(-300, 300, (n, D)), rng), 40.0 if D == 2 else 60.0, 5, 0.9))
        out.append(Case("negative_%d" % kind, queue(kind, rng.uniform(-900, -700, (n, D)), rng), 20.0, 5, 0.9))
    # POIs at -0.0 and +0.0 (the bbox reads an ordered-int encoding of the float)
    pos = rng.uniform(-30, 30, (300, 2)).astype(F)
    pos[:40:2, 0] = F(-0.0)
    pos[1:40:2, 0] = F(0.0)
    pos[40:80:2, 1] = F(-0.0)
    pos[41:80:2, 1] = F(0.0)
    pos[80] = F(-0.0)
    pos[81] = F(0.0)
    out.append(Case("signed_zero_2", queue(2, pos, rng), 6.0, 5, 0.9))
    pos3 = rng.uniform(-15, 15, (600, 3)).astype(F)
    pos3[:60, 2] = np.where(np.arange(60) % 2, F(0.0), F(-0.0))
    pos3[60] = F(-0.0)
    out.append(Case("signed_zero_3", queue(3, pos3, rng), 6.0, 5, 0.9))
    # zero extent along one axis
    row = np.stack([rng.uniform(0, 500, 300), np.full(300, 77.0)], 1)
    out.append(Case("one_row_2", queue(2, row, rng), 20.0, 3, 0.9))
    plane = np.stack([rng.uniform(0, 80, 800), rng.uniform(0, 80, 800), np.full(800, -5.0)], 1)
    out.append(Case("one_plane_3", queue(3, plane, rng), 12.0, 5, 0.9))
    # a single POI; every POI at one position
    out.append(Case("single_2", queue(2, [[10.0, 20.0]], rng), 20.0, 1, 0.9))
    out.append(Case("single_3", queue(3, [[10.0, 20.0, 30.0]], rng), 20.0, 1, 0.9))
    out.append(Case("one_position_2", queue(2, np.full((12, 2), 33.5), rng), 20.0, 5, 0.9))
    out.append(Case("one_position_3", queue(3, np.full((12, 3), -3.5), rng), 20.0, 5, 0.9))
    return out


def knn_cases(seed=0):
    out = []
    for k in (6, 7, 9, 10, 13):  # ties at the k-th distance: 4 at 3, 4 at 3*sqrt(2), 4 at 6, 8 at 3*sqrt(5)
        pos, rng = lattice(2, 14, 3.0, seed + k)
        out.append(Case("lattice2_k%d" % k, queue(2, pos, rng, bad=0.0), 2.0, k, 0.9))
        pos, rng = lattice(23, 14, 3.0, seed + k)
        out.append(Case("lattice2s_k%d" % k, queue(23, pos, rng, bad=0.0), 2.0, k, 0.9))
    for k in (8, 20):
        pos, rng = lattice(3, 7, 3.0, seed + k)
        out.append(Case("lattice3_k%d" % k, queue(3, pos, rng, bad=0.0), 2.0, k, 0.9))
    rng = np.random.default_rng(seed)
    out.append(Case("k_above_n_2", queue(2, rng.uniform(0, 50, (9, 2)), rng, bad=0.0), 5.0, 12, 0.9))
    out.append(Case("k_above_n_3", queue(3, rng.uniform(0, 50, (9, 3)), rng, bad=0.0), 5.0, 12, 0.9))
    # sparse: most POIs fall back, and a third of the fallback sets hold POIs below the threshold
    out.append(Case("fallback_low_zncc_2", queue(2, rng.uniform(0, 1500, (1500, 2)), rng, bad=0.35), 20.0, 6, 0.9))
    out.append(Case("fallback_low_zncc_3", queue(3, rng.uniform(0, 300, (1500, 3)), rng, bad=0.35), 15.0, 6, 0.9))
    # non-finite coordinates, at the first and the last index too: never a neighbour, never fitted
    for kind in (2, 3, 23):
        D = 3 if kind == 3 else 2
        q = queue(kind, rng.uniform(0, 200 if D == 2 else 60, (700, D)), rng)
        bad = np.r_[0, rng.choice(np.arange(1, 699), 80, replace=False), 699]
        vals = np.array([np.nan, np.inf, -np.inf], F)
        for t, i in enumerate(bad):
            q[i, t % D if t % 4 else D - 1] = vals[t % 3]
        out.append(Case("nonfinite_%d" % kind, q, 15.0, 8, 0.9))
    return out


def rank_cases(seed=0):
    rng = np.random.default_rng(seed)
    out = []
    row = np.stack([np.arange(60) * 2.0, np.full(60, 5.0)], 1)
    out.append(Case("rank_row_2", queue(2, row, rng, bad=0.0), 7.0, 3, 0.9))
    t = rng.uniform(0, 100, 120)
    out.append(Case("rank_diagonal_2", queue(2, np.stack([t, t], 1), rng, bad=0.0), 9.0, 3, 0.9))
    t3 = rng.uniform(0, 100, 120)
    out.append(Case("rank_diagonal_3", queue(3, np.stack([t3, t3, 0.5 * t3], 1), rng, bad=0.0), 9.0, 3, 0.9))
    dup = np.repeat(rng.uniform(0, 60, (80, 2)), 3, 0)
    out.append(Case("rank_duplicates_2", queue(2, dup, rng, bad=0.0), 8.0, 5, 0.9))
    dup3 = np.repeat(np.round(rng.uniform(0, 30, (150, 3))), 2, 0)
    out.append(Case("rank_duplicates_3", queue(3, dup3, rng, bad=0.0), 6.0, 5, 0.9))
    a, b = rng.uniform(0, 60, (2, 600))
    out.append(Case("rank_coplanar_3", queue(3, np.stack([a, b, 0.5 * a - 0.25 * b + 3], 1), rng, bad=0.0), 9.0, 5, 0.9))
    out.append(Case("rank_k2_2", queue(2, rng.uniform(0, 300, (300, 2)), rng, bad=0.1), 12.0, 2, 0.9))
    out.append(Case("rank_k2_3", queue(3, rng.uniform(0, 100, (300, 3)), rng, bad=0.1), 10.0, 2, 0.9))
    return out


def value_cases(seed=0):
    """Radius and threshold values at their edges."""
    rng = np.random.default_rng(seed)
    out = []
    for kind in (2, 3, 23):
        D = 3 if kind == 3 else 2
        q = queue(kind, rng.uniform(0, 120 if D == 2 else 40, (250, D)), rng)
        for r in (0.0, -20.0, 20.0, np.inf, -np.inf, np.nan, 1e-30, 1e20):
            out.append(Case("radius_%d_%g" % (kind, r), q, r, 5, 0.9))
        z = layout(q)["zncc"][0]
        qz = q.copy()
        thr = F(0.95)
        qz[::5, z] = thr                      # exactly at the threshold: passes
        qz[1::7, z] = np.nan                  # NaN ZNCC: fails
        out.append(Case("zncc_equal_nan_%d" % kind, qz, 15.0 if D == 2 else 10.0, 5, float(thr)))
        out.append(Case("threshold_minus_inf_%d" % kind, qz, 15.0 if D == 2 else 10.0, 5, -np.inf))
        out.append(Case("threshold_inf_%d" % kind, q, 15.0, 5, np.inf))
    q = queue(23, rng.uniform(0, 150, (400, 2)), rng, bad=0.0)
    for k, col in enumerate((5, 6, 7)):    # one of the three ZNCCs fails
        q[k::9, col] = 0.5
    out.append(Case("poi2ds_one_zncc_fails", q, 15.0, 5, 0.9))
    return out


def growth_cases(seed=0):
    """Extents that force the kernel's grid to grow its cell, and one far outlier."""
    rng = np.random.default_rng(seed)
    out = []
    a = rng.uniform(0, 150, (600, 2))
    out.append(Case("growth_2d_xy", queue(2, np.concatenate([a, a[:300] + 2e6]), rng), 20.0, 5, 0.9))
    out.append(Case("growth_none_2d_x", queue(2, np.concatenate([a, a[:300] + [2e6, 0]]), rng), 20.0, 5, 0.9))
    # 65 537 x 65 537 cells of the radius: without growth the cell ids would wrap past 2^32 to a count that sorts on 18 bits
    far = np.concatenate([a[:300] + 1310560.0, [[0.0, 0.0], [1310710.0, 1310710.0]]])
    out.append(Case("growth_2d_wrap", queue(2, np.concatenate([a, far]), rng), 20.0, 5, 0.9))
    b = rng.uniform(0, 25, (1500, 3))
    corner = np.array([[0, 0, 0], [3000, 3000, 3000]], np.float64)
    out.append(Case("growth_3d", queue(3, np.concatenate([b, b[:500] + 2975, corner]), rng), 1.5, 5, 0.9))
    out.append(Case("growth_3d_r4", queue(3, np.concatenate([b, b[:500] + 2975, corner]), rng), 4.0, 5, 0.9))
    for kind in (2, 3):
        D = 3 if kind == 3 else 2
        q = queue(kind, rng.uniform(0, 150 if D == 2 else 40, (500, D)), rng)
        q[137, :D] = F(1e30)
        z = layout(q)["zncc"][0]
        q[137, z] = 0.5   # a neighbour candidate only: its own fallback set lies at an overflowing distance
        out.append(Case("outlier_1e30_%d" % kind, q, 15.0, 5, 0.9))
    return out


def small_cases():
    cb = [cell_boundary(kind, r)[0] for kind in (2, 3, 23) for r in (20.0, 7.5, 1.0)]
    return cb + coordinate_cases() + knn_cases() + rank_cases() + value_cases() + growth_cases()
