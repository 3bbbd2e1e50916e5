"""A float64 witness of EpipolarSearch::compute(queue) (reference src/oc_epipolar_search.cpp:133-205), candidate by candidate.

candidates() restates the candidate sweep of opencorr_b200/csrc/epipolar.cu (epipolar_candidates_kernel) in numpy float32 scalars,
one rounding per operation and in the kernel's order; `(int)` truncates toward zero.  witness() registers every candidate that
passes the border test with the float64 oracle's ICGN2D1 and applies the selection rule: the first maximum of ZNCC in slot order,
a slot that fails the border test never wins.  Slot 0 is the centre of the search region (never border-tested), slots 2k - 1 and
2k are x_view2 + k * step and x_view2 - k * step.

Vertical epipolar lines (e[1] == 0) are not covered: the reference converts an infinite or NaN slope to int there, which is
undefined behaviour, so there is no result to match."""
import numpy as np

from oracle.oracle import Oracle2D

GAP = 1e-5  # ZNCC gap between the best and the runner-up below which the winner is decided by rounding
F32 = np.float32
P2_N = 25


def slot_count(radius, step):
    return 1 + 2 * len(range(step, radius, step))


def rectified_f():
    """Epipolar lines y' = y."""
    return np.array([[0, 0, 0], [0, 0, -1], [0, 1, 0]], np.float32)


def sloped_f(slope, dy=0.0):
    """Epipolar line of (x, y): y' = slope * (x' - x) + y + dy."""
    return np.array([[0, 0, slope], [0, 0, -1], [-slope, 1, dy]], np.float32)


def candidates(poi, F, par_x, par_y, radius, step, rx, ry, w, h):
    """[(u, v, valid)] for every slot of one POI record, in slot order."""
    F = [F32(f) for f in np.asarray(F, np.float32).reshape(9)]
    ax = [F32(a) for a in np.asarray(par_x, np.float32).reshape(3)]
    ay = [F32(a) for a in np.asarray(par_y, np.float32).reshape(3)]
    px, py, pu, pv = F32(poi[0]), F32(poi[1]), F32(poi[2]), F32(poi[8])
    with np.errstate(over="ignore", invalid="ignore"):
        cxh, cyh = F32(w // 2), F32(h // 2)
        dxc, dyc = px - cxh, py - cyh
        parx = (ax[0] * dxc + ax[1] * dyc) + ax[2]
        pary = (ay[0] * dxc + ay[1] * dyc) + ay[2]
        v0, v1 = px + pu, py + pv
        e = [(F[3 * k] * v0 + F[3 * k + 1] * v1) + F[3 * k + 2] for k in range(3)]
        slope = -e[0] / e[1]
        intercept = -e[2] / e[1]
        num = slope * (((py + pv) + pary) - intercept)
        num = ((num + px) + pu) + parx
        x_view2 = int(num / (slope * slope + F32(1)))
        out = []
        for slot in range(slot_count(radius, step)):
            x_trial, valid = x_view2, True
            if slot > 0:
                k = (slot + 1) >> 1
                x_trial = x_view2 + k * step if slot & 1 else x_view2 - k * step
            y_trial = int(slope * F32(x_trial) + intercept)
            if slot > 0:
                valid = x_trial - rx > 0 and x_trial + rx < w - 1 and y_trial - ry > 0 and y_trial + ry < h - 1
            out.append((F32(F32(x_trial) - px), F32(F32(y_trial) - py), valid))
    return out


def candidate_queue(q, F, par_x, par_y, radius, step, rx, ry, w, h):
    """(records [n, slots, 25] as the candidate kernel writes them, valid [n, slots])."""
    s = slot_count(radius, step)
    cand = np.zeros((len(q), s, P2_N), np.float32)
    valid = np.zeros((len(q), s), bool)
    for i, poi in enumerate(q):
        for j, (u, v, ok) in enumerate(candidates(poi, F, par_x, par_y, radius, step, rx, ry, w, h)):
            cand[i, j, 0:2] = poi[0:2]
            cand[i, j, 2], cand[i, j, 8] = u, v
            valid[i, j] = ok
    cand[~valid, 16] = -np.inf
    return cand, valid


def witness(ref, tar, q, F, par_x, par_y, radius, step, rx, ry, conv, stop, oracle=None):
    """Returns (records [n, 25], gap [n], near [n] sets of slots within GAP of the best, cand [n, slots, 25], valid [n, slots]).
    gap: best minus runner-up ZNCC over the valid slots (inf with a single valid slot)."""
    h, w = ref.shape
    o = oracle if oracle is not None else Oracle2D(ref, tar)
    cand, valid = candidate_queue(q, F, par_x, par_y, radius, step, rx, ry, w, h)
    flat = np.ascontiguousarray(cand[valid])
    o.icgn2d1(flat, rx, ry, conv, stop, exact=True)
    cand[valid] = flat
    z = np.where(valid, cand[:, :, 16].astype(np.float64), -np.inf)
    out = q.copy()
    gap = np.full(len(q), np.inf)
    near = []
    for i in range(len(q)):
        zi = z[i]
        best = int(np.flatnonzero(zi == zi.max())[0])  # the first maximum in slot order
        out[i, 2:14] = cand[i, best, 2:14]
        out[i, 14:20] = cand[i, best, 14:20]
        rest = np.delete(zi, best)
        if len(rest) and np.isfinite(rest.max()):
            gap[i] = zi[best] - rest.max()
        near.append(set(np.flatnonzero(valid[i] & (zi >= zi[best] - GAP)).tolist()))
    return out, gap, near, cand, valid
