"""CPU only: the float64 witness of tests/epipolar_cases.py against the oracle's EpipolarSearch, and the oracle's single-POI Strain
against its own queue mode.  These pin the two references before test_gpu_epipolar_geometry.py and test_gpu_strain_single.py hold
the GPU to them."""
import numpy as np
import pytest

import opencorr_b200 as ob
from opencorr_b200 import synth
from oracle import oracle
from oracle.oracle import Oracle2D
import epipolar_cases as ec


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def rig_fundamental(width, height):
    """F of the synth.stereo_rig cameras (view 1 pixel -> epipolar line in view 2), K2^-T [t2]x R2 K1^-1 in float32."""
    intr, extr = synth.stereo_rig(width, height)
    K = np.array([[intr[0, 0], 0, intr[0, 3]], [0, intr[0, 1], intr[0, 4]], [0, 0, 1]], np.float64)
    R = synth._rotation(extr[1, 3:6].astype(np.float64))
    t = extr[1, 0:3].astype(np.float64)
    tx = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
    F = np.linalg.inv(K).T @ tx @ R @ np.linalg.inv(K)
    return (F / np.abs(F).max()).astype(np.float32)


def _pin(ref, tar, xy, F, par_x, par_y, radius, step, rx, ry, conv=0.001, stop=10, min_decisive=0.6):
    q = ob.make_poi2d(xy)
    o = Oracle2D(ref, tar)
    out, gap, near, cand, valid = ec.witness(ref, tar, q, F, par_x, par_y, radius, step, rx, ry, conv, stop, oracle=o)
    b = o.epipolar_search(q.copy(), F, par_x, par_y, radius, step, rx, ry, conv, stop, exact=True)
    dec = gap > ec.GAP
    assert dec.mean() >= min_decisive, dec.mean()
    bad = np.flatnonzero(dec & (_bits(out) != _bits(b)).any(1))
    assert len(bad) == 0, (bad[:8], out[bad[:2]], b[bad[:2]])
    # a non-decisive POI: the oracle's winner is one of the near slots
    for i in np.flatnonzero(~dec):
        assert any(np.array_equal(_bits(cand[i, s, 2:20]), _bits(b[i, 2:20])) for s in near[i]), i
    keep = [0, 1, 20, 21, 22, 23, 24]
    assert np.array_equal(_bits(b[:, keep]), _bits(q[:, keep]))
    return out, gap, valid


def test_witness_matches_oracle_rectified():
    ref, tar = synth.speckle_pair_2d(320, 256)
    xy = np.array([[x, y] for y in (30, 128, 200) for x in (24, 90, 160, 250, 300)], np.float32)
    out, gap, valid = _pin(ref, tar, xy, ec.rectified_f(), [0.001, 0, 2.0], [0, 0.002, 0.5], 25, 6, 12, 10)
    assert (~valid).any() and valid[:, 1:].any()   # POIs near the borders lose slots to the border test


def test_witness_matches_oracle_stereo_rig():
    w, h = 384, 320
    d = synth.speckle_stereo_series(w, h, 1)
    F = rig_fundamental(w, h)
    xy = synth.grid_2d(60, 60, 5, 4, 60, 60)
    out, gap, valid = _pin(d["ref1"], d["r2"], xy, F, [0, 0, 4.0], [0, 0, 0], 25, 6, 14, 14)
    e = np.c_[xy, np.ones(len(xy))] @ F.astype(np.float64).T
    slopes = -e[:, 0] / e[:, 1]
    assert np.abs(slopes).max() > 1e-3      # not a rectified pair: the lines tilt, and differ from POI to POI
    assert np.ptp(slopes) > 1e-4


def test_candidates_steep_negative_and_truncation():
    """The candidate positions themselves: a steep line steps y by |slope| * step, a negative x_view2 truncates toward zero."""
    q = ob.make_poi2d(np.array([[100, 120]], np.float32))
    c = ec.candidates(q[0], ec.sloped_f(-3.0), [0, 0, 0], [0, 0, 0], 7, 2, 8, 8, 256, 256)
    assert len(c) == 7
    assert [(float(u), float(v)) for u, v, _ in c[:3]] == [(0, 0), (2, -6), (-2, 6)]
    c = ec.candidates(q[0], ec.rectified_f(), [0, 0, -100.5], [0, 0, 0], 3, 1, 8, 8, 256, 256)
    assert float(c[0][0]) == -100.0   # x_view2 = (int)(-0.5) = 0, not -1
    assert not c[1][2] and not c[2][2]


@pytest.mark.parametrize("dim", [2, 3])
@pytest.mark.parametrize("approximation", [1, 2])
def test_oracle_strain_single_matches_queue(dim, approximation):
    rng = np.random.default_rng(5 + dim)
    n = 400
    if dim == 2:
        q = ob.make_poi2d(rng.uniform(0, 150, (n, 2)).astype(np.float32))
        q[:, 2] = 0.01 * q[:, 0] - 0.002 * q[:, 1] + rng.normal(0, 0.01, n)
        q[:, 8] = 0.003 * q[:, 0] + 0.02 * q[:, 1] + rng.normal(0, 0.01, n)
        zc, sc = 16, slice(20, 23)
    else:
        q = ob.make_poi3d(rng.uniform(0, 60, (n, 3)).astype(np.float32))
        q[:, 3], q[:, 7], q[:, 11] = (q[:, :3] @ rng.normal(0, 0.01, (3, 3))).T
        zc, sc = 18, slice(22, 28)
    q[:, zc] = rng.uniform(0.8, 1.0, n)
    full = oracle.strain(q.copy(), 20.0, 5, 0.9, approximation, exact=True)
    good = np.flatnonzero(q[:, zc] >= 0.9)
    for i in (good[0], good[len(good) // 2], good[-1]):
        one = oracle.strain(q.copy(), 20.0, 5, 0.9, approximation, exact=True, only=int(i))
        expect = q.copy()
        expect[i] = full[i]
        assert np.array_equal(_bits(one), _bits(expect)), i
    assert np.any(one[i, sc] != 0)
    # below the threshold: computed anyway in single mode, skipped by the queue mode
    lows = np.flatnonzero(q[:, zc] < 0.9)
    low = int(lows[np.argmin(np.abs(q[lows, :dim] - q[:, :dim].mean(0)).sum(1))])  # in the middle of the patch
    assert np.all(full[low, sc] == 0)
    one = oracle.strain(q.copy(), 20.0, 5, 0.9, approximation, exact=True, only=low)
    assert np.any(one[low, sc] != 0)
    assert np.array_equal(_bits(np.delete(one, low, 0)), _bits(np.delete(q, low, 0)))
