"""CPU oracle of the stereo-reconstruction module (oracle/oc_stereo.cpp) against the reference's shipped stereo tables:
Calibration::prepare / undistort (src/oc_calibration.cpp:161-264) and Stereovision::reconstruct (src/oc_stereovision.cpp:70-133),
fed with the tables' own 2D points, in the faithful (float32) and exact (float64) flavours."""
import numpy as np
import pytest

import stereo_cases as sc
from oracle import stereo as so

TOL = 5e-4  # mm


@pytest.fixture(scope="module")
def data():
    return sc.load()


def _oracle_rig(d, name, exact):
    c1, c2, (h, w) = sc.rig(d, name)
    o1 = so.CalibOracle(c1.intrinsic_vector(), h, w, exact=exact)
    o2 = so.CalibOracle(c2.intrinsic_vector(), h, w, exact=exact)
    return o1, c1.projection_vector(), o2, c2.projection_vector()


@pytest.mark.parametrize("exact", [False, True])
def test_step18_table(data, exact):
    o1, p1, o2, p2 = _oracle_rig(data, "step18", exact)
    pts1, pts2, ref = sc.step18_points(data)
    out = so.reconstruct(o1, p1, o2, p2, pts1, pts2)
    err = np.abs(out.astype(np.float64) - ref)
    assert err.max(axis=0).max() <= TOL, err.max(axis=0)
    assert np.median(err[:, 2]) <= 1e-4, np.median(err[:, 2])
    # the rows whose r2 lies outside the image went through undistort's clamp, and r2 was clamped in place
    w, h = (int(v) for v in data["step18_size"][::-1])
    r2 = data["step18_r2"]
    outside = (r2[:, 0] < 0) | (r2[:, 1] < 0) | (r2[:, 0] > w - 2) | (r2[:, 1] > h - 2)
    assert outside.sum() > 0
    assert (pts2[:, 0] >= 0).all() and (pts2[:, 0] <= w - 2).all() and (pts2[:, 1] >= 0).all() and (pts2[:, 1] <= h - 2).all()
    assert np.array_equal(pts2[~outside], r2[~outside])


@pytest.mark.parametrize("exact", [False, True])
def test_gt4_table(data, exact):
    o1, p1, o2, p2 = _oracle_rig(data, "gt4", exact)
    r1, r2, t1, t2, ref, tar = sc.gt4_points(data)
    ref_o = so.reconstruct(o1, p1, o2, p2, r1, r2).astype(np.float64)
    tar_o = so.reconstruct(o1, p1, o2, p2, t1, t2).astype(np.float64)
    assert np.abs(ref_o - ref).max() <= TOL
    assert np.abs(tar_o - tar).max() <= TOL
    # u, v, w = tar - ref
    assert np.abs((tar_o - ref_o) - (tar.astype(np.float64) - ref)).max() <= TOL


@pytest.mark.parametrize("case", sc.SYNTHETIC, ids=[c[0] for c in sc.SYNTHETIC])
def test_faithful_map_matches_numpy(case):
    name, intr, h, w, conv, it = case
    mx, my = so.CalibOracle(intr, h, w, conv, it).map()
    nx, ny = sc.numpy_map(intr, h, w, conv, it)
    assert np.array_equal(mx, nx, equal_nan=True) and np.array_equal(my, ny, equal_nan=True)
    if name == "isinf_reset":
        assert np.isinf(my).any()


def test_nan_pair_gives_zero_and_is_left_alone(data):
    o1, p1, o2, p2 = _oracle_rig(data, "gt4", False)
    r1, r2 = sc.gt4_points(data)[:2]
    r1, r2 = r1[:8].copy(), r2[:8].copy()
    r1[2, 0] = np.nan
    r2[5, 1] = np.nan
    a1, a2 = r1.copy(), r2.copy()
    out = so.reconstruct(o1, p1, o2, p2, r1, r2)
    assert (out[[2, 5]] == 0).all() and (out[[0, 1, 3, 4, 6, 7], 2] > 300).all()
    assert np.array_equal(r1, a1, equal_nan=True) and np.array_equal(r2, a2, equal_nan=True)
