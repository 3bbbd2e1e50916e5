"""Stereo reconstruction on the GPU: Calibration::prepare / undistort (reference src/oc_calibration.cpp:161-264) and
Stereovision::reconstruct (src/oc_stereovision.cpp:70-133) against the faithful CPU oracle (oracle/oc_stereo.cpp) and the
reference's shipped Step18 and GT4 stereo tables.

Maps and undistorted coordinates are float32 in the reference's operation order on both sides, so they must agree bit for bit
(NaN payloads aside: a NaN equals a NaN).  The GPU solves the 4x3 system in FP64, the faithful oracle by float32 column-pivoting
QR as the reference does, so 3D points are compared with tolerances: to the tables, and to a float64 least-squares solve of the
oracle's own float32 system within one float32 ulp."""
import ctypes

import numpy as np
import pytest

import opencorr_b200 as ob
import stereo_cases as sc
from opencorr_b200 import _capi
from oracle import stereo as so

pytestmark = pytest.mark.gpu

TOL = 5e-4  # mm


@pytest.fixture(scope="module")
def data():
    return sc.load()


def _same(a, b):
    return a.shape == b.shape and np.array_equal(a, b, equal_nan=True)


def _prepared_rig(d, name, engine):
    c1, c2, (h, w) = sc.rig(d, name, engine)
    c1.prepare(h, w)
    c2.prepare(h, w)
    sv = ob.Stereovision(c1, c2, 0, engine)
    sv.prepare()
    return c1, c2, sv, (h, w)


@pytest.mark.parametrize("name", ["step18", "gt4"])
def test_example_maps_bit_identical(data, engine, name):
    c1, c2, _, (h, w) = _prepared_rig(data, name, engine)
    for cam in (c1, c2):
        gx, gy = cam.get_map()
        ox, oy = so.CalibOracle(cam.intrinsic_vector(), h, w).map()
        assert gx.shape == (h, w) and _same(gx, ox) and _same(gy, oy)


@pytest.mark.parametrize("case", sc.SYNTHETIC, ids=[c[0] for c in sc.SYNTHETIC])
def test_synthetic_maps_bit_identical(engine, case):
    name, intr, h, w, conv, it = case
    cam = sc.camera(intr, [0] * 6, engine)
    cam.setUndistortion(conv, it)
    assert cam.getConvergence() == conv and cam.getIteration() == it
    cam.prepare(h, w)
    gx, gy = cam.get_map()
    ox, oy = so.CalibOracle(intr, h, w, conv, it).map()
    assert _same(gx, ox) and _same(gy, oy)
    if name == "isinf_reset":
        assert np.isinf(gy).any()


def test_undistort_bit_identical_with_clamp(data, engine):
    c1, c2, _, (h, w) = _prepared_rig(data, "step18", engine)
    pts1, pts2, _ = sc.step18_points(data)
    outside = (pts2[:, 0] < 0) | (pts2[:, 1] < 0) | (pts2[:, 0] > w - 2) | (pts2[:, 1] > h - 2)
    assert outside.sum() > 0
    for cam, pts in ((c1, pts1), (c2, pts2)):
        g, o = pts.copy(), pts.copy()
        ug = cam.undistort(g)
        uo = so.CalibOracle(cam.intrinsic_vector(), h, w).undistort(o)
        assert _same(ug, uo) and _same(g, o)
    # intrinsics changed after prepare(): the lookup uses the current ones, the map stays
    c2.intrinsics["cx"] += 1.5
    g, o = pts2.copy(), pts2.copy()
    ug = c2.undistort(g)
    oc = so.CalibOracle(data["step18_intrinsics"][1], h, w)
    uo = oc.undistort(o, c2.intrinsic_vector())
    assert _same(ug, uo)


@pytest.mark.parametrize("name", ["step18", "gt4"])
def test_reconstruct_tables(data, engine, name):
    _, _, sv, _ = _prepared_rig(data, name, engine)
    if name == "step18":
        pts1, pts2, ref = sc.step18_points(data)
        pairs = [(pts1, pts2, ref)]
    else:
        r1, r2, t1, t2, ref, tar = sc.gt4_points(data)
        pairs = [(r1, r2, ref), (t1, t2, tar)]
    outs = []
    for a, b, table in pairs:
        out = sv.reconstruct(a, b).astype(np.float64)
        err = np.abs(out - table)
        assert err.max() <= TOL, err.max(axis=0)
        assert np.median(err[:, 2]) <= 1e-4
        outs.append(out)
    if name == "gt4":  # derived displacements u, v, w
        r1, r2, t1, t2, ref, tar = sc.gt4_points(data)
        assert np.abs((outs[1] - outs[0]) - (tar.astype(np.float64) - ref)).max() <= TOL


def _lstsq64(A, b):
    """float64 least squares of a stack of 4x3 systems (QR)."""
    q, r = np.linalg.qr(A.astype(np.float64))
    qtb = np.einsum("nij,ni->nj", q, b.astype(np.float64))
    return np.linalg.solve(r, qtb[..., None])[..., 0]


@pytest.mark.parametrize("name", ["step18", "gt4"])
def test_reconstruct_within_one_ulp_of_float64_solve(data, engine, name):
    c1, c2, sv, (h, w) = _prepared_rig(data, name, engine)
    pts1, pts2 = (sc.step18_points(data) if name == "step18" else sc.gt4_points(data))[:2]
    g1, g2, o1, o2 = pts1.copy(), pts2.copy(), pts1.copy(), pts2.copy()
    out = sv.reconstruct(g1, g2)
    oc1 = so.CalibOracle(c1.intrinsic_vector(), h, w)
    oc2 = so.CalibOracle(c2.intrinsic_vector(), h, w)
    _, A, b = so.reconstruct(oc1, c1.projection_vector(), oc2, c2.projection_vector(), o1, o2, with_system=True)
    assert _same(g1, o1) and _same(g2, o2)  # the same clamping, hence the same undistorted points and system
    x = _lstsq64(A, b)
    ulp = np.spacing(np.abs(x.astype(np.float32)))
    assert (np.abs(out.astype(np.float64) - x) <= ulp).all()


def test_nan_pairs(data, engine):
    _, _, sv, _ = _prepared_rig(data, "gt4", engine)
    r1, r2 = (a[:64].copy() for a in sc.gt4_points(data)[:2])
    r1[3, 0] = np.nan
    r2[10, 1] = np.nan
    r1[20] = np.nan
    r2[20] = np.nan
    r2[30, 0] = -50.0  # a clamped neighbour of the NaN rows
    a1, a2 = r1.copy(), r2.copy()
    out = sv.reconstruct(r1, r2)
    nan_rows = [3, 10, 20]
    assert (out[nan_rows] == 0).all()
    assert _same(r1[nan_rows], a1[nan_rows]) and _same(r2[nan_rows], a2[nan_rows])
    assert r2[30, 0] == 0.0 and (out[np.setdiff1d(np.arange(64), nan_rows), 2] > 300).all()


def _raw_reconstruct(eng, calib1, calib2, cams, pts1, pts2, out, n):
    i1, p1 = cams[0].intrinsic_vector(), cams[0].projection_vector()
    i2, p2 = cams[1].intrinsic_vector(), cams[1].projection_vector()
    vp = lambda a: ctypes.c_void_p(a.ctypes.data) if a is not None else None  # noqa: E731
    return eng._lib.ocb_stereo_reconstruct(eng._ctx, calib1, vp(i1), vp(p1), calib2, vp(i2), vp(p2), vp(pts1), vp(pts2), vp(out), n)


def test_errors_leave_the_queue_unchanged(data, engine):
    c1, c2, sv, (h, w) = _prepared_rig(data, "gt4", engine)
    r1, r2 = (a[:16].copy() for a in sc.gt4_points(data)[:2])
    r2[0, 0] = 5000.0  # would be clamped by a successful call
    a1, a2 = r1.copy(), r2.copy()
    out = np.full((16, 3), 7.0, np.float32)
    lib = engine._lib

    rc = _raw_reconstruct(engine, None, c2._calib, (c1, c2), r1, r2, out, 16)
    assert rc == _capi.OCB_ERR_ARG and "null calibration handle" in _capi.last_error(engine._ctx)

    rc = _raw_reconstruct(engine, c1._calib, c2._calib, (c1, c2), None, r2, out, 16)
    assert rc == _capi.OCB_ERR_ARG and "bad arguments" in _capi.last_error(engine._ctx)
    assert _raw_reconstruct(engine, c1._calib, c2._calib, (c1, c2), None, None, None, 0) == _capi.OCB_OK  # n = 0: nothing to do

    bad = sc.camera(data["gt4_intrinsics"][0], data["gt4_extrinsics"][0], engine)
    with pytest.raises(ob.OpenCorrB200Error, match="image size 1 x 5 is below 2 x 2"):
        bad.prepare(5, 1)
    with pytest.raises(ob.OpenCorrB200Error, match="prepare\\(height, width\\) has not been called"):
        bad.undistort(r1.copy())

    other = ob.Engine(0)
    try:
        foreign = sc.camera(data["gt4_intrinsics"][1], data["gt4_extrinsics"][1], other)
        foreign.prepare(h, w)
        rc = _raw_reconstruct(engine, c1._calib, foreign._calib, (c1, foreign), r1, r2, out, 16)
        assert rc == _capi.OCB_ERR_ARG and "calibration handle belongs to another context" in _capi.last_error(engine._ctx)
        with pytest.raises(ob.OpenCorrB200Error, match="prepared on different engines"):
            ob.Stereovision(c1, foreign).reconstruct(r1, r2)
        mx = np.empty((h, w), np.float32)
        rc = lib.ocb_calib_get_map(engine._ctx, foreign._calib, ctypes.c_void_p(mx.ctypes.data), None)
        assert rc == _capi.OCB_ERR_ARG and "calib_get_map: calibration handle belongs to another context" in _capi.last_error(engine._ctx)
        foreign._release()
    finally:
        other.close()
    assert _same(r1, a1) and _same(r2, a2) and (out == 7.0).all()
    # the context still works afterwards
    good = sv.reconstruct(r1, r2)
    assert r2[0, 0] == w - 2 and np.isfinite(good).all()


def test_dev_variant_bit_identical(data, engine):
    torch = pytest.importorskip("torch")
    c1, c2, sv, _ = _prepared_rig(data, "step18", engine)
    pts1, pts2, _ = sc.step18_points(data)
    h1, h2 = pts1.copy(), pts2.copy()
    host = sv.reconstruct(h1, h2)
    d1, d2 = torch.from_numpy(pts1.copy()).cuda(), torch.from_numpy(pts2.copy()).cuda()
    d3 = torch.empty((len(pts1), 3), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    engine.set_stream(torch.cuda.current_stream().cuda_stream)
    try:
        sv.reconstruct_dev(d1.data_ptr(), d2.data_ptr(), d3.data_ptr(), len(pts1))
        torch.cuda.synchronize()
    finally:
        engine.use_own_stream()
    assert _same(d3.cpu().numpy(), host) and _same(d1.cpu().numpy(), h1) and _same(d2.cpu().numpy(), h2)


def test_group_context_bit_identical(data, engine):
    devices = list(range(_capi.load().ocb_device_count()))
    grp = ob.Engine(devices)
    try:
        res = []
        for eng in (engine, grp):
            c1, c2, sv, _ = _prepared_rig(data, "gt4", eng)
            r1, r2, t1, t2 = (a.copy() for a in sc.gt4_points(data)[:4])
            res.append((sv.reconstruct(r1, r2), sv.reconstruct(t1, t2), r1, r2, t1, t2, c2.get_map()[1]))
            u = c1.undistort(t1.copy())
            res[-1] += (u,)
        for a, b in zip(*res):
            assert _same(a, b)
        with pytest.raises(ob.OpenCorrB200Error, match="single-device context"):
            sv.reconstruct_dev(0, 0, 0, 1)
    finally:
        grp.close()
