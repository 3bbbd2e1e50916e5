"""Stereo DIC over a load series of stereo pairs (ocb_stereo_series): both views of every frame registered against reference
view 1, each frame seeded by the previous one, and triangulated into POI2DS records.

out1 and out2 must be, byte for byte, two ocb_icgn2d_series calls on (ref1, tars1) and (ref1, tars2); out2ds must be, byte for
byte, the host assembly of the reference's example (Stereovision.reconstruct on copies of the points plus numpy float32
arithmetic).  Against data: the float64 oracle frame by frame, the synthetic ground truth and the reference's GT4 table, within
the bounds test_stereo_series_host.py measures on the CPU."""
import ctypes

import numpy as np
import pytest

import opencorr_b200 as ob
import stereo_cases as sc
import stereo_series_cases as ssc
from opencorr_b200 import _capi, synth
from oracle.oracle import Oracle2D
from util import compare_2d

pytestmark = pytest.mark.gpu


def assert_same(a, b, label):
    """Byte equality; a NaN equals any NaN (the device's NaN has another payload than numpy's)."""
    assert a.shape == b.shape, label
    bad = (a.view(np.uint32) != b.view(np.uint32)) & ~(np.isnan(a) & np.isnan(b))
    assert not bad.any(), "%s: %d floats differ, first at %s" % (label, bad.sum(), np.argwhere(bad)[:5].tolist())


_series = {}


def series(width):
    """The synthetic stereo series at this width (384: TMA staging; 387: W % 4 != 0, gathers) and its grid points."""
    if width not in _series:
        xy = synth.grid_2d(40, 40, 13, 11, 25, 22)
        _series[width] = (synth.speckle_stereo_series(width, ssc.SYN_H, ssc.SYN_F, points=xy), xy)
    return _series[width]


def prepared_rig(engine, width, height, intrinsics=None, extrinsics=None):
    if intrinsics is None:
        intrinsics, extrinsics = synth.stereo_rig(width, height)
    c1, c2 = sc.camera(intrinsics[0], extrinsics[0], engine), sc.camera(intrinsics[1], extrinsics[1], engine)
    c1.prepare(height, width)
    c2.prepare(height, width)
    rig = ob.Stereovision(c1, c2, 0, engine)
    rig.prepare()
    return rig


def stereo_match(engine, r1, r2, xy, r, guess=None, stop=10):
    """The r1 -> r2 records from the pair calls: ICGN2D2 from the rounded guess, or from FFT-CC without one."""
    q = ob.make_poi2d(xy) if guess is None else ssc.translation_seeds(xy, guess)
    engine.set_images_2d(r1, r2)
    if guess is None:
        engine.fftcc2d(q, r, r)
    engine.icgn2d_prepare()
    engine.icgn2d2(q, r, r, ssc.CONV, stop)
    return q


def recipe(engine, d, xy, stereo, r):
    """Frame-0 seeds as INTEGRATION.md describes them: FFT-CC on (r1, tars1[0]), then stereo's u, v added for view 2."""
    s1 = ob.make_poi2d(xy)
    engine.set_images_2d(d["ref1"], d["tars1"][0])
    engine.fftcc2d(s1, r, r)
    return s1, ssc.recipe_seeds2(s1, stereo)


def _grid(kind, r, width):
    if kind == "short":
        return synth.grid_2d(60, 55, 6, 5, 48, 41)
    return synth.grid_2d(r + 4, r + 4, (width - 2 * r - 12) // 3, 70, 3, 4)  # thousands of POIs: one warp per POI


def _setup(engine, width, kind, r):
    d, _ = series(width)
    xy = _grid(kind, r, width)
    stereo = stereo_match(engine, d["ref1"], d["r2"], xy, r)
    s1, s2 = recipe(engine, d, xy, stereo, r)
    return d, xy, stereo, s1, s2


@pytest.mark.parametrize("width", [384, 387], ids=["tma", "gather"])
@pytest.mark.parametrize("kind", ["short", "long"])
@pytest.mark.parametrize("r", [12, 16])
@pytest.mark.parametrize("order1,order2", [(1, 2), (2, 2), (1, 1)])
def test_views_equal_2d_series_and_records_equal_host_assembly(engine, width, kind, r, order1, order2):
    d, xy, stereo, s1, s2 = _setup(engine, width, kind, r)
    rig = prepared_rig(engine, width, ssc.SYN_H)
    for F in (1, 4):
        engine.set_stereo_series(d["ref1"], d["tars1"][:F], d["tars2"][:F])
        out1, out2, out2ds = engine.stereo_series(rig, stereo, s1, s2, order1, order2, r, r, ssc.CONV, 10)
        engine.set_series_2d(d["ref1"], d["tars1"][:F])
        assert_same(out1, engine.icgn2d_series(order1, s1, r, r, ssc.CONV, 10), "view 1, F %d" % F)
        engine.set_series_2d(d["ref1"], d["tars2"][:F])
        assert_same(out2, engine.icgn2d_series(order2, s2, r, r, ssc.CONV, 10), "view 2, F %d" % F)
        assert_same(out2ds, ssc.assemble(rig.reconstruct, stereo, s1, out1, out2), "POI2DS records, F %d" % F)
        assert (out1[-1][:, 16] >= 0).mean() > 0.8 and (out2[-1][:, 16] >= 0).mean() > 0.8


def test_equals_loop_of_dev_pair_calls(engine):
    torch = pytest.importorskip("torch")
    d, xy, stereo, s1, s2 = _setup(engine, 384, "short", 16)
    rig = prepared_rig(engine, 384, ssc.SYN_H)
    engine.set_stereo_series(d["ref1"], d["tars1"], d["tars2"])
    out1, out2, out2ds = engine.stereo_series(rig, stereo, s1, s2, 1, 2, 16, 16, ssc.CONV, 10)
    d_ref = torch.from_numpy(d["ref1"]).cuda()
    n = len(xy)
    for view, (tars, seeds, order, out) in enumerate(((d["tars1"], s1, 1, out1), (d["tars2"], s2, 2, out2))):
        q = torch.from_numpy(seeds).cuda()
        for f in range(ssc.SYN_F):
            d_tar = torch.from_numpy(tars[f]).cuda()
            torch.cuda.synchronize()
            engine.set_images_2d_dev(d_ref.data_ptr(), d_tar.data_ptr(), 384, ssc.SYN_H)
            engine.icgn2d_prepare()
            (engine.icgn2d1_dev if order == 1 else engine.icgn2d2_dev)(q.data_ptr(), n, 16, 16, ssc.CONV, 10)
            engine.sync()
            assert_same(q.cpu().numpy(), out[f], "view %d frame %d" % (view + 1, f))
    d_out1, d_out2 = torch.from_numpy(out1).cuda(), torch.from_numpy(out2).cuda()
    pts = lambda o: torch.stack([o[:, 0] + o[:, 2], o[:, 1] + o[:, 8]], 1).contiguous()  # noqa: E731
    for f in range(ssc.SYN_F):  # the device-resident triangulation of the loop gives the same tar_coor
        p1, p2 = pts(d_out1[f]), pts(d_out2[f])
        xyz = torch.empty((n, 3), dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        rig.reconstruct_dev(p1.data_ptr(), p2.data_ptr(), xyz.data_ptr(), n)
        engine.sync()
        assert_same(xyz.cpu().numpy(), out2ds[f, :, 17:20], "tar_coor frame %d" % f)


def test_records_at_the_edges(engine):
    """Points clamped at the image border, a POI whose subset leaves the image mid-series, a failed stereo record and NaN
    coordinates: out2ds is still the host assembly, byte for byte."""
    d, xy, stereo, s1, s2 = _setup(engine, 384, "short", 16)
    w, h = 384, ssc.SYN_H
    n = len(xy)
    stereo, s1, s2 = stereo.copy(), s1.copy(), s2.copy()
    stereo[0, 2] = -stereo[0, 0] - 3.5          # r2 left of the image: clamped to x = 0
    stereo[1, 8] = h + 7.25 - stereo[1, 1]      # r2 below the image: clamped to y = h - 2
    stereo[2, 16] = -1.0                        # a failed stereo match: its code is carried into r1r2
    stereo[3, 8] = np.nan                       # a NaN coordinate: ref_coor (0, 0, 0)
    s2[4, 2] = np.nan                           # a NaN guess in view 2
    # the series moves these subsets right, out of the image: frame 0 still registers some of them
    edge = np.array([[w - 21.0, 150.0], [w - 22.0, 200.0], [w - 23.0, 250.0]], np.float32)
    stereo = np.concatenate([stereo, stereo_match(engine, d["ref1"], d["r2"], edge, 16)])
    e1, e2 = recipe(engine, d, edge, stereo[n:], 16)
    s1, s2 = np.concatenate([s1, e1]), np.concatenate([s2, e2])
    rig = prepared_rig(engine, w, h)
    engine.set_stereo_series(d["ref1"], d["tars1"], d["tars2"])
    out1, out2, out2ds = engine.stereo_series(rig, stereo, s1, s2, 1, 2, 16, 16, ssc.CONV, 10)
    assert_same(out2ds, ssc.assemble(rig.reconstruct, stereo, s1, out1, out2), "edge records")
    assert (out2ds[:, 0, 8] < 0).all() and (out2ds[:, 1, 9] > h - 2).all()   # stored unclamped
    assert (out2ds[:, 2, 5] == -1).all()
    assert (out2ds[:, 3, 14:17] == 0).all() and np.isnan(out2ds[:, 3, 9]).all()
    left = out1[:, n:, 16] < 0
    assert (left[-1] & ~left[0]).any()  # lost in a later frame, with its code in r1t1
    assert_same(out2ds[:, n:, 6], out1[:, n:, 16], "r1t1 codes")


def test_synthetic_series_against_oracle_and_truth(engine):
    d, xy = series(384)
    rig = prepared_rig(engine, 384, ssc.SYN_H)
    stereo = stereo_match(engine, d["ref1"], d["r2"], xy, 16)
    s1, s2 = recipe(engine, d, xy, stereo, 16)
    engine.set_stereo_series(d["ref1"], d["tars1"], d["tars2"])
    out1, out2, out2ds = engine.stereo_series(rig, stereo, s1, s2, 1, 2, 16, 16, ssc.CONV, 10)
    for f in range(ssc.SYN_F):
        for view, (tars, seeds, out, order) in enumerate(((d["tars1"], s1, out1, 1), (d["tars2"], s2, out2, 2))):
            q = (seeds if f == 0 else out[f - 1]).copy()
            o = Oracle2D(d["ref1"], tars[f])
            (o.icgn2d1 if order == 1 else o.icgn2d2)(q, 16, 16, ssc.CONV, 10, exact=True)
            compare_2d(out[f], q, "view %d frame %d" % (view + 1, f), order=order)
        assert (out2ds[f, :, 6:8] > 0.99).all()
        assert np.abs(out2ds[f, :, 10:12] - d["t1_true"][f]).max() < ssc.SYN_PX_BOUND
        assert np.abs(out2ds[f, :, 12:14] - d["t2_true"][f]).max() < ssc.SYN_PX_BOUND
        true = d["displaced"][f] - d["material"]
        assert (np.abs(out2ds[f, :, 2:5] - true).max(0) < ssc.SYN_DISP_BOUND).all(), f


def test_gt4_table(engine):
    g = ssc.gt4()
    t, xy = g["table"], g["xy"]
    h, w = g["size"]
    r, stop = ssc.GT4_R, ssc.GT4_STOP
    rig = prepared_rig(engine, w, h, g["intrinsics"], g["extrinsics"])
    stereo = stereo_match(engine, g["r1"], g["r2"], xy, r, t[:, 8:10], stop)
    s1 = ssc.translation_seeds(xy, t[:, 10:12])
    engine.set_stereo_series(g["r1"], g["t1"][None], g["t2"][None])
    _, _, rec = engine.stereo_series(rig, stereo, s1, ssc.recipe_seeds2(s1, stereo), 1, 2, r, r, ssc.CONV, stop)
    rec = rec[0]
    ok = rec[:, 7] >= 0
    assert (~ok).sum() <= ssc.GT4_MAX_CAPPED and (rec[:, 5:7] >= 0).all()
    assert np.abs(rec[:, 8:12] - t[:, 8:12]).max() < ssc.GT4_PX_BOUND
    assert np.abs(rec[ok, 12:14] - t[ok, 12:14]).max() < ssc.GT4_PX_BOUND
    assert np.abs(rec[:, 5:7] - t[:, 5:7]).max() < ssc.GT4_ZNCC_BOUND and np.abs(rec[ok, 7] - t[ok, 7]).max() < ssc.GT4_ZNCC_BOUND
    assert np.abs(rec[:, 14:17] - t[:, 14:17]).max() < ssc.GT4_XYZ_BOUND
    assert np.abs(rec[ok, 17:20] - t[ok, 17:20]).max() < ssc.GT4_XYZ_BOUND and np.abs(rec[ok, 2:5] - t[ok, 2:5]).max() < ssc.GT4_XYZ_BOUND


def test_chunks(engine):
    d, xy, stereo, s1, s2 = _setup(engine, 384, "short", 16)
    rig = prepared_rig(engine, 384, ssc.SYN_H)
    engine.set_stereo_series(d["ref1"], d["tars1"], d["tars2"])
    whole = engine.stereo_series(rig, stereo, s1, s2, 1, 2, 16, 16, ssc.CONV, 10)
    engine.set_stereo_series(d["ref1"], d["tars1"][:2], d["tars2"][:2])
    a = engine.stereo_series(rig, stereo, s1, s2, 1, 2, 16, 16, ssc.CONV, 10)
    engine.set_stereo_series(d["ref1"], d["tars1"][2:], d["tars2"][2:])
    b = engine.stereo_series(rig, stereo, a[0][-1].copy(), a[1][-1].copy(), 1, 2, 16, 16, ssc.CONV, 10)
    for k, name in enumerate(("out1", "out2", "out2ds")):
        assert_same(np.concatenate([a[k], b[k]]), whole[k], "two chunks, " + name)


def test_errors_leave_outputs_untouched():
    eng = ob.Engine(0)
    lib, ctx = eng._lib, eng._ctx
    d, xy = series(384)
    xy = xy[:4]
    n = len(xy)
    rig = prepared_rig(eng, 384, ssc.SYN_H)
    other = ob.Engine(0)
    rig_other = prepared_rig(other, 384, ssc.SYN_H)
    h1, i1, p1, h2, i2, p2 = rig._cameras()
    recs = ob.make_poi2d(xy)
    outs = [np.full((2, n, 25), 7.0, np.float32), np.full((2, n, 25), 7.0, np.float32), np.full((2, n, 28), 7.0, np.float32)]
    vp = lambda a: ctypes.c_void_p(a.ctypes.data) if a is not None else None  # noqa: E731

    def call(o1=1, o2=2, r=8, st=recs, count=n, c1=h1, intr1=i1, out2ds=outs[2]):
        return lib.ocb_stereo_series(ctx, c1, vp(intr1), vp(p1), h2, vp(i2), vp(p2), o1, o2, vp(st), vp(recs), vp(recs), vp(outs[0]),
                                     vp(outs[1]), vp(out2ds), count, r, r, ssc.CONV, 10)

    tars = np.ascontiguousarray(d["tars1"][:2])
    assert call() == _capi.OCB_ERR_STATE
    assert lib.ocb_set_stereo_series_2d(ctx, vp(d["ref1"]), vp(tars), None, 2, 384, ssc.SYN_H) == _capi.OCB_ERR_ARG
    assert lib.ocb_set_stereo_series_2d(ctx, vp(d["ref1"]), vp(tars), vp(tars), 0, 384, ssc.SYN_H) == _capi.OCB_ERR_ARG
    assert call() == _capi.OCB_ERR_STATE
    assert lib.ocb_set_stereo_series_2d(ctx, vp(d["ref1"]), vp(tars), vp(tars), 2, 384, ssc.SYN_H) == _capi.OCB_OK
    assert call(o1=3) == _capi.OCB_ERR_ARG and call(o2=0) == _capi.OCB_ERR_ARG
    assert call(st=None) == _capi.OCB_ERR_ARG and call(out2ds=None) == _capi.OCB_ERR_ARG and call(intr1=None) == _capi.OCB_ERR_ARG
    assert call(c1=None) == _capi.OCB_ERR_ARG
    assert call(c1=rig_other._cameras()[0]) == _capi.OCB_ERR_ARG
    assert "another context" in _capi.last_error(ctx)
    assert call(count=1 << 40) == _capi.OCB_ERR_ARG
    assert call(r=200) == _capi.OCB_ERR_UNSUPPORTED
    assert "exceeds the shared-memory design limit" in _capi.last_error(ctx)
    assert lib.ocb_stereo_series_dev(ctx, h1, vp(i1), vp(p1), h2, vp(i2), vp(p2), 1, 2, None, None, None, None, None, None, 5, 8, 8, ssc.CONV,
                                     10) == _capi.OCB_ERR_ARG
    for o in outs:
        assert (o == 7.0).all()
    assert call() == _capi.OCB_OK
    assert not (outs[2] == 7.0).all()
    del rig, rig_other
    other.close()
    eng.close()


def test_independent_of_pair_and_2d_series_state(engine):
    d, xy, stereo, s1, s2 = _setup(engine, 384, "short", 16)
    rig = prepared_rig(engine, 384, ssc.SYN_H)
    engine.set_stereo_series(d["ref1"], d["tars1"], d["tars2"])
    first = engine.stereo_series(rig, stereo, s1, s2, 1, 2, 16, 16, ssc.CONV, 10)
    # pair state and a 2D series set after the stereo series do not change it ...
    engine.set_images_2d(d["r2"], d["tars2"][-1])
    engine.icgn2d_prepare()
    pair_before = s1.copy()
    engine.icgn2d1(pair_before, 16, 16, ssc.CONV, 10)
    engine.set_series_2d(d["tars1"][-1], d["tars2"][::-1].copy())
    series_before = engine.icgn2d_series(2, s2, 16, 16, ssc.CONV, 10)
    again = engine.stereo_series(rig, stereo, s1, s2, 1, 2, 16, 16, ssc.CONV, 10)
    for k in range(3):
        assert_same(again[k], first[k], "stereo series after pair and 2D series calls")
    # ... and it changes neither of them
    pair_after = s1.copy()
    engine.icgn2d1(pair_after, 16, 16, ssc.CONV, 10)
    assert_same(pair_after, pair_before, "pair call after a stereo series call")
    assert_same(engine.icgn2d_series(2, s2, 16, 16, ssc.CONV, 10), series_before, "2D series after a stereo series call")


def test_dev_variants_match_host(engine):
    torch = pytest.importorskip("torch")
    d, xy, stereo, s1, s2 = _setup(engine, 384, "short", 16)
    rig = prepared_rig(engine, 384, ssc.SYN_H)
    engine.set_stereo_series(d["ref1"], d["tars1"], d["tars2"])
    host = engine.stereo_series(rig, stereo, s1, s2, 1, 2, 16, 16, ssc.CONV, 10)
    F, n = ssc.SYN_F, len(xy)
    dev = [torch.from_numpy(a).cuda() for a in (d["ref1"], d["tars1"], d["tars2"], stereo, s1, s2)]
    outs = [torch.empty((F, n, k), dtype=torch.float32, device="cuda") for k in (25, 25, 28)]
    torch.cuda.synchronize()
    engine.set_stereo_series_dev(dev[0].data_ptr(), dev[1].data_ptr(), dev[2].data_ptr(), F, 384, ssc.SYN_H)
    engine.stereo_series_dev(rig, dev[3].data_ptr(), dev[4].data_ptr(), dev[5].data_ptr(), *(o.data_ptr() for o in outs), n, 1, 2, 16, 16,
                             ssc.CONV, 10)
    engine.sync()
    for k in range(3):
        assert_same(outs[k].cpu().numpy(), host[k], "device-pointer variant %d" % k)
    assert_same(dev[4].cpu().numpy(), s1, "seeds untouched")


def test_group_context():
    if _capi.load().ocb_device_count() < 2:
        pytest.skip("needs two GPUs")
    single = ob.Engine(0)
    d, xy, stereo, s1, s2 = _setup(single, 384, "short", 16)
    rig = prepared_rig(single, 384, ssc.SYN_H)
    single.set_stereo_series(d["ref1"], d["tars1"], d["tars2"])
    expect = single.stereo_series(rig, stereo, s1, s2, 1, 2, 16, 16, ssc.CONV, 10)
    group = ob.Engine([0, 1])
    grig = prepared_rig(group, 384, ssc.SYN_H)
    group.set_stereo_series(d["ref1"], d["tars1"], d["tars2"])
    got = group.stereo_series(grig, stereo, s1, s2, 1, 2, 16, 16, ssc.CONV, 10)
    for k in range(3):
        assert_same(got[k], expect[k], "group context %d" % k)
    del grig, rig
    group.close()
    single.close()
