"""GPU: Strain over a series (ocb_strain2d_series, ocb_strain3d_series, ocb_strain2ds_series and their _dev variants).  Frame f's
records after the call must be, bit for bit, what the pair call leaves on frame f alone, for every case of tests/strain_cases.py,
every approximation and every radius, with displacements, ZNCC flags and (POI2DS) ref_coor varying from frame to frame on the
same positions; lists longer than the series kernel keeps (STRAIN_LIST = 32 indices per lane, 1024 per warp) as well.  A frame
whose positions differ from frame 0's is refused and nothing is written."""
import ctypes

import numpy as np
import pytest

import opencorr_b200 as ob
from opencorr_b200 import _capi, synth
import strain_cases as sc

pytestmark = pytest.mark.gpu

TOL = {25: 2e-6, 31: 2e-6, 28: 1e-5}  # test_gpu_strain_geometry.py
CASES = {c.name: c for c in sc.small_cases()}
KIND = {25: 2, 31: 3, 28: 23}
DEV_KIND = {25: "2d", 31: "3d", 28: "2ds"}
LIST_WARP = 32 * 32  # the series kernel's list capacity per warp (strain.cu STRAIN_LIST x 32 lanes)


def frames(q, n_frames, seed=0):
    """Frame 0 = q; frame f > 0 = q with displacements, ZNCCs and (POI2DS) ref_coor drawn again from seed + f."""
    out = [q.copy()]
    for f in range(1, n_frames):
        out.append(sc.fill(q.copy(), np.random.default_rng(seed + 1000 * f)))
    return np.stack(out)


def pair_loop(engine, qs, radius, k_min, thr, approximation):
    out = qs.copy()
    for f in range(len(qs)):
        engine.strain(out[f], radius, k_min, thr, approximation)
    return out


def series(engine, qs, radius, k_min, thr, approximation):
    out = qs.copy()
    engine.strain_series(out, radius, k_min, thr, approximation)
    return out


def assert_same(a, b, label):
    assert a.shape == b.shape, label
    bad = sc.bits(a) != sc.bits(b)
    assert not bad.any(), "%s: %d floats differ, first at %s" % (label, bad.sum(), np.argwhere(bad)[:5].tolist())


def check_loop(engine, qs, radius, k_min, thr, label, approximations=(0, 1, 2)):
    for a in approximations:
        assert_same(series(engine, qs, radius, k_min, thr, a), pair_loop(engine, qs, radius, k_min, thr, a), "%s approx=%d" % (label, a))


def dev_series(engine, d, qs, radius, k_min, thr, approximation):
    engine.strain_series_dev(DEV_KIND[qs.shape[2]], d.data_ptr(), qs.shape[0], qs.shape[1], radius, k_min, thr, approximation)


# ------------------------------------------------------------------------------------------------ equality with the loop
@pytest.mark.parametrize("n_frames", [1, 3])
@pytest.mark.parametrize("name", sorted(CASES))
def test_equals_loop_of_pair_calls(engine, name, n_frames):
    """Every case of strain_cases (all three kinds, every radius edge: +-inf, 0, NaN, negative, 1e-30, 1e20; non-finite positions,
    the same in every frame; k-nearest ties), approximations 0, 1 and 2."""
    c = CASES[name]
    check_loop(engine, frames(c.q, n_frames, seed=len(name)), c.radius, c.k_min, c.thr, name)


@pytest.mark.parametrize("name", ["nonfinite_2", "nonfinite_3", "nonfinite_23", "radius_2_inf", "radius_3_nan", "radius_23_-20",
                                  "lattice2s_k10", "fallback_low_zncc_3"])
def test_device_pointer_entry_points(engine, name):
    torch = pytest.importorskip("torch")
    c = CASES[name]
    qs = frames(c.q, 3, seed=7)
    for a in (1, 2):
        expect = pair_loop(engine, qs, c.radius, c.k_min, c.thr, a)
        d = torch.from_numpy(qs.copy()).cuda()
        torch.cuda.synchronize()
        dev_series(engine, d, qs, c.radius, c.k_min, c.thr, a)
        engine.sync()
        assert_same(d.cpu().numpy(), expect, "%s approx=%d" % (name, a))


def test_flags_per_frame(engine):
    """A POI below the threshold in frame 1 only is skipped in frame 1 only, and left out of its neighbours' fits there only."""
    for kind in (2, 3, 23):
        c = sc.uniform(kind, 600, 120 if kind != 3 else 40, 15.0 if kind != 3 else 10.0, seed=5, bad=0.0)
        qs = frames(c.q, 3, seed=11)
        z = sc.layout(c.q)["zncc"]
        qs[:, :, list(z)] = 0.95
        qs[1, ::7, z[0]] = 0.5
        got = series(engine, qs, c.radius, c.k_min, c.thr, 1)
        assert_same(got, pair_loop(engine, qs, c.radius, c.k_min, c.thr, 1), "kind %d" % kind)
        sl = sc.layout(c.q)["strain"]
        assert (sc.bits(got[1, ::7, sl]) == sc.bits(qs[1, ::7, sl])).all(), kind  # skipped in frame 1
        assert (sc.bits(got[[0, 2]][:, ::7, sl]) != sc.bits(qs[[0, 2]][:, ::7, sl])).any(-1).all(), kind  # fitted in frames 0 and 2


# ------------------------------------------------------------------------------------------------ list capacity
def _one_run(kind, n, seed):
    """n POIs in a small box: with an infinite radius every POI lies in one cell run, so lane 0 of every warp meets ceil(n / 32)
    neighbours; with a NaN radius every POI takes the k-nearest path."""
    rng = np.random.default_rng(seed)
    D = 3 if kind == 3 else 2
    return sc.queue(kind, rng.uniform(0, 50, (n, D)), rng)


@pytest.mark.parametrize("kind", [2, 3, 23])
def test_radius_lists_at_and_past_capacity(engine, kind):
    for n, label in ((LIST_WARP, "met"), (LIST_WARP + 1, "exceeded")):
        qs = frames(_one_run(kind, n, 3), 3, seed=13)
        for r in (np.inf, -np.inf):
            check_loop(engine, qs, r, 5, 0.9, "kind %d %s r %g" % (kind, label, r), (1, 2))


@pytest.mark.parametrize("kind", [2, 3, 23])
def test_nearest_lists_at_and_past_capacity(engine, kind):
    qs = frames(_one_run(kind, LIST_WARP + 40, 4), 2, seed=17)
    for k, label in ((LIST_WARP, "met"), (LIST_WARP + 1, "exceeded")):
        check_loop(engine, qs, np.nan, k, 0.9, "kind %d %s" % (kind, label), (1,))
        check_loop(engine, qs, 0.0, k, 0.9, "kind %d %s r 0" % (kind, label), (2,))


# ------------------------------------------------------------------------------------------------ size and witness
def _sm_count():
    torch = pytest.importorskip("torch")
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("kind", [2, 3, 23])
def test_queue_longer_than_the_resident_warps_8_frames(engine, kind):
    n = 64 * _sm_count() + 777
    if kind == 3:
        c = sc.uniform(3, n, (n * 4 / 3 * np.pi * 1000 / 10.0) ** (1 / 3), 10.0, seed=22)
    else:
        c = sc.uniform(kind, n, np.sqrt(n * np.pi * 400 / 10.0), 20.0, seed=21)
    c.q[[0, -1], 0] = np.nan
    check_loop(engine, frames(c.q, 8, seed=3), c.radius, c.k_min, c.thr, "kind %d" % kind, (1, 2))


@pytest.mark.parametrize("name", ["cell_boundary_2_r7.5", "fallback_low_zncc_3", "box_pm300_23"])
def test_every_frame_against_the_witness(engine, name):
    c = CASES[name]
    qs = frames(c.q, 3, seed=5)
    got = series(engine, qs, c.radius, c.k_min, c.thr, 2)
    for f in range(len(qs)):
        sc.compare(got[f], qs[f], sc.witness(qs[f], c.radius, c.k_min, c.thr, 2), TOL[c.q.shape[1]], "%s frame %d" % (name, f))


# ------------------------------------------------------------------------------------------------ errors and launches
def _call(engine, kind, ptr, n_frames, n, dev=False):
    fn = getattr(engine._lib, "ocb_strain%s_series%s" % (kind, "_dev" if dev else ""))
    return fn(engine._ctx, ptr, n_frames, n, 15.0, 5, 0.9, 1)


@pytest.mark.parametrize("name", ["box_pm300_2", "box_pm300_3", "box_pm300_23"])
def test_positions_that_move_are_refused(engine, name):
    torch = pytest.importorskip("torch")
    c = CASES[name]
    kind = DEV_KIND[c.q.shape[1]]
    base = frames(c.q, 4, seed=9)
    flipped = base.copy()
    flipped[2, 17, 0] = np.frombuffer((sc.bits(flipped[2, 17, :1]) ^ np.uint32(1)).tobytes(), np.float32)[0]
    nan_y = base.copy()
    nan_y[1, 40, 1] = np.nan
    for label, qs in (("flipped x bit", flipped), ("NaN y", nan_y)):
        host = qs.copy()
        assert _call(engine, kind, ctypes.c_void_p(host.ctypes.data), 4, len(c.q)) == _capi.OCB_ERR_ARG, label
        assert_same(host, qs, label + " host")
        d = torch.from_numpy(qs.copy()).cuda()
        torch.cuda.synchronize()
        assert _call(engine, kind, ctypes.c_void_p(d.data_ptr()), 4, len(c.q), dev=True) == _capi.OCB_ERR_ARG, label
        engine.sync()
        assert_same(d.cpu().numpy(), qs, label + " dev")
    # NaN in the same place in every frame is a position like any other
    same_nan = base.copy()
    same_nan[:, 40, 1] = np.nan
    check_loop(engine, same_nan, c.radius, c.k_min, c.thr, name + " same NaN", (1,))


def test_bad_arguments_are_refused(engine):
    q = np.zeros((2, 4, 25), np.float32)
    for dev in (False, True):
        assert _call(engine, "2d", None, 2, 4, dev) == _capi.OCB_ERR_ARG
        assert _call(engine, "3d", None, 1, 1, dev) == _capi.OCB_ERR_ARG
        for n_frames, n in ((1 << 62, 4), (2, 1 << 62), ((1 << 64) // 100 + 1, 1)):
            assert _call(engine, "2d", ctypes.c_void_p(q.ctypes.data), n_frames, n, dev) == _capi.OCB_ERR_ARG, (n_frames, n, dev)
        assert _call(engine, "2ds", None, 0, 4, dev) == _capi.OCB_OK  # nothing to do
        assert _call(engine, "2ds", None, 3, 0, dev) == _capi.OCB_OK
    with pytest.raises(ValueError):
        engine.strain_series(q[0], 15.0, 5)


def test_launches_do_not_depend_on_the_frame_count(engine):
    c = CASES["box_pm300_2"]
    counts = []
    for n_frames in (1, 8):
        qs = frames(c.q, n_frames)
        before = engine.launch_count()
        engine.strain_series(qs, c.radius, c.k_min, c.thr, 1)
        counts.append(engine.launch_count() - before)
    assert counts[0] == counts[1] > 0, counts


# ------------------------------------------------------------------------------------------------ after the series calls
def test_after_icgn2d_series(engine):
    import subset_series_cases as ssc
    ref, tars = ssc.render_series(384, 320, 5)
    xy = synth.grid_2d(30, 30, 36, 29, 9, 9)
    seeds = ssc.fftcc_seeds(engine, ref, tars[0], xy, 16)
    engine.set_series_2d(ref, tars)
    out = engine.icgn2d_series(1, seeds, 16, 16, ssc.CONV, ssc.STOP)
    out[..., 20:23] = sc.SENTINEL
    assert (out[..., 16] >= 0.9).mean() > 0.5
    check_loop(engine, out, 20.0, 5, 0.9, "icgn2d_series", (1, 2))


def test_after_icgn3d_series(engine):
    DX, DY, DZ = 103, 100, 98
    ref, tars = synth.speckle_series_3d(DX, DY, DZ, 4)
    rng = np.random.default_rng(3)
    xyz = rng.integers(12, np.array([DX, DY, DZ]) - 16, size=(300, 3)).astype(np.float32)
    q = ob.make_poi3d(xyz)
    engine.set_images_3d(ref, tars[0])
    engine.fftcc3d(q, 8, 8, 8)
    engine.set_series_3d(ref, tars)
    out = engine.icgn3d_series(q, 8, 8, 8, 0.001, 20)
    out[..., 22:28] = sc.SENTINEL
    assert (out[..., 18] >= 0.9).mean() > 0.5
    check_loop(engine, out, 20.0, 5, 0.9, "icgn3d_series", (1, 2))


def test_after_stereo_series(engine):
    import stereo_cases as stc
    import stereo_series_cases as sts
    w, h = 384, sts.SYN_H
    xy = synth.grid_2d(20, 20, 114, 70, 3, 4)
    d = synth.speckle_stereo_series(w, h, sts.SYN_F, points=synth.grid_2d(40, 40, 13, 11, 25, 22))
    stereo = ob.make_poi2d(xy)
    engine.set_images_2d(d["ref1"], d["r2"])
    engine.fftcc2d(stereo, 16, 16)
    engine.icgn2d_prepare()
    engine.icgn2d2(stereo, 16, 16, sts.CONV, 10)
    s1 = ob.make_poi2d(xy)
    engine.set_images_2d(d["ref1"], d["tars1"][0])
    engine.fftcc2d(s1, 16, 16)
    intrinsics, extrinsics = synth.stereo_rig(w, h)
    c1, c2 = stc.camera(intrinsics[0], extrinsics[0], engine), stc.camera(intrinsics[1], extrinsics[1], engine)
    c1.prepare(h, w)
    c2.prepare(h, w)
    rig = ob.Stereovision(c1, c2, 0, engine)
    rig.prepare()
    engine.set_stereo_series(d["ref1"], d["tars1"], d["tars2"])
    _, _, out2ds = engine.stereo_series(rig, stereo, s1, sts.recipe_seeds2(s1, stereo), 1, 2, 16, 16, sts.CONV, 10)
    good = (out2ds[..., 5:8] >= 0.9).all(-1).mean()
    assert good > 0.5, good
    check_loop(engine, out2ds, 20.0, 5, 0.9, "stereo_series", (1, 2))


def test_group_context(engine):
    n_dev = _capi.load().ocb_device_count()
    grp = ob.Engine(list(range(n_dev)))
    try:
        for name in ("growth_2d_xy", "cell_boundary_3_r20", "nonfinite_23"):
            c = CASES[name]
            qs = frames(c.q, 3, seed=2)
            assert_same(series(grp, qs, c.radius, c.k_min, c.thr, 2), series(engine, qs, c.radius, c.k_min, c.thr, 2), name)
    finally:
        grp.close()
