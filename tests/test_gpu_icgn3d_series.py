"""ICGN3D1 over a volume series (ocb_icgn3d_series): every frame's records must be, bit for bit, what the loop of pair calls
    set_images_3d(ref, tars[f]); icgn3d_prepare(); icgn3d1(q, ...)
gives when one queue q is carried from frame to frame.  The series builds the reference's gradients and each POI's setup pass
once per call (ICGN3D_SETUP_STORE) and restores the setup state in every frame (ICGN3D_SETUP_LOAD)."""
import ctypes

import numpy as np
import pytest

import opencorr_b200 as ob
from opencorr_b200 import _capi, synth
from oracle.oracle import Oracle3D
import util

pytestmark = pytest.mark.gpu

CONV, STOP = 0.001, 20
DX, DY, DZ = 103, 100, 98  # dim_x % 4 != 0; room for a 61^3 subvolume plus the synthetic displacement
FRAMES = 4


@pytest.fixture(scope="module")
def series():
    return synth.speckle_series_3d(DX, DY, DZ, FRAMES)


def _pois(r, n, seed):
    """n integer POIs whose subvolume stays inside the volume in every frame (v < 0 near y = 0, w < 2.5)."""
    rng = np.random.default_rng(seed)
    r = np.array(r)
    lo, hi = r + 3, np.array([DX, DY, DZ]) - 1 - r - 4
    return rng.integers(lo, hi + 1, size=(n, 3)).astype(np.float32)


def fftcc_seeds(eng, ref, tar, xyz, r):
    q = ob.make_poi3d(xyz)
    eng.set_images_3d(ref, tar)
    eng.fftcc3d(q, *r)
    return q


def pair_loop(eng, ref, tars, seeds, r, stop=STOP):
    q = seeds.copy()
    out = []
    for f in range(len(tars)):
        eng.set_images_3d(ref, tars[f])
        eng.icgn3d_prepare()
        eng.icgn3d1(q, *r, CONV, stop)
        out.append(q.copy())
    return np.stack(out)


def assert_same(a, b, label):
    assert a.shape == b.shape, label
    bad = a.view(np.uint32) != b.view(np.uint32)
    assert not bad.any(), "%s: %d floats differ, first at %s" % (label, bad.sum(), np.argwhere(bad)[:5].tolist())


# radii, POIs; the launch plan each selects (ocb::icgn3d1_plan) in the comment
CASES = [
    ((8, 8, 8), 24),    # <0,256>, one slab
    ((8, 8, 8), 300),   # <0,256>: more POIs than the 2 x 132 resident CTAs
    ((16, 16, 16), 16), # <16,256>, 3 slabs, one tail column
    ((10, 6, 9), 20),   # <0,256>, non-cubic
    ((24, 24, 24), 6),  # <0,512>, 17 tail columns
    ((30, 30, 30), 3),  # <30,512>
]


@pytest.mark.parametrize("tma", [True, False], ids=["tma", "no_tma"])
@pytest.mark.parametrize("r,n", CASES, ids=["r=(%d,%d,%d) n=%d" % (r + (n,)) for r, n in CASES])
def test_series_equals_pair_loop(engine, series, monkeypatch, r, n, tma):
    if not tma:
        monkeypatch.setenv("OCB_NO_TMA", "1")
    ref, tars = series
    seeds = fftcc_seeds(engine, ref, tars[0], _pois(r, n, seed=sum(r) + n), r)
    for n_frames in (1, FRAMES):
        expect = pair_loop(engine, ref, tars[:n_frames], seeds, r)
        engine.set_series_3d(ref, tars[:n_frames])
        before = seeds.copy()
        got = engine.icgn3d_series(seeds, *r, CONV, STOP)
        assert_same(seeds, before, "seeds changed")
        assert_same(got, expect, "r=%s n=%d F=%d" % (r, n, n_frames))
        assert (got[-1][:, 18] >= 0).mean() > 0.8


def test_series_matches_oracle_and_ground_truth(engine, series):
    ref, tars = series
    r = (16, 16, 16)
    xyz = _pois(r, 12, seed=7)
    seeds = fftcc_seeds(engine, ref, tars[0], xyz, r)
    engine.set_series_3d(ref, tars)
    got = engine.icgn3d_series(seeds, *r, CONV, STOP)
    n = len(xyz)
    for f in range(FRAMES):
        q = (seeds if f == 0 else got[f - 1]).copy()  # each frame from the same seeds as the GPU's
        Oracle3D(ref, tars[f]).icgn3d1(q, *r, CONV, STOP, exact=True)
        stats = util.compare_3d(got[f], q, "frame %d" % f, max_iter_mismatch_frac=max(1.0, 0.02 * n) / n)
        print("frame %d: %s" % (f, stats))
    last = got[-1]
    ok = last[:, 18] >= 0
    assert ok.mean() > 0.9
    u, v, w = synth.displacement_3d(xyz[:, 0], xyz[:, 1], xyz[:, 2], DX, DY, DZ)
    for col, truth in ((3, u), (7, v), (11, w)):
        assert np.abs(last[ok, col] - truth[ok]).max() < 0.05


def test_series_sentinels(engine, series):
    """POIs that leave the volume mid-series, stop at the iteration limit (-4), are refused by the guard or arrive with a
    negative or NaN ZNCC keep their code and that frame's record in every later frame, exactly as the pair loop does."""
    ref, tars = series
    r = (12, 12, 12)
    # rows 9 ... 15: subvolumes 0 ... 6 layers below the top of the volume, whose top layers leave it as w grows by about 0.6
    # voxel per frame
    top = [[40 + 3 * k, 50, DZ - 1 - 12 - k] for k in range(7)]
    xyz = np.array([[40, 40, 40], [60, 50, 45], [50, 50, 50], [45, 55, 52], [55, 45, 50], [40, 60, 55], [50, 40, 60], [45, 45, 42],
                    [58, 58, 48]] + top, np.float32)
    seeds = fftcc_seeds(engine, ref, tars[0], xyz, r)
    seeds[4, 3] = DX + 5.0  # |u| >= dim_x: the guard rejects it
    seeds[5, 18] = -1.0     # arrives negative
    seeds[6, 3] = np.nan    # NaN guess
    seeds[7, 18] = np.nan   # NaN ZNCC with coordinates outside the volume: the guard keeps the NaN
    seeds[7, 0] = -5.0
    seeds[8, 3] += 3.5      # far from the optimum: runs into the iteration limit at stop = 2
    for stop in (STOP, 2):
        expect = pair_loop(engine, ref, tars, seeds, r, stop)
        engine.set_series_3d(ref, tars)
        got = engine.icgn3d_series(seeds, *r, CONV, stop)
        assert_same(got, expect, "stop %g" % stop)
        codes = got[:, :, 18]
        assert (codes[:, 4] == -3).all() and (codes[:, 5] == -1).all() and (codes[:, 6] == -3).all()
        assert np.isnan(codes[:, 7]).all() and (got[:, 7, 0] == -5.0).all()
        if stop == 2:
            assert (codes == -4).any()
        else:
            first_fail = [np.nonzero(codes[:, i] < 0)[0] for i in range(9, 16)]
            assert any(len(ff) and 0 < ff[0] < FRAMES for ff in first_fail), "no POI left the volume mid-series: %s" % codes[:, 9:16].T
        for i in range(len(xyz)):
            neg = np.nonzero(~(codes[:, i] >= 0))[0]
            if len(neg):
                f0 = neg[0]
                for f in range(f0 + 1, FRAMES):
                    assert_same(got[f, i], got[f0, i], "POI %d frame %d" % (i, f))


def test_series_chunks_u8_and_device_pointers(engine, series):
    ref, tars = series
    r = (16, 16, 16)
    seeds = fftcc_seeds(engine, ref, tars[0], _pois(r, 16, seed=3), r)
    engine.set_series_3d(ref, tars)
    whole = engine.icgn3d_series(seeds, *r, CONV, STOP)
    engine.set_series_3d(ref, tars[:2])
    a = engine.icgn3d_series(seeds, *r, CONV, STOP)
    engine.set_series_3d(ref, tars[2:])
    b = engine.icgn3d_series(a[-1].copy(), *r, CONV, STOP)
    assert_same(np.concatenate([a, b]), whole, "two chunks")

    assert np.array_equal(ref, np.round(ref)) and ref.max() <= 255  # synth volumes are 8-bit valued
    engine.set_series_3d(ref.astype(np.uint8), tars.astype(np.uint8))
    assert_same(engine.icgn3d_series(seeds, *r, CONV, STOP), whole, "8-bit stack")

    torch = pytest.importorskip("torch")
    d_ref, d_tars, d_seeds = (torch.from_numpy(x).cuda() for x in (ref, tars, seeds))
    d_out = torch.empty((FRAMES, len(seeds), ob.POI3D_FLOATS), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    engine.set_series_3d_dev(d_ref.data_ptr(), d_tars.data_ptr(), FRAMES, DX, DY, DZ)
    engine.icgn3d_series_dev(d_seeds.data_ptr(), d_out.data_ptr(), len(seeds), *r, CONV, STOP)
    engine.sync()
    assert_same(d_out.cpu().numpy(), whole, "device-pointer variant")
    assert_same(d_seeds.cpu().numpy(), seeds, "device seeds changed")


def test_series_errors_leave_out_untouched():
    eng = ob.Engine(0)
    lib, ctx = eng._lib, eng._ctx
    ref, tars = synth.speckle_series_3d(40, 36, 32, 2)
    seeds = ob.make_poi3d(synth.grid_3d(18, 16, 14, 2, 2, 2, 4, 4, 4))
    n = len(seeds)
    out = np.full((2, n, ob.POI3D_FLOATS), 7.0, np.float32)
    vp = lambda a: ctypes.c_void_p(a.ctypes.data)

    def call(r=(6, 6, 6), s=seeds, o=out, count=n):
        return lib.ocb_icgn3d_series(ctx, vp(s) if s is not None else None, vp(o) if o is not None else None, count, *r, CONV, STOP)

    assert call() == _capi.OCB_ERR_STATE
    assert lib.ocb_set_series_3d(ctx, vp(ref), vp(tars), 0, 40, 36, 32) == _capi.OCB_ERR_ARG
    assert lib.ocb_set_series_3d(ctx, vp(ref), None, 2, 40, 36, 32) == _capi.OCB_ERR_ARG
    assert lib.ocb_set_series_3d(ctx, vp(ref), vp(tars), 2, 40, 36, 14) == _capi.OCB_ERR_ARG
    assert lib.ocb_set_series_3d(ctx, vp(ref), vp(tars), 2, 1 << 30, 1 << 30, 1 << 30) == _capi.OCB_ERR_ARG  # size overflow
    assert lib.ocb_set_series_3d_u8(ctx, vp(ref), vp(tars), 1 << 30, 1 << 30, 1 << 30, 1 << 30) == _capi.OCB_ERR_ARG
    assert lib.ocb_set_series_3d_dev(ctx, None, None, 2, 40, 36, 32) == _capi.OCB_ERR_ARG
    assert call() == _capi.OCB_ERR_STATE  # the refused calls set nothing
    assert lib.ocb_set_series_3d(ctx, vp(ref), vp(tars), 2, 40, 36, 32) == _capi.OCB_OK
    assert call(s=None) == _capi.OCB_ERR_ARG
    assert call(o=None) == _capi.OCB_ERR_ARG
    assert call(r=(0, 6, 6)) == _capi.OCB_ERR_ARG
    assert call(count=1 << 40) == _capi.OCB_ERR_ARG
    assert call(r=(44, 44, 44)) == _capi.OCB_ERR_UNSUPPORTED
    assert "exceeds the shared-memory design limit" in _capi.last_error(ctx)
    assert lib.ocb_icgn3d_series_dev(ctx, None, None, 5, 6, 6, 6, CONV, STOP) == _capi.OCB_ERR_ARG
    assert (out == 7.0).all()
    assert call() == _capi.OCB_OK
    assert not (out == 7.0).all()
    eng.close()


def test_pair_calls_unaffected_by_series(engine, series):
    ref, tars = series
    r = (16, 16, 16)
    seeds = fftcc_seeds(engine, ref, tars[-1], _pois(r, 16, seed=5), r)
    engine.icgn3d_prepare()
    before = seeds.copy()
    engine.icgn3d1(before, *r, CONV, STOP)
    engine.set_series_3d(ref[:, ::-1].copy(), tars[:, :, ::-1].copy())
    engine.icgn3d_series(seeds, *r, CONV, STOP)
    after = seeds.copy()
    engine.icgn3d1(after, *r, CONV, STOP)  # the pair (ref, tars[-1]) is still set and prepared
    assert_same(after, before, "pair call after a series call")


def test_series_group(series):
    if _capi.load().ocb_device_count() < 2:
        pytest.skip("needs two GPUs")
    ref, tars = series
    r = (16, 16, 16)
    single = ob.Engine(0)
    seeds = fftcc_seeds(single, ref, tars[0], _pois(r, 16, seed=3), r)
    single.set_series_3d(ref, tars)
    expect = single.icgn3d_series(seeds, *r, CONV, STOP)
    group = ob.Engine([0, 1])
    group.set_series_3d(ref, tars)
    assert_same(group.icgn3d_series(seeds, *r, CONV, STOP), expect, "group context")
    group.close()
    single.close()
