"""IC-GN over an image series with recovery of unreliable POIs (ocb_icgn2d_series_recover): out, recovered and remaining must be,
byte for byte, what the loop of existing calls
    set_images_2d(ref, tars[f]); icgn2d_prepare(); icgn2d<order>_dev(q); icgn2d_recover_dev(q)
gives when one queue q is carried from frame to frame (series_recover_cases.dev_loop)."""
import ctypes

import numpy as np
import pytest

import opencorr_b200 as ob
from opencorr_b200 import _capi, synth
import series_recover_cases as src
import subset_series_cases as sc
from util import assert_same

pytestmark = pytest.mark.gpu
P = src.Params()


@pytest.fixture(scope="module")
def occluded():
    return src.occluded_series()


@pytest.fixture(scope="module")
def occluded2():
    return src.occluded_series(second_order=True)


def _grid(kind, r):
    return sc.short_grid() if kind == "short" else sc.long_grid(r)


def _seeds(eng, ref, tars, xy, r):
    """FFT-CC seeds with a garbage-seeded block"""
    return src.garbage(sc.fftcc_seeds(eng, ref, tars[0], xy, r), src.in_region(xy, (250, 80, 300, 130)))


def _call(eng, order, seeds, r, p=P, dev=False):
    """the series recovery call, host or device pointers: (out, recovered, remaining)"""
    if not dev:
        return eng.icgn2d_series_recover(order, seeds, r, r, *p.recover_args())
    import torch
    d_seeds = torch.from_numpy(seeds).cuda()
    d_out = torch.full((eng._frames["2d"], len(seeds), 25), 7.0, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    rec, left = eng.icgn2d_series_recover_dev(order, d_seeds.data_ptr(), d_out.data_ptr(), len(seeds), r, r, *p.recover_args())
    assert_same(d_seeds.cpu().numpy(), seeds, "device seeds changed")
    return d_out.cpu().numpy(), rec, left


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
@pytest.mark.parametrize("tma", [True, False], ids=["tma", "no_tma"])
@pytest.mark.parametrize("kind", ["short", "long"])
@pytest.mark.parametrize("order,r", [(1, 12), (1, 16), (2, 12), (2, 16)])
def test_equals_the_loop(engine, occluded, occluded2, monkeypatch, order, r, kind, tma, dev):
    if not tma:
        monkeypatch.setenv("OCB_NO_TMA", "1")
    ref, _, tars = occluded if order == 1 else occluded2
    xy = _grid(kind, r)
    seeds = _seeds(engine, ref, tars, xy, r)
    for n_frames in (1, len(tars)):
        expect = src.dev_loop(engine, 2, order, ref, tars[:n_frames], seeds, r, P)
        engine.set_series_2d(ref, tars[:n_frames])
        got = _call(engine, order, seeds, r, dev=dev)
        label = "order %d r %d %s F %d" % (order, r, kind, n_frames)
        assert_same(got[0], expect[0], label)
        assert np.array_equal(got[1], expect[1]) and np.array_equal(got[2], expect[2]), (label, got[1:], expect[1:])
        assert got[1].shape == (n_frames, P.max_rounds) and got[2].shape == (n_frames,)
        assert got[1][0].sum() > 0, "the garbage-seeded block is recovered in frame 0"


def test_occlusion_recovered_in_the_next_frame(engine, occluded):
    """The plain series loses the POIs whose subsets frame K covers for good; the call gets them back in frame K + 1, where they
    match the clean series."""
    ref, clean, tars = occluded
    xy = synth.grid_2d(40, 40, 14, 11, 24, 24)
    block = src.in_region(xy, src.BLOCK)
    p = src.Params(zncc_low=0.9, radius=40.0)
    seeds = sc.fftcc_seeds(engine, ref, tars[0], xy, 16)
    engine.set_series_2d(ref, tars)
    plain = sc.Method("icgn", 1).series(engine, seeds, 16)
    k = src.K
    assert (~(plain[k:, block, 16] >= 0.9)).all(), "control: the plain series loses the block from frame K on"
    got, rec, left = engine.icgn2d_series_recover(1, seeds, 16, 16, *p.recover_args())
    expect = src.dev_loop(engine, 2, 1, ref, tars, seeds, 16, p)
    assert_same(got, expect[0], "occlusion")
    assert np.array_equal(rec, expect[1]) and np.array_equal(left, expect[2])
    assert left[k] >= block.sum() and rec[k + 1].sum() >= block.sum(), (rec, left)
    engine.set_series_2d(ref, clean)
    reference = sc.Method("icgn", 1).series(engine, seeds, 16)
    for f in range(k + 1, len(tars)):
        assert (got[f][block, 16] >= 0.9).all(), "frame %d" % f
        for col in (2, 8):  # the clean series' optimum, reached from the neighbours' fit
            assert np.abs(got[f][block, col] - reference[f][block, col]).max() < 0.01


def test_dead_region_never_recovered(engine, occluded):
    """A region of zero pixels in every frame, covering the subsets of a block of POIs and no other POI's subset: the block's
    POIs take one round per frame, recover none, and stay unreliable."""
    ref, clean, _ = occluded
    xy = synth.grid_2d(40, 40, 7, 6, 48, 48)  # 48 px apart: 15 px between neighbouring r = 16 subsets
    block = src.in_region(xy, src.BLOCK)
    region = tuple(xy[block].min(0)) + tuple(xy[block].max(0) + 1)
    boxes = np.array([src.occlusion_box(region, f, src.FRAMES, 16, margin=3) for f in range(src.FRAMES)])
    x0, y0 = boxes[:, :2].min(0)
    x1, y1 = boxes[:, 2:].max(0)
    tars = clean.copy()
    tars[:, y0:y1, x0:x1] = 0
    seeds = sc.fftcc_seeds(engine, ref, clean[0], xy, 16)
    engine.set_series_2d(ref, tars)
    got, rec, left = engine.icgn2d_series_recover(1, seeds, 16, 16, *P.recover_args())
    expect = src.dev_loop(engine, 2, 1, ref, tars, seeds, 16, P)
    assert_same(got, expect[0], "dead region")
    assert np.array_equal(rec, expect[1]) and np.array_equal(left, expect[2])
    assert block.sum() == 4 and (rec == 0).all(), rec
    assert (left == block.sum()).all(), left


@pytest.mark.parametrize("order", [1, 2])
def test_no_rounds_or_nothing_unreliable_is_the_plain_series(engine, occluded, occluded2, order):
    ref, _, tars = occluded if order == 1 else occluded2
    seeds = _seeds(engine, ref, tars, sc.long_grid(16), 16)
    seeds[::7, 16] = -1.0  # failed seeds
    engine.set_series_2d(ref, tars)
    plain = sc.Method("icgn", order).series(engine, seeds, 16)
    got, rec, left = engine.icgn2d_series_recover(order, seeds, 16, 16, *src.Params(max_rounds=0).recover_args())
    assert_same(got, plain, "max_rounds 0")
    assert rec.shape == (len(tars), 0) and (left > 0).all()
    p = src.Params(zncc_low=-10.0, conv=1e30)  # below every code; conv is also IC-GN's convergence criterion
    got, rec, left = engine.icgn2d_series_recover(order, seeds, 16, 16, *p.recover_args())
    assert_same(got, engine.icgn2d_series(order, seeds, 16, 16, p.conv, p.stop), "nothing unreliable")
    assert (rec == 0).all() and (left == 0).all()


def test_launches_do_not_depend_on_n(engine, occluded):
    """Launches per call depend on the frames and rounds, not on the number of POIs."""
    ref, clean, _ = occluded
    engine.set_series_2d(ref, clean)
    counts = []
    for xy in (sc.short_grid(), synth.grid_2d(60, 55, 24, 20, 12, 10)):  # 30 and 480 POIs inside the same area
        seeds = sc.fftcc_seeds(engine, ref, clean[0], xy, 16)
        seeds[0, 2] += 23.0  # one garbage seed, recovered in frame 0's first round
        engine.set_series_2d(ref, clean)
        before = engine.launch_count()
        _, rec, left = engine.icgn2d_series_recover(1, seeds, 16, 16, *P.recover_args())
        counts.append((engine.launch_count() - before, rec.tolist(), left.tolist()))
    assert counts[0][1] == counts[1][1] and counts[0][0] == counts[1][0], counts


def test_pair_state_untouched(engine, occluded):
    ref, _, tars = occluded
    seeds = sc.fftcc_seeds(engine, ref, tars[-1], sc.short_grid(), 16)
    before = seeds.copy()
    engine.icgn2d_prepare()
    engine.icgn2d1(before, 16, 16, P.conv, P.stop)
    engine.set_series_2d(ref[::-1].copy(), tars[:, ::-1].copy())
    engine.icgn2d_series_recover(1, seeds, 16, 16, *P.recover_args())
    after = seeds.copy()
    engine.icgn2d1(after, 16, 16, P.conv, P.stop)  # the pair (ref, tars[-1]) is still set and prepared
    assert_same(after, before, "pair call after a series recovery call")


def test_group_context(engine, occluded):
    ref, _, tars = occluded
    seeds = _seeds(engine, ref, tars, sc.short_grid(), 16)
    engine.set_series_2d(ref, tars)
    expect = engine.icgn2d_series_recover(1, seeds, 16, 16, *P.recover_args())
    grp = ob.Engine(list(range(_capi.load().ocb_device_count())))
    try:
        grp.set_series_2d(ref, tars)
        got = grp.icgn2d_series_recover(1, seeds, 16, 16, *P.recover_args())
        assert_same(got[0], expect[0], "group context")
        assert np.array_equal(got[1], expect[1]) and np.array_equal(got[2], expect[2])
        with pytest.raises(_capi.OpenCorrB200Error):
            grp.icgn2d_series_recover_dev(1, 0, 0, 0, 16, 16, *P.recover_args())
    finally:
        grp.close()


def test_refusals_write_nothing():
    eng = ob.Engine(0)
    lib, ctx = eng._lib, eng._ctx
    ref, tars = sc.render_series(96, 80, 2)
    seeds = ob.make_poi2d(synth.grid_2d(40, 40, 2, 2, 10, 10))
    n = len(seeds)
    out = np.full((2, n, 25), 7.0, np.float32)
    rec = np.full((2, 3), 99, np.uint64)
    left = np.full(2, 99, np.uint64)
    vp = lambda a: None if a is None else ctypes.c_void_p(a.ctypes.data)

    def call(order=1, r=8, s=seeds, o=out, count=n, conv=0.001, high=0.9, low=0.5, rounds=3, fn=lib.ocb_icgn2d_series_recover):
        return fn(ctx, order, vp(s), vp(o), count, r, r, conv, 10.0, 20.0, 9, high, low, rounds, vp(rec), vp(left))

    assert call() == _capi.OCB_ERR_STATE  # no series
    assert lib.ocb_set_series_2d(ctx, vp(ref), vp(tars), 2, 96, 80) == _capi.OCB_OK
    for kw in [dict(r=0), dict(s=None), dict(o=None), dict(count=1 << 40), dict(order=0), dict(order=3), dict(rounds=-1),
               dict(conv=float("nan")), dict(high=float("nan")), dict(low=float("nan"))]:
        assert call(**kw) == _capi.OCB_ERR_ARG, kw
    assert call(r=200) == _capi.OCB_ERR_UNSUPPORTED and "exceeds the shared-memory design limit" in _capi.last_error(ctx)
    assert call(s=None, o=None, fn=lib.ocb_icgn2d_series_recover_dev) == _capi.OCB_ERR_ARG
    assert (out == 7.0).all() and (rec == 99).all() and (left == 99).all()
    assert call() == _capi.OCB_OK and not (out == 7.0).all() and (rec < 99).all() and (left < 99).all()  # still usable
    eng.close()
