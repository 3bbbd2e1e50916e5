"""IC-GN over an image series (ocb_icgn2d_series): every frame's records must be, bit for bit, what the loop of pair calls
    set_images_2d(ref, tars[f]); icgn2d_prepare(); icgn2d1/2(q, ...)
gives when one queue q is carried from frame to frame."""
import ctypes

import numpy as np
import pytest

import opencorr_b200 as ob
from opencorr_b200 import _capi, synth
from oracle.oracle import Oracle2D
from util import compare_2d

pytestmark = pytest.mark.gpu

CONV, STOP = 0.001, 10


def render_series(width, height, n_frames, second_order=False, rho=2.0, seed=synth.REF_SEED):
    """ref and n_frames targets: the speckles of synth.speckle_pair_2d moved by (f + 1) / n_frames of its displacement field,
    so the last frame carries the full field."""
    rng = np.random.default_rng(seed)
    n = int(0.5 * width * height / (np.pi * rho * rho))
    cx = rng.uniform(-8, width + 8, n)
    cy = rng.uniform(-8, height + 8, n)
    amp = rng.uniform(0.4, 1.0, n)
    u, v = synth.displacement_2d(cx, cy, width, height, second_order)

    def image(s):
        im = synth._render((height, width), np.stack([cy + s * v, cx + s * u], 1), amp, rho)
        return np.round(np.clip(synth.BACKGROUND + (255.0 - synth.BACKGROUND) * im, 0, 255)).astype(np.float32)

    return image(0.0), np.stack([image((f + 1) / n_frames) for f in range(n_frames)])


def pair_loop(eng, ref, tars, seeds, order, rx, ry, stop=STOP):
    q = seeds.copy()
    out = []
    for f in range(len(tars)):
        eng.set_images_2d(ref, tars[f])
        eng.icgn2d_prepare()
        (eng.icgn2d1 if order == 1 else eng.icgn2d2)(q, rx, ry, CONV, stop)
        out.append(q.copy())
    return np.stack(out)


def assert_same(a, b, label):
    assert a.shape == b.shape, label
    bad = a.view(np.uint32) != b.view(np.uint32)
    assert not bad.any(), "%s: %d floats differ, first at %s" % (label, bad.sum(), np.argwhere(bad)[:5].tolist())


@pytest.fixture(scope="module")
def series():
    ref, tars = render_series(384, 320, 5)
    return ref, tars


@pytest.fixture(scope="module")
def series2():
    ref, tars = render_series(384, 320, 5, second_order=True)
    return ref, tars


def fftcc_seeds(eng, ref, tar, xy, r):
    q = ob.make_poi2d(xy)
    eng.set_images_2d(ref, tar)
    eng.fftcc2d(q, r, r)
    return q


# order, radius, POIs: few POIs run two warps per POI, many run one (icgn2d_launch's rule)
CASES = [(1, 16, "short"), (1, 16, "long"), (1, 23, "short"), (1, 23, "long"), (2, 20, "short"), (2, 20, "long"), (2, 12, "short"),
         (2, 12, "long")]


def _grid(kind, r):
    if kind == "short":
        return synth.grid_2d(60, 55, 6, 5, 48, 41)
    return synth.grid_2d(r + 4, r + 4, 112, 70, 3, 4)  # 7840 POIs: more than the resident slots at these radii


@pytest.mark.parametrize("tma", [True, False], ids=["tma", "no_tma"])
@pytest.mark.parametrize("order,r,kind", CASES)
def test_series_equals_pair_loop(engine, series, series2, monkeypatch, order, r, kind, tma):
    if not tma:
        monkeypatch.setenv("OCB_NO_TMA", "1")
    ref, tars = series if order == 1 else series2
    xy = _grid(kind, r)
    seeds = fftcc_seeds(engine, ref, tars[0], xy, r)
    for n_frames in (1, 5):
        expect = pair_loop(engine, ref, tars[:n_frames], seeds, order, r, r)
        engine.set_series_2d(ref, tars[:n_frames])
        got = engine.icgn2d_series(order, seeds, r, r, CONV, STOP)
        assert_same(got, expect, "order %d r %d %s F %d" % (order, r, kind, n_frames))
        assert (got[-1][:, 16] >= 0).mean() > 0.8


@pytest.mark.parametrize("order,r", [(1, 16), (2, 20)])
def test_series_matches_oracle_and_ground_truth(engine, series, series2, order, r):
    ref, tars = series if order == 1 else series2
    xy = synth.grid_2d(40, 40, 12, 10, 27, 24)
    seeds = fftcc_seeds(engine, ref, tars[0], xy, r)
    engine.set_series_2d(ref, tars)
    got = engine.icgn2d_series(order, seeds, r, r, CONV, STOP)
    for f in range(len(tars)):
        q = (seeds if f == 0 else got[f - 1]).copy()  # each frame from the same seeds as the GPU's
        o = Oracle2D(ref, tars[f])
        (o.icgn2d1 if order == 1 else o.icgn2d2)(q, r, r, CONV, STOP, exact=True)
        compare_2d(got[f], q, "frame %d" % f, order=order)
    last = got[-1]
    ok = last[:, 16] >= 0
    assert ok.mean() > 0.95
    u_true, v_true = synth.displacement_2d(xy[:, 0], xy[:, 1], ref.shape[1], ref.shape[0], second_order=order == 2)
    assert np.abs(last[ok, 2] - u_true[ok]).max() < 0.05 and np.abs(last[ok, 8] - v_true[ok]).max() < 0.05


def test_series_sentinels(engine, series):
    """POIs that leave the image mid-series, stop at the iteration limit (-4) or arrive with a negative ZNCC keep their code
    and a copy of that frame's record in every later frame, exactly as the pair loop does."""
    ref, tars = series
    h, w = ref.shape
    xy = np.array([[100, 100], [200, 150], [w - 17, 100], [w - 40, 200], [150, 160], [300, 250], [120, 260], [60, 60]], np.float32)
    seeds = fftcc_seeds(engine, ref, tars[0], xy, 16)
    seeds[2, 2] = 2.0          # the subset leaves the image as the series moves right
    seeds[3, 2] = w + 5.0      # |u| >= width: the guard rejects it
    seeds[4, 16] = -1.0        # arrives negative
    seeds[5, 2] += 7.5         # far from the optimum: runs into the iteration limit
    seeds[6, 8] = np.nan       # NaN guess
    for stop in (STOP, 2):
        expect = pair_loop(engine, ref, tars, seeds, 1, 16, 16, stop)
        engine.set_series_2d(ref, tars)
        got = engine.icgn2d_series(1, seeds, 16, 16, CONV, stop)
        assert_same(got, expect, "stop %g" % stop)
        codes = got[:, :, 16]
        assert (codes[:, 3] == -3).all() and (codes[:, 4] == -1).all()
        if stop == 2:
            assert (codes == -4).any()
        for i in range(len(xy)):
            neg = np.nonzero(codes[:, i] < 0)[0]
            if len(neg):
                f0 = neg[0]
                for f in range(f0 + 1, len(tars)):
                    assert_same(got[f, i], got[f0, i], "POI %d frame %d" % (i, f))


def test_series_chunks(engine, series):
    ref, tars = series
    xy = synth.grid_2d(60, 55, 6, 5, 48, 41)
    seeds = fftcc_seeds(engine, ref, tars[0], xy, 16)
    engine.set_series_2d(ref, tars)
    whole = engine.icgn2d_series(1, seeds, 16, 16, CONV, STOP)
    engine.set_series_2d(ref, tars[:2])
    a = engine.icgn2d_series(1, seeds, 16, 16, CONV, STOP)
    engine.set_series_2d(ref, tars[2:])
    b = engine.icgn2d_series(1, a[-1].copy(), 16, 16, CONV, STOP)
    assert_same(np.concatenate([a, b]), whole, "two chunks")


def test_series_errors_leave_out_untouched():
    eng = ob.Engine(0)
    lib, ctx = eng._lib, eng._ctx
    ref, tars = render_series(96, 80, 2)
    seeds = ob.make_poi2d(synth.grid_2d(40, 40, 2, 2, 10, 10))
    n = len(seeds)
    out = np.full((2, n, 25), 7.0, np.float32)
    vp = lambda a: ctypes.c_void_p(a.ctypes.data)

    def call(order=1, r=8, s=seeds, o=out, count=n):
        return lib.ocb_icgn2d_series(ctx, order, vp(s) if s is not None else None, vp(o) if o is not None else None, count, r, r,
                                     CONV, STOP)

    assert call() == _capi.OCB_ERR_STATE
    assert lib.ocb_set_series_2d(ctx, vp(ref), vp(tars), 0, 96, 80) == _capi.OCB_ERR_ARG
    assert lib.ocb_set_series_2d(ctx, vp(ref), None, 2, 96, 80) == _capi.OCB_ERR_ARG
    assert call() == _capi.OCB_ERR_STATE  # the refused calls set nothing
    assert lib.ocb_set_series_2d(ctx, vp(ref), vp(tars), 2, 96, 80) == _capi.OCB_OK
    assert call(order=3) == _capi.OCB_ERR_ARG
    assert call(s=None) == _capi.OCB_ERR_ARG
    assert call(o=None) == _capi.OCB_ERR_ARG
    assert call(count=1 << 40) == _capi.OCB_ERR_ARG
    assert call(r=200) == _capi.OCB_ERR_UNSUPPORTED
    assert "exceeds the shared-memory design limit" in _capi.last_error(ctx)
    assert lib.ocb_icgn2d_series_dev(ctx, 1, None, None, 5, 8, 8, CONV, STOP) == _capi.OCB_ERR_ARG
    assert (out == 7.0).all()
    assert call() == _capi.OCB_OK
    assert not (out == 7.0).all()
    eng.close()


def test_pair_calls_unaffected_by_series(engine, series):
    ref, tars = series
    xy = synth.grid_2d(60, 55, 6, 5, 48, 41)
    seeds = fftcc_seeds(engine, ref, tars[-1], xy, 16)
    engine.icgn2d_prepare()
    before = seeds.copy()
    engine.icgn2d1(before, 16, 16, CONV, STOP)
    engine.set_series_2d(ref[::-1].copy(), tars[:, ::-1].copy())
    engine.icgn2d_series(2, seeds, 16, 16, CONV, STOP)
    after = seeds.copy()
    engine.icgn2d1(after, 16, 16, CONV, STOP)  # the pair (ref, tars[-1]) is still set and prepared
    assert_same(after, before, "pair call after a series call")


def test_series_dev_matches_host(engine, series):
    torch = pytest.importorskip("torch")
    ref, tars = series
    xy = synth.grid_2d(60, 55, 6, 5, 48, 41)
    seeds = fftcc_seeds(engine, ref, tars[0], xy, 16)
    engine.set_series_2d(ref, tars)
    host = engine.icgn2d_series(1, seeds, 16, 16, CONV, STOP)
    d_ref, d_tars, d_seeds = (torch.from_numpy(a).cuda() for a in (ref, tars, seeds))
    d_out = torch.empty((len(tars), len(seeds), 25), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    engine.set_series_2d_dev(d_ref.data_ptr(), d_tars.data_ptr(), len(tars), ref.shape[1], ref.shape[0])
    engine.icgn2d_series_dev(1, d_seeds.data_ptr(), d_out.data_ptr(), len(seeds), 16, 16, CONV, STOP)
    engine.sync()
    assert_same(d_out.cpu().numpy(), host, "device-pointer variant")


def test_series_group(series):
    if _capi.load().ocb_device_count() < 2:
        pytest.skip("needs two GPUs")
    ref, tars = series
    xy = synth.grid_2d(60, 55, 6, 5, 48, 41)
    single = ob.Engine(0)
    seeds = fftcc_seeds(single, ref, tars[0], xy, 16)
    single.set_series_2d(ref, tars)
    expect = single.icgn2d_series(1, seeds, 16, 16, CONV, STOP)
    group = ob.Engine([0, 1])
    group.set_series_2d(ref, tars)
    assert_same(group.icgn2d_series(1, seeds, 16, 16, CONV, STOP), expect, "group context")
    group.close()
    single.close()
