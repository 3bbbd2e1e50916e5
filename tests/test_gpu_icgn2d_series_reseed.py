"""IC-GN over an image series that re-seeds lost POIs (ocb_icgn2d_series_reseed).  The records must be, bit for bit, what this
loop of pair calls gives when the warps per POI are forced (OCB_ICGN2D_WPP):
    for f: set_images_2d(ref, tars[f]); icgn2d_prepare(); icgn2d1/2(q)
           lost = !(q.zncc >= zncc_min); sub = lost POIs rebuilt from their seeds at their latest good translation
           fftcc2d(sub); icgn2d1/2(sub); q[lost] = sub
and, when nothing is lost, what icgn2d_series gives."""
import ctypes

import numpy as np
import pytest

import opencorr_b200 as ob
from opencorr_b200 import _capi, synth

pytestmark = pytest.mark.gpu

CONV, STOP = 0.001, 10
W, H, FRAMES = 387, 320, 6  # W % 4 != 0: frame pointers of the stack are not 16-byte aligned


def render_series(width, height, n_frames, second_order=False, jump=None, rho=2.0, seed=synth.REF_SEED):
    """ref and n_frames targets: the speckles of synth.speckle_pair_2d moved by (f + 1) / n_frames of its displacement field.
    jump = (k, x0, y0, x1, y1, du, dv): from frame k on, the speckles whose reference centre lies in the box move by (du, dv) more."""
    rng = np.random.default_rng(seed)
    n = int(0.5 * width * height / (np.pi * rho * rho))
    cx = rng.uniform(-8, width + 8, n)
    cy = rng.uniform(-8, height + 8, n)
    amp = rng.uniform(0.4, 1.0, n)
    u, v = synth.displacement_2d(cx, cy, width, height, second_order)

    def image(s, f):
        du = np.zeros_like(cx)
        dv = np.zeros_like(cy)
        if jump is not None and f >= jump[0]:
            k, x0, y0, x1, y1, ju, jv = jump
            inside = (cx >= x0) & (cx < x1) & (cy >= y0) & (cy < y1)
            du[inside], dv[inside] = ju, jv
        im = synth._render((height, width), np.stack([cy + s * v + dv, cx + s * u + du], 1), amp, rho)
        return np.round(np.clip(synth.BACKGROUND + (255.0 - synth.BACKGROUND) * im, 0, 255)).astype(np.float32)

    return image(0.0, -1), np.stack([image((f + 1) / n_frames, f) for f in range(n_frames)])


def occlude(tars, k, box):
    """Cover box = (x0, y0, x1, y1) of frame k with speckles from elsewhere in the same frame (decorrelated from the subsets)."""
    x0, y0, x1, y1 = box
    out = tars.copy()
    out[k, y0:y1, x0:x1] = np.roll(tars[k], (tars.shape[1] // 2, tars.shape[2] // 2), (0, 1))[y0:y1, x0:x1]
    return out


def subset_box(xy, r, u, v, margin=4):
    """The target-frame box covering the subsets of the POIs xy displaced by about (u, v)."""
    return (int(xy[:, 0].min() + u - r - margin), int(xy[:, 1].min() + v - r - margin), int(xy[:, 0].max() + u + r + margin + 1),
            int(xy[:, 1].max() + v + r + margin + 1))


def pair_loop(eng, ref, tars, seeds, order, r, fr, zncc_min):
    icgn = eng.icgn2d1 if order == 1 else eng.icgn2d2
    q = seeds.copy()
    anchor = seeds[:, [2, 8]].copy()
    out, counts = [], []
    for f in range(len(tars)):
        eng.set_images_2d(ref, tars[f])
        eng.icgn2d_prepare()
        icgn(q, r, r, CONV, STOP)
        if f > 0:
            good = out[-1][:, 16] >= zncc_min
            anchor[good] = out[-1][good][:, [2, 8]]
        lost = np.nonzero(~(q[:, 16] >= zncc_min))[0]
        if len(lost):
            sub = np.zeros((len(lost), ob.POI2D_FLOATS), np.float32)
            for c in (0, 1, 23, 24):
                sub[:, c] = seeds[lost, c]
            sub[:, [2, 8]] = anchor[lost]
            eng.fftcc2d(sub, fr, fr)
            icgn(sub, r, r, CONV, STOP)
            q[lost] = sub
        out.append(q.copy())
        counts.append(len(lost))
    return np.stack(out), np.array(counts, np.int64)


def assert_same(a, b, label):
    assert a.shape == b.shape, label
    bad = a.view(np.uint32) != b.view(np.uint32)
    assert not bad.any(), "%s: %d floats differ, first at %s" % (label, bad.sum(), np.argwhere(bad)[:5].tolist())


def fftcc_seeds(eng, ref, tar, xy, r):
    q = ob.make_poi2d(xy)
    eng.set_images_2d(ref, tar)
    eng.fftcc2d(q, r, r)
    return q


@pytest.fixture(scope="module")
def series():
    return render_series(384, 320, 5)


@pytest.fixture(scope="module")
def series2():
    return render_series(384, 320, 5, second_order=True)


# order, radius, POIs: few POIs run two warps per POI, many run one
NOTHING_LOST = [(1, 16, "short"), (1, 16, "long"), (1, 23, "short"), (1, 23, "long"), (2, 20, "short"), (2, 20, "long"), (2, 23, "short"),
                (2, 23, "long")]


@pytest.mark.parametrize("tma", [True, False], ids=["tma", "no_tma"])
@pytest.mark.parametrize("order,r,kind", NOTHING_LOST)
def test_nothing_lost_equals_plain_series(engine, series, series2, monkeypatch, order, r, kind, tma):
    if not tma:
        monkeypatch.setenv("OCB_NO_TMA", "1")
    ref, tars = series if order == 1 else series2
    xy = synth.grid_2d(60, 55, 6, 5, 48, 41) if kind == "short" else synth.grid_2d(r + 4, r + 4, 112, 70, 3, 4)
    seeds = fftcc_seeds(engine, ref, tars[0], xy, 16)
    seeds[::7, 16] = -1.0  # failed seeds stay failed: -10 is below every code
    engine.set_series_2d(ref, tars)
    expect = engine.icgn2d_series(order, seeds, r, r, CONV, STOP)
    got, counts = engine.icgn2d_series_reseed(order, seeds, r, r, CONV, STOP, 16, 16, -10.0)
    assert_same(got, expect, "order %d r %d %s" % (order, r, kind))
    assert counts.shape == (len(tars),) and (counts == 0).all()


@pytest.fixture(scope="module")
def lossy():
    """Frame 2 occludes a 2 x 2 block of POIs, frame 5 (the last) another one; three seeds arrive failed."""
    ref, tars = render_series(W, H, FRAMES)
    xy = synth.grid_2d(50, 50, 8, 6, 40, 40)
    blocks = []
    for k, (bx, by) in ((2, (130, 130)), (5, (250, 170))):
        sel = (xy[:, 0] >= bx) & (xy[:, 0] < bx + 80) & (xy[:, 1] >= by) & (xy[:, 1] < by + 80)
        u, v = synth.displacement_2d(bx + 20.0, by + 20.0, W, H)
        s = (k + 1) / FRAMES
        tars = occlude(tars, k, subset_box(xy[sel], 20, s * u, s * v))
        blocks.append(sel)
    return ref, tars, xy, blocks


@pytest.mark.parametrize("wpp", ["1", "2"])
@pytest.mark.parametrize("fr", [16, 10, 7], ids=["fft_w32", "fft_reg", "fft_generic"])
@pytest.mark.parametrize("order", [1, 2])
def test_reseed_equals_pair_loop(engine, lossy, monkeypatch, order, fr, wpp):
    monkeypatch.setenv("OCB_ICGN2D_WPP", wpp)
    ref, tars, xy, blocks = lossy
    r = 16 if order == 1 else 20
    seeds = fftcc_seeds(engine, ref, tars[0], xy, 16)
    seeds[[3, 17, 40], 16] = -1.0
    for n_frames in (1, FRAMES):
        expect, expect_counts = pair_loop(engine, ref, tars[:n_frames], seeds, order, r, fr, 0.9)
        engine.set_series_2d(ref, tars[:n_frames])
        got, counts = engine.icgn2d_series_reseed(order, seeds, r, r, CONV, STOP, fr, fr, 0.9)
        assert_same(got, expect, "order %d fft r %d F %d" % (order, fr, n_frames))
        assert np.array_equal(counts, expect_counts), (counts, expect_counts)
        assert counts[0] >= 3
        if n_frames == FRAMES:
            assert counts[2] >= blocks[0].sum() and counts[5] >= blocks[1].sum()  # the last frame is re-seeded too


def test_transient_occlusion_recovers(engine):
    ref, clean = render_series(W, H, FRAMES)
    xy = synth.grid_2d(40, 40, 7, 6, 48, 48)
    block = (xy[:, 0] >= 130) & (xy[:, 0] < 200) & (xy[:, 1] >= 130) & (xy[:, 1] < 200)
    k = 2
    u, v = synth.displacement_2d(xy[block, 0], xy[block, 1], W, H)
    s = (k + 1) / FRAMES
    tars = occlude(clean, k, subset_box(xy[block], 16, s * u.mean(), s * v.mean()))
    seeds = fftcc_seeds(engine, ref, tars[0], xy, 16)
    engine.set_series_2d(ref, tars)
    plain = engine.icgn2d_series(1, seeds, 16, 16, CONV, STOP)
    assert (~(plain[k, block, 16] >= 0.9)).all(), "control: IC-GN alone loses the block in the occluded frame"
    got, counts = engine.icgn2d_series_reseed(1, seeds, 16, 16, CONV, STOP, 16, 16, 0.9)
    assert counts[k] == block.sum() and counts[k + 1] == block.sum(), counts
    assert counts.sum() == 2 * block.sum(), counts
    engine.set_series_2d(ref, clean)
    reference = engine.icgn2d_series(1, seeds, 16, 16, CONV, STOP)
    for f in range(k + 1, FRAMES):
        assert (got[f][:, 16] >= 0.9).all(), "frame %d" % f
        for col in (2, 8):  # the clean series' records: the same optimum, reached from another start
            assert np.abs(got[f][block, col] - reference[f][block, col]).max() < 0.01
        uf, vf = synth.displacement_2d(xy[:, 0], xy[:, 1], W, H)
        s = (f + 1) / FRAMES
        assert np.abs(got[f][:, 2] - s * uf).max() < 0.05 and np.abs(got[f][:, 8] - s * vf).max() < 0.05
    outside = ~block
    assert_same(got[:, outside], plain[:, outside], "POIs that are never lost")


def test_local_jump_recovered_by_fftcc(engine):
    k, box, du, dv = 3, (130, 100, 330, 260), 7.0, -5.0
    ref, tars = render_series(W, H, FRAMES, jump=(k,) + box + (du, dv))
    xy = synth.grid_2d(40, 40, 8, 6, 44, 44)
    m = 16 + 10
    inside = (xy[:, 0] >= box[0] + m) & (xy[:, 0] < box[2] - m - 8) & (xy[:, 1] >= box[1] + m) & (xy[:, 1] < box[3] - m)
    assert inside.sum() >= 4
    seeds = fftcc_seeds(engine, ref, tars[0], xy, 16)
    engine.set_series_2d(ref, tars)
    plain = engine.icgn2d_series(1, seeds, 16, 16, CONV, STOP)
    assert (~(plain[k, inside, 16] >= 0.9)).all(), "control: IC-GN alone loses the jumped POIs"
    got, counts = engine.icgn2d_series_reseed(1, seeds, 16, 16, CONV, STOP, 16, 16, 0.9)
    assert counts[k] >= inside.sum()
    uf, vf = synth.displacement_2d(xy[inside, 0], xy[inside, 1], W, H)
    for f in range(k, FRAMES):
        s = (f + 1) / FRAMES
        rec = got[f][inside]
        assert (rec[:, 16] >= 0.9).all(), "frame %d" % f
        assert np.abs(rec[:, 2] - (s * uf + du)).max() < 0.05 and np.abs(rec[:, 8] - (s * vf + dv)).max() < 0.05


def test_failed_seeds_reseeded_in_frame_0(engine, series):
    ref, tars = series
    xy = synth.grid_2d(60, 55, 6, 5, 48, 41)
    seeds = fftcc_seeds(engine, ref, tars[0], xy, 16)
    failed = np.array([1, 8, 20])
    seeds[failed, 16] = -1.0
    engine.set_series_2d(ref, tars)
    got, counts = engine.icgn2d_series_reseed(1, seeds, 16, 16, CONV, STOP, 16, 16, 0.5)
    assert counts[0] == len(failed) and counts[1:].sum() == 0, counts
    assert (got[:, :, 16] >= 0.5).all()
    ok = seeds.copy()
    ok[failed, 16] = 0.0
    ok[failed, 2:14] = 0.0
    ok[failed, 2], ok[failed, 8] = seeds[failed, 2], seeds[failed, 8]
    plain = engine.icgn2d_series(1, ok, 16, 16, CONV, STOP)
    assert np.abs(got[-1][:, [2, 8]] - plain[-1][:, [2, 8]]).max() < 0.01


def test_errors_leave_out_and_counts_untouched():
    eng = ob.Engine(0)
    lib, ctx = eng._lib, eng._ctx
    ref, tars = render_series(96, 80, 2)
    seeds = ob.make_poi2d(synth.grid_2d(40, 40, 2, 2, 10, 10))
    n = len(seeds)
    out = np.full((2, n, 25), 7.0, np.float32)
    counts = np.full(2, 99, np.uint64)
    vp = lambda a: ctypes.c_void_p(a.ctypes.data)

    def call(order=1, r=8, fr=8, zmin=0.5, s=seeds, o=out, count=n):
        return lib.ocb_icgn2d_series_reseed(ctx, order, vp(s) if s is not None else None, vp(o) if o is not None else None, count, r, r, CONV,
                                            STOP, fr, fr, zmin, vp(counts))

    assert call() == _capi.OCB_ERR_STATE
    assert lib.ocb_set_series_2d(ctx, vp(ref), vp(tars), 2, 96, 80) == _capi.OCB_OK
    assert call(order=3) == _capi.OCB_ERR_ARG
    assert call(s=None) == _capi.OCB_ERR_ARG
    assert call(o=None) == _capi.OCB_ERR_ARG
    assert call(count=1 << 40) == _capi.OCB_ERR_ARG
    assert call(zmin=float("nan")) == _capi.OCB_ERR_ARG
    assert call(fr=0) == _capi.OCB_ERR_ARG
    assert call(fr=37) == _capi.OCB_ERR_UNSUPPORTED
    assert "prime factor > 31" in _capi.last_error(ctx)
    assert call(r=200) == _capi.OCB_ERR_UNSUPPORTED
    assert "exceeds the shared-memory design limit" in _capi.last_error(ctx)
    assert lib.ocb_icgn2d_series_reseed_dev(ctx, 1, None, None, 5, 8, 8, CONV, STOP, 8, 8, 0.5, vp(counts)) == _capi.OCB_ERR_ARG
    assert (out == 7.0).all() and (counts == 99).all()
    assert call() == _capi.OCB_OK
    assert not (out == 7.0).all() and (counts < 99).all()
    eng.close()


def test_pair_calls_unaffected(engine, lossy):
    ref, tars, xy, _ = lossy
    seeds = fftcc_seeds(engine, ref, tars[-1], xy, 16)
    engine.icgn2d_prepare()
    before = seeds.copy()
    engine.icgn2d1(before, 16, 16, CONV, STOP)
    engine.set_series_2d(ref, tars)
    _, counts = engine.icgn2d_series_reseed(1, seeds, 16, 16, CONV, STOP, 10, 10, 0.9)
    assert counts.sum() > 0
    after = seeds.copy()
    engine.icgn2d1(after, 16, 16, CONV, STOP)  # the pair (ref, tars[-1]) is still set and prepared
    assert_same(after, before, "pair call after a re-seeding series call")


def test_dev_matches_host(engine, lossy):
    torch = pytest.importorskip("torch")
    ref, tars, xy, _ = lossy
    seeds = fftcc_seeds(engine, ref, tars[0], xy, 16)
    engine.set_series_2d(ref, tars)
    host, host_counts = engine.icgn2d_series_reseed(2, seeds, 20, 20, CONV, STOP, 16, 16, 0.9)
    assert host_counts.sum() > 0
    d_ref, d_tars, d_seeds = (torch.from_numpy(a).cuda() for a in (ref, tars, seeds))
    d_out = torch.empty((len(tars), len(seeds), 25), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    engine.set_series_2d_dev(d_ref.data_ptr(), d_tars.data_ptr(), len(tars), W, H)
    counts = engine.icgn2d_series_reseed_dev(2, d_seeds.data_ptr(), d_out.data_ptr(), len(seeds), 20, 20, CONV, STOP, 16, 16, 0.9)
    assert_same(d_out.cpu().numpy(), host, "device-pointer variant")
    assert np.array_equal(counts, host_counts)
    assert_same(d_seeds.cpu().numpy(), seeds, "device seeds changed")


def test_group(lossy):
    if _capi.load().ocb_device_count() < 2:
        pytest.skip("needs two GPUs")
    ref, tars, xy, _ = lossy
    single = ob.Engine(0)
    seeds = fftcc_seeds(single, ref, tars[0], xy, 16)
    single.set_series_2d(ref, tars)
    expect, expect_counts = single.icgn2d_series_reseed(1, seeds, 16, 16, CONV, STOP, 16, 16, 0.9)
    group = ob.Engine([0, 1])
    group.set_series_2d(ref, tars)
    got, counts = group.icgn2d_series_reseed(1, seeds, 16, 16, CONV, STOP, 16, 16, 0.9)
    assert_same(got, expect, "group context")
    assert np.array_equal(counts, expect_counts)
    group.close()
    single.close()
