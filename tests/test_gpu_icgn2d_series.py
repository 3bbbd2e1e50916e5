"""IC-GN over an image series (ocb_icgn2d_series, ocb_icgn2d_series_reseed): every frame's records must be, bit for bit, what the
loop of pair calls
    set_images_2d(ref, tars[f]); icgn2d_prepare(); icgn2d1/2(q, ...)
gives when one queue q is carried from frame to frame.  The re-seeding call must give, with the warps per POI forced
(OCB_ICGN2D_WPP), what that loop gives when it also rebuilds the POIs lost in frame f from their seeds at their latest good
translation and runs fftcc2d and icgn2d1/2 on them against frame f (subset_series_cases.reseed_pair_loop), and, when nothing
is lost, what icgn2d_series gives."""
import numpy as np
import pytest

import opencorr_b200 as ob
from opencorr_b200 import _capi, synth
import subset_series_cases as sc
from util import assert_same

pytestmark = pytest.mark.gpu

W, H, FRAMES = 387, 320, 6  # W % 4 != 0: frame pointers of the stack are not 16-byte aligned
ICGN1 = sc.Method("icgn", 1)


@pytest.fixture(scope="module")
def series():
    return sc.render_series(384, 320, 5)


@pytest.fixture(scope="module")
def series2():
    return sc.render_series(384, 320, 5, second_order=True)


def _grid(kind, r):
    return sc.short_grid() if kind == "short" else sc.long_grid(r)


# order, radius, POIs: few POIs run two warps per POI, many run one (icgn2d_launch's rule)
CASES = [(1, 16, "short"), (1, 16, "long"), (1, 23, "short"), (1, 23, "long"), (2, 20, "short"), (2, 20, "long"), (2, 12, "short"),
         (2, 12, "long")]
NOTHING_LOST = [(1, 16, "short"), (1, 16, "long"), (1, 23, "short"), (1, 23, "long"), (2, 20, "short"), (2, 20, "long"), (2, 23, "short"),
                (2, 23, "long")]


@pytest.mark.parametrize("tma", [True, False], ids=["tma", "no_tma"])
@pytest.mark.parametrize("order,r,kind", CASES)
def test_series_equals_pair_loop(engine, series, series2, monkeypatch, order, r, kind, tma):
    if not tma:
        monkeypatch.setenv("OCB_NO_TMA", "1")
    ref, tars = series if order == 1 else series2
    sc.check_equals_pair_loop(engine, sc.Method("icgn", order), ref, tars, _grid(kind, r), r, "r %d %s" % (r, kind), fft_r=r)


@pytest.mark.parametrize("order,r", [(1, 16), (2, 20)])
def test_series_matches_oracle_and_ground_truth(engine, series, series2, order, r):
    ref, tars = series if order == 1 else series2
    sc.check_oracle_and_ground_truth(engine, sc.Method("icgn", order), ref, tars, r, second_order=order == 2, fft_r=r, every_frame=True)


def test_series_sentinels(engine, series):
    """POIs that leave the image mid-series, stop at the iteration limit (-4) or arrive with a negative ZNCC keep their code
    and a copy of that frame's record in every later frame, exactly as the pair loop does."""
    ref, tars = series
    h, w = ref.shape
    xy = np.array([[100, 100], [200, 150], [w - 17, 100], [w - 40, 200], [150, 160], [300, 250], [120, 260], [60, 60]], np.float32)
    seeds = sc.fftcc_seeds(engine, ref, tars[0], xy, 16)
    seeds[2, 2] = 2.0          # the subset leaves the image as the series moves right
    seeds[3, 2] = w + 5.0      # |u| >= width: the guard rejects it
    seeds[4, 16] = -1.0        # arrives negative
    seeds[5, 2] += 7.5         # far from the optimum: runs into the iteration limit
    seeds[6, 8] = np.nan       # NaN guess
    for stop in (sc.STOP, 2):
        expect = sc.pair_loop(engine, ICGN1, ref, tars, seeds, 16, stop)
        engine.set_series_2d(ref, tars)
        got = ICGN1.series(engine, seeds, 16, stop)
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
    sc.check_chunks(engine, ICGN1, *series, 16)


def test_series_errors_leave_out_untouched():
    sc.check_errors_leave_out_untouched(ICGN1)


def test_series_errors_leave_out_untouched_order_2():
    sc.check_errors_leave_out_untouched(sc.Method("icgn", 2))


def test_pair_calls_unaffected_by_series(engine, series):
    sc.check_pair_state_undisturbed(engine, ICGN1, *series, 16, series_method=sc.Method("icgn", 2))


def test_series_dev_matches_host(engine, series):
    torch = pytest.importorskip("torch")
    ref, tars = series
    seeds = sc.fftcc_seeds(engine, ref, tars[0], sc.short_grid(), 16)
    engine.set_series_2d(ref, tars)
    host = ICGN1.series(engine, seeds, 16)
    d_ref, d_tars, d_seeds = (torch.from_numpy(a).cuda() for a in (ref, tars, seeds))
    d_out = torch.empty((len(tars), len(seeds), 25), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    engine.set_series_2d_dev(d_ref.data_ptr(), d_tars.data_ptr(), len(tars), ref.shape[1], ref.shape[0])
    ICGN1.series_dev(engine, d_seeds.data_ptr(), d_out.data_ptr(), len(seeds), 16)
    engine.sync()
    assert_same(d_out.cpu().numpy(), host, "device-pointer variant")


def test_series_group(series):
    if _capi.load().ocb_device_count() < 2:
        pytest.skip("needs two GPUs")
    ref, tars = series
    single = ob.Engine(0)
    seeds = sc.fftcc_seeds(single, ref, tars[0], sc.short_grid(), 16)
    single.set_series_2d(ref, tars)
    expect = ICGN1.series(single, seeds, 16)
    group = ob.Engine([0, 1])
    group.set_series_2d(ref, tars)
    assert_same(ICGN1.series(group, seeds, 16), expect, "group context")
    group.close()
    single.close()


@pytest.mark.parametrize("tma", [True, False], ids=["tma", "no_tma"])
@pytest.mark.parametrize("order,r,kind", NOTHING_LOST)
def test_reseed_nothing_lost_equals_plain_series(engine, series, series2, monkeypatch, order, r, kind, tma):
    if not tma:
        monkeypatch.setenv("OCB_NO_TMA", "1")
    ref, tars = series if order == 1 else series2
    sc.check_nothing_lost(engine, sc.Method("icgn", order), ref, tars, _grid(kind, r), r)


def subset_box(xy, r, u, v, margin=4):
    """The target-frame box covering the subsets of the POIs xy displaced by about (u, v)."""
    return (int(xy[:, 0].min() + u - r - margin), int(xy[:, 1].min() + v - r - margin), int(xy[:, 0].max() + u + r + margin + 1),
            int(xy[:, 1].max() + v + r + margin + 1))


@pytest.fixture(scope="module")
def lossy():
    """Frame 2 occludes a 2 x 2 block of POIs, frame 5 (the last) another one; three seeds arrive failed."""
    ref, tars = sc.render_series(W, H, FRAMES)
    xy = synth.grid_2d(50, 50, 8, 6, 40, 40)
    occluded = []
    for k, (bx, by) in ((2, (130, 130)), (5, (250, 170))):
        sel = (xy[:, 0] >= bx) & (xy[:, 0] < bx + 80) & (xy[:, 1] >= by) & (xy[:, 1] < by + 80)
        u, v = synth.displacement_2d(bx + 20.0, by + 20.0, W, H)
        s = (k + 1) / FRAMES
        tars = sc.occlude(tars, k, subset_box(xy[sel], 20, s * u, s * v))
        occluded.append((k, sel))
    return ref, tars, xy, occluded


@pytest.mark.parametrize("wpp", ["1", "2"])
@pytest.mark.parametrize("fr", [16, 10, 7], ids=["fft_w32", "fft_reg", "fft_generic"])
@pytest.mark.parametrize("order", [1, 2])
def test_reseed_equals_pair_loop(engine, lossy, monkeypatch, order, fr, wpp):
    monkeypatch.setenv("OCB_ICGN2D_WPP", wpp)
    sc.check_reseed_equals_pair_loop(engine, sc.Method("icgn", order), lossy, 16 if order == 1 else 20, fr)


def test_transient_occlusion_recovers(engine):
    ref, clean = sc.render_series(W, H, FRAMES)
    xy = synth.grid_2d(40, 40, 7, 6, 48, 48)
    block = (xy[:, 0] >= 130) & (xy[:, 0] < 200) & (xy[:, 1] >= 130) & (xy[:, 1] < 200)
    k = 2
    u, v = synth.displacement_2d(xy[block, 0], xy[block, 1], W, H)
    s = (k + 1) / FRAMES
    tars = sc.occlude(clean, k, subset_box(xy[block], 16, s * u.mean(), s * v.mean()))
    seeds = sc.fftcc_seeds(engine, ref, tars[0], xy, 16)
    engine.set_series_2d(ref, tars)
    plain = ICGN1.series(engine, seeds, 16)
    assert (~(plain[k, block, 16] >= 0.9)).all(), "control: IC-GN alone loses the block in the occluded frame"
    got, counts = ICGN1.series_reseed(engine, seeds, 16, 16, 0.9)
    assert counts[k] == block.sum() and counts[k + 1] == block.sum(), counts
    assert counts.sum() == 2 * block.sum(), counts
    engine.set_series_2d(ref, clean)
    reference = ICGN1.series(engine, seeds, 16)
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
    ref, tars = sc.render_series(W, H, FRAMES, jump=(k,) + box + (du, dv))
    xy = synth.grid_2d(40, 40, 8, 6, 44, 44)
    m = 16 + 10
    inside = (xy[:, 0] >= box[0] + m) & (xy[:, 0] < box[2] - m - 8) & (xy[:, 1] >= box[1] + m) & (xy[:, 1] < box[3] - m)
    assert inside.sum() >= 4
    seeds = sc.fftcc_seeds(engine, ref, tars[0], xy, 16)
    engine.set_series_2d(ref, tars)
    plain = ICGN1.series(engine, seeds, 16)
    assert (~(plain[k, inside, 16] >= 0.9)).all(), "control: IC-GN alone loses the jumped POIs"
    got, counts = ICGN1.series_reseed(engine, seeds, 16, 16, 0.9)
    assert counts[k] >= inside.sum()
    uf, vf = synth.displacement_2d(xy[inside, 0], xy[inside, 1], W, H)
    for f in range(k, FRAMES):
        s = (f + 1) / FRAMES
        rec = got[f][inside]
        assert (rec[:, 16] >= 0.9).all(), "frame %d" % f
        assert np.abs(rec[:, 2] - (s * uf + du)).max() < 0.05 and np.abs(rec[:, 8] - (s * vf + dv)).max() < 0.05


def test_failed_seeds_reseeded_in_frame_0(engine, series):
    ref, tars = series
    seeds = sc.fftcc_seeds(engine, ref, tars[0], sc.short_grid(), 16)
    failed = np.array([1, 8, 20])
    seeds[failed, 16] = -1.0
    engine.set_series_2d(ref, tars)
    got, counts = ICGN1.series_reseed(engine, seeds, 16, 16, 0.5)
    assert counts[0] == len(failed) and counts[1:].sum() == 0, counts
    assert (got[:, :, 16] >= 0.5).all()
    ok = seeds.copy()
    ok[failed, 16] = 0.0
    ok[failed, 2:14] = 0.0
    ok[failed, 2], ok[failed, 8] = seeds[failed, 2], seeds[failed, 8]
    plain = ICGN1.series(engine, ok, 16)
    assert np.abs(got[-1][:, [2, 8]] - plain[-1][:, [2, 8]]).max() < 0.01


def test_reseed_pair_calls_unaffected(engine, lossy):
    ref, tars, xy, _ = lossy
    seeds = sc.fftcc_seeds(engine, ref, tars[-1], xy, 16)
    before = seeds.copy()
    ICGN1.pair(engine, before, 16)
    engine.set_series_2d(ref, tars)
    _, counts = ICGN1.series_reseed(engine, seeds, 16, 10, 0.9)
    assert counts.sum() > 0
    after = seeds.copy()
    ICGN1.pair(engine, after, 16, prepare=False)  # the pair (ref, tars[-1]) is still set and prepared
    assert_same(after, before, "pair call after a re-seeding series call")


def test_reseed_dev_matches_host(engine, lossy):
    torch = pytest.importorskip("torch")
    icgn2 = sc.Method("icgn", 2)
    ref, tars, xy, _ = lossy
    seeds = sc.fftcc_seeds(engine, ref, tars[0], xy, 16)
    engine.set_series_2d(ref, tars)
    host, host_counts = icgn2.series_reseed(engine, seeds, 20, 16, 0.9)
    assert host_counts.sum() > 0
    d_ref, d_tars, d_seeds = (torch.from_numpy(a).cuda() for a in (ref, tars, seeds))
    d_out = torch.empty((len(tars), len(seeds), 25), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    engine.set_series_2d_dev(d_ref.data_ptr(), d_tars.data_ptr(), len(tars), W, H)
    counts = icgn2.series_reseed_dev(engine, d_seeds.data_ptr(), d_out.data_ptr(), len(seeds), 20, 16, 0.9)
    assert_same(d_out.cpu().numpy(), host, "device-pointer variant")
    assert np.array_equal(counts, host_counts)
    assert_same(d_seeds.cpu().numpy(), seeds, "device seeds changed")


def test_reseed_group(lossy):
    if _capi.load().ocb_device_count() < 2:
        pytest.skip("needs two GPUs")
    ref, tars, xy, _ = lossy
    single = ob.Engine(0)
    seeds = sc.fftcc_seeds(single, ref, tars[0], xy, 16)
    single.set_series_2d(ref, tars)
    expect, expect_counts = ICGN1.series_reseed(single, seeds, 16, 16, 0.9)
    group = ob.Engine([0, 1])
    group.set_series_2d(ref, tars)
    got, counts = ICGN1.series_reseed(group, seeds, 16, 16, 0.9)
    assert_same(got, expect, "group context")
    assert np.array_equal(counts, expect_counts)
    group.close()
    single.close()
