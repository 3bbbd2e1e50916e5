"""IC-LM over an image series (ocb_iclm2d_series, ocb_iclm2d_series_reseed): every frame's records must be, bit for bit, what the
loop of pair calls
    set_images_2d(ref, tars[f]); icgn2d_prepare(); iclm2d(order, q, ..., damping)
gives when one queue q is carried from frame to frame, with the warps per POI forced (OCB_ICGN2D_WPP) so that the pair calls
split their sums as the series launch over all POIs does."""
import pytest

from opencorr_b200 import _capi
import subset_series_cases as sc

pytestmark = pytest.mark.gpu

W_TMA, W_GATHER, H = 384, 387, 320  # 387 % 4 != 0: the frames of the stack are not 16-byte aligned, so tiles are gathered


@pytest.fixture(scope="module")
def stacks():
    return {(w, o): sc.render_series(w, H, 5, second_order=o == 2) for w in (W_TMA, W_GATHER) for o in (1, 2)}


@pytest.mark.parametrize("staging", ["tma", "gather"])
@pytest.mark.parametrize("wpp", ["1", "2"])
@pytest.mark.parametrize("r", [12, 16, 20, 23])
@pytest.mark.parametrize("order", [1, 2])
def test_series_equals_pair_loop(engine, stacks, monkeypatch, order, r, wpp, staging):
    monkeypatch.setenv("OCB_ICGN2D_WPP", wpp)
    ref, tars = stacks[(W_TMA if staging == "tma" else W_GATHER, order)]
    damping = sc.OTHER_DAMPING if r == 20 else sc.DAMPING
    sc.check_equals_pair_loop(engine, sc.Method("iclm", order, damping), ref, tars, sc.short_grid(), r, "r %d wpp %s %s" % (r, wpp, staging))


@pytest.mark.parametrize("order,r", [(1, 16), (2, 20)])
def test_series_equals_pair_loop_long_queue(engine, stacks, monkeypatch, order, r):
    """7840 POIs: one warp per POI, persistent warps pulling POIs from the queue"""
    monkeypatch.setenv("OCB_ICGN2D_WPP", "1")
    ref, tars = stacks[(W_TMA, order)]
    sc.check_equals_pair_loop(engine, sc.Method("iclm", order), ref, tars, sc.long_grid(r), r, "long queue")


@pytest.mark.parametrize("order", [1, 2])
def test_series_sentinels(engine, stacks, monkeypatch, order):
    monkeypatch.setenv("OCB_ICGN2D_WPP", "1")
    ref, tars = stacks[(W_TMA, order)]
    sc.check_sentinels(engine, sc.Method("iclm", order), ref, tars, 16)


def test_series_chunks(engine, stacks):
    ref, tars = stacks[(W_TMA, 1)]
    sc.check_chunks(engine, sc.Method("iclm", 1), ref, tars, 16)


def test_series_errors_leave_out_untouched():
    sc.check_errors_leave_out_untouched(sc.Method("iclm", 1))


def test_pair_state_undisturbed(engine, stacks):
    ref, tars = stacks[(W_TMA, 1)]
    sc.check_pair_state_undisturbed(engine, sc.Method("iclm", 2), ref, tars, 16)


def test_series_dev_matches_host(engine, stacks):
    pytest.importorskip("torch")
    ref, tars = stacks[(W_GATHER, 2)]
    sc.check_dev_matches_host(engine, sc.Method("iclm", 2, sc.OTHER_DAMPING), ref, tars, 20)


def test_series_group(stacks):
    if _capi.load().ocb_device_count() < 2:
        pytest.skip("needs two GPUs")
    ref, tars = stacks[(W_TMA, 1)]
    sc.check_group(sc.Method("iclm", 1), ref, tars, 16)


@pytest.mark.parametrize("order,r", [(1, 16), (1, 23), (2, 20)])
def test_reseed_nothing_lost_equals_plain_series(engine, stacks, order, r):
    ref, tars = stacks[(W_TMA, order)]
    for grid in (sc.short_grid(), sc.long_grid(r)):
        sc.check_nothing_lost(engine, sc.Method("iclm", order), ref, tars, grid, r)


@pytest.fixture(scope="module")
def lossy():
    return sc.lossy_series()


@pytest.mark.parametrize("wpp", ["1", "2"])
@pytest.mark.parametrize("order", [1, 2])
def test_reseed_equals_pair_loop(engine, lossy, monkeypatch, order, wpp):
    monkeypatch.setenv("OCB_ICGN2D_WPP", wpp)
    sc.check_reseed_equals_pair_loop(engine, sc.Method("iclm", order), lossy, 16 if order == 1 else 20, 16)


@pytest.mark.parametrize("order,r", [(1, 16), (2, 20)])
def test_series_matches_oracle_and_ground_truth(engine, stacks, order, r):
    ref, tars = stacks[(W_TMA, order)]
    sc.check_oracle_and_ground_truth(engine, sc.Method("iclm", order), ref, tars, r, second_order=order == 2)
