"""NR2D1 over an image series (ocb_nr2d1_series, ocb_nr2d1_series_reseed): every frame's records must be, bit for bit, what the
loop of pair calls
    set_images_2d(ref, tars[f]); nr2d_prepare(); nr2d1(q, ...)
gives when one queue q is carried from frame to frame."""
import numpy as np
import pytest

from opencorr_b200 import _capi, synth
import subset_series_cases as sc
from util import assert_same

pytestmark = pytest.mark.gpu

W_TMA, W_GATHER, H = 384, 387, 320  # 387 % 4 != 0: the frames of the stack are not 16-byte aligned, so tiles are gathered
NR = sc.Method("nr")


@pytest.fixture(scope="module")
def stacks():
    return {w: sc.render_series(w, H, 5) for w in (W_TMA, W_GATHER)}


@pytest.mark.parametrize("staging", ["tma", "gather"])
@pytest.mark.parametrize("r", [12, 16, 23])
def test_series_equals_pair_loop(engine, stacks, staging, r):
    ref, tars = stacks[W_TMA if staging == "tma" else W_GATHER]
    sc.check_equals_pair_loop(engine, NR, ref, tars, sc.short_grid(), r, "r %d %s" % (r, staging))


def test_series_equals_pair_loop_long_queue(engine, stacks):
    ref, tars = stacks[W_TMA]
    sc.check_equals_pair_loop(engine, NR, ref, tars, sc.long_grid(16), 16, "long queue")


@pytest.mark.parametrize("staging", ["tma", "gather"])
def test_global_fallback_reads_the_frame(engine, staging):
    """A vertical stretch that grows frame by frame (0.03 per frame) carries the warped subsets of later frames past the staged
    tile, so those samples and their gradients come from global memory: from frame f, as the pair call on frame f reads them."""
    ref, tars = sc.render_series(W_TMA if staging == "tma" else W_GATHER, H, 5, vy_step=0.03)
    xy = synth.grid_2d(60, 70, 6, 4, 48, 48)
    sc.check_equals_pair_loop(engine, NR, ref, tars, xy, 16, "stretch %s" % staging)
    sc.check_oracle_and_ground_truth(engine, NR, ref, tars, 16, vy_step=0.03, bound=0.1)


def test_series_sentinels(engine, stacks):
    ref, tars = stacks[W_TMA]
    sc.check_sentinels(engine, NR, ref, tars, 16)


def test_failed_codes_follow_the_pair_guard(engine, stacks):
    """The guard writes -1; the -4 test runs on guarded records too, so a failed POI's code can change from frame to frame."""
    ref, tars = stacks[W_TMA]
    seeds = sc.fftcc_seeds(engine, ref, tars[0], sc.short_grid(), 16)
    seeds[0, 16] = -1.0
    seeds[1, 16], seeds[1, 17], seeds[1, 18] = -1.0, 20.0, 1.0  # at the iteration limit and not converged: -4 on every frame
    seeds[2, 8] = np.nan
    expect = sc.pair_loop(engine, NR, ref, tars, seeds, 16)
    engine.set_series_2d(ref, tars)
    got = NR.series(engine, seeds, 16)
    assert_same(got, expect, "failed seeds")
    assert (got[:, 0, 16] == -1).all() and (got[:, 1, 16] == -4).all() and (got[:, 2, 16] == -5).all()


def test_series_chunks(engine, stacks):
    ref, tars = stacks[W_TMA]
    sc.check_chunks(engine, NR, ref, tars, 16)


def test_series_errors_leave_out_untouched():
    sc.check_errors_leave_out_untouched(NR)


def test_pair_state_undisturbed(engine, stacks):
    ref, tars = stacks[W_TMA]
    sc.check_pair_state_undisturbed(engine, NR, ref, tars, 16)


def test_series_dev_matches_host(engine, stacks):
    pytest.importorskip("torch")
    ref, tars = stacks[W_GATHER]
    sc.check_dev_matches_host(engine, NR, ref, tars, 16)


def test_series_group(stacks):
    if _capi.load().ocb_device_count() < 2:
        pytest.skip("needs two GPUs")
    ref, tars = stacks[W_TMA]
    sc.check_group(NR, ref, tars, 16)


@pytest.mark.parametrize("r", [12, 16, 23])
def test_reseed_nothing_lost_equals_plain_series(engine, stacks, r):
    ref, tars = stacks[W_TMA]
    for grid in (sc.short_grid(), sc.long_grid(r)):
        sc.check_nothing_lost(engine, NR, ref, tars, grid, r)


@pytest.fixture(scope="module")
def lossy():
    return sc.lossy_series()


@pytest.mark.parametrize("fr", [16, 10, 7], ids=["fft_w32", "fft_reg", "fft_generic"])
def test_reseed_equals_pair_loop(engine, lossy, fr):
    sc.check_reseed_equals_pair_loop(engine, NR, lossy, 16, fr)


def test_series_matches_oracle_and_ground_truth(engine, stacks):
    ref, tars = stacks[W_TMA]
    sc.check_oracle_and_ground_truth(engine, NR, ref, tars, 16)
