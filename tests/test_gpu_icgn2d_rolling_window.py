"""icgn2d.cu's sampling loop keeps each lane's 4x4 pixel block in registers and reads only the new bottom row when a row's
block is the previous one moved down a pixel row; other rows reload the whole block.  On sheared and stretched guesses most
batches of rows reload, and every record must stay byte-identical (compared as uint32, so NaNs compare too) to the records
of a library that reads the full block at every sample, recorded in tests/golden/icgn2d_rolling_window_parent.npz by
tests/golden/make_icgn2d_rolling_window_golden.py.  The cases are listed in tests/rolling_window_cases.py."""
import os

import numpy as np
import pytest

import opencorr_b200 as ob
import rolling_window_cases as rw

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "icgn2d_rolling_window_parent.npz")
IMAGES = os.path.join(HERE, "golden", "icgn2d_whole_pixel_parent.npz")


@pytest.fixture(scope="module")
def fixture():
    return dict(np.load(GOLDEN))


@pytest.fixture(scope="module")
def images():
    return dict(np.load(IMAGES))


@pytest.mark.parametrize("name", list(rw.CASES))
def test_first_pass_reloads(fixture, name):
    """The guesses keep most first passes on the branch-free loop, and most of those passes have batches that reload, so the
    records below depend on the reload path and on the rolling one alike."""
    seeds = ob.make_poi2d(rw.CASES[name][5])
    seeds[:, [2, 8]] = fixture[name + "_seed_uv"]
    steps = rw.first_pass_steps(seeds, name)
    assert len(steps) >= 0.5 * len(seeds), "%s: only %d of %d first passes take the branch-free loop" % (name, len(steps), len(seeds))
    assert (steps[:, 1] > 0).mean() >= 0.5, name + ": too few first passes reload"
    assert (steps[:, 1] < steps[:, 2]).mean() >= 0.3, name + ": too few first passes keep the rolling window"


def test_fixture_keeps_pois(fixture):
    for name in rw.CASES:
        z = fixture[name][:, 16]
        assert (z >= 0).sum() >= 0.5 * len(z), name


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(rw.CASES))
def test_records_byte_identical(engine, fixture, images, name):
    s, q = rw.run(engine, images, name)
    assert np.array_equal(s[:, [2, 8]], fixture[name + "_seed_uv"]), name + ": FFT-CC seeds differ from the fixture's"
    want = fixture[name]
    differ = np.flatnonzero((q.view(np.uint32) != want.view(np.uint32)).any(1))
    assert len(differ) == 0, "%s: %d of %d records differ, first POIs %s\ngot  %s\nwant %s" % (
        name, len(differ), len(q), differ[:8].tolist(), q[differ[0]].tolist(), want[differ[0]].tolist())
