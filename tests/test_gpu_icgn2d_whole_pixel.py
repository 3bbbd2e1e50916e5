"""Pass 1 of a POI seeded by FFT-CC samples the target at whole pixels, where the bicubic interpolant returns the pixel itself;
icgn2d.cu then reads the samples straight from the target tile.  Every record must stay byte-identical (compared as uint32, so
NaNs compare too) to the records of the full evaluation, recorded in tests/golden/icgn2d_whole_pixel_parent.npz by
tests/golden/make_icgn2d_whole_pixel_golden.py.  The cases are listed in tests/whole_pixel_cases.py."""
import os

import numpy as np
import pytest

import whole_pixel_cases as wp

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "icgn2d_whole_pixel_parent.npz")


@pytest.fixture(scope="module")
def fixture():
    return dict(np.load(GOLDEN))


def test_fixture_exercises_the_cases(fixture):
    """The cases reach what they are there for: POIs rejected at the border and kept, black-background POIs rejected by the
    negative-sample rule and kept, and the float target's three non-finite pixels."""
    z = fixture["icgn1_r16"][:, 16]
    assert (z == -3).sum() > 10 and (z >= 0).sum() > 280
    z = fixture["black1_r16"][:, 16]
    assert (z == -3).sum() > 100 and (z >= 0).sum() > 20
    e = fixture["float_edits"]
    assert np.isnan(e[0, 2]) and e[1, 2] == np.inf and e[2, 2] == -np.inf
    assert fixture["icgn1_r16_stop1"][:, 17].max() == 1 and fixture["icgn2_r20_stop1"][:, 17].max() == 1


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(wp.CASES))
def test_records_byte_identical(engine, fixture, name):
    s, q = wp.run(engine, fixture, name)
    assert np.array_equal(s[:, [2, 8]], fixture[name + "_seed_uv"]), name + ": FFT-CC seeds differ from the fixture's"
    want = fixture[name]
    differ = np.flatnonzero((q.view(np.uint32) != want.view(np.uint32)).any(1))
    assert len(differ) == 0, "%s: %d of %d records differ, first POIs %s\ngot  %s\nwant %s" % (
        name, len(differ), len(q), differ[:8].tolist(), q[differ[0]].tolist(), want[differ[0]].tolist())
