"""The r = 16 IC-GN kernel samples its tail column (the 33rd) without per-sample tests when the pass's corner test holds.
Guesses that put every tail sample's support against the staged tile's right edge must give records byte-identical (compared
as uint32) to those of a library that tests each tail sample, recorded in tests/golden/icgn2d_tail_edge_parent.npz by
tests/golden/make_icgn2d_tail_edge_golden.py.  The cases are described in tests/tail_edge_cases.py."""
import os

import numpy as np
import pytest

import opencorr_b200 as ob
import tail_edge_cases as te

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "icgn2d_tail_edge_parent.npz")
IMAGES = os.path.join(HERE, "golden", "icgn2d_whole_pixel_parent.npz")


@pytest.fixture(scope="module")
def fixture():
    return dict(np.load(GOLDEN))


def test_guesses_reach_tile_edge(fixture):
    """Most POIs get a guess whose first pass passes the corner test with the tail's support on the tile's last column, and
    most of those POIs are kept, so the records depend on the tail samples."""
    seeds = ob.make_poi2d(te.XY)
    seeds[:, [2, 8]] = fixture["seed_uv"]
    q, edge = te.guess(seeds)
    assert edge.mean() >= 0.8
    for k in np.flatnonzero(edge):
        cx = float(q[k, 0]) + float(q[k, 2])
        xlo, xhi = te.tile_x(cx)
        x_tail = cx + (1.0 + float(q[k, 3])) * te.R
        assert np.floor(x_tail) + 2 == xhi + 1 and cx - (1.0 + float(q[k, 3])) * te.R >= xlo
    assert (fixture["records"][edge, 16] >= 0).mean() >= 0.8


@pytest.mark.gpu
def test_records_byte_identical(engine, fixture):
    s, q, _ = te.run(engine, dict(np.load(IMAGES)))
    assert np.array_equal(s[:, [2, 8]], fixture["seed_uv"]), "FFT-CC seeds differ from the fixture's"
    want = fixture["records"]
    differ = np.flatnonzero((q.view(np.uint32) != want.view(np.uint32)).any(1))
    assert len(differ) == 0, "%d of %d records differ, first POIs %s\ngot  %s\nwant %s" % (
        len(differ), len(q), differ[:8].tolist(), q[differ[0]].tolist(), want[differ[0]].tolist())
