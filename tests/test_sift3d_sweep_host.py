"""CPU: the float64 matching witness (tests/sift3d_match_witness.py) pinned to the oracle's monodirectionalMatch on hand-built
descriptor sets, and every SWEEP case of sift3d_cases.py reaching its branch on the oracle alone, with the match split evaluated
for an H100's 132 SMs.  A case that stops reaching its branch fails here, before it runs on a GPU."""
import numpy as np
import pytest

import sift3d_cases as sc
import sift3d_match_witness as wit
from oracle import sift3d as s3


def _unit_rows(rng, n):
    d = rng.random((n, 768)).astype(np.float32)
    return (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)


def _pin(d1, d2, ratio):
    """witness == oracle: the same pairs in the same order, no marginal row; returns the pairs"""
    pairs, top2, _ = s3.match(d1, d2, ratio)
    got, info = wit.match(d1, d2, ratio)
    assert not info["marginal"].any(), np.nonzero(info["marginal"])[0]
    assert np.array_equal(got, pairs.astype(np.int64)), (got.tolist(), pairs.tolist())
    assert np.array_equal(info["index0"], top2[:, 1].astype(np.int64))
    return got


def _near(base, rng, scale):
    d = base + scale * rng.standard_normal(base.shape).astype(np.float32)
    return np.abs(d).astype(np.float32)


def test_witness_ties_keep_the_first_index():
    rng = np.random.default_rng(11)
    t = _unit_rows(rng, 200)
    t[150] = t[20]  # a tie across 64-column tiles
    t[23] = t[20]  # and within one
    # rows near t[20], t[40], t[60], and one equal to t[20]: d0 = d1 = 0 fails the test at any ratio, so that the others,
    # which pass at 1.2, are returned
    r = np.concatenate([_near(t[[20, 40, 60]], rng, 1e-3), t[[20]]])
    pairs = _pin(r, t, 1.2)
    info = wit.match(r, t, 1.2)[1]
    assert info["index0"][0] == 20 and info["d0"][0] == info["d1"][0] > 0
    assert info["index0"][3] == 20 and info["d0"][3] == info["d1"][3] == 0
    assert pairs.tolist() == [[2, 60], [1, 40], [0, 20]]


def test_witness_empty_and_single_target():
    rng = np.random.default_rng(12)
    r = _unit_rows(rng, 5)
    for ratio in (0.85, 1.0, 1.2):
        assert len(_pin(r, np.zeros((0, 768), np.float32), ratio)) == 0  # n2 = 0: nothing, at every ratio
    one = _unit_rows(rng, 1)
    # n2 = 1: d1 stays FLT_MAX, every row passes, and so nothing is returned (:1309-1317) ...
    assert len(_pin(r, one, 0.85)) == 0
    # ... unless a row fails: a NaN component makes its distance NaN, which the scan never keeps.  The other four form one
    # many-to-one run on target 0, which keeps the row next to it
    r[2, 5] = np.nan
    r[0] = _near(one, rng, 1e-3)[0]
    assert _pin(r, one, 0.85).tolist() == [[0, 0]]


def test_witness_quirks():
    rng = np.random.default_rng(13)
    t = _unit_rows(rng, 300)
    r = _near(t[rng.permutation(300)[:120]], rng, 0.02)
    # every row passes at ratio 1.2: nothing returned; no row passes at NaN
    assert len(_pin(r, t, 1.2)) == 0 and len(_pin(r, t, float("nan"))) == 0
    # many-to-one runs: rows near the same target, only the nearest of each run survives and the run's first slot carries it
    between = 0.51 * t[100:110] + 0.49 * t[200:210]  # nearer t[100 + k], but d0 / d1 = 0.92 fails the test
    r3 = np.concatenate([r, _near(t[[5, 5, 5, 9]], rng, 0.01), between])
    pairs = _pin(r3, t, 0.95)
    tars = pairs[:, 1]
    assert len(tars) == len(set(tars.tolist())) and np.all(np.diff(tars) < 0)


@pytest.mark.parametrize("name", list(sc.SWEEP))
def test_sweep_case_reaches_its_branch(name):
    print(sc.reach(name, sc.SPLIT_SM))
