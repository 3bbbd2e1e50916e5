"""CPU only: the grid-free float64 RegionFit witness of tests/region_fit_cases.py against the oracle's RegionFit on every case.
The exact (float64) oracle must write the same POIs and agree to 1e-9 of the POI's largest written value, or one float32
rounding of it (both solve in float64 and round once); the faithful float32 oracle -- the reference's
Eigen::MatrixXf arithmetic -- must write the same POIs and stay within FAITHFUL_TOL, its measured worst case over these cases
(2.4e-3 of a value's magnitude above 1, on k-nearest fits far outside the reliable set, where float32 offsets of hundreds
of pixels cost the QR its precision) with a margin of four.  This pins the witness before
test_gpu_region_fit.py holds the GPU to it."""
import numpy as np
import pytest

from oracle import region_fit as oracle
import region_fit_cases as rc
import strain_cases as sc

CASES = {c.name: c for c in rc.small_cases()}
FAITHFUL_TOL = 1e-2


def _oracle(c, exact):
    return oracle.region_fit(c.rel.copy(), c.q.copy(), c.radius, c.k_min, exact=exact)


@pytest.mark.parametrize("name", sorted(CASES))
def test_witness_matches_exact_oracle(name):
    c = CASES[name]
    w = rc.witness(c.rel, c.q, c.radius, c.k_min)
    o = _oracle(c, True)
    n, _ = rc.compare(o, c.q, w, np.inf, name)
    assert n == int(w.computed.sum())
    idx = np.flatnonzero(w.computed)
    fields = list(rc.layout(c.q)["fields"])
    a, b = o[idx][:, fields].astype(np.float64), w.out[idx][:, fields].astype(np.float64)
    scale = np.maximum(np.abs(a), np.abs(b)).max(1, keepdims=True)
    allowed = np.maximum(1e-9 * scale, np.spacing(scale.astype(np.float32)).astype(np.float64))
    d = np.abs(a - b) / allowed
    for t, i in enumerate(idx):
        if int(i) in w.alts:  # the oracle may take either branch of a near tie
            d[t] = np.min(np.abs(a[t] - w.alts[int(i)]) / allowed[t], 0)
    assert len(idx) == 0 or d.max() <= 1, (name, idx[np.argmax(d.max(1))], d.max())


@pytest.mark.parametrize("name", sorted(CASES))
def test_faithful_oracle_within_bound(name):
    c = CASES[name]
    w = rc.witness(c.rel, c.q, c.radius, c.k_min)
    rc.compare(_oracle(c, False), c.q, w, FAITHFUL_TOL, name)


def test_cases_reach_their_edges():
    """The generators build what their names promise."""
    c = CASES["outside_2_r10"]
    w = rc.witness(c.rel, c.q, c.radius, c.k_min)
    lo, hi = c.rel[:, :2].min(0), c.rel[:, :2].max(0)
    out = ~((c.q[:, :2] >= lo) & (c.q[:, :2] <= hi)).all(1)
    # queries outside the box that find neighbours within the radius, and queries that fall back
    assert (out & w.computed & ~w.fallback).sum() > 20 and (out & w.fallback).sum() > 10
    for name in ("cell_boundary_2_r20", "cell_boundary_3_r7.5"):
        c = CASES[name]
        D = 3 if c.q.shape[1] == 31 else 2
        r2 = np.float32(np.float32(c.radius) ** 2)
        d = sc.dist2(c.q[:, None, :D], c.rel[None, :, :D])
        assert (d == r2).sum() >= 8 and ((d < r2) & (d >= r2 * np.float32(1 - 1e-6))).sum() >= 8, name
    for name in ("knn_2_n6_k9", "knn_3_n9_k12"):  # fewer reliable POIs than k_min: nothing is written
        c = CASES[name]
        assert not rc.witness(c.rel, c.q, c.radius, c.k_min).computed.any(), name
    for name in ("knn_2_n9_k9", "knn_3_n16_k12", "empty_reliable_2_k0", "kmin_nan_radius_3_0", "reliable_all_nonfinite_2_k0"):
        c = CASES[name]
        w = rc.witness(c.rel, c.q, c.radius, c.k_min)
        assert w.computed.sum() == np.isfinite(c.q[:, :2]).all(1).sum(), name
    assert not rc.witness(CASES["empty_reliable_3_k5"].rel, CASES["empty_reliable_3_k5"].q, 10.0, 5).computed.any()
    assert len(rc.witness(CASES["rank_diagonal_2"].rel, CASES["rank_diagonal_2"].q, 9.0, 3).alts) > 0


def test_negative_radius_is_its_magnitude():
    for D in (2, 3):
        c = CASES["radius_%d_-12" % D]
        a = oracle.region_fit(c.rel.copy(), c.q.copy(), -12.0, 5, exact=True)
        b = oracle.region_fit(c.rel.copy(), c.q.copy(), 12.0, 5, exact=True)
        assert np.array_equal(sc.bits(a), sc.bits(b))
