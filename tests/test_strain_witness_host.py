"""CPU only: the grid-free float64 witness of tests/strain_cases.py against the oracle's Strain, on every generated case.  Both
solve in float64 and round once to float, so the same POIs must be fitted and strains must agree to 2 float32 ulps (of the
largest strain of the POI); a disagreement is a bug in one of them.  This pins the witness before test_gpu_strain_geometry.py
holds the GPU to it."""
import numpy as np
import pytest

from oracle import oracle
import strain_cases as sc

CASES = {c.name: c for c in sc.small_cases()}


def _pin(c, approximation, only=None):
    w = sc.witness(c.q, c.radius, c.k_min, c.thr, approximation, only=only)
    o = oracle.strain(c.q.copy(), c.radius, c.k_min, c.thr, approximation, exact=True, only=only)
    n, _ = sc.compare(o, c.q, w, np.inf, c.name)
    sl = sc.layout(c.q)["strain"]
    idx = np.flatnonzero(w.computed)
    a, b = o[idx, sl].astype(np.float64), w.out[idx, sl].astype(np.float64)
    ulp = np.spacing(np.maximum(np.abs(a), np.abs(b)).max(1, keepdims=True).astype(np.float32)).astype(np.float64)
    d = np.abs(a - b) / ulp
    for t, i in enumerate(idx):
        if int(i) in w.alts:
            d[t] = np.min(np.abs(a[t] - w.alts[int(i)]) / ulp[t], 0)  # the oracle may take either branch, per field as well
    assert len(idx) == 0 or d.max() <= 2, (c.name, idx[np.argmax(d.max(1))], d.max())
    return n, w


@pytest.mark.parametrize("approximation", [1, 2])
@pytest.mark.parametrize("name", sorted(CASES))
def test_witness_matches_oracle(name, approximation):
    c = CASES[name]
    n, w = _pin(c, approximation)
    assert n == int(w.computed.sum())


def test_cases_reach_their_edges():
    """The generators build what their names promise."""
    for name in ("cell_boundary_2_r20", "cell_boundary_3_r7.5", "cell_boundary_23_r1"):
        c = CASES[name]
        w = sc.witness(c.q, c.radius, c.k_min, c.thr, 1)
        assert w.computed.sum() > 0.8 * len(c.q)
        r2 = np.float32(np.float32(c.radius) ** 2)
        D = 3 if c.q.shape[1] == 31 else 2
        d = sc.dist2(c.q[:, None, :D], c.q[None, :, :D])
        assert (d == r2).sum() >= 8 and ((d < r2) & (d >= r2 * np.float32(1 - 1e-6))).sum() >= 8, name  # on the radius, a few ulps in
    for k in (6, 7, 9, 10, 13):  # the POI itself, then shells of 4, 4, 4 and 8: k = 6, 7 and 10 cut a shell, 9 and 13 close one
        c = CASES["lattice2_k%d" % k]
        pos = c.q[:, :2]
        centre = np.argmin(np.abs(pos - pos.mean(0)).sum(1))
        d = np.sort(sc.dist2(pos[centre], pos))
        assert (d[k - 1] == d[k]) == (k in (6, 7, 10)), k
    assert len(sc.witness(CASES["rank_diagonal_2"].q, 9.0, 3, 0.9).alts) > 0
    assert sc.witness(CASES["fallback_low_zncc_2"].q, 20.0, 6, 0.9).fallback.sum() > 500


@pytest.mark.parametrize("approximation", [0, 3])
def test_other_approximations_write_nothing(approximation):
    c = CASES["box_pm300_2"]
    o = oracle.strain(c.q.copy(), c.radius, c.k_min, c.thr, approximation, exact=True)
    assert np.array_equal(sc.bits(o), sc.bits(c.q))


@pytest.mark.parametrize("name", ["nonfinite_2", "nonfinite_3", "fallback_low_zncc_2", "rank_duplicates_3"])
def test_single_poi_matches_oracle(name):
    c = CASES[name]
    z = sc.layout(c.q)["zncc"][0]
    rng = np.random.default_rng(0)
    for i in [0, len(c.q) - 1, int(np.argmin(c.q[:, z]))] + rng.integers(0, len(c.q), 4).tolist():
        _pin(c, 2, only=i)


def test_negative_radius_is_its_magnitude():
    for kind in (2, 3, 23):
        c = CASES["radius_%d_-20" % kind]
        a = oracle.strain(c.q.copy(), -20.0, 5, 0.9, 1, exact=True)
        b = oracle.strain(c.q.copy(), 20.0, 5, 0.9, 1, exact=True)
        assert np.array_equal(sc.bits(a), sc.bits(b))
