"""GPU: Strain (strain.cu) held to the grid-free float64 witness of tests/strain_cases.py at the geometry the kernel's uniform
grid has to get right: POIs on both sides of computed cell edges with neighbours one ulp inside and exactly on the radius,
negative, mixed-sign and signed-zero coordinates, zero extent, grids that must grow their cell, queues longer than the kernels'
thread grids, k-nearest ties on lattices, rank-deficient fits, edge values of the radius and the threshold, and every entry
point.  For every case the set of fitted POIs is exactly the witness's, strains agree within 2e-6 (POI2D, POI3D) or 1e-5 (POI2DS:
ill-conditioned 3D fit coordinates, as in test_gpu_nr_strain.py), and every other field is bit-identical to the input."""
import ctypes

import numpy as np
import pytest

import opencorr_b200 as ob
from opencorr_b200 import _capi
import strain_cases as sc

pytestmark = pytest.mark.gpu

TOL = {25: 2e-6, 31: 2e-6, 28: 1e-5}
CASES = {c.name: c for c in sc.small_cases()}


def _strain(engine, q, c, approximation=1):
    got = q.copy()
    engine.strain(got, c.radius, c.k_min, c.thr, approximation)
    return got


def _check(engine, c, approximation=1, q=None, subset=None):
    q = c.q if q is None else q
    got = _strain(engine, q, c, approximation)
    w = sc.witness(q, c.radius, c.k_min, c.thr, approximation, subset=subset)
    n, d = sc.compare(got, q, w, TOL[q.shape[1]], c.name)
    print("%s approx=%d: %d POIs, %d fitted, %d by k-nearest, %d non-decisive, max |de| %.2e" % (
        c.name, approximation, len(q), n, int((w.fallback & w.computed).sum()), len(w.alts), d))
    return got, w


def _sm_count():
    torch = pytest.importorskip("torch")
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("approximation", [1, 2])
@pytest.mark.parametrize("name", sorted(CASES))
def test_case(engine, name, approximation):
    _check(engine, CASES[name], approximation)


def test_negative_radius_is_its_magnitude(engine):
    for kind in (2, 3, 23):
        c = CASES["radius_%d_-20" % kind]
        a = _strain(engine, c.q, c)
        b = _strain(engine, c.q, c._replace(radius=20.0))
        assert np.array_equal(sc.bits(a), sc.bits(b)), kind


@pytest.mark.parametrize("approximation", [0, 3])
def test_other_approximations_write_nothing(engine, approximation):
    for name in ("box_pm300_2", "box_pm300_3", "box_pm300_23"):
        c = CASES[name]
        assert np.array_equal(sc.bits(_strain(engine, c.q, c, approximation)), sc.bits(c.q))


# ------------------------------------------------------------------------------------------------ queue length
@pytest.mark.parametrize("kind", [2, 3])
def test_queue_longer_than_the_resident_warps(engine, kind):
    """More valid POIs than the 8 x SM-count blocks of 8 warps: the warp-stride loop of strain_kernel runs."""
    n = 64 * _sm_count() + 777
    if kind == 2:
        c = sc.uniform(2, n, np.sqrt(n * np.pi * 400 / 10.0), 20.0, seed=21)
    else:
        c = sc.uniform(3, n, (n * 4 / 3 * np.pi * 1000 / 10.0) ** (1 / 3), 10.0, seed=22)
    c.q[[0, -1], 0] = np.nan  # non-finite POIs sort last: the valid count is less than n
    _check(engine, c, 1)


def _fallback_and_sample(q, radius, k_min, seed, size=5000):
    from scipy.spatial import cKDTree
    pos = q[:, :2].astype(np.float64)
    fin = np.flatnonzero(np.isfinite(pos).all(1))
    cnt = cKDTree(pos[fin]).query_ball_point(pos[fin], radius * 1.001, return_length=True)
    fb = fin[cnt < k_min + 2]
    rng = np.random.default_rng(seed)
    return np.union1d(fb, rng.choice(len(q), size, replace=False)), len(fb)


def test_queue_longer_than_the_thread_grid(engine):
    """More POIs than the bbox, keys and gather kernels' 8 x SM-count blocks of 256 threads; checked on every k-nearest POI and a
    seeded sample, then once more on the same queue shuffled (ties go to the lower original index, so the two runs differ)."""
    n = 2048 * _sm_count() + 4099
    c = sc.uniform(2, n, np.sqrt(n * np.pi * 400 / 12.0), 20.0, seed=23)
    c.q[[0, n // 2, n - 1], 1] = np.inf
    subset, n_fb = _fallback_and_sample(c.q, 20.0, 5, 0)
    assert n_fb > 200
    got, w = _check(engine, c, 1, subset=subset)
    assert (w.fallback & w.checked).sum() > 200
    perm = np.random.default_rng(1).permutation(n)
    shuffled = c.q[perm].copy()
    inv = np.argsort(perm)
    _check(engine, c, 2, q=shuffled, subset=inv[subset])


# ------------------------------------------------------------------------------------------------ entry points
def _dev_call(engine, kind, d, n, c, approximation):
    fn = {2: engine._lib.ocb_strain2d_dev, 3: engine._lib.ocb_strain3d_dev, 23: engine._lib.ocb_strain2ds_dev}[kind]
    return fn(engine._ctx, ctypes.c_void_p(d.data_ptr()), n, float(c.radius), int(c.k_min), float(c.thr), int(approximation))


@pytest.mark.parametrize("kind", [2, 3, 23])
def test_device_pointer_entry_points(engine, kind):
    torch = pytest.importorskip("torch")
    for name in ("nonfinite_%d" % kind, "cell_boundary_%d_r7.5" % kind):
        c = CASES[name]
        host = _strain(engine, c.q, c, 2)
        d = torch.from_numpy(c.q.copy()).cuda()
        torch.cuda.synchronize()
        assert _dev_call(engine, kind, d, len(c.q), c, 2) == _capi.OCB_OK, _capi.last_error(engine._ctx)
        engine.sync()
        assert np.array_equal(sc.bits(d.cpu().numpy()), sc.bits(host)), name


@pytest.mark.parametrize("kind", [2, 3])
def test_single_poi_on_the_sweeps(engine, kind):
    """Strain::compute(POI*, queue) on centres of the boundary sweep, a k-nearest POI and a POI below the threshold."""
    fn = engine._lib.ocb_strain2d_single if kind == 2 else engine._lib.ocb_strain3d_single
    for name in ("cell_boundary_%d_r1" % kind, "fallback_low_zncc_%d" % kind):
        c = CASES[name]
        z = sc.layout(c.q)["zncc"][0]
        w = sc.witness(c.q, c.radius, c.k_min, c.thr, 1)
        picks = [1, 2, len(c.q) - 1, int(np.flatnonzero(w.fallback)[0]), int(np.argmin(c.q[:, z]))]
        for i in picks:
            got = c.q.copy()
            rc = fn(engine._ctx, ctypes.c_void_p(got.ctypes.data), len(got), i, float(c.radius), int(c.k_min), float(c.thr), 1)
            assert rc == _capi.OCB_OK, _capi.last_error(engine._ctx)
            sc.compare(got, c.q, sc.witness(c.q, c.radius, c.k_min, c.thr, 1, only=i), TOL[c.q.shape[1]], "%s only=%d" % (name, i))


def test_group_context(engine):
    """A group context runs Strain on its first member: the records are those of a single-device context."""
    n_dev = _capi.load().ocb_device_count()
    grp = ob.Engine(list(range(n_dev)))
    try:
        for name in ("growth_2d_xy", "cell_boundary_3_r20", "nonfinite_23"):
            c = CASES[name]
            a = _strain(engine, c.q, c, 2)
            b = _strain(grp, c.q, c, 2)
            assert np.array_equal(sc.bits(a), sc.bits(b)), name
        print("group context: %d member(s)" % n_dev)
    finally:
        grp.close()
