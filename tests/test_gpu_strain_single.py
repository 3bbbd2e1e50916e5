"""GPU: Strain's single-POI overloads, Strain::compute(POI2D*, queue) / (POI3D*, queue) (include/opencorr/opencorr.h,
ocb_strain2d_single / ocb_strain3d_single), against the queue call and the float64 oracle's single-POI mode.

The selected POI is processed whatever its own ZNCC, as in the reference (src/oc_strain.cpp:158-237, :373-474): its neighbours
still have to pass the threshold.  Every byte outside that POI's strain fields must be left alone."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import opencorr_b200 as ob
from opencorr_b200 import _capi
from oracle import oracle

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RADIUS, K, THR = 20.0, 5, 0.9
TOL = 2e-6  # FP64 normal equations vs FP64 Householder QR, as in test_gpu_nr_strain.py


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _single(engine, dim, q, index, approximation):
    fn = engine._lib.ocb_strain2d_single if dim == 2 else engine._lib.ocb_strain3d_single
    fn.restype = ctypes.c_int
    fn.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_float, ctypes.c_int, ctypes.c_float, ctypes.c_int]
    return fn(engine._ctx, ctypes.c_void_p(q.ctypes.data), q.shape[0], index, RADIUS, K, THR, approximation)


def make_queue(dim, seed=1):
    """A dense patch, an isolated POI (k-nearest fallback), a cluster whose neighbours mostly fail the threshold, a NaN POI.
    Returns (queue, named indices, ZNCC column, strain columns)."""
    rng = np.random.default_rng(seed)
    n, extent = 300, 150.0 if dim == 2 else 60.0
    pts = [rng.uniform(0, extent, (n, dim))]
    lone = np.full(dim, 400.0)
    d = rng.normal(size=(6, dim))
    ring = lone + d / np.linalg.norm(d, axis=1, keepdims=True) * rng.uniform(25, 45, (6, 1))   # outside the radius
    few = np.full(dim, 600.0) + rng.uniform(-4, 4, (6, dim))                                   # six within the radius, four below THR
    pts += [lone[None], ring, few, np.full((1, dim), 50.0), rng.uniform(0, extent, (1, dim))]
    xyz = np.concatenate(pts).astype(np.float32)
    if dim == 2:
        q = ob.make_poi2d(xyz)
        q[:, 2] = 0.01 * xyz[:, 0] - 0.002 * xyz[:, 1] + rng.normal(0, 0.01, len(q))
        q[:, 8] = 0.003 * xyz[:, 0] + 0.02 * xyz[:, 1] + rng.normal(0, 0.01, len(q))
        zc, sc = 16, slice(20, 23)
    else:
        q = ob.make_poi3d(xyz)
        q[:, 3], q[:, 7], q[:, 11] = (xyz @ rng.normal(0, 0.01, (3, 3)) + rng.normal(0, 0.01, (len(q), 3))).T
        zc, sc = 18, slice(22, 28)
    q[:, zc] = rng.uniform(0.91, 1.0, len(q))
    q[:n:7, zc] = rng.uniform(0.5, 0.89, len(q[:n:7]))
    i_lone, i_few = n, n + 7
    q[i_few + 1:i_few + 5, zc] = 0.5
    i_nan = len(q) - 2
    q[i_nan, 1] = np.nan
    good = np.flatnonzero(q[:n, zc] >= THR)
    idx = dict(good=int(good[len(good) // 2]), low=int(np.flatnonzero(q[:n, zc] < THR)[3]), knn=i_lone, few=i_few, nan=i_nan, first=0,
               last=len(q) - 1)
    q[-1, zc] = 0.3  # the last POI is below the threshold too
    return q, idx, zc, sc


@pytest.mark.parametrize("dim", [2, 3])
@pytest.mark.parametrize("approximation", [1, 2])
def test_single_poi(engine, dim, approximation):
    q, idx, zc, sc = make_queue(dim, seed=dim + 10 * approximation)
    full = q.copy()
    s = ob.Strain(RADIUS, K, engine=engine)
    s.set_zncc_threshold(THR)
    s.set_approximation(approximation)
    s.compute(full)
    for name, i in idx.items():
        got = q.copy()
        assert _single(engine, dim, got, i, approximation) == _capi.OCB_OK, _capi.last_error(engine._ctx)
        ref = oracle.strain(q.copy(), RADIUS, K, THR, approximation, exact=True, only=i)
        others = np.delete(np.arange(len(q)), i)
        assert np.array_equal(_bits(got[others]), _bits(q[others])), "%s: another POI changed" % name
        outside = np.delete(np.arange(q.shape[1]), np.arange(sc.start, sc.stop))
        assert np.array_equal(_bits(got[i, outside]), _bits(q[i, outside])), "%s: a field other than the strain changed" % name
        computed = bool(np.any(got[i, sc] != 0))
        assert computed == bool(np.any(ref[i, sc] != 0)), name
        d = np.abs(got[i, sc] - ref[i, sc]).max()
        assert d < TOL, (name, d)
        if q[i, zc] >= THR and np.isfinite(q[i, :dim]).all():
            assert np.array_equal(_bits(got[i]), _bits(full[i])), "%s: differs from the queue call" % name
        print("dim=%d approx=%d %s (POI %d, ZNCC %.2f): computed=%s max|de| vs oracle=%.2e" % (dim, approximation, name, i, q[i, zc], computed, d))
        expect = dict(good=True, low=True, knn=True, few=False, nan=False, first=True, last=True)[name]
        assert computed == expect, name
        if name in ("low", "last"):
            assert np.all(full[i, sc] == 0)  # the queue call skips it
    bad = q.copy()
    assert _single(engine, dim, bad, len(q), approximation) == _capi.OCB_ERR_ARG
    assert np.array_equal(_bits(bad), _bits(q))


def test_shim_single_overload(engine, tmp_path):
    """Strain::compute(POI2D*, queue) of the C++ shim is the ctypes call."""
    exe = tmp_path / "strain_single_shim_test"
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    lib = os.path.join(ROOT, "opencorr_b200", "lib")
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-fopenmp", "-I" + os.path.join(ROOT, "include", "opencorr"), "-o", str(exe),
                           os.path.join(ROOT, "tests", "native", "strain_single_shim_test.cpp"), "-L" + lib, "-lopencorr_b200", "-Wl,-rpath," + lib])
    q, idx, _, _ = make_queue(2, seed=5)
    (tmp_path / "in.bin").write_bytes(q.tobytes())
    for name in ("low", "good"):
        out = subprocess.run([str(exe), str(tmp_path / "in.bin"), str(tmp_path / "out.bin"), str(idx[name]), str(RADIUS), str(K), str(THR), "2"],
                             capture_output=True, text=True, timeout=300)
        assert out.returncode == 0, out.stderr
        shim = np.frombuffer((tmp_path / "out.bin").read_bytes(), np.float32).reshape(q.shape)
        got = q.copy()
        assert _single(engine, 2, got, idx[name], 2) == _capi.OCB_OK
        assert np.any(got[idx[name], 20:23] != 0)
        assert np.array_equal(_bits(shim), _bits(got)), name
