"""ctypes front-end of the stereo-reconstruction oracle (oracle/oc_stereo.cpp).

TEST INFRASTRUCTURE ONLY, like oracle.py: importable from tests/, __graft_entry__ and bench.py; the product package never imports it.

Intrinsics are the 13 floats of CameraIntrinsics (fx fy fs cx cy k1..k6 p1 p2), projections 3x4 row-major float32, points
float32 [n, 2] mutated in place (clamped) as the reference's Point2D& arguments are.
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "oc_stereo.cpp")
_LIB_PATH = os.path.join(_HERE, "liboc_stereo.so")
# the same arithmetic rules as oracle/Makefile: no fast-math, no FMA contraction
_CXXFLAGS = ["-O3", "-std=c++17", "-fPIC", "-fopenmp", "-ffp-contract=off", "-Wall", "-shared"]
_lib = None

_f32p = ctypes.POINTER(ctypes.c_float)
_vp = ctypes.c_void_p


def _cxx():
    return "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"


def build(force=False):
    """Compile oracle/oc_stereo.cpp -> oracle/liboc_stereo.so."""
    if force or not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < os.path.getmtime(_SRC):
        subprocess.check_call([_cxx()] + _CXXFLAGS + ["-o", _LIB_PATH, _SRC])
    return _LIB_PATH


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            build()
        L = ctypes.CDLL(_LIB_PATH)
        L.ocs_calib_create.restype = _vp
        L.ocs_calib_create.argtypes = [_f32p, ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_int, ctypes.c_int, ctypes.c_int]
        L.ocs_calib_destroy.argtypes = [_vp]
        L.ocs_calib_get_map.argtypes = [_vp, _f32p, _f32p]
        L.ocs_undistort.argtypes = [_vp, _f32p, _f32p, _f32p, ctypes.c_long, ctypes.c_int]
        L.ocs_reconstruct.restype = ctypes.c_int
        L.ocs_reconstruct.argtypes = [_vp, _f32p, _f32p, _vp, _f32p, _f32p, _f32p, _f32p, _f32p, _f32p, _f32p, ctypes.c_long, ctypes.c_int]
        L.ocs_max_threads.restype = ctypes.c_int
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(_f32p)


def _c32(a, n=None):
    a = np.ascontiguousarray(a, dtype=np.float32)
    return a if n is None else a.reshape(n)


def _check_points(p):
    assert isinstance(p, np.ndarray) and p.dtype == np.float32 and p.ndim == 2 and p.shape[1] == 2 and p.flags.c_contiguous


def _threads(threads):
    return threads if threads > 0 else max(1, int(lib().ocs_max_threads()) - 1)


class CalibOracle:
    """Calibration::prepare(height, width) of one camera (src/oc_calibration.cpp:161-219); exact=True keeps float64 maps."""

    def __init__(self, intrinsics, height, width, convergence=0.001, iteration=40, exact=False, threads=0):
        self.intrinsics = _c32(intrinsics, 13)
        self.height, self.width, self.exact = int(height), int(width), bool(exact)
        self.threads = _threads(threads)
        self._h = lib().ocs_calib_create(_p(self.intrinsics), self.height, self.width, float(convergence), int(iteration), self.threads,
                                         int(self.exact))
        assert self._h, "image size below 2 x 2"

    def __del__(self):
        if getattr(self, "_h", None):
            lib().ocs_calib_destroy(self._h)
            self._h = None

    def map(self):
        """(map_x, map_y) float32 [height, width] (the exact flavour's rounded to float)."""
        mx = np.empty((self.height, self.width), np.float32)
        my = np.empty((self.height, self.width), np.float32)
        lib().ocs_calib_get_map(self._h, _p(mx), _p(my))
        return mx, my

    def undistort(self, pts, intrinsics=None):
        """Calibration::undistort (:221-264) for float32 [n, 2] points, clamped in place; returns the sensor coordinates [n, 2]."""
        _check_points(pts)
        intr = self.intrinsics if intrinsics is None else _c32(intrinsics, 13)
        out = np.empty_like(pts)
        lib().ocs_undistort(self._h, _p(intr), _p(pts), _p(out), pts.shape[0], self.threads)
        return out


def reconstruct(cam1, projection1, cam2, projection2, pts1, pts2, intrinsics1=None, intrinsics2=None, with_system=False):
    """Stereovision::reconstruct(queue, queue, queue) (src/oc_stereovision.cpp:70-133) on two CalibOracle of the same flavour.
    Returns pts3d [n, 3]; with_system=True also returns the float32 systems A [n, 4, 3] and b [n, 4] (zero for NaN pairs)."""
    _check_points(pts1)
    _check_points(pts2)
    assert pts1.shape == pts2.shape and cam1.exact == cam2.exact
    n = pts1.shape[0]
    i1 = cam1.intrinsics if intrinsics1 is None else _c32(intrinsics1, 13)
    i2 = cam2.intrinsics if intrinsics2 is None else _c32(intrinsics2, 13)
    p1, p2 = _c32(projection1, 12), _c32(projection2, 12)
    out = np.empty((n, 3), np.float32)
    A = np.empty((n, 4, 3), np.float32) if with_system else None
    b = np.empty((n, 4), np.float32) if with_system else None
    rc = lib().ocs_reconstruct(cam1._h, _p(i1), _p(p1), cam2._h, _p(i2), _p(p2), _p(pts1), _p(pts2), _p(out),
                               _p(A) if with_system else None, _p(b) if with_system else None, n, cam1.threads)
    assert rc == 0
    return (out, A, b) if with_system else out
