"""ctypes front-end of the RegionFit oracle (oracle/oc_region_fit.cpp, which compiles in oracle/oc_oracle.cpp).

TEST INFRASTRUCTURE ONLY, like oracle.py: importable from tests/, __graft_entry__ and tools/; the product package never imports it.
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRCS = [os.path.join(_HERE, "oc_region_fit.cpp"), os.path.join(_HERE, "oc_oracle.cpp")]
_LIB_PATH = os.path.join(_HERE, "liboc_region_fit.so")
# the same arithmetic rules as oracle/Makefile: no fast-math, no FMA contraction
_CXXFLAGS = ["-O3", "-std=c++17", "-fPIC", "-fopenmp", "-ffp-contract=off", "-fcx-limited-range", "-Wall", "-Wno-unused-variable",
             "-Wno-sign-compare", "-Wno-unused-function", "-shared"]
_lib = None

_f32p = ctypes.POINTER(ctypes.c_float)


def _cxx():
    return "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"


def build(force=False):
    """Compile oracle/oc_region_fit.cpp -> oracle/liboc_region_fit.so."""
    if force or not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < max(os.path.getmtime(s) for s in _SRCS):
        subprocess.check_call([_cxx()] + _CXXFLAGS + ["-o", _LIB_PATH, _SRCS[0]])
    return _LIB_PATH


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            build()
        L = ctypes.CDLL(_LIB_PATH)
        L.oco_region_fit.restype = ctypes.c_int
        L.oco_region_fit.argtypes = [_f32p, ctypes.c_long, _f32p, ctypes.c_long, ctypes.c_int, ctypes.c_float, ctypes.c_int, ctypes.c_int,
                                     ctypes.c_int]
        L.oco_max_threads.restype = ctypes.c_int
        _lib = L
    return _lib


def max_threads():
    return int(lib().oco_max_threads())


def region_fit(reliable, pois, radius, min_neighbors, threads=0, exact=False):
    """RegionFit2D / RegionFit3D setNeighbor(reliable) + compute(queue) (reference src/oc_region_fit.cpp) on a POI2D [n,25] or
    POI3D [n,31] queue, in place; reliable: records of the same kind.  exact: the fit in float64 instead of float."""
    assert pois.dtype == np.float32 and pois.flags.c_contiguous and pois.shape[1] in (25, 31)
    reliable = np.ascontiguousarray(reliable, dtype=np.float32)
    assert reliable.ndim == 2 and reliable.shape[1] == pois.shape[1]
    threads = threads if threads > 0 else max(1, max_threads() - 1)
    rc = lib().oco_region_fit(reliable.ctypes.data_as(_f32p), reliable.shape[0], pois.ctypes.data_as(_f32p), pois.shape[0],
                              2 if pois.shape[1] == 25 else 3, radius, min_neighbors, threads, int(exact))
    assert rc == 0
    return pois
