"""ctypes front-end of the SIFT3D oracle (oracle/oc_sift3d.cpp).

TEST INFRASTRUCTURE ONLY, like oracle.py: importable from tests/, __graft_entry__ and tools/; the product package never imports it.

Volumes are float32 [z, y, x].  config is the 10 floats of Sift3dConfig in field order (n_octave_layers, n_octave,
min_dimension, alpha, beta, gamma, sigma_source, sigma_base, gradient_threshold, truncate_threshold); n_octave is computed.
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "oc_sift3d.cpp")
_HDR = os.path.join(_HERE, "..", "opencorr_b200", "csrc", "sift3d_common.h")
_LIB_PATH = os.path.join(_HERE, "liboc_sift3d.so")
# the same arithmetic rules as oracle/Makefile: no fast-math, no FMA contraction
_CXXFLAGS = ["-O3", "-std=c++17", "-fPIC", "-fopenmp", "-ffp-contract=off", "-Wall", "-shared"]
_lib = None

_f32p = ctypes.POINTER(ctypes.c_float)
_f64p = ctypes.POINTER(ctypes.c_double)
_i32p = ctypes.POINTER(ctypes.c_int)
_vp = ctypes.c_void_p

KP_FLOATS = 18
DESC = 768


def default_config():
    """SIFT3D::SIFT3D() defaults (src/oc_sift.cpp:142-158)."""
    return np.array([3, 0, 8, 0.1, 0.9, 0.4, 1.15, 1.6, 1e-10, np.float32(0.2) * 128 / 768], np.float32)


def _cxx():
    return "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"


def build(force=False):
    """Compile oracle/oc_sift3d.cpp -> oracle/liboc_sift3d.so."""
    newest = max(os.path.getmtime(_SRC), os.path.getmtime(_HDR))
    if force or not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < newest:
        subprocess.check_call([_cxx()] + _CXXFLAGS + ["-o", _LIB_PATH, _SRC])
    return _LIB_PATH


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            build()
        L = ctypes.CDLL(_LIB_PATH)
        L.os3_max_threads.restype = ctypes.c_int
        L.os3_extract.restype = _vp
        L.os3_extract.argtypes = [_f32p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _f32p, _f32p, ctypes.c_int]
        L.os3_counts.argtypes = [_vp, ctypes.POINTER(ctypes.c_long)]
        L.os3_get.argtypes = [_vp, _i32p, _f32p, _f32p, _f32p, _f64p, _i32p]
        L.os3_free.argtypes = [_vp]
        L.os3_match.restype = ctypes.c_long
        L.os3_match.argtypes = [_f32p, ctypes.c_long, _f32p, ctypes.c_long, ctypes.c_float, ctypes.c_int, _f32p, _f64p, _i32p]
        L.os3_blur.argtypes = [_f32p, _f32p, ctypes.c_int, ctypes.c_int, ctypes.c_int, _f32p, ctypes.c_float]
        L.os3_blur_kernel.argtypes = [ctypes.c_float, _f32p, _i32p, _f32p]
        L.os3_eig3.argtypes = [_f32p, _f32p, _f32p]
        L.os3_ico_face.restype = ctypes.c_int
        L.os3_ico_face.argtypes = [_f32p, _f32p]
        L.os3_exp.restype = ctypes.c_float
        L.os3_exp.argtypes = [ctypes.c_float]
        _lib = L
    return _lib


def _p(a, t=_f32p):
    return a.ctypes.data_as(t)


def _threads(threads):
    return threads if threads > 0 else max(1, int(lib().os3_max_threads()) - 1)


class Features:
    """One volume's SIFT3D products: n_octave, cand [n, 5] int32 (octave, layer, z, y, x), max_abs [n_octave * (L - 1)],
    kp [k, 18] float32, desc [k, 768] float32, margin [n] float64 (orientation decision margins), kept [n] int32."""

    def __init__(self, vol, config=None, unit=(1.0, 1.0, 1.0), threads=0):
        vol = np.ascontiguousarray(vol, dtype=np.float32)
        assert vol.ndim == 3
        cfg = np.ascontiguousarray(default_config() if config is None else config, dtype=np.float32)
        u = np.ascontiguousarray(unit, dtype=np.float32)
        dz, dy, dx = vol.shape
        h = lib().os3_extract(_p(vol), dx, dy, dz, _p(cfg), _p(u), _threads(threads))
        try:
            c = (ctypes.c_long * 4)()
            lib().os3_counts(h, c)
            self.n_octave = int(c[0])
            self.cand = np.empty((c[1], 5), np.int32)
            self.max_abs = np.empty(c[2], np.float32)
            self.kp = np.empty((c[3], KP_FLOATS), np.float32)
            self.desc = np.empty((c[3], DESC), np.float32)
            self.margin = np.empty(c[1], np.float64)
            self.kept = np.empty(c[1], np.int32)
            lib().os3_get(h, _p(self.cand, _i32p), _p(self.max_abs), _p(self.kp), _p(self.desc), _p(self.margin, _f64p),
                          _p(self.kept, _i32p))
        finally:
            lib().os3_free(h)


def match(desc1, desc2, ratio=0.85, threads=0):
    """monodirectionalMatch on two descriptor sets: returns (pairs [m, 2] int32 (ref, tar) in output order, top2 [n1, 3]
    float32 (d0, index0, d1), ratio_margin [n1] float64)."""
    d1 = np.ascontiguousarray(desc1, dtype=np.float32).reshape(-1, DESC)
    d2 = np.ascontiguousarray(desc2, dtype=np.float32).reshape(-1, DESC)
    n1 = d1.shape[0]
    top2 = np.empty((n1, 3), np.float32)
    margin = np.empty(n1, np.float64)
    pairs = np.empty((max(n1, 1), 2), np.int32)
    n = lib().os3_match(_p(d1), n1, _p(d2), d2.shape[0], float(ratio), _threads(threads), _p(top2), _p(margin, _f64p), _p(pairs, _i32p))
    return pairs[:n].copy(), top2, margin


def sift3d(ref, tar, config=None, unit=(1.0, 1.0, 1.0), ratio=0.85, threads=0):
    """SIFT3D::compute() on a pair: returns (ref Features, tar Features, pairs, ref_matched [m, 3], tar_matched [m, 3])."""
    fr = Features(ref, config, unit, threads)
    ft = Features(tar, config, unit, threads)
    pairs, _, _ = match(fr.desc, ft.desc, ratio, threads)
    return fr, ft, pairs, fr.kp[pairs[:, 0], 3:6], ft.kp[pairs[:, 1], 3:6]


def blur(vol, sigma, unit=(1.0, 1.0, 1.0)):
    vol = np.ascontiguousarray(vol, dtype=np.float32)
    out = np.empty_like(vol)
    u = np.ascontiguousarray(unit, dtype=np.float32)
    dz, dy, dx = vol.shape
    lib().os3_blur(_p(vol), _p(out), dx, dy, dz, _p(u), float(sigma))
    return out


def blur_kernel(sigma, unit=(1.0, 1.0, 1.0)):
    """(radius [3], weights: list of 3 arrays w[0..radius])."""
    u = np.ascontiguousarray(unit, dtype=np.float32)
    r = np.zeros(3, np.int32)
    w = np.zeros((3, 65), np.float32)
    lib().os3_blur_kernel(float(sigma), _p(u), _p(r, _i32p), _p(w))
    return r, [w[a, :r[a] + 1].copy() for a in range(3)]


def eig3(m):
    m = np.ascontiguousarray(m, dtype=np.float32).reshape(9)
    val = np.empty(3, np.float32)
    vec = np.empty((3, 3), np.float32)
    lib().os3_eig3(_p(m), _p(val), _p(vec))
    return val, vec


def ico_face(g):
    g = np.ascontiguousarray(g, dtype=np.float32).reshape(3)
    b = np.zeros(3, np.float32)
    f = lib().os3_ico_face(_p(g), _p(b))
    return f, b
