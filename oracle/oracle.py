"""ctypes front-end of the CPU oracle (oracle/oc_oracle.cpp).

TEST INFRASTRUCTURE ONLY: importable from tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs.  The product package (opencorr_b200/) must never import it.

POI arrays are float32 [n, 25] (2D) / [n, 31] (3D): the reference's POI2D / POI3D records
(src/oc_poi.h:102-136,187-222) viewed as floats.
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "liboc_oracle.so")
_lib = None

_f32p = ctypes.POINTER(ctypes.c_float)


def build(force=False):
    """Compile oracle/oc_oracle.cpp -> oracle/liboc_oracle.so (g++ -O3 -fopenmp, no fast-math)."""
    src = os.path.join(_HERE, "oc_oracle.cpp")
    if force or not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "-B" if force else "-s"], stdout=subprocess.DEVNULL)
    return _LIB_PATH


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            build()
        L = ctypes.CDLL(_LIB_PATH)
        L.oco_create2d.restype = ctypes.c_void_p
        L.oco_create2d.argtypes = [_f32p, _f32p, ctypes.c_int, ctypes.c_int, ctypes.c_int]
        L.oco_destroy2d.argtypes = [ctypes.c_void_p]
        L.oco_prepare2d.argtypes = [ctypes.c_void_p]
        L.oco_get_gradient2d.argtypes = [ctypes.c_void_p, _f32p, _f32p]
        L.oco_bicubic_eval.argtypes = [ctypes.c_void_p, _f32p, ctypes.c_long, _f32p, ctypes.c_int]
        L.oco_fftcc2d.argtypes = [ctypes.c_void_p, _f32p, ctypes.c_long, ctypes.c_int, ctypes.c_int, ctypes.c_int]
        for f in (L.oco_icgn2d1, L.oco_icgn2d2):
            f.restype = ctypes.c_int
            f.argtypes = [ctypes.c_void_p, _f32p, ctypes.c_long, ctypes.c_int, ctypes.c_int,
                          ctypes.c_float, ctypes.c_float, ctypes.c_int]
        L.oco_icgn2d_ex.restype = ctypes.c_int
        L.oco_icgn2d_ex.argtypes = [ctypes.c_void_p, ctypes.c_int, _f32p, ctypes.c_long, ctypes.c_int, ctypes.c_int,
                                    ctypes.c_float, ctypes.c_float, _f32p, ctypes.c_int, ctypes.c_int]
        L.oco_iclm2d.restype = ctypes.c_int
        L.oco_iclm2d.argtypes = [ctypes.c_void_p, ctypes.c_int, _f32p, ctypes.c_long, ctypes.c_int, ctypes.c_int,
                                 ctypes.c_float, ctypes.c_float, _f32p, ctypes.c_int]
        L.oco_prepare_nr2d.argtypes = [ctypes.c_void_p]
        L.oco_nr2d1.restype = ctypes.c_int
        L.oco_nr2d1.argtypes = [ctypes.c_void_p, _f32p, ctypes.c_long, ctypes.c_int, ctypes.c_int,
                                ctypes.c_float, ctypes.c_float, ctypes.c_int]
        L.oco_create3d.restype = ctypes.c_void_p
        L.oco_create3d.argtypes = [_f32p, _f32p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int]
        L.oco_destroy3d.argtypes = [ctypes.c_void_p]
        L.oco_prepare3d.argtypes = [ctypes.c_void_p]
        L.oco_get_gradient3d.argtypes = [ctypes.c_void_p, _f32p, _f32p, _f32p]
        L.oco_get_coefficient3d.argtypes = [ctypes.c_void_p, _f32p]
        L.oco_tricubic_eval.argtypes = [ctypes.c_void_p, _f32p, ctypes.c_long, _f32p, ctypes.c_int]
        L.oco_fftcc3d.argtypes = [ctypes.c_void_p, _f32p, ctypes.c_long, ctypes.c_int, ctypes.c_int,
                                  ctypes.c_int, ctypes.c_int]
        L.oco_icgn3d1.restype = ctypes.c_int
        L.oco_icgn3d1.argtypes = [ctypes.c_void_p, _f32p, ctypes.c_long, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                  ctypes.c_float, ctypes.c_float, ctypes.c_int]
        L.oco_epipolar_search.restype = ctypes.c_int
        L.oco_epipolar_search.argtypes = [ctypes.c_void_p, _f32p, ctypes.c_long, _f32p, _f32p, _f32p, ctypes.c_int, ctypes.c_int,
                                          ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_float, ctypes.c_int]
        L.oco_strain.restype = ctypes.c_int
        L.oco_strain.argtypes = [_f32p, ctypes.c_long, ctypes.c_int, ctypes.c_float, ctypes.c_int, ctypes.c_float,
                                 ctypes.c_int, ctypes.c_int, ctypes.c_int]
        L.oco_strain_single.restype = ctypes.c_int
        L.oco_strain_single.argtypes = [_f32p, ctypes.c_long, ctypes.c_int, ctypes.c_long, ctypes.c_float, ctypes.c_int,
                                        ctypes.c_float, ctypes.c_int, ctypes.c_int, ctypes.c_int]
        L.oco_max_threads.restype = ctypes.c_int
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(_f32p)


def _c32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def set_legacy_no_minus4(on):
    """Pinning aid: drop the '-4 = not converged' rule of 2D IC-GN (the shipped tables predate it); OFF by default."""
    lib().oco_set_legacy_no_minus4(int(bool(on)))


def max_threads():
    return int(lib().oco_max_threads())


def strain(pois, radius, min_neighbors, zncc_threshold=0.9, approximation=1, threads=0, exact=False, only=None):
    """Strain::prepare + Strain::compute(queue) (reference src/oc_strain.cpp) on a POI2D [n,25] / POI3D [n,31] /
    POI2DS [n,28] array.  only=i: Strain::compute(&pois[i], queue) instead, POI i alone whatever its own ZNCC."""
    assert pois.dtype == np.float32 and pois.flags.c_contiguous and pois.shape[1] in (25, 31, 28)
    dim = {25: 2, 31: 3, 28: 23}[pois.shape[1]]  # 28 floats: POI2DS records (stereo DIC)
    threads = threads if threads > 0 else max(1, max_threads() - 1)
    if only is not None:
        assert 0 <= only < pois.shape[0]
    rc = lib().oco_strain_single(_p(pois), pois.shape[0], dim, -1 if only is None else int(only), radius, min_neighbors, zncc_threshold,
                                 approximation, threads, int(exact))
    assert rc == 0
    return pois


class Oracle2D:
    """ref, tar: float32 [H, W] row-major.  Mirrors FFTCC2D / ICGN2D1 / ICGN2D2 of the reference."""

    def __init__(self, ref, tar, threads=0):
        self.ref = _c32(ref)
        self.tar = _c32(tar)
        assert self.ref.shape == self.tar.shape and self.ref.ndim == 2
        self.h, self.w = self.ref.shape
        self.threads = threads if threads > 0 else max(1, max_threads() - 1)
        self._h = lib().oco_create2d(_p(self.ref), _p(self.tar), self.h, self.w, self.threads)
        self._prepared = False
        self._prepared_nr = False

    def __del__(self):
        if getattr(self, "_h", None):
            lib().oco_destroy2d(self._h)
            self._h = None

    def prepare(self):
        lib().oco_prepare2d(self._h)
        self._prepared = True

    def gradients(self):
        assert self._prepared
        gx = np.empty((self.h, self.w), np.float32)
        gy = np.empty((self.h, self.w), np.float32)
        lib().oco_get_gradient2d(self._h, _p(gx), _p(gy))
        return gx, gy

    def bicubic(self, xy, exact=False):
        assert self._prepared
        xy = _c32(xy).reshape(-1, 2)
        out = np.empty(xy.shape[0], np.float32)
        lib().oco_bicubic_eval(self._h, _p(xy), xy.shape[0], _p(out), int(exact))
        return out

    def fftcc2d(self, pois, rx, ry, exact=False):
        assert pois.dtype == np.float32 and pois.flags.c_contiguous and pois.shape[1] == 25
        lib().oco_fftcc2d(self._h, _p(pois), pois.shape[0], rx, ry, int(exact))
        return pois

    def icgn2d1(self, pois, rx, ry, conv=0.001, stop=10, exact=False):
        assert pois.dtype == np.float32 and pois.flags.c_contiguous and pois.shape[1] == 25
        if not self._prepared:
            self.prepare()
        rc = lib().oco_icgn2d1(self._h, _p(pois), pois.shape[0], rx, ry, conv, stop, int(exact))
        assert rc == 0
        return pois

    def icgn2d2(self, pois, rx, ry, conv=0.001, stop=10, exact=False):
        assert pois.dtype == np.float32 and pois.flags.c_contiguous and pois.shape[1] == 25
        if not self._prepared:
            self.prepare()
        rc = lib().oco_icgn2d2(self._h, _p(pois), pois.shape[0], rx, ry, conv, stop, int(exact))
        assert rc == 0
        return pois

    def icgn2d_ex(self, order, pois, rx, ry, conv=0.001, stop=10, center_offsets=None, self_adaptive=False, exact=False):
        """compute(queue, center_offset_queue) and/or the self-adaptive mode (radius read from each POI)."""
        assert pois.dtype == np.float32 and pois.flags.c_contiguous and pois.shape[1] == 25
        if not self._prepared:
            self.prepare()
        off = None
        if center_offsets is not None:
            off = _c32(center_offsets).reshape(-1, 2)
            assert off.shape[0] == pois.shape[0]
        rc = lib().oco_icgn2d_ex(self._h, order, _p(pois), pois.shape[0], rx, ry, conv, stop,
                                 _p(off) if off is not None else None, int(self_adaptive), int(exact))
        assert rc == 0
        return pois


    def iclm2d(self, order, pois, rx, ry, conv=0.001, stop=10, damping=(100.0, 0.1, 10.0), exact=False):
        """ICLM2D1 / ICLM2D2 (inverse-compositional Levenberg-Marquardt), reference src/oc_iclm.cpp."""
        assert pois.dtype == np.float32 and pois.flags.c_contiguous and pois.shape[1] == 25
        if not self._prepared:
            self.prepare()
        d = _c32(damping).reshape(3)
        rc = lib().oco_iclm2d(self._h, order, _p(pois), pois.shape[0], rx, ry, conv, stop, _p(d), int(exact))
        assert rc == 0
        return pois

    def epipolar_search(self, pois, fundamental, parallax_x, parallax_y, search_radius, search_step, rx, ry, conv, stop, exact=False):
        """EpipolarSearch::compute(queue), reference src/oc_epipolar_search.cpp:133-205."""
        assert pois.dtype == np.float32 and pois.flags.c_contiguous and pois.shape[1] == 25
        if not self._prepared:
            self.prepare()
        f = _c32(fundamental).reshape(9)
        ax, ay = _c32(parallax_x).reshape(3), _c32(parallax_y).reshape(3)
        rc = lib().oco_epipolar_search(self._h, _p(pois), pois.shape[0], _p(f), _p(ax), _p(ay), search_radius, search_step,
                                       rx, ry, conv, stop, int(exact))
        assert rc == 0
        return pois

    def nr2d1(self, pois, rx, ry, conv=0.001, stop=10, exact=False):
        """NR2D1 (forward-additive Newton-Raphson), reference src/oc_nr.cpp:119-334."""
        assert pois.dtype == np.float32 and pois.flags.c_contiguous and pois.shape[1] == 25
        if not self._prepared_nr:
            lib().oco_prepare_nr2d(self._h)
            self._prepared_nr = True
        rc = lib().oco_nr2d1(self._h, _p(pois), pois.shape[0], rx, ry, conv, stop, int(exact))
        assert rc == 0
        return pois


class Oracle3D:
    """ref, tar: float32 [Z, Y, X].  Mirrors FFTCC3D / ICGN3D1 of the reference."""

    def __init__(self, ref, tar, threads=0):
        self.ref = _c32(ref)
        self.tar = _c32(tar)
        assert self.ref.shape == self.tar.shape and self.ref.ndim == 3
        self.dz, self.dy, self.dx = self.ref.shape
        self.threads = threads if threads > 0 else max(1, max_threads() - 1)
        self._h = lib().oco_create3d(_p(self.ref), _p(self.tar), self.dx, self.dy, self.dz, self.threads)
        self._prepared = False

    def __del__(self):
        if getattr(self, "_h", None):
            lib().oco_destroy3d(self._h)
            self._h = None

    def prepare(self):
        lib().oco_prepare3d(self._h)
        self._prepared = True

    def gradients(self):
        assert self._prepared
        g = [np.empty((self.dz, self.dy, self.dx), np.float32) for _ in range(3)]
        lib().oco_get_gradient3d(self._h, _p(g[0]), _p(g[1]), _p(g[2]))
        return g

    def coefficients(self):
        assert self._prepared
        c = np.empty((self.dz, self.dy, self.dx), np.float32)
        lib().oco_get_coefficient3d(self._h, _p(c))
        return c

    def tricubic(self, xyz, exact=False):
        assert self._prepared
        xyz = _c32(xyz).reshape(-1, 3)
        out = np.empty(xyz.shape[0], np.float32)
        lib().oco_tricubic_eval(self._h, _p(xyz), xyz.shape[0], _p(out), int(exact))
        return out

    def fftcc3d(self, pois, rx, ry, rz, exact=False):
        assert pois.dtype == np.float32 and pois.flags.c_contiguous and pois.shape[1] == 31
        lib().oco_fftcc3d(self._h, _p(pois), pois.shape[0], rx, ry, rz, int(exact))
        return pois

    def icgn3d1(self, pois, rx, ry, rz, conv=0.001, stop=20, exact=False):
        assert pois.dtype == np.float32 and pois.flags.c_contiguous and pois.shape[1] == 31
        if not self._prepared:
            self.prepare()
        rc = lib().oco_icgn3d1(self._h, _p(pois), pois.shape[0], rx, ry, rz, conv, stop, int(exact))
        assert rc == 0
        return pois
