"""Host-side mirror of the reference's operator interface for the FFT-CC -> IC-GN path.

Class names, constructor arguments and method meaning follow the reference (C++):
  FFTCC2D(int rx, int ry, int threads)                        src/oc_fftcc.h:61
  FFTCC3D(int rx, int ry, int rz, int threads)                src/oc_fftcc.h:82
  ICGN2D1 / ICGN2D2(int rx, int ry, float conv, float stop, int threads)   src/oc_icgn.h:58,113
  ICGN3D1(int rx, int ry, int rz, float conv, float stop, int threads)     src/oc_icgn.h:168
  setImages / setSubset / prepare / compute / setIteration    src/oc_dic.h:56-84, oc_icgn.h:61-76
Python spellings (set_images, ...) are provided next to the reference's camelCase names.

POI queues are numpy float32 arrays [n, 25] (POI2D) or [n, 31] (POI3D) -- the reference's
records viewed as floats (src/oc_poi.h:102-136,187-222) -- mutated in place like
compute(std::vector<POI>&).  Everything runs through the C ABI (include/opencorr_b200.h); the
`thread_number` argument is accepted for signature compatibility and ignored (no CPU threads).
"""
import ctypes

import numpy as np

from . import _capi

# ---- POI record layout (reference src/oc_poi.h) ------------------------------------------------
POI2D_FLOATS = 25
POI3D_FLOATS = 31
POI2DS_FLOATS = 28
_STRAIN_SERIES = {POI2D_FLOATS: "2d", POI3D_FLOATS: "3d", POI2DS_FLOATS: "2ds"}  # record floats -> ocb_strain*_series suffix
P2 = dict(x=0, y=1, u=2, ux=3, uy=4, uxx=5, uxy=6, uyy=7, v=8, vx=9, vy=10, vxx=11, vxy=12, vyy=13,
          u0=14, v0=15, zncc=16, iteration=17, convergence=18, feature=19, exx=20, eyy=21, exy=22,
          subset_rx=23, subset_ry=24)
P3 = dict(x=0, y=1, z=2, u=3, ux=4, uy=5, uz=6, v=7, vx=8, vy=9, vz=10, w=11, wx=12, wy=13, wz=14,
          u0=15, v0=16, w0=17, zncc=18, iteration=19, convergence=20, feature=21,
          exx=22, eyy=23, ezz=24, exy=25, eyz=26, ezx=27, subset_rx=28, subset_ry=29, subset_rz=30)


# ---- SIFT3D (reference src/oc_sift.h:71-155) ----------------------------------------------------
SIFT3D_CONFIG_FLOATS = 10
SIFT3D_KP_FLOATS = 18
# Sift3dConfig in field order, the constructor's defaults (src/oc_sift.cpp:142-152); n_octave is computed by compute()
SIFT3D_CONFIG_FIELDS = ("n_octave_layers", "n_octave", "min_dimension", "alpha", "beta", "gamma", "sigma_source", "sigma_base",
                        "gradient_threshold", "truncate_threshold")
SIFT3D_DEFAULT_CONFIG = np.array([3, 0, 8, 0.1, 0.9, 0.4, 1.15, 1.6, 1e-10, np.float32(0.2) * 128 / 768], np.float32)
SIFT3D_STAGES = ("ref_pyramid", "ref_extrema", "ref_orientation", "ref_descriptors", "tar_pyramid", "tar_extrema",
                 "tar_orientation", "tar_descriptors", "matching", "host_post_pass")


def make_poi2d(xy):
    """POI2D(Point2D) for every row of xy: location set, everything else cleared (oc_poi.h:112-135)."""
    xy = np.asarray(xy, dtype=np.float32).reshape(-1, 2)
    q = np.zeros((xy.shape[0], POI2D_FLOATS), np.float32)
    q[:, 0:2] = xy
    return q


def make_poi3d(xyz):
    xyz = np.asarray(xyz, dtype=np.float32).reshape(-1, 3)
    q = np.zeros((xyz.shape[0], POI3D_FLOATS), np.float32)
    q[:, 0:3] = xyz
    return q


def _vp(a):
    return ctypes.c_void_p(a.ctypes.data)


def _check_queue(q, floats):
    if not isinstance(q, np.ndarray) or q.dtype != np.float32 or q.ndim != 2 or q.shape[1] != floats \
            or not q.flags.c_contiguous:
        raise ValueError("POI queue must be a C-contiguous float32 array of shape [n, %d]" % floats)


def _check_points(p):
    if not isinstance(p, np.ndarray) or p.dtype != np.float32 or p.ndim != 2 or p.shape[1] != 2 or not p.flags.c_contiguous:
        raise ValueError("points must be a C-contiguous float32 array of shape [n, 2] (they are clamped in place)")


class Engine:
    """One GPU context (ocb_ctx), or a GROUP context over several devices: device = -1 / "all" (every visible device) or a
    list of device indices -- host-queue calls then shard the queue over the devices inside the C ABI (one process, G
    devices; include/opencorr_b200.h ocb_create_multi).  Raises OpenCorrB200Error when no H100-class (sm_90) GPU is usable."""

    def __init__(self, device=0):
        self._lib = _capi.load()
        if isinstance(device, str):
            if device != "all":
                raise ValueError("device must be an index, -1 / 'all', or a list of indices")
            device = -1
        if isinstance(device, (list, tuple)):
            devs = (ctypes.c_int * len(device))(*[int(d) for d in device])
            self._ctx = self._lib.ocb_create_multi(devs, len(device))
            self.device = tuple(int(d) for d in device)
        else:
            self._ctx = self._lib.ocb_create(int(device))
            self.device = int(device)
        if not self._ctx:
            raise _capi.OpenCorrB200Error(_capi.OCB_ERR_CUDA, _capi.last_error(None))
        self._keep = []  # host arrays referenced by the last upload
        self._frames = {}  # frame count of each series set on this context: "2d", "3d", "stereo"
        self.image_token = 0  # bumped by every set_images_*: lets an operator see that another one replaced its images

    @property
    def member_count(self):
        """Devices behind this context (1 unless it is a group)."""
        return int(self._lib.ocb_member_count(self._ctx))

    def close(self):
        if getattr(self, "_ctx", None):
            self._lib.ocb_destroy(self._ctx)
            self._ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc):
        _capi.check(rc, self._ctx)

    # images ------------------------------------------------------------------------------------
    def set_images_2d(self, ref, tar):
        """float32 images, or uint8 images (as read from an 8-bit file): the latter are uploaded as
        bytes and widened on the device -- same results, a quarter of the PCIe traffic."""
        ref, tar = np.asarray(ref), np.asarray(tar)
        if ref.ndim != 2 or ref.shape != tar.shape:
            raise ValueError("ref/tar must be 2-D arrays of equal shape")
        h, w = ref.shape
        if ref.dtype == np.uint8 and tar.dtype == np.uint8:
            ref, tar = np.ascontiguousarray(ref), np.ascontiguousarray(tar)
            self._ck(self._lib.ocb_set_images_2d_u8(self._ctx, _vp(ref), _vp(tar), w, h))
        else:
            ref = np.ascontiguousarray(ref, dtype=np.float32)
            tar = np.ascontiguousarray(tar, dtype=np.float32)
            self._ck(self._lib.ocb_set_images_2d(self._ctx, _vp(ref), _vp(tar), w, h, 0))
        self._ck(self._lib.ocb_sync(self._ctx))
        self.image_token += 1

    def set_images_3d(self, ref, tar):
        ref, tar = np.asarray(ref), np.asarray(tar)
        if ref.ndim != 3 or ref.shape != tar.shape:
            raise ValueError("ref/tar must be 3-D arrays [z, y, x] of equal shape")
        dz, dy, dx = ref.shape
        if ref.dtype == np.uint8 and tar.dtype == np.uint8:
            ref, tar = np.ascontiguousarray(ref), np.ascontiguousarray(tar)
            self._ck(self._lib.ocb_set_images_3d_u8(self._ctx, _vp(ref), _vp(tar), dx, dy, dz))
        else:
            ref = np.ascontiguousarray(ref, dtype=np.float32)
            tar = np.ascontiguousarray(tar, dtype=np.float32)
            self._ck(self._lib.ocb_set_images_3d(self._ctx, _vp(ref), _vp(tar), dx, dy, dz))
        self._ck(self._lib.ocb_sync(self._ctx))
        self.image_token += 1

    def set_images_2d_dev(self, d_ref, d_tar, width, height):
        self._ck(self._lib.ocb_set_images_2d_dev(self._ctx, int(d_ref), int(d_tar), width, height))
        self.image_token += 1

    def set_images_3d_dev(self, d_ref, d_tar, dim_x, dim_y, dim_z):
        self._ck(self._lib.ocb_set_images_3d_dev(self._ctx, int(d_ref), int(d_tar), dim_x, dim_y, dim_z))
        self.image_token += 1

    def set_stream(self, cuda_stream):
        """Enqueue on this cudaStream_t handle (0/None = CUDA's legacy default stream)."""
        self._ck(self._lib.ocb_set_stream(self._ctx, int(cuda_stream) if cuda_stream else None))

    def use_own_stream(self):
        self._ck(self._lib.ocb_use_own_stream(self._ctx))

    def sync(self):
        self._ck(self._lib.ocb_sync(self._ctx))

    def launch_count(self):
        return int(self._lib.ocb_launch_count(self._ctx))

    # hot path, host POI queues -------------------------------------------------------------------
    def fftcc2d(self, q, rx, ry):
        _check_queue(q, POI2D_FLOATS)
        self._ck(self._lib.ocb_fftcc2d(self._ctx, _vp(q), q.shape[0], rx, ry))

    def fftcc3d(self, q, rx, ry, rz):
        _check_queue(q, POI3D_FLOATS)
        self._ck(self._lib.ocb_fftcc3d(self._ctx, _vp(q), q.shape[0], rx, ry, rz))

    def icgn2d_prepare(self):
        self._ck(self._lib.ocb_icgn2d_prepare(self._ctx))

    def icgn3d_prepare(self):
        self._ck(self._lib.ocb_icgn3d_prepare(self._ctx))

    def icgn2d1(self, q, rx, ry, conv, stop):
        _check_queue(q, POI2D_FLOATS)
        self._ck(self._lib.ocb_icgn2d1(self._ctx, _vp(q), q.shape[0], rx, ry, conv, stop))

    def icgn2d2(self, q, rx, ry, conv, stop):
        _check_queue(q, POI2D_FLOATS)
        self._ck(self._lib.ocb_icgn2d2(self._ctx, _vp(q), q.shape[0], rx, ry, conv, stop))

    def icgn2d_ex(self, order, q, rx, ry, conv, stop, center_offsets=None, self_adaptive=False):
        """Offset-centre and/or self-adaptive overloads (reference src/oc_icgn.cpp:353-557, :910-1136)."""
        _check_queue(q, POI2D_FLOATS)
        off = None
        if center_offsets is not None:
            off = np.ascontiguousarray(center_offsets, dtype=np.float32).reshape(-1, 2)
            if off.shape[0] != q.shape[0]:
                raise ValueError("center_offsets must hold one (x, y) pair per POI")
        self._ck(self._lib.ocb_icgn2d_ex(self._ctx, int(order), _vp(q), q.shape[0], rx, ry, conv, stop,
                                         _vp(off) if off is not None else None, int(bool(self_adaptive))))

    def set_series_2d(self, ref, tars):
        """An image series for icgn2d_series: ref (H, W) and tars (F, H, W), float32.  Kept apart from set_images_2d's pair."""
        ref = np.ascontiguousarray(ref, dtype=np.float32)
        tars = np.ascontiguousarray(tars, dtype=np.float32)
        if ref.ndim != 2 or tars.ndim != 3 or tars.shape[1:] != ref.shape:
            raise ValueError("ref must be (H, W) and tars (F, H, W)")
        f, h, w = tars.shape
        self._ck(self._lib.ocb_set_series_2d(self._ctx, _vp(ref), _vp(tars), f, w, h))
        self._ck(self._lib.ocb_sync(self._ctx))
        self._frames["2d"] = f

    def icgn2d_series(self, order, seeds, rx, ry, conv, stop):
        """ICGN2D1 (order 1) / ICGN2D2 (order 2) over the series set by set_series_2d, frame f seeded by frame f - 1's records
        (frame 0 by `seeds`, [n, 25]).  Returns the records of every frame, float32 (F, n, 25); seeds are not changed."""
        _check_queue(seeds, POI2D_FLOATS)
        out = np.empty((self._series_frames("2d", "icgn2d_series"), seeds.shape[0], POI2D_FLOATS), np.float32)
        self._ck(self._lib.ocb_icgn2d_series(self._ctx, int(order), _vp(seeds), _vp(out), seeds.shape[0], rx, ry, conv, stop))
        return out

    def _series_frames(self, kind, call):
        """The frame count of the series of this kind; without one, the error the C call would return."""
        if kind not in self._frames:
            raise _capi.OpenCorrB200Error(_capi.OCB_ERR_STATE, call + ": no series set")
        return self._frames[kind]

    def set_series_3d(self, ref, tars):
        """A volume series for icgn3d_series: ref (Z, Y, X) and tars (F, Z, Y, X).  uint8 volumes stay 8-bit on the device (one
        byte per voxel and frame); anything else becomes float32.  Kept apart from set_images_3d's pair."""
        ref, tars = np.asarray(ref), np.asarray(tars)
        if ref.ndim != 3 or tars.ndim != 4 or tars.shape[1:] != ref.shape:
            raise ValueError("ref must be (Z, Y, X) and tars (F, Z, Y, X)")
        f, dz, dy, dx = tars.shape
        if ref.dtype == np.uint8 and tars.dtype == np.uint8:
            ref, tars = np.ascontiguousarray(ref), np.ascontiguousarray(tars)
            self._ck(self._lib.ocb_set_series_3d_u8(self._ctx, _vp(ref), _vp(tars), f, dx, dy, dz))
        else:
            ref = np.ascontiguousarray(ref, dtype=np.float32)
            tars = np.ascontiguousarray(tars, dtype=np.float32)
            self._ck(self._lib.ocb_set_series_3d(self._ctx, _vp(ref), _vp(tars), f, dx, dy, dz))
        self._ck(self._lib.ocb_sync(self._ctx))
        self._frames["3d"] = f

    def icgn3d_series(self, seeds, rx, ry, rz, conv, stop):
        """ICGN3D1 over the series set by set_series_3d, frame f seeded by frame f - 1's records (frame 0 by `seeds`, [n, 31]).
        Returns the records of every frame, float32 (F, n, 31); seeds are not changed."""
        _check_queue(seeds, POI3D_FLOATS)
        out = np.empty((self._series_frames("3d", "icgn3d_series"), seeds.shape[0], POI3D_FLOATS), np.float32)
        self._ck(self._lib.ocb_icgn3d_series(self._ctx, _vp(seeds), _vp(out), seeds.shape[0], rx, ry, rz, conv, stop))
        return out

    def icgn2d_series_reseed(self, order, seeds, rx, ry, conv, stop, fft_rx, fft_ry, zncc_min):
        """icgn2d_series that re-seeds lost POIs: a POI whose frame-f record has !(zncc >= zncc_min) is rebuilt from its seed at
        its latest good translation and registered again in frame f by FFTCC2D (radii fft_rx, fft_ry) and IC-GN.  Returns
        (records float32 (F, n, 25), reseeded int64 (F,): the POIs re-seeded in each frame)."""
        _check_queue(seeds, POI2D_FLOATS)
        n_frames = self._series_frames("2d", "icgn2d_series_reseed")
        out = np.empty((n_frames, seeds.shape[0], POI2D_FLOATS), np.float32)
        counts = np.zeros(n_frames, np.uint64)
        self._ck(self._lib.ocb_icgn2d_series_reseed(self._ctx, int(order), _vp(seeds), _vp(out), seeds.shape[0], rx, ry, conv, stop, int(fft_rx),
                                                    int(fft_ry), float(zncc_min), _vp(counts)))
        return out, counts.astype(np.int64)

    def iclm2d_series(self, order, seeds, rx, ry, conv, stop, damping=(100.0, 0.1, 10.0)):
        """ICLM2D1 (order 1) / ICLM2D2 (order 2) over the series set by set_series_2d, frame f seeded by frame f - 1's records
        (frame 0 by `seeds`, [n, 25]); damping = (lambda, alpha, beta), restarted in every frame.  Returns the records of every
        frame, float32 (F, n, 25); seeds are not changed."""
        _check_queue(seeds, POI2D_FLOATS)
        out = np.empty((self._series_frames("2d", "iclm2d_series"), seeds.shape[0], POI2D_FLOATS), np.float32)
        self._ck(self._lib.ocb_iclm2d_series(self._ctx, int(order), _vp(seeds), _vp(out), seeds.shape[0], rx, ry, conv, stop, float(damping[0]),
                                             float(damping[1]), float(damping[2])))
        return out

    def iclm2d_series_reseed(self, order, seeds, rx, ry, conv, stop, fft_rx, fft_ry, zncc_min, damping=(100.0, 0.1, 10.0)):
        """iclm2d_series that re-seeds lost POIs with FFTCC2D and IC-LM in the frame where they are lost (see
        icgn2d_series_reseed).  Returns (records float32 (F, n, 25), reseeded int64 (F,))."""
        _check_queue(seeds, POI2D_FLOATS)
        n_frames = self._series_frames("2d", "iclm2d_series_reseed")
        out = np.empty((n_frames, seeds.shape[0], POI2D_FLOATS), np.float32)
        counts = np.zeros(n_frames, np.uint64)
        self._ck(self._lib.ocb_iclm2d_series_reseed(self._ctx, int(order), _vp(seeds), _vp(out), seeds.shape[0], rx, ry, conv, stop,
                                                    float(damping[0]), float(damping[1]), float(damping[2]), int(fft_rx), int(fft_ry),
                                                    float(zncc_min), _vp(counts)))
        return out, counts.astype(np.int64)

    def nr2d1_series(self, seeds, rx, ry, conv, stop):
        """NR2D1 over the series set by set_series_2d, frame f seeded by frame f - 1's records (frame 0 by `seeds`, [n, 25]).
        Returns the records of every frame, float32 (F, n, 25); seeds are not changed."""
        _check_queue(seeds, POI2D_FLOATS)
        out = np.empty((self._series_frames("2d", "nr2d1_series"), seeds.shape[0], POI2D_FLOATS), np.float32)
        self._ck(self._lib.ocb_nr2d1_series(self._ctx, _vp(seeds), _vp(out), seeds.shape[0], rx, ry, conv, stop))
        return out

    def nr2d1_series_reseed(self, seeds, rx, ry, conv, stop, fft_rx, fft_ry, zncc_min):
        """nr2d1_series that re-seeds lost POIs with FFTCC2D and NR2D1 in the frame where they are lost (see
        icgn2d_series_reseed).  Returns (records float32 (F, n, 25), reseeded int64 (F,))."""
        _check_queue(seeds, POI2D_FLOATS)
        n_frames = self._series_frames("2d", "nr2d1_series_reseed")
        out = np.empty((n_frames, seeds.shape[0], POI2D_FLOATS), np.float32)
        counts = np.zeros(n_frames, np.uint64)
        self._ck(self._lib.ocb_nr2d1_series_reseed(self._ctx, _vp(seeds), _vp(out), seeds.shape[0], rx, ry, conv, stop, int(fft_rx), int(fft_ry),
                                                   float(zncc_min), _vp(counts)))
        return out, counts.astype(np.int64)

    def icgn3d_series_reseed(self, seeds, rx, ry, rz, conv, stop, fft_rx, fft_ry, fft_rz, zncc_min):
        """icgn3d_series that re-seeds lost POIs with FFTCC3D (radii fft_rx, fft_ry, fft_rz) in the frame where they are lost (see
        icgn2d_series_reseed).  Returns (records float32 (F, n, 31), reseeded int64 (F,))."""
        _check_queue(seeds, POI3D_FLOATS)
        n_frames = self._series_frames("3d", "icgn3d_series_reseed")
        out = np.empty((n_frames, seeds.shape[0], POI3D_FLOATS), np.float32)
        counts = np.zeros(n_frames, np.uint64)
        self._ck(self._lib.ocb_icgn3d_series_reseed(self._ctx, _vp(seeds), _vp(out), seeds.shape[0], rx, ry, rz, conv, stop, int(fft_rx), int(fft_ry),
                                                    int(fft_rz), float(zncc_min), _vp(counts)))
        return out, counts.astype(np.int64)

    def icgn2d_series_recover(self, order, seeds, rx, ry, conv, stop, radius, min_neighbors, zncc_high, zncc_low, max_rounds):
        """icgn2d_series that recovers unreliable POIs in the frame where they fail: each frame's records go through icgn2d_recover's
        rounds of RegionFit2D and ICGN2D<order> against that frame, and frame f + 1 starts from the recovered records
        (include/opencorr_b200.h ocb_icgn2d_series_recover).  Returns (records float32 (F, n, 25), recovered int64 (F, max_rounds):
        the POIs accepted in each round of each frame, remaining int64 (F,): the POIs still unreliable at the end of each frame)."""
        _check_queue(seeds, POI2D_FLOATS)
        n_frames = self._series_frames("2d", "icgn2d_series_recover")
        out = np.empty((n_frames, seeds.shape[0], POI2D_FLOATS), np.float32)
        return self._series_recover(self._lib.ocb_icgn2d_series_recover, (int(order), _vp(seeds), _vp(out), seeds.shape[0], rx, ry), n_frames, out,
                                    conv, stop, radius, min_neighbors, zncc_high, zncc_low, max_rounds)

    def icgn3d_series_recover(self, seeds, rx, ry, rz, conv, stop, radius, min_neighbors, zncc_high, zncc_low, max_rounds):
        """icgn2d_series_recover over the volume series, with RegionFit3D and ICGN3D1.  Returns (records float32 (F, n, 31),
        recovered int64 (F, max_rounds), remaining int64 (F,))."""
        _check_queue(seeds, POI3D_FLOATS)
        n_frames = self._series_frames("3d", "icgn3d_series_recover")
        out = np.empty((n_frames, seeds.shape[0], POI3D_FLOATS), np.float32)
        return self._series_recover(self._lib.ocb_icgn3d_series_recover, (_vp(seeds), _vp(out), seeds.shape[0], rx, ry, rz), n_frames, out, conv,
                                    stop, radius, min_neighbors, zncc_high, zncc_low, max_rounds)

    def icgn2d_series_recover_dev(self, order, d_seeds, d_out, n, rx, ry, conv, stop, radius, min_neighbors, zncc_high, zncc_low, max_rounds):
        """icgn2d_series_recover on device pointers; synchronises the stream.  Returns (recovered (F, max_rounds), remaining (F,))."""
        n_frames = self._series_frames("2d", "icgn2d_series_recover")
        return self._series_recover(self._lib.ocb_icgn2d_series_recover_dev, (int(order), int(d_seeds), int(d_out), n, rx, ry), n_frames, None,
                                    conv, stop, radius, min_neighbors, zncc_high, zncc_low, max_rounds)

    def icgn3d_series_recover_dev(self, d_seeds, d_out, n, rx, ry, rz, conv, stop, radius, min_neighbors, zncc_high, zncc_low, max_rounds):
        """icgn3d_series_recover on device pointers; synchronises the stream.  Returns (recovered (F, max_rounds), remaining (F,))."""
        n_frames = self._series_frames("3d", "icgn3d_series_recover")
        return self._series_recover(self._lib.ocb_icgn3d_series_recover_dev, (int(d_seeds), int(d_out), n, rx, ry, rz), n_frames, None, conv,
                                    stop, radius, min_neighbors, zncc_high, zncc_low, max_rounds)

    def _series_recover(self, fn, head, n_frames, out, conv, stop, radius, min_neighbors, zncc_high, zncc_low, max_rounds):
        if int(max_rounds) < 0:
            raise ValueError("max_rounds must be >= 0")
        recovered = np.zeros((n_frames, int(max_rounds)), np.uint64)
        remaining = np.zeros(n_frames, np.uint64)
        self._ck(fn(self._ctx, *head, float(conv), float(stop), float(radius), int(min_neighbors), float(zncc_high), float(zncc_low),
                    int(max_rounds), _vp(recovered) if recovered.size else None, _vp(remaining)))
        counts = (recovered.astype(np.int64), remaining.astype(np.int64))
        return counts if out is None else (out,) + counts

    def set_stereo_series(self, ref1, tars1, tars2):
        """A stereo load series for stereo_series: reference view 1 (H, W) and the two views of every frame, tars1 and tars2
        (F, H, W), float32.  Kept apart from set_images_2d's pair and set_series_2d's series."""
        ref1 = np.ascontiguousarray(ref1, dtype=np.float32)
        tars1 = np.ascontiguousarray(tars1, dtype=np.float32)
        tars2 = np.ascontiguousarray(tars2, dtype=np.float32)
        if ref1.ndim != 2 or tars1.ndim != 3 or tars1.shape[1:] != ref1.shape or tars2.shape != tars1.shape:
            raise ValueError("ref1 must be (H, W) and tars1, tars2 (F, H, W)")
        f, h, w = tars1.shape
        self._ck(self._lib.ocb_set_stereo_series_2d(self._ctx, _vp(ref1), _vp(tars1), _vp(tars2), f, w, h))
        self._ck(self._lib.ocb_sync(self._ctx))
        self._frames["stereo"] = f

    def stereo_series(self, rig, stereo, seeds1, seeds2, order1, order2, rx, ry, conv, stop):
        """Both views of every frame of the series set by set_stereo_series, registered against reference view 1 and
        triangulated by `rig` (a Stereovision whose cameras were prepared on this engine):
        out1[f] = ICGN2D<order1> of (ref1, tars1[f]) from out1[f - 1] (frame 0: seeds1), out2[f] the same for view 2 with
        order2 and seeds2, and out2ds[f] the POI2DS records of frame f (include/opencorr_b200.h ocb_stereo_series).  stereo:
        the r1 -> r2 records, [n, 25].  Returns (out1 (F, n, 25), out2 (F, n, 25), out2ds (F, n, 28)), float32; the inputs are
        not changed."""
        for q in (stereo, seeds1, seeds2):
            _check_queue(q, POI2D_FLOATS)
        n = seeds1.shape[0]
        if stereo.shape[0] != n or seeds2.shape[0] != n:
            raise ValueError("stereo, seeds1 and seeds2 must hold the same number of POIs")
        rig._engine()
        h1, i1, p1, h2, i2, p2 = rig._cameras()
        f = self._series_frames("stereo", "stereo_series")
        out1 = np.empty((f, n, POI2D_FLOATS), np.float32)
        out2 = np.empty((f, n, POI2D_FLOATS), np.float32)
        out2ds = np.empty((f, n, POI2DS_FLOATS), np.float32)
        self._ck(self._lib.ocb_stereo_series(self._ctx, h1, _vp(i1), _vp(p1), h2, _vp(i2), _vp(p2), int(order1), int(order2), _vp(stereo),
                                             _vp(seeds1), _vp(seeds2), _vp(out1), _vp(out2), _vp(out2ds), n, rx, ry, conv, stop))
        return out1, out2, out2ds

    def iclm2d(self, order, q, rx, ry, conv, stop, damping=(100.0, 0.1, 10.0)):
        """ICLM2D1 / ICLM2D2 (reference src/oc_iclm.cpp); damping = (lambda, alpha, beta)."""
        _check_queue(q, POI2D_FLOATS)
        self._ck(self._lib.ocb_iclm2d(self._ctx, int(order), _vp(q), q.shape[0], rx, ry, conv, stop,
                                      float(damping[0]), float(damping[1]), float(damping[2])))

    def epipolar_search2d(self, q, fundamental, parallax_x, parallax_y, search_radius, search_step, rx, ry, conv, stop):
        """EpipolarSearch::compute(queue) (reference src/oc_epipolar_search.cpp:133-205) as one batch."""
        _check_queue(q, POI2D_FLOATS)
        f = np.ascontiguousarray(fundamental, dtype=np.float32).reshape(9)
        ax = np.ascontiguousarray(parallax_x, dtype=np.float32).reshape(3)
        ay = np.ascontiguousarray(parallax_y, dtype=np.float32).reshape(3)
        self._ck(self._lib.ocb_epipolar_search2d(self._ctx, _vp(q), q.shape[0], _vp(f), _vp(ax), _vp(ay), int(search_radius),
                                                 int(search_step), rx, ry, conv, stop))

    def strain(self, q, radius, min_neighbors, zncc_threshold=0.9, approximation=1):
        """Strain::prepare + compute(queue) (reference src/oc_strain.cpp) on a POI2D [n,25] or POI3D [n,31] queue."""
        if q.ndim == 2 and q.shape[1] == 28:  # POI2DS records (stereo DIC)
            _check_queue(q, 28)
            fn = self._lib.ocb_strain2ds
        elif q.ndim == 2 and q.shape[1] == POI3D_FLOATS:
            _check_queue(q, POI3D_FLOATS)
            fn = self._lib.ocb_strain3d
        else:
            _check_queue(q, POI2D_FLOATS)
            fn = self._lib.ocb_strain2d
        self._ck(fn(self._ctx, _vp(q), q.shape[0], float(radius), int(min_neighbors), float(zncc_threshold), int(approximation)))

    def strain_series(self, q, radius, min_neighbors, zncc_threshold=0.9, approximation=1):
        """strain on every frame of a series, q a C-contiguous float32 [n_frames, n, floats] array of POI2D (25), POI3D (31) or
        POI2DS (28) records whose positions are the same in every frame (include/opencorr_b200.h ocb_strain2d_series): each
        frame's records become those strain leaves on that frame, with each POI's neighbours searched once."""
        if not isinstance(q, np.ndarray) or q.dtype != np.float32 or q.ndim != 3 or q.shape[2] not in _STRAIN_SERIES \
                or not q.flags.c_contiguous:
            raise ValueError("strain_series takes a C-contiguous float32 array of shape [n_frames, n, 25 | 31 | 28]")
        fn = getattr(self._lib, "ocb_strain%s_series" % _STRAIN_SERIES[q.shape[2]])
        self._ck(fn(self._ctx, _vp(q), q.shape[0], q.shape[1], float(radius), int(min_neighbors), float(zncc_threshold), int(approximation)))

    def strain_series_dev(self, kind, d_q, n_frames, n, radius, min_neighbors, zncc_threshold=0.9, approximation=1):
        """strain_series on device records (a pointer as an int); kind "2d", "3d" or "2ds".  Only enqueues."""
        if kind not in _STRAIN_SERIES.values():
            raise ValueError("kind must be '2d', '3d' or '2ds'")
        fn = getattr(self._lib, "ocb_strain%s_series_dev" % kind)
        self._ck(fn(self._ctx, int(d_q), n_frames, n, float(radius), int(min_neighbors), float(zncc_threshold), int(approximation)))

    def region_fit(self, reliable, q, radius, min_neighbors):
        """RegionFit2D / RegionFit3D (reference src/oc_region_fit.cpp) setNeighbor(reliable) + compute(queue): q and reliable are
        both POI2D [n,25] or both POI3D [n,31]; every POI of q with enough reliable neighbours takes their plane fit as its
        first-order deformation, with zncc 0 (include/opencorr_b200.h ocb_region_fit2d)."""
        floats = POI3D_FLOATS if q.ndim == 2 and q.shape[1] == POI3D_FLOATS else POI2D_FLOATS
        _check_queue(q, floats)
        _check_queue(reliable, floats)
        fn = self._lib.ocb_region_fit3d if floats == POI3D_FLOATS else self._lib.ocb_region_fit2d
        self._ck(fn(self._ctx, _vp(reliable), reliable.shape[0], _vp(q), q.shape[0], float(radius), int(min_neighbors)))

    def region_fit_dev(self, kind, d_reliable, n_reliable, d_q, n, radius, min_neighbors):
        """region_fit on device records (pointers as ints); kind "2d" or "3d".  Only enqueues."""
        if kind not in ("2d", "3d"):
            raise ValueError("kind must be '2d' or '3d'")
        fn = getattr(self._lib, "ocb_region_fit%s_dev" % kind)
        self._ck(fn(self._ctx, int(d_reliable), n_reliable, int(d_q), n, float(radius), int(min_neighbors)))

    def icgn2d_recover(self, order, q, rx, ry, conv, stop, radius, min_neighbors, zncc_high, zncc_low, max_rounds):
        """Recover the unreliable POIs of a registered POI2D queue q [n,25] in place: rounds of RegionFit2D over the reliable POIs
        and ICGN2D<order> on the unreliable ones, each POI that passes moved into the reliable set, until a round recovers none
        or max_rounds have run (include/opencorr_b200.h ocb_icgn2d_recover).  Returns (recovered int64 (max_rounds,): the POIs
        accepted in each round, remaining: the POIs still unreliable)."""
        _check_queue(q, POI2D_FLOATS)
        return self._recover(self._lib.ocb_icgn2d_recover, (int(order), _vp(q), q.shape[0], rx, ry), conv, stop, radius, min_neighbors,
                             zncc_high, zncc_low, max_rounds)

    def icgn3d_recover(self, q, rx, ry, rz, conv, stop, radius, min_neighbors, zncc_high, zncc_low, max_rounds):
        """icgn2d_recover for a POI3D queue q [n,31], with RegionFit3D and ICGN3D1.  Returns (recovered, remaining)."""
        _check_queue(q, POI3D_FLOATS)
        return self._recover(self._lib.ocb_icgn3d_recover, (_vp(q), q.shape[0], rx, ry, rz), conv, stop, radius, min_neighbors, zncc_high,
                             zncc_low, max_rounds)

    def icgn2d_recover_dev(self, order, d_q, n, rx, ry, conv, stop, radius, min_neighbors, zncc_high, zncc_low, max_rounds):
        """icgn2d_recover on device records (a pointer as an int); synchronises the stream.  Returns (recovered, remaining)."""
        return self._recover(self._lib.ocb_icgn2d_recover_dev, (int(order), int(d_q), n, rx, ry), conv, stop, radius, min_neighbors,
                             zncc_high, zncc_low, max_rounds)

    def icgn3d_recover_dev(self, d_q, n, rx, ry, rz, conv, stop, radius, min_neighbors, zncc_high, zncc_low, max_rounds):
        """icgn3d_recover on device records (a pointer as an int); synchronises the stream.  Returns (recovered, remaining)."""
        return self._recover(self._lib.ocb_icgn3d_recover_dev, (int(d_q), n, rx, ry, rz), conv, stop, radius, min_neighbors, zncc_high,
                             zncc_low, max_rounds)

    def _recover(self, fn, head, conv, stop, radius, min_neighbors, zncc_high, zncc_low, max_rounds):
        if int(max_rounds) < 0:
            raise ValueError("max_rounds must be >= 0")
        counts = np.zeros(int(max_rounds), np.uint64)
        remaining = ctypes.c_size_t(0)
        self._ck(fn(self._ctx, *head, float(conv), float(stop), float(radius), int(min_neighbors), float(zncc_high), float(zncc_low),
                    int(max_rounds), _vp(counts) if len(counts) else None, ctypes.byref(remaining)))
        return counts.astype(np.int64), int(remaining.value)

    def nr2d_prepare(self):
        self._ck(self._lib.ocb_nr2d_prepare(self._ctx))

    def nr2d1(self, q, rx, ry, conv, stop):
        """NR2D1 (reference src/oc_nr.cpp:160-334)."""
        _check_queue(q, POI2D_FLOATS)
        self._ck(self._lib.ocb_nr2d1(self._ctx, _vp(q), q.shape[0], rx, ry, conv, stop))

    def icgn3d1(self, q, rx, ry, rz, conv, stop):
        _check_queue(q, POI3D_FLOATS)
        self._ck(self._lib.ocb_icgn3d1(self._ctx, _vp(q), q.shape[0], rx, ry, rz, conv, stop))

    # hot path, device-resident POI queues (pointers as ints, e.g. torch.Tensor.data_ptr()) --------
    def fftcc2d_dev(self, d_q, n, rx, ry):
        self._ck(self._lib.ocb_fftcc2d_dev(self._ctx, int(d_q), n, rx, ry))

    def fftcc3d_dev(self, d_q, n, rx, ry, rz):
        self._ck(self._lib.ocb_fftcc3d_dev(self._ctx, int(d_q), n, rx, ry, rz))

    def icgn2d1_dev(self, d_q, n, rx, ry, conv, stop):
        self._ck(self._lib.ocb_icgn2d1_dev(self._ctx, int(d_q), n, rx, ry, conv, stop))

    def icgn2d2_dev(self, d_q, n, rx, ry, conv, stop):
        self._ck(self._lib.ocb_icgn2d2_dev(self._ctx, int(d_q), n, rx, ry, conv, stop))

    def set_series_2d_dev(self, d_ref, d_tars, n_frames, width, height):
        """Device pointers: ref (height x width) and the frame-major stack of n_frames targets; borrowed, not copied."""
        self._ck(self._lib.ocb_set_series_2d_dev(self._ctx, int(d_ref), int(d_tars), n_frames, width, height))
        self._frames["2d"] = int(n_frames)

    def icgn2d_series_dev(self, order, d_seeds, d_out, n, rx, ry, conv, stop):
        """n seed records in, n_frames x n records out (frame-major), device pointers; enqueue only."""
        self._ck(self._lib.ocb_icgn2d_series_dev(self._ctx, int(order), int(d_seeds), int(d_out), n, rx, ry, conv, stop))

    def icgn2d_series_reseed_dev(self, order, d_seeds, d_out, n, rx, ry, conv, stop, fft_rx, fft_ry, zncc_min):
        """icgn2d_series_reseed on device pointers; synchronises the stream.  Returns reseeded, int64 (F,)."""
        counts = np.zeros(self._series_frames("2d", "icgn2d_series_reseed"), np.uint64)
        self._ck(self._lib.ocb_icgn2d_series_reseed_dev(self._ctx, int(order), int(d_seeds), int(d_out), n, rx, ry, conv, stop, int(fft_rx), int(fft_ry),
                                                        float(zncc_min), _vp(counts)))
        return counts.astype(np.int64)

    def iclm2d_series_dev(self, order, d_seeds, d_out, n, rx, ry, conv, stop, damping=(100.0, 0.1, 10.0)):
        """n seed records in, n_frames x n records out (frame-major), device pointers; enqueue only."""
        self._ck(self._lib.ocb_iclm2d_series_dev(self._ctx, int(order), int(d_seeds), int(d_out), n, rx, ry, conv, stop, float(damping[0]),
                                                 float(damping[1]), float(damping[2])))

    def iclm2d_series_reseed_dev(self, order, d_seeds, d_out, n, rx, ry, conv, stop, fft_rx, fft_ry, zncc_min, damping=(100.0, 0.1, 10.0)):
        """iclm2d_series_reseed on device pointers; synchronises the stream.  Returns reseeded, int64 (F,)."""
        counts = np.zeros(self._series_frames("2d", "iclm2d_series_reseed"), np.uint64)
        self._ck(self._lib.ocb_iclm2d_series_reseed_dev(self._ctx, int(order), int(d_seeds), int(d_out), n, rx, ry, conv, stop, float(damping[0]),
                                                        float(damping[1]), float(damping[2]), int(fft_rx), int(fft_ry), float(zncc_min),
                                                        _vp(counts)))
        return counts.astype(np.int64)

    def nr2d1_series_dev(self, d_seeds, d_out, n, rx, ry, conv, stop):
        """n seed records in, n_frames x n records out (frame-major), device pointers; enqueue only."""
        self._ck(self._lib.ocb_nr2d1_series_dev(self._ctx, int(d_seeds), int(d_out), n, rx, ry, conv, stop))

    def nr2d1_series_reseed_dev(self, d_seeds, d_out, n, rx, ry, conv, stop, fft_rx, fft_ry, zncc_min):
        """nr2d1_series_reseed on device pointers; synchronises the stream.  Returns reseeded, int64 (F,)."""
        counts = np.zeros(self._series_frames("2d", "nr2d1_series_reseed"), np.uint64)
        self._ck(self._lib.ocb_nr2d1_series_reseed_dev(self._ctx, int(d_seeds), int(d_out), n, rx, ry, conv, stop, int(fft_rx), int(fft_ry),
                                                       float(zncc_min), _vp(counts)))
        return counts.astype(np.int64)

    def icgn3d1_dev(self, d_q, n, rx, ry, rz, conv, stop):
        self._ck(self._lib.ocb_icgn3d1_dev(self._ctx, int(d_q), n, rx, ry, rz, conv, stop))

    def set_series_3d_dev(self, d_ref, d_tars, n_frames, dim_x, dim_y, dim_z):
        """Device pointers: the float32 reference volume and the frame-major stack of n_frames targets; borrowed, not copied."""
        self._ck(self._lib.ocb_set_series_3d_dev(self._ctx, int(d_ref), int(d_tars), n_frames, dim_x, dim_y, dim_z))
        self._frames["3d"] = int(n_frames)

    def icgn3d_series_dev(self, d_seeds, d_out, n, rx, ry, rz, conv, stop):
        """n seed records in, n_frames x n records out (frame-major), device pointers; enqueue only."""
        self._ck(self._lib.ocb_icgn3d_series_dev(self._ctx, int(d_seeds), int(d_out), n, rx, ry, rz, conv, stop))

    def icgn3d_series_reseed_dev(self, d_seeds, d_out, n, rx, ry, rz, conv, stop, fft_rx, fft_ry, fft_rz, zncc_min):
        """icgn3d_series_reseed on device pointers; synchronises the stream.  Returns reseeded, int64 (F,)."""
        counts = np.zeros(self._series_frames("3d", "icgn3d_series_reseed"), np.uint64)
        self._ck(self._lib.ocb_icgn3d_series_reseed_dev(self._ctx, int(d_seeds), int(d_out), n, rx, ry, rz, conv, stop, int(fft_rx), int(fft_ry),
                                                        int(fft_rz), float(zncc_min), _vp(counts)))
        return counts.astype(np.int64)

    def set_stereo_series_dev(self, d_ref1, d_tars1, d_tars2, n_frames, width, height):
        """Device pointers: reference view 1 (height x width) and the frame-major stacks of view 1 and view 2 (n_frames images
        each); borrowed, not copied."""
        self._ck(self._lib.ocb_set_stereo_series_2d_dev(self._ctx, int(d_ref1), int(d_tars1), int(d_tars2), n_frames, width, height))
        self._frames["stereo"] = int(n_frames)

    def stereo_series_dev(self, rig, d_stereo, d_seeds1, d_seeds2, d_out1, d_out2, d_out2ds, n, order1, order2, rx, ry, conv, stop):
        """stereo_series on device pointers: n records each of stereo, seeds1, seeds2 in; n_frames x n POI2D records into d_out1
        and d_out2 and n_frames x n POI2DS records into d_out2ds (frame-major); enqueue only."""
        rig._engine()
        h1, i1, p1, h2, i2, p2 = rig._cameras()
        self._ck(self._lib.ocb_stereo_series_dev(self._ctx, h1, _vp(i1), _vp(p1), h2, _vp(i2), _vp(p2), int(order1), int(order2), int(d_stereo),
                                                 int(d_seeds1), int(d_seeds2), int(d_out1), int(d_out2), int(d_out2ds), int(n), rx, ry, conv,
                                                 stop))

    # SIFT3D --------------------------------------------------------------------------------------
    def sift3d(self, config=None, unit=(1.0, 1.0, 1.0), matching_ratio=0.85):
        """SIFT3D::compute() on the volumes of set_images_3d: returns (ref_matched_kp, tar_matched_kp, n_octave), the
        matched keypoints as float32 [n, 3] (x, y, z) arrays.  config: the 10 floats of Sift3dConfig in field order
        (SIFT3D_DEFAULT_CONFIG)."""
        cfg = np.ascontiguousarray(SIFT3D_DEFAULT_CONFIG if config is None else config, dtype=np.float32).reshape(SIFT3D_CONFIG_FLOATS)
        u = np.ascontiguousarray(unit, dtype=np.float32).reshape(3)
        n = ctypes.c_size_t(0)
        n_oct = ctypes.c_int(0)
        self._ck(self._lib.ocb_sift3d(self._ctx, _vp(cfg), _vp(u), float(matching_ratio), ctypes.byref(n), ctypes.byref(n_oct)))
        ref = np.empty((n.value, 3), np.float32)
        tar = np.empty((n.value, 3), np.float32)
        self._ck(self._lib.ocb_sift3d_get_matches(self._ctx, _vp(ref), _vp(tar)))
        return ref, tar, int(n_oct.value)

    def sift3d_inspect(self, image):
        """Products of the last sift3d() for image 0 (reference) or 1 (target): dict of cand [n, 5] int32 (octave, layer, z,
        y, x), max_abs [m] float32, kp [k, 18] float32, desc [k, 768] float32."""
        counts = (ctypes.c_size_t * 3)()
        self._ck(self._lib.ocb_sift3d_inspect(self._ctx, int(image), counts, None, None, None, None))
        out = dict(cand=np.empty((counts[0], 5), np.int32), max_abs=np.empty(counts[1], np.float32),
                   kp=np.empty((counts[2], SIFT3D_KP_FLOATS), np.float32), desc=np.empty((counts[2], 768), np.float32))
        self._ck(self._lib.ocb_sift3d_inspect(self._ctx, int(image), counts, _vp(out["cand"]), _vp(out["max_abs"]), _vp(out["kp"]),
                                              _vp(out["desc"])))
        return out

    def sift3d_inspect_counts(self, image):
        """Number of keypoints the last sift3d() kept in image 0 (reference) or 1 (target)."""
        counts = (ctypes.c_size_t * 3)()
        self._ck(self._lib.ocb_sift3d_inspect(self._ctx, int(image), counts, None, None, None, None))
        return int(counts[2])

    def sift3d_stage_times(self):
        """Milliseconds per stage of the last sift3d(), keyed by SIFT3D_STAGES."""
        ms = np.zeros(len(SIFT3D_STAGES), np.float32)
        self._ck(self._lib.ocb_sift3d_stage_times(self._ctx, _vp(ms)))
        return dict(zip(SIFT3D_STAGES, ms.tolist()))


_default_engines = {}


def default_engine(device=0):
    """Process-wide engine per device, shared by the operator objects below (the reference's
    objects all borrow the same Image2D/Image3D; here they share one device copy)."""
    key = tuple(device) if isinstance(device, (list, tuple)) else device
    eng = _default_engines.get(key)
    if eng is None or not eng._ctx:
        eng = Engine(device)
        _default_engines[key] = eng
    return eng


class _DIC:
    def __init__(self, rx, ry, thread_number=0, engine=None):
        self.subset_radius_x = int(rx)
        self.subset_radius_y = int(ry)
        self.thread_number = int(thread_number)
        self.self_adaptive = False
        self.engine = engine if engine is not None else default_engine()
        self.ref_img = None
        self.tar_img = None
        self._token = None      # engine.image_token of this object's own upload
        self._prepared = False  # prepare() has been called since set_images()

    def set_images(self, ref_img, tar_img):
        self.ref_img, self.tar_img = ref_img, tar_img
        self.engine.set_images_2d(ref_img, tar_img)
        self._token = self.engine.image_token
        self._prepared = False

    def _bind(self):
        """The operators of one engine share its device images (like the reference's objects share Image2D pointers), but
        each keeps ITS pair and prepared state (the reference keeps per-object tables): if another object has replaced the
        engine's images since, upload this object's pair again and redo its prepare()."""
        if self.ref_img is None or self._token == self.engine.image_token:
            return
        self.engine.set_images_2d(self.ref_img, self.tar_img)
        self._token = self.engine.image_token
        if self._prepared:
            self._prepare_engine()

    def _prepare_engine(self):
        pass

    def set_subset(self, radius_x, radius_y):
        self.subset_radius_x, self.subset_radius_y = int(radius_x), int(radius_y)

    setImages = set_images
    setSubset = set_subset


class _DVC:
    def __init__(self, rx, ry, rz, thread_number=0, engine=None):
        self.subset_radius_x = int(rx)
        self.subset_radius_y = int(ry)
        self.subset_radius_z = int(rz)
        self.thread_number = int(thread_number)
        self.engine = engine if engine is not None else default_engine()
        self.ref_img = None
        self.tar_img = None
        self._token = None
        self._prepared = False

    def set_images(self, ref_img, tar_img):
        self.ref_img, self.tar_img = ref_img, tar_img
        self.engine.set_images_3d(ref_img, tar_img)
        self._token = self.engine.image_token
        self._prepared = False

    def _bind(self):
        """See _DIC._bind."""
        if self.ref_img is None or self._token == self.engine.image_token:
            return
        self.engine.set_images_3d(self.ref_img, self.tar_img)
        self._token = self.engine.image_token
        if self._prepared:
            self._prepare_engine()

    def _prepare_engine(self):
        pass

    def set_subset(self, radius_x, radius_y, radius_z):
        self.subset_radius_x, self.subset_radius_y, self.subset_radius_z = int(radius_x), int(radius_y), int(radius_z)

    setImages = set_images
    setSubset = set_subset


class FFTCC2D(_DIC):
    def prepare(self):
        pass

    def compute(self, poi_queue):
        self._bind()
        self.engine.fftcc2d(poi_queue, self.subset_radius_x, self.subset_radius_y)
        return poi_queue


class FFTCC3D(_DVC):
    def prepare(self):
        pass

    def compute(self, poi_queue):
        self._bind()
        self.engine.fftcc3d(poi_queue, self.subset_radius_x, self.subset_radius_y, self.subset_radius_z)
        return poi_queue


class _ICGN2D(_DIC):
    _order = 1

    def __init__(self, rx, ry, conv_criterion, stop_condition, thread_number=0, engine=None):
        super().__init__(rx, ry, thread_number, engine)
        self.conv_criterion = float(conv_criterion)
        self.stop_condition = float(stop_condition)

    def set_iteration(self, conv_criterion, stop_condition):
        self.conv_criterion, self.stop_condition = float(conv_criterion), float(stop_condition)

    def _prepare_engine(self):
        self.engine.icgn2d_prepare()

    def prepare(self):
        self._bind()
        self._prepare_engine()
        self._prepared = True

    prepare_ref = prepare
    prepare_tar = prepare

    def compute(self, poi_queue, center_offset_queue=None):
        """compute(queue) and compute(queue, center_offset_queue); honours set_self_adaptive(True)."""
        self._bind()
        if center_offset_queue is None and not self.self_adaptive:
            fn = self.engine.icgn2d1 if self._order == 1 else self.engine.icgn2d2
            fn(poi_queue, self.subset_radius_x, self.subset_radius_y, self.conv_criterion, self.stop_condition)
        else:
            self.engine.icgn2d_ex(self._order, poi_queue, self.subset_radius_x, self.subset_radius_y, self.conv_criterion,
                                  self.stop_condition, center_offset_queue, self.self_adaptive)
        return poi_queue

    def set_self_adaptive(self, is_self_adaptive):
        self.self_adaptive = bool(is_self_adaptive)

    setSelfAdaptive = set_self_adaptive

    setIteration = set_iteration
    prepareRef = prepare_ref
    prepareTar = prepare_tar


class ICGN2D1(_ICGN2D):
    _order = 1


class ICGN2D2(_ICGN2D):
    _order = 2


class _ICLM2D(_ICGN2D):
    """ICLM2D1 / ICLM2D2(int rx, int ry, float conv, float stop, int threads), reference src/oc_iclm.h:56-75,110-130."""

    def __init__(self, rx, ry, conv_criterion, stop_condition, thread_number=0, engine=None):
        super().__init__(rx, ry, conv_criterion, stop_condition, thread_number, engine)
        self.damping = (100.0, 0.1, 10.0)

    def set_damping(self, lambda_, alpha, beta):
        self.damping = (float(lambda_), float(alpha), float(beta))

    def compute(self, poi_queue):
        self._bind()
        self.engine.iclm2d(self._order, poi_queue, self.subset_radius_x, self.subset_radius_y, self.conv_criterion,
                           self.stop_condition, self.damping)
        return poi_queue

    setDamping = set_damping


class ICLM2D1(_ICLM2D):
    _order = 1


class ICLM2D2(_ICLM2D):
    _order = 2


class NR2D1(_DIC):
    """NR2D1(int rx, int ry, float conv, float stop, int threads), reference src/oc_nr.h:46-71."""

    def __init__(self, rx, ry, conv_criterion, stop_condition, thread_number=0, engine=None):
        super().__init__(rx, ry, thread_number, engine)
        self.conv_criterion = float(conv_criterion)
        self.stop_condition = float(stop_condition)

    def set_iteration(self, conv_criterion, stop_condition):
        self.conv_criterion, self.stop_condition = float(conv_criterion), float(stop_condition)

    def _prepare_engine(self):
        self.engine.nr2d_prepare()

    def prepare(self):
        self._bind()
        self._prepare_engine()
        self._prepared = True

    def compute(self, poi_queue):
        self._bind()
        self.engine.nr2d1(poi_queue, self.subset_radius_x, self.subset_radius_y, self.conv_criterion, self.stop_condition)
        return poi_queue

    setIteration = set_iteration


INTRINSIC_NAMES = ("fx", "fy", "fs", "cx", "cy", "k1", "k2", "k3", "k4", "k5", "k6", "p1", "p2")  # CameraIntrinsics order


class Calibration:
    """Calibration(CameraIntrinsics, CameraExtrinsics), reference src/oc_calibration.h:25-98, .cpp:21-264: the intrinsic matrix,
    the rotation matrix from the rotation vector (rx, ry, rz), the translation vector and the projection matrix K [R | t], float32,
    and the lens-distortion correction -- prepare(height, width) builds the map of undistorted image coordinates on the GPU,
    undistort(points) looks points up in it.  The distortion model is (1 + k1 r^2 + k2 r^4 + k3 r^6) / (1 + k4 r^2 + k5 r^4 +
    k6 r^6) with tangential terms p1, p2 and skew fs.  The map stays in device memory (the reference's map_x / map_y Eigen members
    are not exposed); it belongs to `engine` (default: the process-wide engine of device 0)."""

    def __init__(self, fx, fy, fs, cx, cy, tx=0.0, ty=0.0, tz=0.0, rx=0.0, ry=0.0, rz=0.0, k1=0.0, k2=0.0, k3=0.0, k4=0.0, k5=0.0,
                 k6=0.0, p1=0.0, p2=0.0, engine=None):
        self.intrinsics = dict(fx=fx, fy=fy, fs=fs, cx=cx, cy=cy, k1=k1, k2=k2, k3=k3, k4=k4, k5=k5, k6=k6, p1=p1, p2=p2)
        self.extrinsics = dict(tx=tx, ty=ty, tz=tz, rx=rx, ry=ry, rz=rz)
        self.convergence = 0.001  # src/oc_calibration.cpp:21-32
        self.iteration = 40
        self.engine = engine
        self._calib = None  # ocb_calib handle of prepare()
        self._map_engine = None
        self.height = self.width = 0
        self.update_matrices()

    def __del__(self):
        try:
            self._release()
        except Exception:
            pass

    def _release(self):
        if getattr(self, "_calib", None):
            _capi.load().ocb_calib_destroy(self._calib)
            self._calib = None

    def intrinsic_vector(self):
        """The 13 floats of CameraIntrinsics (fx fy fs cx cy k1..k6 p1 p2) as they are now."""
        return np.array([self.intrinsics[k] for k in INTRINSIC_NAMES], np.float32)

    def get_convergence(self):
        return self.convergence

    def get_iteration(self):
        return self.iteration

    def set_undistortion(self, convergence, iteration):
        """setUndistortion (:111-115): stop rules of the fixed-point loop of prepare()."""
        self.convergence, self.iteration = float(convergence), int(iteration)

    def prepare(self, height, width):
        """Calibration::prepare (:161-219): the distortion map of a height x width camera, built on the GPU."""
        eng = self.engine if self.engine is not None else default_engine()
        h = ctypes.c_void_p()
        intr = self.intrinsic_vector()
        rc = eng._lib.ocb_calib_prepare(eng._ctx, _vp(intr), int(height), int(width), float(self.convergence), int(self.iteration),
                                        ctypes.byref(h))
        eng._ck(rc)
        self._release()
        self._calib, self._map_engine = h.value, eng
        self.height, self.width = int(height), int(width)

    def _need_map(self):
        if not self._calib:
            raise _capi.OpenCorrB200Error(_capi.OCB_ERR_STATE, "Calibration: prepare(height, width) has not been called")
        return self._map_engine

    def get_map(self):
        """(map_x, map_y): float32 [height, width] copies of the device map (for tests)."""
        eng = self._need_map()
        mx = np.empty((self.height, self.width), np.float32)
        my = np.empty((self.height, self.width), np.float32)
        eng._ck(eng._lib.ocb_calib_get_map(eng._ctx, self._calib, _vp(mx), _vp(my)))
        return mx, my

    def undistort(self, points):
        """Calibration::undistort (:221-264) for a C-contiguous float32 [n, 2] array: the points are clamped in place to
        [0, W-2] x [0, H-2] (the reference takes Point2D&); returns the sensor coordinates [n, 2]."""
        eng = self._need_map()
        _check_points(points)
        out = np.empty_like(points)
        intr = self.intrinsic_vector()
        eng._ck(eng._lib.ocb_calib_undistort(eng._ctx, self._calib, _vp(intr), _vp(points), _vp(out), points.shape[0]))
        return out

    def projection_vector(self):
        return np.ascontiguousarray(self.projection_matrix, dtype=np.float32).reshape(12)

    def update_matrices(self):
        f32 = np.float32
        i, e = self.intrinsics, self.extrinsics
        self.intrinsic_matrix = np.array([[i["fx"], i["fs"], i["cx"]], [0, i["fy"], i["cy"]], [0, 0, 1]], f32)
        v = np.array([e["rx"], e["ry"], e["rz"]], f32)
        th = f32(np.linalg.norm(v))
        if th == 0:
            self.rotation_matrix = np.eye(3, dtype=f32)
        else:  # Eigen::AngleAxisf::toRotationMatrix, src/oc_calibration.cpp:50-60
            x, y, z = v / th
            c, s = f32(np.cos(th)), f32(np.sin(th))
            t = f32(1) - c
            self.rotation_matrix = np.array([[t * x * x + c, t * x * y - s * z, t * x * z + s * y],
                                             [t * x * y + s * z, t * y * y + c, t * y * z - s * x],
                                             [t * x * z - s * y, t * y * z + s * x, t * z * z + c]], f32)
        self.translation_vector = np.array([e["tx"], e["ty"], e["tz"]], f32)
        # K [R | t] (:69-77), each entry summed over k = 0, 1, 2 in float32
        rt = np.concatenate([self.rotation_matrix, self.translation_vector[:, None]], axis=1)
        p = np.zeros((3, 4), f32)
        for i in range(3):
            for j in range(4):
                v = f32(0)
                for k in range(3):
                    v = f32(v + f32(self.intrinsic_matrix[i, k] * rt[k, j]))
                p[i, j] = v
        self.projection_matrix = p

    updateMatrices = update_matrices
    getConvergence = get_convergence
    getIteration = get_iteration
    setUndistortion = set_undistortion


def _fundamental_matrix(c1, c2):
    """K2^-T [t2]x R2 K1^-1 in float32 (EpipolarSearch::updateFundementalMatrix src/oc_epipolar_search.cpp:110-126, and
    Stereovision::updateFundementalMatrix src/oc_stereovision.cpp:36-54)."""
    f32 = np.float32
    t = c2.translation_vector
    tx = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]], f32)
    e = (tx @ c2.rotation_matrix).astype(f32)
    k2_inv_t = np.linalg.inv(c2.intrinsic_matrix.astype(np.float64)).T.astype(f32)
    k1_inv = np.linalg.inv(c1.intrinsic_matrix.astype(np.float64)).astype(f32)
    return (k2_inv_t @ e @ k1_inv).astype(f32)


class Stereovision:
    """Stereovision(Calibration* view1_cam, Calibration* view2_cam, int thread_number), reference src/oc_stereovision.h,
    .cpp:21-133.  Both cameras must have been prepare()d on the same engine.  reconstruct(pts1, pts2) triangulates every pair
    in one GPU batch: float32 [n, 2] arrays (clamped in place, as the reference's Point2D& arguments are) -> float32 [n, 3];
    a pair with a NaN coordinate gives (0, 0, 0) and is left untouched."""

    def __init__(self, view1_cam, view2_cam, thread_number=0, engine=None):
        self.view1_cam, self.view2_cam = view1_cam, view2_cam
        self.thread_number = int(thread_number)
        self.engine = engine
        self.fundamental_matrix = None

    def update_cameras(self, view1_cam, view2_cam):
        self.view1_cam, self.view2_cam = view1_cam, view2_cam

    def update_fundamental_matrix(self):
        self.fundamental_matrix = _fundamental_matrix(self.view1_cam, self.view2_cam)

    def prepare(self):
        """:56-68: the matrices of both cameras and the fundamental matrix."""
        self.view1_cam.update_matrices()
        self.view2_cam.update_matrices()
        self.update_fundamental_matrix()

    def _engine(self):
        e1, e2 = self.view1_cam._need_map(), self.view2_cam._need_map()
        if e1 is not e2:
            raise _capi.OpenCorrB200Error(_capi.OCB_ERR_ARG, "Stereovision: the two cameras were prepared on different engines")
        if self.engine is not None and self.engine is not e1:
            raise _capi.OpenCorrB200Error(_capi.OCB_ERR_ARG, "Stereovision: the cameras were prepared on another engine")
        return e1

    def _cameras(self):
        """(calib1, intrinsics1, projection1, calib2, intrinsics2, projection2): handles and float32 arrays as they are now."""
        c1, c2 = self.view1_cam, self.view2_cam
        return (c1._calib, c1.intrinsic_vector(), c1.projection_vector(), c2._calib, c2.intrinsic_vector(), c2.projection_vector())

    def reconstruct(self, pts1, pts2):
        """reconstruct(queue, queue, queue) (:126-133); a single pair is an [1, 2] array."""
        eng = self._engine()
        _check_points(pts1)
        _check_points(pts2)
        if pts1.shape != pts2.shape:
            raise ValueError("pts1 and pts2 must have the same shape")
        out = np.empty((pts1.shape[0], 3), np.float32)
        h1, i1, p1, h2, i2, p2 = self._cameras()
        eng._ck(eng._lib.ocb_stereo_reconstruct(eng._ctx, h1, _vp(i1), _vp(p1), h2, _vp(i2), _vp(p2), _vp(pts1), _vp(pts2), _vp(out),
                                                pts1.shape[0]))
        return out

    def reconstruct_dev(self, d_pts1, d_pts2, d_pts3d, n):
        """Device pointers (ints, e.g. torch.Tensor.data_ptr()) of n x 2, n x 2 and n x 3 floats: enqueue only, on a
        single-device engine."""
        eng = self._engine()
        h1, i1, p1, h2, i2, p2 = self._cameras()
        eng._ck(eng._lib.ocb_stereo_reconstruct_dev(eng._ctx, h1, _vp(i1), _vp(p1), h2, _vp(i2), _vp(p2), int(d_pts1), int(d_pts2),
                                                    int(d_pts3d), int(n)))

    updateCameras = update_cameras
    updateFundementalMatrix = update_fundamental_matrix


class EpipolarSearch(_DIC):
    """EpipolarSearch(Calibration& view1_cam, Calibration& view2_cam, int thread_number), reference
    src/oc_epipolar_search.h:30-63.  set_images(view1, view2); the candidate sweep of all POIs runs as one GPU batch."""

    def __init__(self, view1_cam, view2_cam, thread_number=0, engine=None):
        super().__init__(0, 0, thread_number, engine)
        self.view1_cam, self.view2_cam = view1_cam, view2_cam
        self.search_radius, self.search_step = 0, 1
        self.parallax_x = np.zeros(3, np.float32)
        self.parallax_y = np.zeros(3, np.float32)
        self.fundamental_matrix = None
        self._icgn = None

    def set_search(self, search_radius, search_step):
        if search_radius < search_step:
            raise ValueError("Search radius is less than search step")
        self.search_radius, self.search_step = int(search_radius), int(search_step)

    def create_icgn(self, subset_radius_x, subset_radius_y, conv_criterion, stop_condition):
        self._icgn = (int(subset_radius_x), int(subset_radius_y), float(conv_criterion), float(stop_condition))

    def set_parallax(self, *args):
        """set_parallax((px, py))  or  set_parallax(coefficient_x[3], coefficient_y[3])  (src/oc_epipolar_search.cpp:74-95)."""
        if len(args) == 1:
            self.parallax_x = np.array([0, 0, args[0][0]], np.float32)
            self.parallax_y = np.array([0, 0, args[0][1]], np.float32)
        else:
            self.parallax_x = np.asarray(args[0], np.float32).reshape(3)
            self.parallax_y = np.asarray(args[1], np.float32).reshape(3)

    def update_cameras(self, view1_cam, view2_cam):
        self.view1_cam, self.view2_cam = view1_cam, view2_cam

    def update_fundamental_matrix(self):
        """src/oc_epipolar_search.cpp:110-126, float32."""
        self.fundamental_matrix = _fundamental_matrix(self.view1_cam, self.view2_cam)

    def prepare(self):
        self.view1_cam.update_matrices()
        self.view2_cam.update_matrices()
        self.update_fundamental_matrix()
        self._bind()
        self._prepare_engine()
        self._prepared = True

    def _prepare_engine(self):
        self.engine.icgn2d_prepare()

    def compute(self, poi_queue):
        if self._icgn is None or self.fundamental_matrix is None:
            raise _capi.OpenCorrB200Error(_capi.OCB_ERR_STATE, "EpipolarSearch: create_icgn() and prepare() must be called before compute()")
        self._bind()
        rx, ry, conv, stop = self._icgn
        self.engine.epipolar_search2d(poi_queue, self.fundamental_matrix, self.parallax_x, self.parallax_y, self.search_radius,
                                      self.search_step, rx, ry, conv, stop)
        return poi_queue

    setSearch = set_search
    createICGN = create_icgn
    setParallax = set_parallax
    updateCameras = update_cameras
    updateFundementalMatrix = update_fundamental_matrix


class Strain:
    """Strain(float subregion_radius, int neighbor_number_min, int thread_number), reference src/oc_strain.h:33-70."""

    def __init__(self, subregion_radius, neighbor_number_min, thread_number=0, engine=None):
        self.engine = engine if engine is not None else default_engine()
        self.subregion_radius = float(subregion_radius)
        self.neighbor_number_min = int(neighbor_number_min)
        self.zncc_threshold = 0.9  # src/oc_strain.cpp:38-40
        self.description = 1
        self.approximation = 1
        self.thread_number = thread_number

    def set_subregion_radius(self, r):
        self.subregion_radius = float(r)

    def set_neighbor_min(self, k):
        self.neighbor_number_min = int(k)

    def set_zncc_threshold(self, t):
        self.zncc_threshold = float(t)

    def set_description(self, d):
        self.description = int(d)

    def set_approximation(self, a):
        self.approximation = int(a)

    def prepare(self, poi_queue):
        """The reference builds its kd-trees here; the grid binning happens inside compute()."""

    def compute(self, poi_queue):
        self.engine.strain(poi_queue, self.subregion_radius, self.neighbor_number_min, self.zncc_threshold, self.approximation)
        return poi_queue

    setSubregionRadius = set_subregion_radius
    setNeighborMin = set_neighbor_min
    setZnccThreshold = set_zncc_threshold
    setDescription = set_description
    setApproximation = set_approximation


class _RegionFit:
    """RegionFit2D / RegionFit3D(float neighbor_search_radius, int neighbor_number_min, int thread_number), reference
    src/oc_region_fit.h:25-85.  setNeighbor keeps a reference to the reliable queue, which is read when compute runs."""
    _floats = None

    def __init__(self, neighbor_search_radius, neighbor_number_min, thread_number=0, engine=None):
        self.engine = engine if engine is not None else default_engine()
        self.neighbor_search_radius = float(neighbor_search_radius)
        self.neighbor_number_min = int(neighbor_number_min)
        self.thread_number = thread_number
        self.neighbor_reliable = np.zeros((0, self._floats), np.float32)

    def get_search_radius(self):
        return self.neighbor_search_radius

    def get_neighbor_min(self):
        return self.neighbor_number_min

    def set_search_radius(self, r):
        self.neighbor_search_radius = float(r)

    def set_neighbor_min(self, k):
        self.neighbor_number_min = int(k)

    def set_neighbor(self, reliable_pois):
        _check_queue(reliable_pois, self._floats)
        self.neighbor_reliable = reliable_pois

    def prepare(self):
        """The reference builds its kd-trees here; the grid over the reliable set is built inside compute()."""

    def compute(self, poi_queue):
        """compute(std::vector<POI>&) on a queue [n, floats]; a single record [floats] is compute(POI*)."""
        q = poi_queue if poi_queue.ndim == 2 else poi_queue.reshape(1, -1)
        self.engine.region_fit(self.neighbor_reliable, q, self.neighbor_search_radius, self.neighbor_number_min)
        return poi_queue

    getSearchRadius = get_search_radius
    getNeighborMin = get_neighbor_min
    setSearchRadius = set_search_radius
    setNeighborMin = set_neighbor_min
    setNeighbor = set_neighbor


class RegionFit2D(_RegionFit):
    _floats = POI2D_FLOATS


class RegionFit3D(_RegionFit):
    _floats = POI3D_FLOATS


class ICGN3D1(_DVC):
    def __init__(self, rx, ry, rz, conv_criterion, stop_condition, thread_number=0, engine=None):
        super().__init__(rx, ry, rz, thread_number, engine)
        self.conv_criterion = float(conv_criterion)
        self.stop_condition = float(stop_condition)

    def set_iteration(self, conv_criterion, stop_condition):
        self.conv_criterion, self.stop_condition = float(conv_criterion), float(stop_condition)

    def _prepare_engine(self):
        self.engine.icgn3d_prepare()

    def prepare(self):
        self._bind()
        self._prepare_engine()
        self._prepared = True

    prepare_ref = prepare_tar = prepare

    def compute(self, poi_queue):
        self._bind()
        self.engine.icgn3d1(poi_queue, self.subset_radius_x, self.subset_radius_y, self.subset_radius_z,
                            self.conv_criterion, self.stop_condition)
        return poi_queue

    def tables(self):
        """(gx, gy, gz, coefficient) volumes built by prepare() -- for parity tests."""
        dz, dy, dx = np.asarray(self.ref_img).shape
        out = [np.empty((dz, dy, dx), np.float32) for _ in range(4)]
        eng = self.engine
        eng._ck(eng._lib.ocb_get_tables_3d(eng._ctx, _vp(out[0]), _vp(out[1]), _vp(out[2]), _vp(out[3])))
        return out

    setIteration = set_iteration
    prepareRef = prepareTar = prepare


class SIFT3D:
    """SIFT3D (reference src/oc_sift.h:117-155, src/oc_sift.cpp:140-1418): volumetric keypoints of the reference and target
    volumes, matched by descriptor distance with a ratio test.  compute() fills ref_matched_kp / tar_matched_kp, float32
    [n, 3] arrays of (x, y, z) in voxels of the input volumes, and prints the reference's two lines."""

    def __init__(self, engine=None):
        self.engine = engine if engine is not None else default_engine()
        self.sift_config = dict(zip(SIFT3D_CONFIG_FIELDS, SIFT3D_DEFAULT_CONFIG.tolist()))
        for k in ("n_octave_layers", "n_octave", "min_dimension"):
            self.sift_config[k] = int(self.sift_config[k])
        self.matching_ratio = float(np.float32(0.85))
        self.physical_unit = [1.0, 1.0, 1.0]
        self.ref_img = None
        self.tar_img = None
        self._token = None
        self.ref_matched_kp = np.empty((0, 3), np.float32)
        self.tar_matched_kp = np.empty((0, 3), np.float32)

    def set_images(self, ref_img, tar_img):
        self.ref_img, self.tar_img = ref_img, tar_img
        self.engine.set_images_3d(ref_img, tar_img)
        self._token = self.engine.image_token

    def get_sift_config(self):
        return dict(self.sift_config)

    def set_sift_config(self, sift_config):
        self.sift_config = dict(sift_config)

    def get_physical_unit(self, dim):
        return self.physical_unit[dim] if dim in (0, 1, 2) else 0.0

    def set_physical_unit(self, unit_x, unit_y, unit_z):
        self.physical_unit = [float(unit_x), float(unit_y), float(unit_z)]

    def get_matching_ratio(self):
        return self.matching_ratio

    def set_matching_ratio(self, matching_ratio):
        self.matching_ratio = float(matching_ratio)

    def prepare(self):
        """The icosahedron of prepare() is built into the kernels; nothing to do."""

    def clear(self):
        self.ref_matched_kp = np.empty((0, 3), np.float32)
        self.tar_matched_kp = np.empty((0, 3), np.float32)

    def compute(self):
        if self.ref_img is None:
            raise _capi.OpenCorrB200Error(_capi.OCB_ERR_STATE, "SIFT3D: set_images() has not been called")
        if self._token != self.engine.image_token:  # another operator replaced the engine's volumes
            self.set_images(self.ref_img, self.tar_img)
        cfg = np.array([self.sift_config[k] for k in SIFT3D_CONFIG_FIELDS], np.float32)
        self.clear()
        self.ref_matched_kp, self.tar_matched_kp, n_octave = self.engine.sift3d(cfg, self.physical_unit, self.matching_ratio)
        self.sift_config["n_octave"] = n_octave
        counts = [self.engine.sift3d_inspect_counts(i) for i in (0, 1)]
        print("%d features are extracted from the reference image." % counts[0])
        print("%d features are extracted from the target image." % counts[1])

    setImages = set_images
    getSiftConfig = get_sift_config
    setSiftConfig = set_sift_config
    getPhysicalUnit = get_physical_unit
    setPhysicalUnit = set_physical_unit
    getMatchingRatio = get_matching_ratio
    setMatchingRatio = set_matching_ratio
