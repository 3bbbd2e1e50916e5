"""An engine keeps its device buffers (image pairs, POI staging, offsets, candidates, FFT scratch, Strain workspace, 3D tables,
stereo points) across calls and only grows them.  Every call below runs on one long-lived engine, in sequences that re-use
and grow these buffers (small -> large -> small), and must give records bit-identical to a fresh engine that made only that
call.  The 2D queue cases also run with a page-locked queue (ocb_host_alloc), which the in-place kernels read and write
through PCIe: the records must be bit-identical to the pageable run."""
import ctypes

import numpy as np
import pytest

import opencorr_b200 as ob
import stereo_cases as sc
import util
from opencorr_b200 import _capi, synth

pytestmark = pytest.mark.gpu

SMALL, LARGE, SMALLER = 600, 20400, 400  # LARGE >= 16 384: the chunked host-queue path
FM = np.array([[0, 0, 0], [0, 0, -1], [0, 1, 0]], np.float32)  # rectified pair: epipolar lines y' = y
W2, H2 = 1280, 1024


def _fresh(setup, call, q):
    eng = ob.Engine(0)
    try:
        setup(eng)
        return call(eng, q)
    finally:
        eng.close()


def _same(a, b):
    return all(np.array_equal(x, y, equal_nan=True) for x, y in zip(a, b))


# ------------------------------------------------------------------------------------------------ image pairs
def _upload_2d(kind, ref, tar):
    def up(eng):
        if kind == "u8":
            eng.set_images_2d(ref.astype(np.uint8), tar.astype(np.uint8))
        elif kind == "col_major":  # element (r, c) at c * h + r
            h, w = ref.shape
            rt, tt = np.ascontiguousarray(ref.T), np.ascontiguousarray(tar.T)
            assert eng._lib.ocb_set_images_2d(eng._ctx, ctypes.c_void_p(rt.ctypes.data), ctypes.c_void_p(tt.ctypes.data), w, h, 1) == 0
            eng.sync()
        else:
            eng.set_images_2d(ref, tar)
    return up


def _probe_2d(eng, _):
    q = ob.make_poi2d(synth.grid_2d(24, 24, 15, 15, 14, 14))
    eng.fftcc2d(q, 16, 16)
    eng.icgn2d_prepare()
    eng.icgn2d1(q, 16, 16, 0.001, 10)
    return (q,)


def _probe_3d(eng, _):
    q = ob.make_poi3d(synth.grid_3d(16, 16, 16, 4, 4, 4, 8, 8, 8))
    eng.fftcc3d(q, 8, 8, 8)
    eng.icgn3d_prepare()
    eng.icgn3d1(q, 8, 8, 8, 0.001, 20)
    return (q,)


@pytest.mark.parametrize("kind", ["float", "col_major", "u8"])
def test_image_pair_2d_small_large_small(kind):
    seq = ob.Engine(0)
    try:
        for w, h in ((256, 256), (W2, H2), (320, 288)):  # the large pair takes the banded upload of row-major float images
            up = _upload_2d(kind, *synth.speckle_pair_2d(w, h))
            up(seq)
            assert _same(_probe_2d(seq, None), _fresh(up, _probe_2d, None)), (w, h)
    finally:
        seq.close()


@pytest.mark.parametrize("cast", [np.float32, np.uint8])
def test_image_pair_3d_small_large_small(cast):
    seq = ob.Engine(0)
    try:
        for dims in ((64, 60, 56), (112, 104, 96), (72, 64, 60)):
            ref, tar = synth.speckle_pair_3d(*dims)
            up = lambda eng: eng.set_images_3d(ref.astype(cast), tar.astype(cast))  # noqa: E731
            up(seq)
            assert _same(_probe_3d(seq, None), _fresh(up, _probe_3d, None)), dims
    finally:
        seq.close()


# ------------------------------------------------------------------------------------------------ host queues
@pytest.fixture(scope="module")
def pair2d():
    return synth.speckle_pair_2d(W2, H2)


@pytest.fixture(scope="module")
def seed2d(pair2d):
    """LARGE POI2D records with the FFT-CC initial guess (one set of grid positions, repeated)."""
    q = ob.make_poi2d(synth.grid_2d(40, 40, 170, 120, 7, 7))
    eng = ob.Engine(0)
    try:
        eng.set_images_2d(*pair2d)
        eng.fftcc2d(q, 16, 16)
    finally:
        eng.close()
    return q


def _offsets(n):
    return np.random.default_rng(n).uniform(-3, 3, (n, 2)).astype(np.float32)


def _self_adaptive(eng, q):
    q[:, 23:25] = np.array([[12, 12], [16, 16], [10, 18]], np.float32)[np.arange(len(q)) % 3]
    eng.icgn2d_ex(1, q, 16, 16, 0.001, 10, center_offsets=_offsets(len(q)), self_adaptive=True)


CALLS_2D = {
    "fftcc2d_w32": lambda eng, q: eng.fftcc2d(q, 16, 16),
    "fftcc2d_reg": lambda eng, q: eng.fftcc2d(q, 12, 12),
    "icgn2d1": lambda eng, q: eng.icgn2d1(q, 16, 16, 0.001, 10),
    "icgn2d2": lambda eng, q: eng.icgn2d2(q, 16, 16, 0.001, 10),
    "icgn2d_ex_offsets": lambda eng, q: eng.icgn2d_ex(2, q, 16, 16, 0.001, 10, center_offsets=_offsets(len(q))),
    "icgn2d_ex_self_adaptive": _self_adaptive,
    "iclm2d": lambda eng, q: eng.iclm2d(1, q, 16, 16, 0.001, 10),
    "nr2d1": lambda eng, q: eng.nr2d1(q, 16, 16, 0.001, 10),
    "epipolar_search2d": lambda eng, q: eng.epipolar_search2d(q, FM, [0.001, 0, 1.5], [0, 0.002, 0.5], 24, 3, 12, 10, 0.05, 5),
}


def _queue_2d(seed, n):
    q = np.resize(seed, (n, seed.shape[1]))
    q[:, 16] = 0
    return q


@pytest.mark.parametrize("name", list(CALLS_2D))
def test_queue_2d_small_large_small(pair2d, seed2d, name):
    """Each size runs on the long-lived engine (whose buffers were sized by the previous call), on a fresh engine, and on the
    long-lived engine again with a page-locked copy of the queue."""
    call = CALLS_2D[name]
    lib = _capi.load()

    def setup(eng):
        eng.set_images_2d(*pair2d)
        eng.icgn2d_prepare()
        eng.nr2d_prepare()

    def run(eng, q):
        call(eng, q)
        return (q,)

    seq = ob.Engine(0)
    try:
        setup(seq)
        for n in (SMALL, LARGE, SMALLER):
            q0 = _queue_2d(seed2d, n)
            got = run(seq, q0.copy())
            assert not np.array_equal(got[0], q0) and _same(got, _fresh(setup, run, q0.copy())), n
            p = lib.ocb_host_alloc(q0.nbytes)
            assert p
            try:
                pinned = np.frombuffer((ctypes.c_byte * q0.nbytes).from_address(p), np.float32).reshape(q0.shape)
                pinned[...] = q0
                call(seq, pinned)
                assert np.array_equal(pinned, got[0], equal_nan=True), n
                del pinned
            finally:
                lib.ocb_host_free(p)
    finally:
        seq.close()


@pytest.fixture(scope="module")
def pair3d():
    return synth.speckle_pair_3d(96, 88, 80)


CALLS_3D = {
    "fftcc3d": lambda eng, q: eng.fftcc3d(q, 8, 8, 8),
    "icgn3d1": lambda eng, q: eng.icgn3d1(q, 8, 8, 8, 0.001, 20),
}


@pytest.mark.parametrize("name", list(CALLS_3D))
def test_queue_3d_small_large_small(pair3d, name):
    call = CALLS_3D[name]
    base = ob.make_poi3d(synth.grid_3d(20, 20, 20, 9, 8, 7, 6, 6, 6))

    def setup(eng):
        eng.set_images_3d(*pair3d)
        eng.icgn3d_prepare()

    def run(eng, q):
        call(eng, q)
        return (q,)

    seq = ob.Engine(0)
    try:
        setup(seq)
        for n in (SMALL, LARGE, SMALLER):
            q0 = np.resize(base, (n, base.shape[1]))
            q0[:, 15:18] = np.array([1, -1, 0], np.float32)  # an integer guess for ICGN3D1
            got = run(seq, q0.copy())
            assert not np.array_equal(got[0], q0) and _same(got, _fresh(setup, run, q0.copy())), n
    finally:
        seq.close()


def _strain_queues():
    """POI2D, POI3D and POI2DS queues of LARGE distinct positions with smooth displacements."""
    rng = np.random.default_rng(5)
    xy = synth.grid_2d(10, 10, 170, 120, 7, 7)
    q2 = ob.make_poi2d(xy)
    q2[:, 2] = 1e-3 * xy[:, 0] + rng.normal(0, 0.005, len(xy))
    q2[:, 8] = 0.5 * np.sin(xy[:, 1] / 40.0) + rng.normal(0, 0.005, len(xy))
    q2[:, 16] = 0.97
    xyz = rng.uniform(0, 600, (LARGE, 3)).astype(np.float32)
    q3 = ob.make_poi3d(xyz)
    disp = xyz @ rng.normal(0, 0.01, (3, 3)).T
    q3[:, 3], q3[:, 7], q3[:, 11] = disp[:, 0], disp[:, 1], disp[:, 2]
    q3[:, 18] = 0.95
    s, _, _ = util.gt4_stereo_queue()
    tiles = -(-LARGE // len(s))
    q23 = np.concatenate([s + np.array([5000.0 * k] + [0] * 27, np.float32) for k in range(tiles)])[:LARGE]  # tiles far apart
    return {"strain2d": q2, "strain3d": q3, "strain2ds": np.ascontiguousarray(q23)}


@pytest.mark.parametrize("name", ["strain2d", "strain3d", "strain2ds"])
def test_strain_small_large_small(name):
    base = _strain_queues()[name]

    def run(eng, q):
        ob.Strain(20.0, 5, engine=eng).compute(q)
        return (q,)

    seq = ob.Engine(0)
    try:
        for n in (SMALL, LARGE, SMALLER):
            q0 = np.ascontiguousarray(base[:n])
            assert _same(run(seq, q0.copy()), _fresh(lambda e: None, run, q0.copy())), n
    finally:
        seq.close()


# ------------------------------------------------------------------------------------------------ FFT scratch across kernels
def test_fftcc3d_scratch_across_kernel_paths(pair3d):
    """r = 16 (32-point register kernel), r = 12 (register codelets), then generic windows (14 = 2 * 7 points, and a non-cubic
    one) on one engine: each kernel sizes the shared FFT scratch differently."""
    base = ob.make_poi3d(synth.grid_3d(20, 20, 20, 9, 8, 7, 6, 6, 6))

    def setup(eng):
        eng.set_images_3d(*pair3d)

    seq = ob.Engine(0)
    try:
        setup(seq)
        for r, n in (((16, 16, 16), 504), ((12, 12, 12), 300), ((7, 7, 7), 504), ((10, 10, 12), 504), ((16, 16, 16), 100)):
            run = lambda eng, q: (eng.fftcc3d(q, *r), q)[1:]  # noqa: E731
            q0 = np.resize(base, (n, base.shape[1]))
            assert _same(run(seq, q0.copy()), _fresh(setup, run, q0.copy())), r
    finally:
        seq.close()


# ------------------------------------------------------------------------------------------------ stereo
def test_stereo_growing_point_counts():
    d = sc.load()
    r1, r2, _, _, _, _ = sc.gt4_points(d)

    def rig(eng):
        c1, c2, (h, w) = sc.rig(d, "gt4", eng)
        c1.prepare(h, w)
        c2.prepare(h, w)
        sv = ob.Stereovision(c1, c2, 0, eng)
        sv.prepare()
        return c1, sv

    def run(cams, n):
        c1, sv = cams
        a, b, u = r1[:n].copy(), r2[:n].copy(), r2[:n].copy()
        return a, b, sv.reconstruct(a, b), u, c1.undistort(u)

    seq = ob.Engine(0)
    try:
        cams = rig(seq)
        for n in (100, 2000, len(r1), 500):
            got = run(cams, n)
            fresh = ob.Engine(0)
            try:
                want = run(rig(fresh), n)
            finally:
                fresh.close()
            assert _same(got, want), n
    finally:
        seq.close()
