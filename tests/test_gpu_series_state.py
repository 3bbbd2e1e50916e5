"""Series and image-pair setters that fail part-way leave no state behind (include/opencorr_b200.h): a setter refused by its
argument checks changes nothing, and one whose device allocation fails (OCB_ERR_CUDA) leaves no series or pair set, so the
next call is refused with OCB_ERR_STATE instead of reading freed memory.

The failing setters ask for terabytes, more than any device has.  Their host buffers are small: the allocation fails before
any copy reads them."""
import ctypes

import numpy as np
import pytest

import opencorr_b200 as ob
import stereo_cases as sc
from opencorr_b200 import _capi, synth
from opencorr_b200.api import POI2DS_FLOATS

pytestmark = pytest.mark.gpu

CONV, STOP = 0.001, 10
W, H, F = 96, 80, 2
HUGE_2D = (1 << 18, 1024, 1024)   # frames, width, height: 1 TiB of floats per stack
HUGE_3D = (1 << 22, 64, 64, 64)   # frames, dim_x, dim_y, dim_z: 4 TiB of floats, 1 TiB of bytes


def vp(a):
    return ctypes.c_void_p(a.ctypes.data) if a is not None else None


@pytest.fixture
def eng():
    e = ob.Engine(0)
    yield e
    e.close()


def series_2d():
    ref, tar = synth.speckle_pair_2d(W, H)
    return ref, np.ascontiguousarray(np.stack([tar] * F))


def series_3d():
    ref, tars = synth.speckle_series_3d(24, 24, 24, F)
    return np.ascontiguousarray(ref, np.float32), np.ascontiguousarray(tars, np.float32)


def test_series_2d(eng):
    lib, ctx = eng._lib, eng._ctx
    ref, tars = series_2d()
    seeds = ob.make_poi2d(synth.grid_2d(30, 30, 2, 2, 20, 20))
    n = len(seeds)

    def call(count=n):
        out = np.full((F, n, ob.POI2D_FLOATS), 7.0, np.float32)
        return lib.ocb_icgn2d_series(ctx, 1, vp(seeds), vp(out), count, 8, 8, CONV, STOP), out

    assert lib.ocb_set_series_2d(ctx, vp(ref), vp(tars), F, W, H) == _capi.OCB_OK
    rc, before = call()
    assert rc == _capi.OCB_OK
    assert lib.ocb_set_series_2d(ctx, vp(ref), vp(tars), 0, W, H) == _capi.OCB_ERR_ARG
    assert lib.ocb_set_series_2d(ctx, vp(ref), None, F, W, H) == _capi.OCB_ERR_ARG
    rc, after = call()
    assert rc == _capi.OCB_OK and np.array_equal(before.view(np.uint32), after.view(np.uint32))
    assert lib.ocb_set_series_2d(ctx, vp(ref), vp(tars), *HUGE_2D) == _capi.OCB_ERR_CUDA
    assert call(0)[0] == _capi.OCB_ERR_STATE


@pytest.mark.parametrize("u8", [False, True])
def test_series_3d(eng, u8):
    lib, ctx = eng._lib, eng._ctx
    ref, tars = series_3d()
    if u8:
        ref, tars = ref.astype(np.uint8), tars.astype(np.uint8)
    setter = lib.ocb_set_series_3d_u8 if u8 else lib.ocb_set_series_3d
    seeds = ob.make_poi3d(synth.grid_3d(10, 10, 10, 2, 2, 2, 4, 4, 4))
    n = len(seeds)

    def call(count=n):
        out = np.full((F, n, ob.POI3D_FLOATS), 7.0, np.float32)
        return lib.ocb_icgn3d_series(ctx, vp(seeds), vp(out), count, 5, 5, 5, CONV, 20), out

    assert setter(ctx, vp(ref), vp(tars), F, 24, 24, 24) == _capi.OCB_OK
    rc, before = call()
    assert rc == _capi.OCB_OK
    assert setter(ctx, vp(ref), vp(tars), F, 24, 24, 14) == _capi.OCB_ERR_ARG
    assert setter(ctx, None, vp(tars), F, 24, 24, 24) == _capi.OCB_ERR_ARG
    rc, after = call()
    assert rc == _capi.OCB_OK and np.array_equal(before.view(np.uint32), after.view(np.uint32))
    assert setter(ctx, vp(ref), vp(tars), *HUGE_3D) == _capi.OCB_ERR_CUDA
    assert call(0)[0] == _capi.OCB_ERR_STATE


def test_stereo_series(eng):
    """Pins what the stereo setter already did before the series shared one setter path."""
    lib, ctx = eng._lib, eng._ctx
    intrinsics, extrinsics = synth.stereo_rig(W, H)
    c1, c2 = sc.camera(intrinsics[0], extrinsics[0], eng), sc.camera(intrinsics[1], extrinsics[1], eng)
    c1.prepare(H, W)
    c2.prepare(H, W)
    rig = ob.Stereovision(c1, c2, 0, eng)
    rig.prepare()
    h1, i1, p1, h2, i2, p2 = rig._cameras()
    ref, tars = series_2d()
    recs = ob.make_poi2d(synth.grid_2d(30, 30, 2, 2, 20, 20))
    n = len(recs)

    def call(count=n):
        outs = [np.full((F, n, ob.POI2D_FLOATS), 7.0, np.float32), np.full((F, n, ob.POI2D_FLOATS), 7.0, np.float32),
                np.full((F, n, POI2DS_FLOATS), 7.0, np.float32)]
        rc = lib.ocb_stereo_series(ctx, h1, vp(i1), vp(p1), h2, vp(i2), vp(p2), 1, 2, vp(recs), vp(recs), vp(recs), vp(outs[0]), vp(outs[1]),
                                   vp(outs[2]), count, 8, 8, CONV, STOP)
        return rc, np.concatenate([o.reshape(-1) for o in outs])

    assert lib.ocb_set_stereo_series_2d(ctx, vp(ref), vp(tars), vp(tars), F, W, H) == _capi.OCB_OK
    rc, before = call()
    assert rc == _capi.OCB_OK
    assert lib.ocb_set_stereo_series_2d(ctx, vp(ref), vp(tars), None, F, W, H) == _capi.OCB_ERR_ARG
    assert lib.ocb_set_stereo_series_2d(ctx, vp(ref), vp(tars), vp(tars), F, 4, H) == _capi.OCB_ERR_ARG
    rc, after = call()
    assert rc == _capi.OCB_OK and np.array_equal(before.view(np.uint32), after.view(np.uint32))
    assert lib.ocb_set_stereo_series_2d(ctx, vp(ref), vp(tars), vp(tars), *HUGE_2D) == _capi.OCB_ERR_CUDA
    assert call(0)[0] == _capi.OCB_ERR_STATE
    del rig


def test_images_2d(eng):
    lib, ctx = eng._lib, eng._ctx
    ref, tar = synth.speckle_pair_2d(W, H)
    xy = synth.grid_2d(30, 30, 2, 2, 20, 20)

    def fftcc():
        q = ob.make_poi2d(xy)
        return lib.ocb_fftcc2d(ctx, vp(q), len(q), 8, 8), q

    assert lib.ocb_set_images_2d(ctx, vp(ref), vp(tar), W, H, 0) == _capi.OCB_OK
    rc, before = fftcc()
    assert rc == _capi.OCB_OK
    assert lib.ocb_set_images_2d(ctx, vp(ref), vp(tar), 4, H, 0) == _capi.OCB_ERR_ARG
    assert lib.ocb_set_images_2d(ctx, None, vp(tar), W, H, 0) == _capi.OCB_ERR_ARG
    rc, after = fftcc()
    assert rc == _capi.OCB_OK and np.array_equal(before.view(np.uint32), after.view(np.uint32))
    assert lib.ocb_set_images_2d(ctx, vp(ref), vp(tar), 1 << 19, 1 << 19, 0) == _capi.OCB_ERR_CUDA
    assert lib.ocb_fftcc2d_dev(ctx, None, 0, 8, 8) == _capi.OCB_ERR_STATE
    assert lib.ocb_icgn2d_prepare(ctx) == _capi.OCB_ERR_STATE


def test_images_3d(eng):
    lib, ctx = eng._lib, eng._ctx
    ref, tar = synth.speckle_pair_3d(24, 24, 24)
    xyz = synth.grid_3d(10, 10, 10, 2, 2, 2, 4, 4, 4)

    def fftcc():
        q = ob.make_poi3d(xyz)
        return lib.ocb_fftcc3d(ctx, vp(q), len(q), 4, 4, 4), q

    assert lib.ocb_set_images_3d(ctx, vp(ref), vp(tar), 24, 24, 24) == _capi.OCB_OK
    rc, before = fftcc()
    assert rc == _capi.OCB_OK
    assert lib.ocb_set_images_3d(ctx, vp(ref), vp(tar), 24, 24, 14) == _capi.OCB_ERR_ARG
    rc, after = fftcc()
    assert rc == _capi.OCB_OK and np.array_equal(before.view(np.uint32), after.view(np.uint32))
    assert lib.ocb_set_images_3d(ctx, vp(ref), vp(tar), 1 << 13, 1 << 13, 1 << 13) == _capi.OCB_ERR_CUDA
    assert lib.ocb_fftcc3d_dev(ctx, None, 0, 4, 4, 4) == _capi.OCB_ERR_STATE
    assert lib.ocb_icgn3d_prepare(ctx) == _capi.OCB_ERR_STATE
