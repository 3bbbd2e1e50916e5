"""ICGN3D1 over a volume series with recovery of unreliable POIs (ocb_icgn3d_series_recover): out, recovered and remaining must be,
byte for byte, what the loop of existing calls
    set_images_3d(ref, tars[f]); icgn3d_prepare(); icgn3d1_dev(q); icgn3d_recover_dev(q)
gives when one queue q is carried from frame to frame (series_recover_cases.dev_loop)."""
import ctypes

import numpy as np
import pytest

import opencorr_b200 as ob
from opencorr_b200 import _capi, synth
import series_recover_cases as src
from util import assert_same

pytestmark = pytest.mark.gpu

DX, DY, DZ = 103, 100, 98  # dim_x % 4 != 0
FRAMES, K = 4, 1
R = (8, 8, 8)
P = src.Params(stop=20, radius=20.0, k_min=12, zncc_low=0.9)


def _ball(xyz, centre, radius):
    return ((xyz - np.array(centre)) ** 2).sum(1) < radius ** 2


def _occlude(tars, k, sel_xyz, r, margin=3):
    """Cover the subvolumes of the POIs sel_xyz in frame k with voxels from elsewhere in the same frame."""
    s = (k + 1) / len(tars)
    u, v, w = synth.displacement_3d(sel_xyz[:, 0], sel_xyz[:, 1], sel_xyz[:, 2], DX, DY, DZ)
    p = sel_xyz + s * np.stack([u, v, w], 1)
    x0, y0, z0 = np.maximum(np.floor(p - r - margin).min(0).astype(int), 0)
    x1, y1, z1 = np.minimum(np.ceil(p + r + margin + 1).max(0).astype(int), [DX, DY, DZ])
    out = tars.copy()
    out[k, z0:z1, y0:y1, x0:x1] = np.roll(tars[k], (DZ // 2, DY // 2, DX // 2), (0, 1, 2))[z0:z1, y0:y1, x0:x1]
    return out


@pytest.fixture(scope="module")
def volumes():
    """(ref, clean stack, stack whose frame K covers a ball of POIs, POIs, the ball)"""
    ref, clean = synth.speckle_series_3d(DX, DY, DZ, FRAMES)
    xyz = synth.grid_3d(16, 16, 16, 9, 9, 9, 8, 8, 8)
    ball = _ball(xyz, (48, 48, 48), 13)
    return ref, clean, _occlude(clean, K, xyz[ball], 8), xyz, ball


def _seeds(eng, ref, tar, xyz, garbage=None):
    q = ob.make_poi3d(xyz)
    eng.set_images_3d(ref, tar)
    eng.fftcc3d(q, *R)
    if garbage is not None:
        q[garbage, 3], q[garbage, 7], q[garbage, 11] = 11.0, -9.0, 13.0
    return q


def _dev_call(eng, seeds, n_frames, p=P):
    import torch
    d_seeds = torch.from_numpy(seeds).cuda()
    d_out = torch.full((n_frames, len(seeds), ob.POI3D_FLOATS), 7.0, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    rec, left = eng.icgn3d_series_recover_dev(d_seeds.data_ptr(), d_out.data_ptr(), len(seeds), *R, *p.recover_args())
    assert_same(d_seeds.cpu().numpy(), seeds, "device seeds changed")
    return d_out.cpu().numpy(), rec, left


@pytest.mark.parametrize("stack", ["float", "u8", "dev"])
def test_equals_the_loop(engine, volumes, stack):
    ref, _, tars, xyz, _ = volumes
    seeds = _seeds(engine, ref, tars[0], xyz, _ball(xyz, (72, 40, 64), 9))
    for n_frames in (1, FRAMES):
        expect = src.dev_loop(engine, 3, 1, ref, tars[:n_frames], seeds, R, P)
        if stack == "u8":
            engine.set_series_3d(ref.astype(np.uint8), tars[:n_frames].astype(np.uint8))
        else:
            engine.set_series_3d(ref, tars[:n_frames])
        got = _dev_call(engine, seeds, n_frames) if stack == "dev" else engine.icgn3d_series_recover(seeds, *R, *P.recover_args())
        label = "%s F %d" % (stack, n_frames)
        assert_same(got[0], expect[0], label)
        assert np.array_equal(got[1], expect[1]) and np.array_equal(got[2], expect[2]), (label, got[1:], expect[1:])
        assert got[1][0].sum() > 0, "the garbage-seeded ball is recovered in frame 0"


def test_occluded_ball_recovered_in_the_next_frame(engine, volumes):
    ref, clean, tars, xyz, ball = volumes
    seeds = _seeds(engine, ref, tars[0], xyz)
    engine.set_series_3d(ref, tars)
    plain = engine.icgn3d_series(seeds, *R, P.conv, P.stop)
    assert (~(plain[K:, ball, 18] >= 0.9)).all(), "control: the plain series loses the ball from frame K on"
    got, rec, left = engine.icgn3d_series_recover(seeds, *R, *P.recover_args())
    assert left[K] >= ball.sum() and rec[K + 1].sum() >= ball.sum(), (rec, left)
    engine.set_series_3d(ref, clean)
    reference = engine.icgn3d_series(seeds, *R, P.conv, P.stop)
    for f in range(K + 1, FRAMES):
        assert (got[f][ball, 18] >= 0.9).all(), "frame %d" % f
        for col in (3, 7, 11):
            assert np.abs(got[f][ball, col] - reference[f][ball, col]).max() < 0.01


def test_no_rounds_or_nothing_unreliable_is_the_plain_series(engine, volumes):
    ref, _, tars, xyz, _ = volumes
    seeds = _seeds(engine, ref, tars[0], xyz, _ball(xyz, (72, 40, 64), 9))
    engine.set_series_3d(ref, tars)
    plain = engine.icgn3d_series(seeds, *R, P.conv, P.stop)
    got, rec, left = engine.icgn3d_series_recover(seeds, *R, *src.Params(stop=20, max_rounds=0).recover_args())
    assert_same(got, plain, "max_rounds 0")
    assert rec.shape == (FRAMES, 0) and (left > 0).all()
    got, rec, left = engine.icgn3d_series_recover(seeds, *R, *src.Params(stop=20, zncc_low=-10.0, conv=1e30).recover_args())
    assert (rec == 0).all() and (left == 0).all()
    assert_same(got, engine.icgn3d_series(seeds, *R, 1e30, P.stop), "nothing unreliable")


def test_pair_state_untouched_and_group(engine, volumes):
    ref, _, tars, xyz, _ = volumes
    seeds = _seeds(engine, ref, tars[-1], xyz[::9])
    engine.icgn3d_prepare()
    before = seeds.copy()
    engine.icgn3d1(before, *R, P.conv, P.stop)
    engine.set_series_3d(ref, tars)
    expect = engine.icgn3d_series_recover(seeds, *R, *P.recover_args())
    after = seeds.copy()
    engine.icgn3d1(after, *R, P.conv, P.stop)  # the pair (ref, tars[-1]) is still set and prepared
    assert_same(after, before, "pair call after a series recovery call")
    grp = ob.Engine(list(range(_capi.load().ocb_device_count())))
    try:
        grp.set_series_3d(ref, tars)
        got = grp.icgn3d_series_recover(seeds, *R, *P.recover_args())
        assert_same(got[0], expect[0], "group context")
        assert np.array_equal(got[1], expect[1]) and np.array_equal(got[2], expect[2])
    finally:
        grp.close()


def test_refusals_write_nothing():
    eng = ob.Engine(0)
    lib, ctx = eng._lib, eng._ctx
    ref, tars = synth.speckle_series_3d(40, 36, 32, 2)
    seeds = ob.make_poi3d(synth.grid_3d(18, 16, 14, 2, 2, 2, 4, 4, 4))
    n = len(seeds)
    out = np.full((2, n, ob.POI3D_FLOATS), 7.0, np.float32)
    rec = np.full((2, 3), 99, np.uint64)
    left = np.full(2, 99, np.uint64)
    vp = lambda a: None if a is None else ctypes.c_void_p(a.ctypes.data)

    def call(r=(6, 6, 6), s=seeds, o=out, count=n, conv=0.001, high=0.9, low=0.5, rounds=3, fn=lib.ocb_icgn3d_series_recover):
        return fn(ctx, vp(s), vp(o), count, *r, conv, 20.0, 20.0, 12, high, low, rounds, vp(rec), vp(left))

    assert call() == _capi.OCB_ERR_STATE
    assert lib.ocb_set_series_3d(ctx, vp(ref), vp(tars), 2, 40, 36, 32) == _capi.OCB_OK
    for kw in [dict(r=(0, 6, 6)), dict(s=None), dict(o=None), dict(count=1 << 40), dict(rounds=-1), dict(conv=float("nan")),
               dict(high=float("nan")), dict(low=float("nan"))]:
        assert call(**kw) == _capi.OCB_ERR_ARG, kw
    assert call(r=(44, 44, 44)) == _capi.OCB_ERR_UNSUPPORTED and "exceeds the shared-memory design limit" in _capi.last_error(ctx)
    assert call(s=None, o=None, fn=lib.ocb_icgn3d_series_recover_dev) == _capi.OCB_ERR_ARG
    assert (out == 7.0).all() and (rec == 99).all() and (left == 99).all()
    assert call() == _capi.OCB_OK and not (out == 7.0).all() and (rec < 99).all() and (left < 99).all()
    eng.close()
