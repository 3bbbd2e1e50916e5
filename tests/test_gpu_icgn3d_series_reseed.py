"""ICGN3D1 over a volume series that re-seeds lost POIs (ocb_icgn3d_series_reseed).  The records must be, bit for bit, what this
loop of pair calls gives:
    for f: set_images_3d(ref, tars[f]); icgn3d_prepare(); icgn3d1(q)
           lost = !(q.zncc >= zncc_min); sub = lost POIs rebuilt from their seeds at their latest good translation
           fftcc3d(sub); icgn3d1(sub); q[lost] = sub
and, when nothing is lost, what icgn3d_series gives."""
import ctypes

import numpy as np
import pytest

import opencorr_b200 as ob
from opencorr_b200 import _capi, synth

pytestmark = pytest.mark.gpu

CONV, STOP = 0.001, 20
DX, DY, DZ = 103, 100, 98  # dim_x % 4 != 0
FRAMES = 4
DISP = (3, 7, 11)  # u, v, w in a POI3D record


@pytest.fixture(scope="module")
def series():
    return synth.speckle_series_3d(DX, DY, DZ, FRAMES)


def occlude(tars, k, box):
    """Cover box = (x0, y0, z0, x1, y1, z1) of frame k with speckles from elsewhere in the same frame."""
    x0, y0, z0, x1, y1, z1 = box
    out = tars.copy()
    out[k, z0:z1, y0:y1, x0:x1] = np.roll(tars[k], (DZ // 2, DY // 2, DX // 2), (0, 1, 2))[z0:z1, y0:y1, x0:x1]
    return out


def block_box(xyz, r, k, margin=3):
    s = (k + 1) / FRAMES
    u, v, w = synth.displacement_3d(xyz[:, 0], xyz[:, 1], xyz[:, 2], DX, DY, DZ)
    lo = np.floor(xyz + s * np.stack([u, v, w], 1) - r - margin).min(0).astype(int)
    hi = np.ceil(xyz + s * np.stack([u, v, w], 1) + r + margin + 1).max(0).astype(int)
    return tuple(np.maximum(lo, 0)) + tuple(np.minimum(hi, [DX, DY, DZ]))


def fftcc_seeds(eng, ref, tar, xyz, r):
    q = ob.make_poi3d(xyz)
    eng.set_images_3d(ref, tar)
    eng.fftcc3d(q, *r)
    return q


def pair_loop(eng, ref, tars, seeds, r, fr, zncc_min):
    q = seeds.copy()
    anchor = seeds[:, DISP].copy()
    out, counts = [], []
    for f in range(len(tars)):
        eng.set_images_3d(ref, tars[f])
        eng.icgn3d_prepare()
        eng.icgn3d1(q, *r, CONV, STOP)
        if f > 0:
            good = out[-1][:, 18] >= zncc_min
            anchor[good] = out[-1][good][:, DISP]
        lost = np.nonzero(~(q[:, 18] >= zncc_min))[0]
        if len(lost):
            sub = np.zeros((len(lost), ob.POI3D_FLOATS), np.float32)
            for c in (0, 1, 2, 28, 29, 30):
                sub[:, c] = seeds[lost, c]
            sub[:, DISP] = anchor[lost]
            eng.fftcc3d(sub, *fr)
            eng.icgn3d1(sub, *r, CONV, STOP)
            q[lost] = sub
        out.append(q.copy())
        counts.append(len(lost))
    return np.stack(out), np.array(counts, np.int64)


def assert_same(a, b, label):
    assert a.shape == b.shape, label
    bad = a.view(np.uint32) != b.view(np.uint32)
    assert not bad.any(), "%s: %d floats differ, first at %s" % (label, bad.sum(), np.argwhere(bad)[:5].tolist())


def grid(r):
    """POIs whose subvolumes stay inside the volume in every frame: r = 8, 3 x 3 x 3 POIs 25 voxels apart (8 voxels between the
    subvolumes); r = 24, 2 x 2 x 2 POIs."""
    if r == 8:
        return synth.grid_3d(14, 14, 14, 3, 3, 3, 25, 25, 25)
    return synth.grid_3d(27, 27, 27, 2, 2, 2, 42, 42, 42)


@pytest.fixture(scope="module")
def lossy(series):
    """Frame 1 occludes the column of POIs at the smallest x and y (r = 8 grid, 3 POIs along z); frame 3 (the last) the POI at
    the far corner."""
    ref, tars = series
    xyz = grid(8)
    col = (xyz[:, 0] == xyz[:, 0].min()) & (xyz[:, 1] == xyz[:, 1].min())
    corner = (xyz[:, 0] == xyz[:, 0].max()) & (xyz[:, 1] == xyz[:, 1].max()) & (xyz[:, 2] == xyz[:, 2].max())
    tars = occlude(tars, 1, block_box(xyz[col], 8, 1))
    tars = occlude(tars, 3, block_box(xyz[corner], 8, 3))
    return ref, tars, xyz, col, corner


CASES = [((8, 8, 8), (7, 7, 7)), ((8, 8, 8), (10, 10, 10)), ((8, 8, 8), (16, 16, 16)), ((24, 24, 24), (10, 10, 10))]


@pytest.mark.parametrize("u8", [False, True], ids=["float", "u8"])
@pytest.mark.parametrize("r,fr", CASES, ids=["r8 fft7", "r8 fft10", "r8 fft16", "r24 fft10 (512 threads)"])
def test_reseed_equals_pair_loop(engine, series, lossy, r, fr, u8):
    ref, tars, xyz, col, corner = lossy
    if r[0] > 12:
        xyz = grid(r[0])
        tars = occlude(series[1], 1, block_box(xyz[:1], r[0], 1))
    seeds = fftcc_seeds(engine, ref, tars[0], xyz, fr)
    seeds[-2, 18] = -1.0  # refused by the guard in frame 0, good once re-seeded: needs the neutral seeds' setup state
    for n_frames in (1, FRAMES):
        expect, expect_counts = pair_loop(engine, ref, tars[:n_frames], seeds, r, fr, 0.9)
        if u8:
            engine.set_series_3d(ref.astype(np.uint8), tars[:n_frames].astype(np.uint8))
        else:
            engine.set_series_3d(ref, tars[:n_frames])
        before = seeds.copy()
        got, counts = engine.icgn3d_series_reseed(seeds, *r, CONV, STOP, *fr, 0.9)
        assert_same(seeds, before, "seeds changed")
        assert_same(got, expect, "r=%s fft=%s F=%d" % (r, fr, n_frames))
        assert np.array_equal(counts, expect_counts), (counts, expect_counts)
        assert counts[0] >= 1
        assert (got[-1][-2:-1, 18] >= 0.9).all()
        if n_frames == FRAMES and r[0] <= 12:
            assert counts[1] >= col.sum() and counts[3] >= corner.sum(), counts


@pytest.mark.parametrize("r,n", [((8, 8, 8), 40), ((16, 16, 16), 16), ((24, 24, 24), 6)])
def test_nothing_lost_equals_plain_series(engine, series, r, n):
    ref, tars = series
    rng = np.random.default_rng(sum(r) + n)
    lo, hi = np.array(r) + 3, np.array([DX, DY, DZ]) - 1 - np.array(r) - 4
    seeds = fftcc_seeds(engine, ref, tars[0], rng.integers(lo, hi + 1, size=(n, 3)).astype(np.float32), r)
    seeds[0, 18] = -1.0
    engine.set_series_3d(ref, tars)
    expect = engine.icgn3d_series(seeds, *r, CONV, STOP)
    got, counts = engine.icgn3d_series_reseed(seeds, *r, CONV, STOP, 16, 16, 16, -10.0)
    assert_same(got, expect, "r=%s" % (r,))
    assert (counts == 0).all()


def test_occlusion_recovers(engine, series, lossy):
    ref, tars, xyz, col, corner = lossy
    seeds = fftcc_seeds(engine, ref, tars[0], xyz, (16, 16, 16))
    engine.set_series_3d(ref, tars[:3])
    plain = engine.icgn3d_series(seeds, 8, 8, 8, CONV, STOP)
    assert (~(plain[1, col, 18] >= 0.9)).all(), "control: IC-GN alone loses the column in the occluded frame"
    got, counts = engine.icgn3d_series_reseed(seeds, 8, 8, 8, CONV, STOP, 16, 16, 16, 0.9)
    assert counts[1] == col.sum(), counts
    engine.set_series_3d(ref, series[1][:3])
    clean = engine.icgn3d_series(seeds, 8, 8, 8, CONV, STOP)
    assert (got[2][:, 18] >= 0.9).all()
    u, v, w = synth.displacement_3d(xyz[:, 0], xyz[:, 1], xyz[:, 2], DX, DY, DZ)
    s = 3 / FRAMES
    for c, truth in zip(DISP, (u, v, w)):
        assert np.abs(got[2][col, c] - clean[2][col, c]).max() < 0.01
        assert np.abs(got[2][:, c] - s * truth).max() < 0.05


def test_errors_and_dev(engine, series, lossy):
    ref, tars, xyz, _, _ = lossy
    eng = ob.Engine(0)
    lib, ctx = eng._lib, eng._ctx
    seeds = fftcc_seeds(eng, ref, tars[0], xyz, (16, 16, 16))
    n = len(seeds)
    out = np.full((FRAMES, n, ob.POI3D_FLOATS), 7.0, np.float32)
    counts = np.full(FRAMES, 99, np.uint64)
    vp = lambda a: ctypes.c_void_p(a.ctypes.data)

    def call(r=(8, 8, 8), fr=(16, 16, 16), zmin=0.9, s=seeds, o=out, count=n):
        return lib.ocb_icgn3d_series_reseed(ctx, vp(s) if s is not None else None, vp(o) if o is not None else None, count, *r, CONV, STOP, *fr,
                                            zmin, vp(counts))

    assert call() == _capi.OCB_ERR_STATE
    eng.set_series_3d(ref, tars)
    assert call(s=None) == _capi.OCB_ERR_ARG
    assert call(r=(0, 8, 8)) == _capi.OCB_ERR_ARG
    assert call(count=1 << 40) == _capi.OCB_ERR_ARG
    assert call(zmin=float("nan")) == _capi.OCB_ERR_ARG
    assert call(fr=(16, 0, 16)) == _capi.OCB_ERR_ARG
    assert call(fr=(37, 37, 37)) == _capi.OCB_ERR_UNSUPPORTED
    assert "prime factor > 31" in _capi.last_error(ctx)
    assert call(r=(44, 44, 44)) == _capi.OCB_ERR_UNSUPPORTED
    assert "exceeds the shared-memory design limit" in _capi.last_error(ctx)
    assert lib.ocb_icgn3d_series_reseed_dev(ctx, None, None, 5, 8, 8, 8, CONV, STOP, 16, 16, 16, 0.9, vp(counts)) == _capi.OCB_ERR_ARG
    assert (out == 7.0).all() and (counts == 99).all()
    assert call() == _capi.OCB_OK
    host = out.copy()
    assert counts[1] > 0 and counts[1] < 99

    # a pair call after a re-seeding call returns what it returned before
    eng.set_images_3d(ref, tars[2])
    eng.icgn3d_prepare()
    before = seeds.copy()
    eng.icgn3d1(before, 8, 8, 8, CONV, STOP)
    eng.set_series_3d(ref, tars)
    eng.icgn3d_series_reseed(seeds, 8, 8, 8, CONV, STOP, 16, 16, 16, 0.9)
    after = seeds.copy()
    eng.icgn3d1(after, 8, 8, 8, CONV, STOP)
    assert_same(after, before, "pair call after a re-seeding series call")

    torch = pytest.importorskip("torch")
    d_ref, d_tars, d_seeds = (torch.from_numpy(a).cuda() for a in (ref, tars, seeds))
    d_out = torch.empty((FRAMES, n, ob.POI3D_FLOATS), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    eng.set_series_3d_dev(d_ref.data_ptr(), d_tars.data_ptr(), FRAMES, DX, DY, DZ)
    dev_counts = eng.icgn3d_series_reseed_dev(d_seeds.data_ptr(), d_out.data_ptr(), n, 8, 8, 8, CONV, STOP, 16, 16, 16, 0.9)
    assert_same(d_out.cpu().numpy(), host, "device-pointer variant")
    assert np.array_equal(dev_counts, counts.astype(np.int64))
    eng.close()


def test_group(lossy):
    if _capi.load().ocb_device_count() < 2:
        pytest.skip("needs two GPUs")
    ref, tars, xyz, _, _ = lossy
    single = ob.Engine(0)
    seeds = fftcc_seeds(single, ref, tars[0], xyz, (16, 16, 16))
    single.set_series_3d(ref, tars)
    expect, expect_counts = single.icgn3d_series_reseed(seeds, 8, 8, 8, CONV, STOP, 16, 16, 16, 0.9)
    group = ob.Engine([0, 1])
    group.set_series_3d(ref, tars)
    got, counts = group.icgn3d_series_reseed(seeds, 8, 8, 8, CONV, STOP, 16, 16, 16, 0.9)
    assert_same(got, expect, "group context")
    assert np.array_equal(counts, expect_counts)
    group.close()
    single.close()
