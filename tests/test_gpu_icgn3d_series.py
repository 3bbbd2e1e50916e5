"""ICGN3D1 over a volume series (ocb_icgn3d_series, ocb_icgn3d_series_reseed): every frame's records must be, bit for bit, what
the loop of pair calls
    set_images_3d(ref, tars[f]); icgn3d_prepare(); icgn3d1(q, ...)
gives when one queue q is carried from frame to frame.  The series builds the reference's gradients and each POI's setup pass
once per call (ICGN3D_SETUP_STORE) and restores the setup state in every frame (ICGN3D_SETUP_LOAD).  The re-seeding call must
give what this loop of pair calls gives:
    for f: set_images_3d(ref, tars[f]); icgn3d_prepare(); icgn3d1(q)
           lost = !(q.zncc >= zncc_min); sub = lost POIs rebuilt from their seeds at their latest good translation
           fftcc3d(sub); icgn3d1(sub); q[lost] = sub
and, when nothing is lost, what icgn3d_series gives."""
import ctypes

import numpy as np
import pytest

import opencorr_b200 as ob
from opencorr_b200 import _capi, synth
from oracle.oracle import Oracle3D
import util
from util import assert_same

pytestmark = pytest.mark.gpu

CONV, STOP = 0.001, 20
DX, DY, DZ = 103, 100, 98  # dim_x % 4 != 0; room for a 61^3 subvolume plus the synthetic displacement
FRAMES = 4
DISP = (3, 7, 11)  # u, v, w in a POI3D record


@pytest.fixture(scope="module")
def series():
    return synth.speckle_series_3d(DX, DY, DZ, FRAMES)


def _pois(r, n, seed):
    """n integer POIs whose subvolume stays inside the volume in every frame (v < 0 near y = 0, w < 2.5)."""
    rng = np.random.default_rng(seed)
    r = np.array(r)
    lo, hi = r + 3, np.array([DX, DY, DZ]) - 1 - r - 4
    return rng.integers(lo, hi + 1, size=(n, 3)).astype(np.float32)


def fftcc_seeds(eng, ref, tar, xyz, r):
    q = ob.make_poi3d(xyz)
    eng.set_images_3d(ref, tar)
    eng.fftcc3d(q, *r)
    return q


def pair_loop(eng, ref, tars, seeds, r, stop=STOP):
    q = seeds.copy()
    out = []
    for f in range(len(tars)):
        eng.set_images_3d(ref, tars[f])
        eng.icgn3d_prepare()
        eng.icgn3d1(q, *r, CONV, stop)
        out.append(q.copy())
    return np.stack(out)


# radii, POIs; the launch plan each selects (ocb::icgn3d1_plan) in the comment
CASES = [
    ((8, 8, 8), 24),    # <0,256>, one slab
    ((8, 8, 8), 300),   # <0,256>: more POIs than the 2 x 132 resident CTAs
    ((16, 16, 16), 16), # <16,256>, 3 slabs, one tail column
    ((10, 6, 9), 20),   # <0,256>, non-cubic
    ((24, 24, 24), 6),  # <0,512>, 17 tail columns
    ((30, 30, 30), 3),  # <30,512>
]


@pytest.mark.parametrize("tma", [True, False], ids=["tma", "no_tma"])
@pytest.mark.parametrize("r,n", CASES, ids=["r=(%d,%d,%d) n=%d" % (r + (n,)) for r, n in CASES])
def test_series_equals_pair_loop(engine, series, monkeypatch, r, n, tma):
    if not tma:
        monkeypatch.setenv("OCB_NO_TMA", "1")
    ref, tars = series
    seeds = fftcc_seeds(engine, ref, tars[0], _pois(r, n, seed=sum(r) + n), r)
    for n_frames in (1, FRAMES):
        expect = pair_loop(engine, ref, tars[:n_frames], seeds, r)
        engine.set_series_3d(ref, tars[:n_frames])
        before = seeds.copy()
        got = engine.icgn3d_series(seeds, *r, CONV, STOP)
        assert_same(seeds, before, "seeds changed")
        assert_same(got, expect, "r=%s n=%d F=%d" % (r, n, n_frames))
        assert (got[-1][:, 18] >= 0).mean() > 0.8


def test_series_matches_oracle_and_ground_truth(engine, series):
    ref, tars = series
    r = (16, 16, 16)
    xyz = _pois(r, 12, seed=7)
    seeds = fftcc_seeds(engine, ref, tars[0], xyz, r)
    engine.set_series_3d(ref, tars)
    got = engine.icgn3d_series(seeds, *r, CONV, STOP)
    n = len(xyz)
    for f in range(FRAMES):
        q = (seeds if f == 0 else got[f - 1]).copy()  # each frame from the same seeds as the GPU's
        Oracle3D(ref, tars[f]).icgn3d1(q, *r, CONV, STOP, exact=True)
        stats = util.compare_3d(got[f], q, "frame %d" % f, max_iter_mismatch_frac=max(1.0, 0.02 * n) / n)
        print("frame %d: %s" % (f, stats))
    last = got[-1]
    ok = last[:, 18] >= 0
    assert ok.mean() > 0.9
    u, v, w = synth.displacement_3d(xyz[:, 0], xyz[:, 1], xyz[:, 2], DX, DY, DZ)
    for col, truth in ((3, u), (7, v), (11, w)):
        assert np.abs(last[ok, col] - truth[ok]).max() < 0.05


def test_series_sentinels(engine, series):
    """POIs that leave the volume mid-series, stop at the iteration limit (-4), are refused by the guard or arrive with a
    negative or NaN ZNCC keep their code and that frame's record in every later frame, exactly as the pair loop does."""
    ref, tars = series
    r = (12, 12, 12)
    # rows 9 ... 15: subvolumes 0 ... 6 layers below the top of the volume, whose top layers leave it as w grows by about 0.6
    # voxel per frame
    top = [[40 + 3 * k, 50, DZ - 1 - 12 - k] for k in range(7)]
    xyz = np.array([[40, 40, 40], [60, 50, 45], [50, 50, 50], [45, 55, 52], [55, 45, 50], [40, 60, 55], [50, 40, 60], [45, 45, 42],
                    [58, 58, 48]] + top, np.float32)
    seeds = fftcc_seeds(engine, ref, tars[0], xyz, r)
    seeds[4, 3] = DX + 5.0  # |u| >= dim_x: the guard rejects it
    seeds[5, 18] = -1.0     # arrives negative
    seeds[6, 3] = np.nan    # NaN guess
    seeds[7, 18] = np.nan   # NaN ZNCC with coordinates outside the volume: the guard keeps the NaN
    seeds[7, 0] = -5.0
    seeds[8, 3] += 3.5      # far from the optimum: runs into the iteration limit at stop = 2
    for stop in (STOP, 2):
        expect = pair_loop(engine, ref, tars, seeds, r, stop)
        engine.set_series_3d(ref, tars)
        got = engine.icgn3d_series(seeds, *r, CONV, stop)
        assert_same(got, expect, "stop %g" % stop)
        codes = got[:, :, 18]
        assert (codes[:, 4] == -3).all() and (codes[:, 5] == -1).all() and (codes[:, 6] == -3).all()
        assert np.isnan(codes[:, 7]).all() and (got[:, 7, 0] == -5.0).all()
        if stop == 2:
            assert (codes == -4).any()
        else:
            first_fail = [np.nonzero(codes[:, i] < 0)[0] for i in range(9, 16)]
            assert any(len(ff) and 0 < ff[0] < FRAMES for ff in first_fail), "no POI left the volume mid-series: %s" % codes[:, 9:16].T
        for i in range(len(xyz)):
            neg = np.nonzero(~(codes[:, i] >= 0))[0]
            if len(neg):
                f0 = neg[0]
                for f in range(f0 + 1, FRAMES):
                    assert_same(got[f, i], got[f0, i], "POI %d frame %d" % (i, f))


def test_series_chunks_u8_and_device_pointers(engine, series):
    ref, tars = series
    r = (16, 16, 16)
    seeds = fftcc_seeds(engine, ref, tars[0], _pois(r, 16, seed=3), r)
    engine.set_series_3d(ref, tars)
    whole = engine.icgn3d_series(seeds, *r, CONV, STOP)
    engine.set_series_3d(ref, tars[:2])
    a = engine.icgn3d_series(seeds, *r, CONV, STOP)
    engine.set_series_3d(ref, tars[2:])
    b = engine.icgn3d_series(a[-1].copy(), *r, CONV, STOP)
    assert_same(np.concatenate([a, b]), whole, "two chunks")

    assert np.array_equal(ref, np.round(ref)) and ref.max() <= 255  # synth volumes are 8-bit valued
    engine.set_series_3d(ref.astype(np.uint8), tars.astype(np.uint8))
    assert_same(engine.icgn3d_series(seeds, *r, CONV, STOP), whole, "8-bit stack")

    torch = pytest.importorskip("torch")
    d_ref, d_tars, d_seeds = (torch.from_numpy(x).cuda() for x in (ref, tars, seeds))
    d_out = torch.empty((FRAMES, len(seeds), ob.POI3D_FLOATS), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    engine.set_series_3d_dev(d_ref.data_ptr(), d_tars.data_ptr(), FRAMES, DX, DY, DZ)
    engine.icgn3d_series_dev(d_seeds.data_ptr(), d_out.data_ptr(), len(seeds), *r, CONV, STOP)
    engine.sync()
    assert_same(d_out.cpu().numpy(), whole, "device-pointer variant")
    assert_same(d_seeds.cpu().numpy(), seeds, "device seeds changed")


def test_series_errors_leave_out_untouched():
    eng = ob.Engine(0)
    lib, ctx = eng._lib, eng._ctx
    ref, tars = synth.speckle_series_3d(40, 36, 32, 2)
    seeds = ob.make_poi3d(synth.grid_3d(18, 16, 14, 2, 2, 2, 4, 4, 4))
    n = len(seeds)
    out = np.full((2, n, ob.POI3D_FLOATS), 7.0, np.float32)
    vp = lambda a: ctypes.c_void_p(a.ctypes.data)

    def call(r=(6, 6, 6), s=seeds, o=out, count=n):
        return lib.ocb_icgn3d_series(ctx, vp(s) if s is not None else None, vp(o) if o is not None else None, count, *r, CONV, STOP)

    assert call() == _capi.OCB_ERR_STATE
    assert lib.ocb_set_series_3d(ctx, vp(ref), vp(tars), 0, 40, 36, 32) == _capi.OCB_ERR_ARG
    assert lib.ocb_set_series_3d(ctx, vp(ref), None, 2, 40, 36, 32) == _capi.OCB_ERR_ARG
    assert lib.ocb_set_series_3d(ctx, vp(ref), vp(tars), 2, 40, 36, 14) == _capi.OCB_ERR_ARG
    assert lib.ocb_set_series_3d(ctx, vp(ref), vp(tars), 2, 1 << 30, 1 << 30, 1 << 30) == _capi.OCB_ERR_ARG  # size overflow
    assert lib.ocb_set_series_3d_u8(ctx, vp(ref), vp(tars), 1 << 30, 1 << 30, 1 << 30, 1 << 30) == _capi.OCB_ERR_ARG
    assert lib.ocb_set_series_3d_dev(ctx, None, None, 2, 40, 36, 32) == _capi.OCB_ERR_ARG
    assert call() == _capi.OCB_ERR_STATE  # the refused calls set nothing
    assert lib.ocb_set_series_3d(ctx, vp(ref), vp(tars), 2, 40, 36, 32) == _capi.OCB_OK
    assert call(s=None) == _capi.OCB_ERR_ARG
    assert call(o=None) == _capi.OCB_ERR_ARG
    assert call(r=(0, 6, 6)) == _capi.OCB_ERR_ARG
    assert call(count=1 << 40) == _capi.OCB_ERR_ARG
    assert call(r=(44, 44, 44)) == _capi.OCB_ERR_UNSUPPORTED
    assert "exceeds the shared-memory design limit" in _capi.last_error(ctx)
    assert lib.ocb_icgn3d_series_dev(ctx, None, None, 5, 6, 6, 6, CONV, STOP) == _capi.OCB_ERR_ARG
    assert (out == 7.0).all()
    assert call() == _capi.OCB_OK
    assert not (out == 7.0).all()
    eng.close()


def test_pair_calls_unaffected_by_series(engine, series):
    ref, tars = series
    r = (16, 16, 16)
    seeds = fftcc_seeds(engine, ref, tars[-1], _pois(r, 16, seed=5), r)
    engine.icgn3d_prepare()
    before = seeds.copy()
    engine.icgn3d1(before, *r, CONV, STOP)
    engine.set_series_3d(ref[:, ::-1].copy(), tars[:, :, ::-1].copy())
    engine.icgn3d_series(seeds, *r, CONV, STOP)
    after = seeds.copy()
    engine.icgn3d1(after, *r, CONV, STOP)  # the pair (ref, tars[-1]) is still set and prepared
    assert_same(after, before, "pair call after a series call")


def test_series_group(series):
    if _capi.load().ocb_device_count() < 2:
        pytest.skip("needs two GPUs")
    ref, tars = series
    r = (16, 16, 16)
    single = ob.Engine(0)
    seeds = fftcc_seeds(single, ref, tars[0], _pois(r, 16, seed=3), r)
    single.set_series_3d(ref, tars)
    expect = single.icgn3d_series(seeds, *r, CONV, STOP)
    group = ob.Engine([0, 1])
    group.set_series_3d(ref, tars)
    assert_same(group.icgn3d_series(seeds, *r, CONV, STOP), expect, "group context")
    group.close()
    single.close()


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


def reseed_pair_loop(eng, ref, tars, seeds, r, fr, zncc_min):
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


RESEED_CASES = [((8, 8, 8), (7, 7, 7)), ((8, 8, 8), (10, 10, 10)), ((8, 8, 8), (16, 16, 16)), ((24, 24, 24), (10, 10, 10))]


@pytest.mark.parametrize("u8", [False, True], ids=["float", "u8"])
@pytest.mark.parametrize("r,fr", RESEED_CASES, ids=["r8 fft7", "r8 fft10", "r8 fft16", "r24 fft10 (512 threads)"])
def test_reseed_equals_pair_loop(engine, series, lossy, r, fr, u8):
    ref, tars, xyz, col, corner = lossy
    if r[0] > 12:
        xyz = grid(r[0])
        tars = occlude(series[1], 1, block_box(xyz[:1], r[0], 1))
    seeds = fftcc_seeds(engine, ref, tars[0], xyz, fr)
    seeds[-2, 18] = -1.0  # refused by the guard in frame 0, good once re-seeded: needs the neutral seeds' setup state
    for n_frames in (1, FRAMES):
        expect, expect_counts = reseed_pair_loop(engine, ref, tars[:n_frames], seeds, r, fr, 0.9)
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
def test_reseed_nothing_lost_equals_plain_series(engine, series, r, n):
    ref, tars = series
    seeds = fftcc_seeds(engine, ref, tars[0], _pois(r, n, seed=sum(r) + n), r)
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


def test_reseed_errors_and_dev(engine, series, lossy):
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


def test_reseed_group(lossy):
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
