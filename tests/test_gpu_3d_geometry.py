"""GPU: FFTCC3D -> ICGN3D1 at every launch geometry the library selects, against the float64 oracle (Oracle3D, exact=1).

ocb::icgn3d1_plan (opencorr_b200/csrc/ocb_kernels.h) picks the ICGN3D1 kernel variant (<RC, THREADS>), the z-slab thickness and
the slab count from the subvolume radii; test_icgn3d_plan_host.py checks on the CPU that every radius set below lands in the
branch its case is meant to cover (single slab, several slabs, a thinner last slab, tail columns beyond 32, one 512-thread CTA
per SM, rejection).  The FFTCC3D leg of each case runs the generic Stockham kernel wherever the window leaves the register
kernels (radices 7, 11 and 13, windows over 64 points, non-cubic windows).

Tolerances: 1e-4 voxel and 1e-5 ZNCC (all 12 parameters within 1e-4) on POIs whose iteration counts agree; at most
max(1, 2 %) POIs per case may take one iteration more or less (||dp|| within float noise of the convergence criterion).
Each case prints one line with its largest deviations."""
import numpy as np
import pytest

import opencorr_b200 as ob
from opencorr_b200 import synth
from oracle.oracle import Oracle3D
import util

pytestmark = pytest.mark.gpu

DIM = 104  # sweep volume DIM^3: room for a 87^3 subvolume (r = 43) plus the synthetic displacement

# ICGN3D1 radius sets and POI counts (fewer POIs where a subvolume is large); the plan each one selects is in the comment
SWEEP = [
    ((8, 8, 8), 24),     # <0,256>, one slab
    ((12, 12, 12), 24),  # <0,256>, 2 slabs x 13 (last 12)
    ((16, 16, 16), 16),  # <16,256>, 3 x 11, 1 tail column
    ((16, 16, 15), 16),  # <0,256>, 3 x 11 (last 9), 1 tail column
    ((20, 20, 20), 12),  # <0,256>, 7 x 6 (last 5), 9 tail columns
    ((22, 22, 22), 8),   # <0,512>, 3 x 15, 13 tail columns
    ((24, 24, 24), 6),   # <0,512>, 5 x 10 (last 9), 17 tail columns
    ((30, 30, 30), 3),   # <30,512>, 11 x 6 (last 1), 29 tail columns
    ((40, 40, 40), 2),   # <0,512>, 41 x 2 (last 1), 49 tail columns
    ((24, 8, 30), 8),    # <0,256>, 5 x 13 (last 9), 17 tail columns
    ((30, 30, 12), 5),   # <0,512>, 5 x 5, 29 tail columns
]
SHEAR_RADII = [(16, 16, 16), (14, 14, 14), (24, 24, 24)]
SENTINEL_RADII = [(24, 24, 24), (12, 12, 12)]
LARGE_Z_RADII = [(8, 8, 8), (16, 16, 16)]
LONG_QUEUE_RADII = (22, 22, 22)  # 294 POIs: more than one 512-thread CTA per SM can take at once
LARGEST_RADII = (43, 43, 43)     # the largest cubic subvolume the plan accepts on an H100; r = 44 is rejected
ICGN3D_RADII = ([r for r, _ in SWEEP] + SHEAR_RADII + SENTINEL_RADII + LARGE_Z_RADII + [LONG_QUEUE_RADII, LARGEST_RADII,
                (44, 44, 44)])

INT_COLS = [3, 7, 11, 15, 16, 17]  # FFT-CC integer displacement and u0, v0, w0


@pytest.fixture(scope="module")
def vol():
    return synth.speckle_pair_3d(DIM, DIM, DIM)


def _pois(r, n, seed, dim=DIM):
    """n integer POIs whose subvolume and FFT-CC window (and their image under the synthetic displacement) are inside."""
    rng = np.random.default_rng(seed)
    lo = np.array(r) + 1
    hi = dim - 1 - np.array(r) - 4
    return rng.integers(lo, hi + 1, size=(n, 3)).astype(np.float32)


def _fftcc(engine, ref, tar, xyz, r, label):
    """FFTCC3D on the GPU vs the exact oracle: integer outputs bit-exact, ZNCC within 1e-5.  Returns the GPU records."""
    q = ob.make_poi3d(xyz)
    q_exact = q.copy()
    f = ob.FFTCC3D(*r, engine=engine)
    f.set_images(ref, tar)
    f.compute(q)
    Oracle3D(ref, tar).fftcc3d(q_exact, *r, exact=True)
    assert np.array_equal(q[:, INT_COLS], q_exact[:, INT_COLS]), label + ": FFT-CC integer outputs differ"
    dz = np.abs(q[:, 18] - q_exact[:, 18]).max()
    assert dz < 1e-5, "%s: FFT-CC max |dZNCC| = %.3g" % (label, dz)
    print("%s fftcc3d: n=%d max|dZNCC|=%.2e" % (label, len(q), dz))
    return q


def _icgn_gpu(engine, ref, tar, q, r, stop=20):
    icgn = ob.ICGN3D1(*r, 0.001, stop, engine=engine)
    icgn.set_images(ref, tar)
    icgn.prepare()
    icgn.compute(q)
    return q


def _check(a, b, label, min_valid=0.75, tol=1e-4):
    """a: GPU records, b: exact oracle records (both POI3D [n, 31]); tol bounds the displacement and all 12 parameters."""
    n = len(a)
    flips = int((a[:, 19] != b[:, 19]).sum())
    stats = util.compare_3d(a, b, label, tol_disp=tol, max_iter_mismatch_frac=max(1.0, 0.02 * n) / n)
    ok = (a[:, 18] >= 0) & (b[:, 18] >= 0) & (a[:, 19] == b[:, 19])
    dp = np.abs(a[ok][:, 3:15] - b[ok][:, 3:15]).max() if ok.any() else 0.0
    assert dp < tol, "%s: max |d parameter| = %.3g" % (label, dp)
    assert ok.sum() >= min_valid * n, "%s: only %d of %d POIs compared" % (label, ok.sum(), n)
    print("%s icgn3d1: n=%d compared=%d max|ddisp|=%.2e max|dparam|=%.2e max|dZNCC|=%.2e flips=%d"
          % (label, n, ok.sum(), stats["max_disp"], dp, stats["max_zncc"], flips))


def _label(r):
    return "r=(%d,%d,%d)" % tuple(r)


# ------------------------------------------------------------------------------------------------ radius sweep
@pytest.mark.parametrize("r,n", SWEEP, ids=[_label(r) for r, _ in SWEEP])
def test_radius_sweep(engine, vol, r, n):
    ref, tar = vol
    q = _fftcc(engine, ref, tar, _pois(r, n, seed=sum(r)), r, _label(r))
    a, b = q.copy(), q.copy()
    _icgn_gpu(engine, ref, tar, a, r)
    Oracle3D(ref, tar).icgn3d1(b, *r, 0.001, 20, exact=True)
    _check(a, b, _label(r))


def test_long_queue_is_order_invariant(engine, vol):
    """More POIs than resident CTAs: persistent CTAs pull POIs from a work counter, so a shuffled queue gives the same records."""
    ref, tar = vol
    r = LONG_QUEUE_RADII
    xyz = synth.grid_3d(26, 26, 26, 7, 7, 6, 8, 8, 10)
    assert len(xyz) > 132  # an H100 has 132 SMs, one such CTA each
    q = _fftcc(engine, ref, tar, xyz, r, "long queue")
    a, b = q.copy(), q.copy()
    _icgn_gpu(engine, ref, tar, a, r)
    perm = np.random.default_rng(3).permutation(len(q))
    s = _icgn_gpu(engine, ref, tar, q[perm].copy(), r)
    assert np.array_equal(s, a[perm])
    Oracle3D(ref, tar).icgn3d1(b, *r, 0.001, 20, exact=True)
    _check(a, b, "long queue " + _label(r))


def test_largest_accepted_subvolume(engine, vol):
    """r = 43 (87^3 samples, one-layer slabs) runs; FFTCC3D cannot serve it (86 = 2 x 43), so the guess is the rounded truth."""
    ref, tar = vol
    r = LARGEST_RADII
    xyz = np.array([[50, 52, 49], [52, 50, 51], [51, 51, 50]], np.float32)
    q = ob.make_poi3d(xyz)
    u, v, w = synth.displacement_3d(xyz[:, 0], xyz[:, 1], xyz[:, 2], DIM, DIM, DIM)
    q[:, 3], q[:, 7], q[:, 11] = np.round(u), np.round(v), np.round(w)
    a, b = q.copy(), q.copy()
    _icgn_gpu(engine, ref, tar, a, r)
    Oracle3D(ref, tar).icgn3d1(b, *r, 0.001, 20, exact=True)
    _check(a, b, "largest " + _label(r), min_valid=1.0)


def test_limits_raise_and_leave_the_queue_unchanged(engine, vol):
    ref, tar = vol
    xyz = np.array([[50, 52, 49], [52, 50, 51]], np.float32)
    q = ob.make_poi3d(xyz)
    q[:, 3] = 1.0
    q0 = q.copy()
    icgn = ob.ICGN3D1(44, 44, 44, 0.001, 20, engine=engine)  # no slab of even one layer fits in shared memory
    icgn.set_images(ref, tar)
    icgn.prepare()
    with pytest.raises(ob.OpenCorrB200Error, match="exceeds the shared-memory design limit"):
        icgn.compute(q)
    assert np.array_equal(q, q0)
    # a 90^3 window over the shared-memory opt-in; 74 = 2 x 37
    for r, msg in (((45, 45, 45), "B of shared memory"), ((37, 37, 37), "prime factor > 31"), ((20, 37, 20), "prime factor > 31")):
        f = ob.FFTCC3D(*r, engine=engine)
        f.set_images(ref, tar)
        with pytest.raises(ob.OpenCorrB200Error, match=msg):
            f.compute(q)
        assert np.array_equal(q, q0)
    ref2, tar2 = synth.speckle_pair_2d(256, 256)
    q2 = ob.make_poi2d(np.array([[128, 128], [120, 130]], np.float32))
    q20 = q2.copy()
    for r in ((37, 37), (16, 37)):
        f = ob.FFTCC2D(*r, engine=engine)
        f.set_images(ref2, tar2)
        with pytest.raises(ob.OpenCorrB200Error, match="prime factor > 31"):
            f.compute(q2)
        assert np.array_equal(q2, q20)


# ------------------------------------------------------------------------------------------------ FFTCC3D generic kernel
@pytest.mark.parametrize("r", [(21, 21, 21), (26, 26, 26), (36, 36, 36)], ids=_label)
def test_fftcc3d_generic_radices_and_long_windows(engine, vol, r):
    """42 = 2 3 7, 52 = 4 13 and 72 > 64 points per axis (radix 11 and windows of 80 points run in the sweep)."""
    ref, tar = vol
    _fftcc(engine, ref, tar, _pois(r, 4, seed=7 * r[0]), r, _label(r))


# ------------------------------------------------------------------------------------------------ shear
G_BASE = np.array([[0.025, -0.015, 0.02], [0.018, -0.02, 0.012], [-0.022, 0.016, 0.03]])
# per subvolume radius: |A_ij| up to 0.075 at r = 14 and 16, 0.0375 at r = 24, so that the shear reach of a subset row
# (|A_ij| r summed over j) is 2 to 3 voxels, beyond the tile's 1-voxel margin in y and z at every radius
SHEAR_SCALE = {14: 2.5, 16: 2.5, 24: 1.25}
SHEAR_SLAB_K = {14: 10, 16: 11, 24: 10}  # slab thickness of the plan (checked by test_icgn3d_plan_host.py)
T_TRUE = np.array([1.4, -0.8, 2.3])


def _sheared_target(ref, g):
    """Target = reference resampled (oracle tricubic) under x' = c + t + (I + G)(x - c), all nine gradient terms non-zero."""
    o = Oracle3D(ref, ref)
    o.prepare()
    c = 0.5 * (DIM - 1)
    zz, yy, xx = np.mgrid[0:DIM, 0:DIM, 0:DIM].astype(np.float64)
    dst = np.stack([xx.ravel(), yy.ravel(), zz.ravel()], 1)
    src = (dst - c - T_TRUE) @ np.linalg.inv(np.eye(3) + g).T + c
    tar = o.tricubic(src.astype(np.float32)).reshape(DIM, DIM, DIM)
    return np.where(tar < 0, synth.BACKGROUND, tar).astype(np.float32)  # -1: source point outside the reference


def _tile_replay(q, r, slab_k, dims):
    """Replays icgn3d1_kernel's tile placement (icgn3d.cu: tile origin per iteration and slab, the warp-uniform slab_fast
    bounding-box test, the per-sample tile test of the checked loop) at the warp each POI starts from.  Returns the number of
    slabs that take the checked loop and the number of samples whose 4x4x4 support leaves the staged tile."""
    rx, ry, rz = r
    dx, dy, dz = dims
    margin = 1  # ICGN3D_TILE_MARGIN
    tx, ty, tz = (2 * rx + 1 + 3 + 2 * margin + 3 + 3) & ~3, 2 * ry + 1 + 3 + 2 * margin, slab_k + 3 + 2 * margin
    sz = 2 * rz + 1
    slabs_checked = samples_out = 0
    for p in q.astype(np.float64):
        px, py, pz = p[0:3]
        A = np.array([[1 + p[4], p[5], p[6], p[3]], [p[8], 1 + p[9], p[10], p[7]], [p[12], p[13], 1 + p[14], p[11]]])
        tx0 = (int(np.floor(px + A[0, 3])) - rx - 1 - margin) & ~3
        ty0 = int(np.floor(py + A[1, 3])) - ry - 1 - margin
        xlo, xhi = max(1.0, tx0 + 1.0), min(dx - 2.0, tx0 + tx - 2.0)
        ylo, yhi = max(1.0, ty0 + 1.0), min(dy - 2.0, ty0 + ty - 2.0)
        for zs in range(0, sz, slab_k):
            nz = min(slab_k, sz - zs)
            zl0 = zs - rz
            tz0 = int(np.floor(pz + A[2, 3] + min(A[2, 2] * zl0, A[2, 2] * (zl0 + nz - 1)))) - 1 - margin
            zlo, zhi = max(1.0, tz0 + 1.0), min(dz - 2.0, tz0 + tz - 2.0)
            zh = 0.5 * (nz - 1)
            zc = zl0 + zh
            ctr = np.array([px, py, pz]) + A[:, 2] * zc + A[:, 3]
            ext = np.abs(A[:, 0]) * rx + np.abs(A[:, 1]) * ry + np.abs(A[:, 2]) * zh + 2e-3
            lo, hi = np.array([xlo, ylo, zlo]), np.array([xhi, yhi, zhi])
            if np.all(ctr - ext >= lo) and np.all(ctr + ext < hi):
                continue
            slabs_checked += 1
            zl, yl, xl = np.meshgrid(np.arange(zl0, zl0 + nz), np.arange(-ry, ry + 1), np.arange(-rx, rx + 1), indexing="ij")
            loc = np.stack([xl.ravel(), yl.ravel(), zl.ravel(), np.ones(xl.size)], 0)
            X = (A @ loc) + np.array([[px], [py], [pz]])
            inside = np.all((X >= lo[:, None]) & (X < hi[:, None]), 0)
            samples_out += int((~inside).sum())
    return slabs_checked, samples_out


@pytest.mark.parametrize("r", SHEAR_RADII, ids=_label)
def test_shear_tma_and_staged_loads(engine, vol, monkeypatch, r):
    """Off-diagonal gradients move samples out of the staged tile (whose x, y origin follows the translation only): the
    slab-wide bounding-box test and the checked per-sample fallback decide.  Half the POIs start at the true map, half at
    the rounded true translation with zero gradients.  The TMA and the staged (OCB_NO_TMA) tile loads must give identical records."""
    g = G_BASE * SHEAR_SCALE[r[0]]
    ref = vol[0]
    tar = _sheared_target(ref, g)
    c = 0.5 * (DIM - 1)
    n = {14: 16, 16: 12, 24: 6}[r[0]]
    xyz = _pois(r, n, seed=11 * r[0], dim=DIM)
    xyz = np.clip(xyz, r[0] + 14, DIM - 1 - r[0] - 14)  # keep the sheared subvolume clear of the resampling border
    q = ob.make_poi3d(xyz)
    disp = T_TRUE + (xyz - c) @ g.T
    true_map = np.arange(n) % 2 == 0
    disp[~true_map] = np.round(disp[~true_map])  # an FFT-CC-like start: the translation stops the iterations only once it moves little
    q[:, 3], q[:, 7], q[:, 11] = disp[:, 0], disp[:, 1], disp[:, 2]
    for i in range(3):
        for j in range(3):
            q[true_map, 4 * i + 4 + j] = g[i, j]
    # the case exercises what it is meant to: already at the starting warps, slabs leave the fast path and samples the tile
    slabs_checked, samples_out = _tile_replay(q, r, SHEAR_SLAB_K[r[0]], (DIM, DIM, DIM))
    assert slabs_checked >= 1 and samples_out >= 1, (slabs_checked, samples_out)
    print("shear %s: %d slabs on the checked path, %d samples outside the tile at the starting warps" % (_label(r), slabs_checked, samples_out))
    a, b = q.copy(), q.copy()
    _icgn_gpu(engine, ref, tar, a, r)
    monkeypatch.setenv("OCB_NO_TMA", "1")
    s = _icgn_gpu(engine, ref, tar, q.copy(), r)
    monkeypatch.delenv("OCB_NO_TMA")
    assert np.array_equal(a, s), "TMA and staged tile loads differ"
    Oracle3D(ref, tar).icgn3d1(b, *r, 0.001, 20, exact=True)
    _check(a, b, "shear " + _label(r))
    ok = a[:, 18] > 0.9
    assert ok.sum() >= n // 2
    assert np.abs(a[ok][:, [4, 5, 6, 8, 9, 10, 12, 13, 14]] - g.ravel()).max() < 2e-3  # the shear is recovered


# ------------------------------------------------------------------------------------------------ sentinels
@pytest.mark.parametrize("r", SENTINEL_RADII, ids=_label)
def test_sentinels(engine, vol, r):
    ref, tar = vol
    rx = r[0]
    c = DIM // 2
    xyz = np.array([[rx - 1, c, c], [c, c, c], [c, c, c], [c, c, c], [c, c, c], [c, c, c], [c + 2, c - 1, c + 1],
                    [c - 2, c + 1, c - 1]], np.float32)
    q = ob.make_poi3d(xyz)
    q[:, 3], q[:, 7], q[:, 11] = 1.0, -1.0, 2.0
    q[1, 18] = -1.0              # skipped, keeps its code
    q[2, 18] = -2.0
    q[3, 3] = DIM - c - rx + 3   # the guess pushes the subvolume out of the target -> -3
    q[4, 7] = np.nan             # NaN guess -> -3
    a, b = q.copy(), q.copy()
    _icgn_gpu(engine, ref, tar, a, r)
    Oracle3D(ref, tar).icgn3d1(b, *r, 0.001, 20, exact=True)
    assert list(b[:5, 18]) == [-3, -1, -2, -3, -3]
    assert np.array_equal(a[:5], b[:5], equal_nan=True)
    _check(a[5:], b[5:], "sentinels " + _label(r), min_valid=1.0)
    # stop = 1: one iteration, not converged -> -4; the parameters of that iteration are kept and compared
    a, b = q[5:].copy(), q[5:].copy()
    _icgn_gpu(engine, ref, tar, a, r, stop=1)
    Oracle3D(ref, tar).icgn3d1(b, *r, 0.001, 1, exact=True)
    assert (b[:, 18] == -4).all() and (a[:, 18] == -4).all()
    assert np.array_equal(a[:, 19], b[:, 19])
    d = np.abs(a[:, 3:15] - b[:, 3:15]).max()
    assert d < 1e-4, "stop=1 %s: max |d parameter| = %.3g" % (_label(r), d)
    print("sentinels stop=1 %s: max|dparam|=%.2e" % (_label(r), d))


@pytest.mark.parametrize("r", SENTINEL_RADII, ids=_label)
def test_negative_interpolated_sample_rule(engine, vol, r):
    """Black voids in both volumes: the `any interpolated sample < 0 -> -3` rule must reject exactly the POIs the reference's
    float arithmetic rejects (oracle exact=0); the kept POIs match the exact oracle."""
    from test_gpu_sentinel import _discs
    base_ref, base_tar = vol
    rx = r[0]
    voids = _discs((DIM, DIM, DIM), 30 if rx <= 12 else 6, 3, 7, 5)  # fewer voids for larger subvolumes: some POIs are kept
    ref, tar = np.where(voids, 0, base_ref).astype(np.float32), np.where(voids, 0, base_tar).astype(np.float32)
    step = 6 if rx <= 12 else 8
    lo, hi = rx + 1, DIM - rx - 5
    k = np.arange(lo, hi + 1, step)
    xyz = np.stack(np.meshgrid(k, k, k, indexing="ij"), -1).reshape(-1, 3)[:, ::-1].astype(np.float32)
    if len(xyz) > 64:
        xyz = xyz[np.random.default_rng(1).choice(len(xyz), 64, replace=False)]
    q = ob.make_poi3d(xyz)
    u, v, w = synth.displacement_3d(xyz[:, 0], xyz[:, 1], xyz[:, 2], DIM, DIM, DIM)
    q[:, 3], q[:, 7], q[:, 11] = np.round(u), np.round(v), np.round(w)
    a, b, e = q.copy(), q.copy(), q.copy()
    _icgn_gpu(engine, ref, tar, a, r)
    o = Oracle3D(ref, tar)
    o.icgn3d1(b, *r, 0.001, 20)
    o.icgn3d1(e, *r, 0.001, 20, exact=True)
    differ = np.where((a[:, 18] == -3) != (b[:, 18] == -3))[0]
    assert len(differ) == 0, "%s: -3 decided differently at POIs %s" % (_label(r), differ[:10])
    rej = b[:, 18] == -3
    assert np.array_equal(a[rej], b[rej])
    assert rej.sum() >= 1 and (~rej).sum() >= 1, (rej.sum(), len(rej))
    kept = ~rej & (e[:, 18] != -3)
    _check(a[kept], e[kept], "voids " + _label(r), min_valid=0.5)
    # The first iteration samples the target at integer offsets, where the interpolant of a void is zero up to rounding: a
    # POI whose subvolume touches a void and stays inside the volume has a borderline smallest sample (|min| < 0.125,
    # ICGN3D_NEG_TRIGGER), which the kernel re-decides in icgn3d_exact_negative.  Make sure some POIs go that way.
    off = np.stack(np.meshgrid(np.arange(-r[2], r[2] + 1), np.arange(-r[1], r[1] + 1), np.arange(-rx, rx + 1), indexing="ij"), -1)
    off = off.reshape(-1, 3)[:, ::-1].astype(np.float64)
    tmin = np.array([o.tricubic(p[0:3] + p[[3, 7, 11]] + off).min() for p in q.astype(np.float64)])
    borderline = int(((tmin > -0.1) & (tmin < 0.1)).sum())
    assert borderline >= 1, tmin
    print("voids %s: %d rejected, %d kept, %d with a borderline smallest first sample" % (_label(r), rej.sum(), (~rej).sum(), borderline))


# ------------------------------------------------------------------------------------------------ large coordinates
@pytest.fixture(scope="module")
def tall():
    """48 x 48 x 3100 voxels: a 200-layer speckle block at z = 2900..3099 in a uniform background."""
    ref_b, tar_b = synth.speckle_pair_3d(48, 48, 200)
    ref = np.full((3100, 48, 48), synth.BACKGROUND, np.float32)
    tar = ref.copy()
    ref[2900:], tar[2900:] = ref_b, tar_b
    return ref, tar


@pytest.mark.parametrize("r", LARGE_Z_RADII, ids=_label)
def test_large_z_coordinates(engine, tall, r):
    """z ~ 3000: a float ulp is 2.4e-4 voxel there, so the order `centre + warped offset` matters."""
    ref, tar = tall
    k = np.array([20, 24, 28]) if r[0] == 8 else np.array([22, 26])
    kz = 3000 + (np.array([-8, 0, 8]) if r[0] == 8 else np.array([-4, 4]))
    xyz = np.stack(np.meshgrid(kz, k, k, indexing="ij"), -1).reshape(-1, 3)[:, ::-1].astype(np.float32)
    q = _fftcc(engine, ref, tar, xyz, r, "large z " + _label(r))
    a, b = q.copy(), q.copy()
    _icgn_gpu(engine, ref, tar, a, r)
    Oracle3D(ref, tar).icgn3d1(b, *r, 0.001, 20, exact=True)
    _check(a, b, "large z " + _label(r), tol=1.5e-4)
