"""GPU: RegionFit2D / RegionFit3D (ocb_region_fit2d / 3d and their _dev variants, the Python classes and the C++ shim) against
the float64 witness of tests/region_fit_cases.py on every two-set case: the same POIs written, the written fields within
TOL = 2e-6 max(1, |value|) -- FP64 normal equations against FP64 Householder QR, the tolerance of the Strain tests -- and every
other byte, and every byte of an unwritten POI, as it was.  Then the launch count, the argument checks, a group context, and
the recovery loop RegionFit2D -> ICGN2D2 on a synthetic pair."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import opencorr_b200 as ob
from opencorr_b200 import _capi, synth
import region_fit_cases as rc
import strain_cases as sc

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = {c.name: c for c in rc.small_cases()}
KIND = {25: "2d", 31: "3d"}


def host_fit(engine, c):
    got = c.q.copy()
    engine.region_fit(np.ascontiguousarray(c.rel), got, c.radius, c.k_min)
    return got


def dev_fit(engine, c):
    torch = pytest.importorskip("torch")
    d_q = torch.from_numpy(c.q.copy()).cuda()
    d_rel = torch.from_numpy(np.ascontiguousarray(c.rel)).cuda()
    torch.cuda.synchronize()
    engine.region_fit_dev(KIND[c.q.shape[1]], d_rel.data_ptr() if len(c.rel) else 0, len(c.rel), d_q.data_ptr(), len(c.q), c.radius, c.k_min)
    engine.sync()
    return d_q.cpu().numpy()


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
@pytest.mark.parametrize("name", sorted(CASES))
def test_against_the_witness(engine, name, dev):
    c = CASES[name]
    w = rc.witness(c.rel, c.q, c.radius, c.k_min)
    got = (dev_fit if dev else host_fit)(engine, c)
    n, d = rc.compare(got, c.q, w, rc.TOL, name)
    assert n == int(w.computed.sum())
    print("%s %s: %d of %d written, %d by the k-nearest fallback, max rel diff %.2e" % (name, "dev" if dev else "host", n, len(c.q),
                                                                                        int((w.computed & w.fallback).sum()), d))


@pytest.mark.parametrize("D", [2, 3])
def test_queue_longer_than_the_resident_warps(engine, D):
    """A queue several times the warps one launch holds (the kernel's grid-stride loop), against the witness."""
    rng = np.random.default_rng(D)
    ext = 600.0 if D == 2 else 90.0
    rel = rc.reliable_set(rng.uniform(0, ext, (40000, D)), rng)
    c = rc.Case("long_%d" % D, rel, rc.queue_set(rng.uniform(-5, ext + 5, (60000, D)), rng), 9.0 if D == 2 else 5.0, 9)
    w = rc.witness(c.rel, c.q, c.radius, c.k_min)
    rc.compare(host_fit(engine, c), c.q, w, rc.TOL, c.name)


def test_launch_count_does_not_depend_on_n(engine):
    rng = np.random.default_rng(3)
    counts = []
    for n_rel, n in ((50, 10), (20000, 30000), (0, 5)):
        rel = rc.reliable_set(rng.uniform(0, 300, (n_rel, 2)), rng) if n_rel else np.zeros((0, 25), np.float32)
        q = rc.queue_set(rng.uniform(0, 300, (n, 2)), rng)
        before = engine.launch_count()
        engine.region_fit(rel, q, 12.0, 9)
        counts.append(engine.launch_count() - before)
    assert counts[0] == counts[1] == counts[2] == 5, counts


def _raw(engine, D, dev, rel, n_rel, q, n):
    fn = getattr(engine._lib, "ocb_region_fit%dd%s" % (D, "_dev" if dev else ""))
    return fn(engine._ctx, rel, n_rel, q, n, ctypes.c_float(10.0), 5)


def test_bad_arguments_write_nothing(engine):
    torch = pytest.importorskip("torch")
    c = CASES["uniform_2"]
    for dev in (False, True):
        q = c.q.copy()
        rel = np.ascontiguousarray(c.rel)
        if dev:
            d_q, d_rel = torch.from_numpy(q.copy()).cuda(), torch.from_numpy(rel).cuda()
            qp, rp = ctypes.c_void_p(d_q.data_ptr()), ctypes.c_void_p(d_rel.data_ptr())
        else:
            qp, rp = ctypes.c_void_p(q.ctypes.data), ctypes.c_void_p(rel.ctypes.data)
        for args in ((None, len(rel), qp, len(q)), (rp, len(rel), None, len(q)), (rp, 1 << 31, qp, len(q)), (rp, len(rel), qp, 1 << 31),
                     (rp, 1 << 62, qp, len(q))):
            assert _raw(engine, 2, dev, *args) == _capi.OCB_ERR_ARG, (dev, args)
        assert _raw(engine, 2, dev, rp, len(rel), None, 0) == _capi.OCB_OK  # nothing to do
        if dev:
            engine.sync()
            q = d_q.cpu().numpy()
        assert np.array_equal(sc.bits(q), sc.bits(c.q)), dev
    with pytest.raises(ValueError):
        engine.region_fit(CASES["uniform_3"].rel, c.q.copy(), 10.0, 5)  # 3D reliable records for a 2D queue
    with pytest.raises(ValueError):
        engine.region_fit_dev("2ds", 0, 0, 0, 0, 10.0, 5)


def test_group_context(engine):
    n_dev = _capi.load().ocb_device_count()
    grp = ob.Engine(list(range(n_dev)))
    try:
        for name in ("uniform_2", "cell_boundary_3_r7.5", "outside_grown_2", "nonfinite_3"):
            c = CASES[name]
            assert np.array_equal(sc.bits(host_fit(grp, c)), sc.bits(host_fit(engine, c))), name
        # the device-pointer entry points need a single-device context
        c = CASES["uniform_2"]
        q = c.q.copy()
        assert _raw(grp, 2, True, ctypes.c_void_p(c.rel.ctypes.data), len(c.rel), ctypes.c_void_p(q.ctypes.data), len(q)) == _capi.OCB_ERR_ARG
    finally:
        grp.close()


def test_python_classes(engine):
    for name, cls in (("uniform_2", ob.RegionFit2D), ("uniform_3", ob.RegionFit3D)):
        c = CASES[name]
        fit = cls(c.radius, c.k_min, 4, engine=engine)
        assert (fit.getSearchRadius(), fit.getNeighborMin()) == (c.radius, c.k_min)
        fit.setNeighbor(np.ascontiguousarray(c.rel))
        fit.prepare()
        q = c.q.copy()
        fit.compute(q)
        assert np.array_equal(sc.bits(q), sc.bits(host_fit(engine, c))), name
        one = c.q.copy()
        fit.compute(one[3])  # compute(POI*): that POI alone
        expect = c.q.copy()
        expect[3] = q[3]
        assert np.array_equal(sc.bits(one), sc.bits(expect)), name


def test_shim_both_classes_and_overloads(engine, tmp_path):
    exe = tmp_path / "region_fit_shim_test"
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    lib = os.path.join(ROOT, "opencorr_b200", "lib")
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-fopenmp", "-I" + os.path.join(ROOT, "include", "opencorr"), "-o", str(exe),
                           os.path.join(ROOT, "tests", "native", "region_fit_shim_test.cpp"), "-L" + lib, "-lopencorr_b200", "-Wl,-rpath," + lib])
    for name in ("uniform_2", "knn_fallback_3"):
        c = CASES[name]
        D = 3 if c.q.shape[1] == 31 else 2
        (tmp_path / "rel.bin").write_bytes(np.ascontiguousarray(c.rel).tobytes())
        (tmp_path / "q.bin").write_bytes(c.q.tobytes())
        full = host_fit(engine, c)
        for index in (-1, 0, len(c.q) - 1):
            out = subprocess.run([str(exe), str(D), str(tmp_path / "rel.bin"), str(tmp_path / "q.bin"), str(tmp_path / "out.bin"), str(c.radius),
                                  str(c.k_min), str(index)], capture_output=True, text=True, timeout=300)
            assert out.returncode == 0, out.stderr
            shim = np.frombuffer((tmp_path / "out.bin").read_bytes(), np.float32).reshape(c.q.shape)
            expect = full if index < 0 else np.where(np.arange(len(c.q))[:, None] == index, full, c.q)
            assert np.array_equal(sc.bits(shim), sc.bits(expect)), (name, index)


def test_recovery_loop(engine):
    """FFTCC2D -> ICGN2D2 on a second-order speckle pair; a block of POIs re-seeded with garbage fails ICGN2D2; rounds of
    RegionFit2D over the reliable POIs then ICGN2D2 over the unreliable ones bring the block back to the clean run's records,
    within IC-GN's tolerance of the synthetic truth."""
    W = H = 512
    r, conv, stop = 16, 0.001, 10
    ref, tar = synth.speckle_pair_2d(W, H, second_order=True)
    xy = synth.grid_2d(40, 40, 55, 55, 8, 8)
    engine.set_images_2d(ref, tar)
    engine.icgn2d_prepare()
    clean = ob.make_poi2d(xy)
    engine.fftcc2d(clean, r, r)
    engine.icgn2d2(clean, r, r, conv, stop)
    reliable = lambda q: (q[:, 16] >= 0.9) & (q[:, 18] < conv)
    assert reliable(clean).mean() > 0.95
    gx, gy = (xy[:, 0] - 40) / 8, (xy[:, 1] - 40) / 8
    block = np.flatnonzero((gx >= 20) & (gx < 32) & (gy >= 18) & (gy < 30))
    q = clean.copy()
    q[block, 2:14] = 0
    q[block, 2], q[block, 8] = 23.0, -19.0  # garbage seeds, far beyond the subset
    engine.icgn2d2(q, r, r, conv, stop)
    assert not reliable(q)[block].any()
    fit = ob.RegionFit2D(20.0, 9, 1, engine=engine)
    rounds = 0
    for rounds in range(1, 21):
        bad = np.flatnonzero(~reliable(q))
        if not len(bad):
            break
        rel = np.ascontiguousarray(q[reliable(q)])
        sub = np.ascontiguousarray(q[bad])
        fit.setNeighbor(rel)
        fit.prepare()
        fit.compute(sub)
        engine.icgn2d2(sub, r, r, conv, stop)
        q[bad] = sub
        if not reliable(sub).any():
            break
    assert reliable(q)[block].all(), "%d block POIs still unreliable after %d rounds" % ((~reliable(q)[block]).sum(), rounds)
    u, v = synth.displacement_2d(xy[block, 0].astype(np.float64), xy[block, 1].astype(np.float64), W, H, True)
    err = np.hypot(q[block, 2] - u, q[block, 8] - v).max()
    clean_err = np.hypot(clean[block, 2] - u, clean[block, 8] - v).max()
    diff = np.abs(q[block, 2:14] - clean[block, 2:14]).max()
    print("recovered %d POIs in %d rounds: max |d| vs truth %.2e px (clean run %.2e), max field diff vs clean %.2e"
          % (len(block), rounds, err, clean_err, diff))
    assert err < max(2 * clean_err, 0.01) and np.abs(q[block][:, [2, 8]] - clean[block][:, [2, 8]]).max() < 5e-3, (err, clean_err, diff)
