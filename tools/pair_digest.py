"""What every pair call computes, as digests: one line per call on fixed seeded inputs, with the SHA-256 of each output buffer and
the launches the call made (launch_count() delta).  Two builds of the library (selected with OCB_LIB_PATH) that compute the same
and do the same work print the same lines.

Calls: FFTCC2D (all three kernels), FFTCC3D, ICGN2D1, ICGN2D2, ICGN2D_EX (centre offsets; self-adaptive), ICLM2D, NR2D1,
EpipolarSearch, Strain (2D, 3D, POI2DS, single POI), ICGN3D1 (every kernel variant; sheared guesses) and stereo reconstruction,
with host buffers and with device pointers.  Host queues include one of >= 16384 records (the four-stream pipeline) and one
page-locked queue (read and written in place), and every call that shards a host queue also runs once on a one-member group
context.

    python tools/pair_digest.py > a.txt; OCB_LIB_PATH=other.so python tools/pair_digest.py > b.txt; diff a.txt b.txt
"""
import ctypes
import hashlib
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from opencorr_b200 import _capi, synth  # noqa: E402
from opencorr_b200.api import POI2D_FLOATS, POI2DS_FLOATS, POI3D_FLOATS  # noqa: E402

CONV, STOP = 0.001, 10.0
W, H, D = 512, 384, 64
DL = 96  # room for a 61^3 subvolume
FUND = np.array([0, 0, 0, 0, 0, -1, 0, 1, 0], np.float32)  # a rectified pair
PAR = np.zeros(3, np.float32)
ST = (40.0, 6, 0.5, 1)  # strain: radius, min_neighbors, zncc_threshold, approximation


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()[:16]


def vp(a):
    return ctypes.c_void_p(a.ctypes.data)


class Runner:
    def __init__(self, lib, ctx, label):
        self.lib, self.ctx, self.label = lib, ctx, label

    def host(self, name, call, *queues):
        """call(*pointers) on copies of the host queues; prints their digests"""
        qs = [q.copy() for q in queues]
        b = self.lib.ocb_launch_count(self.ctx)
        rc = call(*[vp(q) for q in qs])
        self.report(name, rc, b, qs)
        return qs

    def pinned(self, name, call, queue):
        """call(pointer) on a page-locked copy of the queue"""
        p = self.lib.ocb_host_alloc(queue.nbytes)
        a = np.ctypeslib.as_array(ctypes.cast(p, ctypes.POINTER(ctypes.c_float)), queue.shape)
        a[...] = queue
        b = self.lib.ocb_launch_count(self.ctx)
        rc = call(ctypes.c_void_p(p))
        self.report(name + " pinned", rc, b, [a.copy()])
        self.lib.ocb_host_free(ctypes.c_void_p(p))

    def dev(self, name, call, *queues):
        """call(*device pointers) on device copies of the queues"""
        ts = [torch.from_numpy(np.ascontiguousarray(q)).cuda() for q in queues]
        torch.cuda.synchronize()
        b = self.lib.ocb_launch_count(self.ctx)
        rc = call(*[ctypes.c_void_p(t.data_ptr()) for t in ts])
        assert self.lib.ocb_sync(self.ctx) == 0
        self.report(name + " dev", rc, b, [t.cpu().numpy() for t in ts])

    def report(self, name, rc, before, outs):
        err = "" if rc == 0 else " error=%s" % self.lib.ocb_last_error(self.ctx).decode()
        print(" ".join(["%s %s" % (self.label, name), "rc=%d" % rc, "launches=%d" % (self.lib.ocb_launch_count(self.ctx) - before)]
                       + [sha(o) for o in outs]) + err, flush=True)


def queue_2d(step=20, margin=40):
    xy = synth.grid_2d(margin, margin, (W - 2 * margin) // step + 1, (H - 2 * margin) // step + 1, step, step)
    q = np.zeros((len(xy), POI2D_FLOATS), np.float32)
    q[:, :2] = xy
    return q


def queue_3d(step=8, margin=16, dim=D):
    k = (dim - 2 * margin) // step + 1
    xyz = synth.grid_3d(margin, margin, margin, k, k, k, step, step, step)
    q = np.zeros((len(xyz), POI3D_FLOATS), np.float32)
    q[:, :3] = xyz
    return q


def setup(lib, ctx):
    ref, tar = synth.speckle_pair_2d(W, H, second_order=True)
    r3, t3 = synth.speckle_pair_3d(D, D, D)
    assert lib.ocb_set_images_2d(ctx, vp(ref), vp(tar), W, H, 0) == 0
    assert lib.ocb_set_images_3d(ctx, vp(r3), vp(t3), D, D, D) == 0
    for prep in (lib.ocb_icgn2d_prepare, lib.ocb_nr2d_prepare, lib.ocb_icgn3d_prepare):
        assert prep(ctx) == 0


def run_2d(run, lib, ctx, group):
    q, big = queue_2d(), queue_2d(step=3, margin=24)
    assert len(big) >= 16384
    n, nb = len(q), len(big)
    seeds = run.host("fftcc2d r=16", lambda p: lib.ocb_fftcc2d(ctx, p, n, 16, 16), q)[0]
    big_seeds = run.host("fftcc2d r=16 n=%d" % nb, lambda p: lib.ocb_fftcc2d(ctx, p, nb, 16, 16), big)[0]
    run.host("fftcc2d r=10", lambda p: lib.ocb_fftcc2d(ctx, p, n, 10, 10), q)
    run.host("fftcc2d r=(12,9)", lambda p: lib.ocb_fftcc2d(ctx, p, n, 12, 9), q)
    offsets = np.tile(np.array([[0.25, -0.5]], np.float32), (n, 1))
    adaptive = seeds.copy()
    adaptive[:, 23], adaptive[:, 24] = np.where(np.arange(n) % 2, 12, 16), np.where(np.arange(n) % 2, 10, 16)
    calls = [
        ("icgn2d1 r=16", lambda c, p, m: lib.ocb_icgn2d1(c, p, m, 16, 16, CONV, STOP), lambda c, p, m: lib.ocb_icgn2d1_dev(c, p, m, 16, 16, CONV, STOP)),
        ("icgn2d1 r=(12,9)", lambda c, p, m: lib.ocb_icgn2d1(c, p, m, 12, 9, CONV, STOP), lambda c, p, m: lib.ocb_icgn2d1_dev(c, p, m, 12, 9, CONV, STOP)),
        ("icgn2d2 r=20", lambda c, p, m: lib.ocb_icgn2d2(c, p, m, 20, 20, CONV, STOP), lambda c, p, m: lib.ocb_icgn2d2_dev(c, p, m, 20, 20, CONV, STOP)),
        ("icgn2d_ex order=2", lambda c, p, m: lib.ocb_icgn2d_ex(c, 2, p, m, 16, 16, CONV, STOP, None, 0),
         lambda c, p, m: lib.ocb_icgn2d_ex_dev(c, 2, p, m, 16, 16, CONV, STOP, None)),
        ("iclm2d order=1", lambda c, p, m: lib.ocb_iclm2d(c, 1, p, m, 16, 16, CONV, STOP, 10.0, 0.5, 4.0),
         lambda c, p, m: lib.ocb_iclm2d_dev(c, 1, p, m, 16, 16, CONV, STOP, 10.0, 0.5, 4.0)),
        ("nr2d1 r=16", lambda c, p, m: lib.ocb_nr2d1(c, p, m, 16, 16, CONV, STOP), lambda c, p, m: lib.ocb_nr2d1_dev(c, p, m, 16, 16, CONV, STOP)),
    ]
    for name, host, dev in calls:
        run.host(name, lambda p: host(ctx, p, n), seeds)
        if group:
            continue
        run.host(name + " n=%d" % nb, lambda p: host(ctx, p, nb), big_seeds)
        run.pinned(name, lambda p: host(ctx, p, n), seeds)
        run.dev(name, lambda p: dev(ctx, p, n), seeds)
    epi = seeds[:64]
    run.host("epipolar_search2d", lambda p: lib.ocb_epipolar_search2d(ctx, p, len(epi), vp(FUND), vp(PAR), vp(PAR), 6, 1, 16, 16, CONV, STOP), epi)
    if group:
        return
    run.pinned("fftcc2d r=16", lambda p: lib.ocb_fftcc2d(ctx, p, n, 16, 16), q)
    run.pinned("fftcc2d r=16 n=%d" % nb, lambda p: lib.ocb_fftcc2d(ctx, p, nb, 16, 16), big)
    run.dev("fftcc2d r=16", lambda p: lib.ocb_fftcc2d_dev(ctx, p, n, 16, 16), q)
    run.dev("fftcc2d r=10", lambda p: lib.ocb_fftcc2d_dev(ctx, p, n, 10, 10), q)
    run.host("icgn2d_ex order=1 offsets", lambda p, o: lib.ocb_icgn2d_ex(ctx, 1, p, n, 16, 16, CONV, STOP, o, 0), seeds, offsets)
    run.dev("icgn2d_ex order=1 offsets", lambda p, o: lib.ocb_icgn2d_ex_dev(ctx, 1, p, n, 16, 16, CONV, STOP, o), seeds, offsets)
    run.host("icgn2d_ex self-adaptive", lambda p: lib.ocb_icgn2d_ex(ctx, 2, p, n, 16, 16, CONV, STOP, None, 1), adaptive)
    run.dev("epipolar_search2d", lambda p: lib.ocb_epipolar_search2d_dev(ctx, p, len(epi), vp(FUND), vp(PAR), vp(PAR), 6, 1, 16, 16, CONV, STOP), epi)
    out = run.host("icgn2d1 r=16 (strain input)", lambda p: lib.ocb_icgn2d1(ctx, p, n, 16, 16, CONV, STOP), seeds)[0]
    out2ds = np.zeros((n, POI2DS_FLOATS), np.float32)
    out2ds[:, :2], out2ds[:, 2:4] = out[:, :2], out[:, 2:3].repeat(2, 1)
    for name, data, host, dev in (("strain2d", out, lib.ocb_strain2d, lib.ocb_strain2d_dev), ("strain2ds", out2ds, lib.ocb_strain2ds, lib.ocb_strain2ds_dev)):
        run.host(name, lambda p: host(ctx, p, n, *ST), data)
        run.dev(name, lambda p: dev(ctx, p, n, *ST), data)
    run.host("strain2d_single", lambda p: lib.ocb_strain2d_single(ctx, p, n, n // 2, *ST), out)


def run_3d(run, lib, ctx, group):
    q = queue_3d()
    n = len(q)
    seeds = run.host("fftcc3d r=8", lambda p: lib.ocb_fftcc3d(ctx, p, n, 8, 8, 8), q)[0]
    out = run.host("icgn3d1 r=8", lambda p: lib.ocb_icgn3d1(ctx, p, n, 8, 8, 8, CONV, 20.0), seeds)[0]
    if group:
        return
    run.host("fftcc3d r=16", lambda p: lib.ocb_fftcc3d(ctx, p, n, 16, 16, 16), q)
    run.host("fftcc3d r=(7,6,5)", lambda p: lib.ocb_fftcc3d(ctx, p, n, 7, 6, 5), q)
    run.dev("fftcc3d r=8", lambda p: lib.ocb_fftcc3d_dev(ctx, p, n, 8, 8, 8), q)
    run.dev("icgn3d1 r=8", lambda p: lib.ocb_icgn3d1_dev(ctx, p, n, 8, 8, 8, CONV, 20.0), seeds)
    run.host("strain3d", lambda p: lib.ocb_strain3d(ctx, p, n, *ST), out)
    run.dev("strain3d", lambda p: lib.ocb_strain3d_dev(ctx, p, n, *ST), out)
    run.host("strain3d_single", lambda p: lib.ocb_strain3d_single(ctx, p, n, 3, *ST), out)


def run_3d_kernels(run, lib, ctx):
    """ICGN3D1 at every kernel it selects, on a DL^3 pair: <16,256> (tail column), a generic <0,512> radius, <30,512>, and a
    queue whose guesses carry shears of three sizes, so that both row-pair samples of a step fall in different blocks (small
    shears) and whole slabs leave the tile (large ones)."""
    r3, t3 = synth.speckle_pair_3d(DL, DL, DL)
    assert lib.ocb_set_images_3d(ctx, vp(r3), vp(t3), DL, DL, DL) == 0
    assert lib.ocb_icgn3d_prepare(ctx) == 0
    q = queue_3d(step=12, margin=32, dim=DL)
    n = len(q)
    seeds = run.host("fftcc3d r=8 D=%d" % DL, lambda p: lib.ocb_fftcc3d(ctx, p, n, 8, 8, 8), q)[0]
    for r in (16, 22, 30):
        run.host("icgn3d1 r=%d" % r, lambda p: lib.ocb_icgn3d1(ctx, p, n, r, r, r, CONV, 20.0), seeds)
    sheared = seeds.copy()
    scale = np.array([0.01, 0.03, 0.15], np.float32)[np.arange(n) % 3]
    for k, g in zip((4, 5, 6, 8, 9, 10, 12, 13, 14), (0.4, -0.6, 0.5, 0.7, 0.3, -0.5, -0.6, 0.8, 0.2)):  # ux uy uz vx vy vz wx wy wz
        sheared[:, k] = scale * g
    for r in (8, 16):
        run.host("icgn3d1 r=%d sheared" % r, lambda p: lib.ocb_icgn3d1(ctx, p, n, r, r, r, CONV, 20.0), sheared)


def run_stereo(run, lib, ctx):
    intr = np.array([900, 905, 0.5, W / 2, H / 2, 0.01, -0.002, 0, 0, 0, 0, 0.001, -0.001], np.float32)
    cal = []
    b = lib.ocb_launch_count(ctx)
    for _ in range(2):
        h = ctypes.c_void_p()
        assert lib.ocb_calib_prepare(ctx, vp(intr), H, W, 0.001, 10, ctypes.byref(h)) == 0
        cal.append(h)
    maps = np.zeros((2, H, W), np.float32)
    assert lib.ocb_calib_get_map(ctx, cal[0], vp(maps[0]), vp(maps[1])) == 0
    run.report("calib_prepare x2", 0, b, [maps])
    p1 = np.array([900, 0, W / 2, 0, 0, 905, H / 2, 0, 0, 0, 1, 0], np.float32)
    p2 = p1.copy()
    p2[3] = -900 * 60.0
    rng = np.random.default_rng(7)
    pts1 = (rng.random((500, 2)) * [W, H]).astype(np.float32)
    pts2 = pts1 + np.float32([-12.5, 0.25])
    pts3 = np.zeros((500, 3), np.float32)
    undist = np.zeros_like(pts1)
    run.host("calib_undistort", lambda p, o: lib.ocb_calib_undistort(ctx, cal[0], vp(intr), p, o, 500), pts1, undist)

    def rec(a, b_, c):
        return lib.ocb_stereo_reconstruct(ctx, cal[0], vp(intr), vp(p1), cal[1], vp(intr), vp(p2), a, b_, c, 500)

    def rec_dev(a, b_, c):
        return lib.ocb_stereo_reconstruct_dev(ctx, cal[0], vp(intr), vp(p1), cal[1], vp(intr), vp(p2), a, b_, c, 500)

    run.host("stereo_reconstruct", rec, pts1, pts2, pts3)
    run.dev("stereo_reconstruct", rec_dev, pts1, pts2, pts3)
    for h in cal:
        lib.ocb_calib_destroy(h)


def main():
    lib = _capi.load()
    ctx = lib.ocb_create(0)
    group = lib.ocb_create_multi((ctypes.c_int * 1)(0), 1)
    for c in (ctx, group):
        setup(lib, c)
    run = Runner(lib, ctx, "single")
    run_2d(run, lib, ctx, False)
    run_3d(run, lib, ctx, False)
    run_3d_kernels(run, lib, ctx)
    run_stereo(run, lib, ctx)
    grun = Runner(lib, group, "group")
    run_2d(grun, lib, group, True)
    run_3d(grun, lib, group, True)
    lib.ocb_destroy(group)
    lib.ocb_destroy(ctx)


if __name__ == "__main__":
    main()
