"""The pair calls (one kernel family on the context's image or volume pair) refuse what they cannot run, each with its code and
message, in the order their checks run: a null context, a null queue with n > 0, a radius below 1, images not set, prepare() not
called, a radius the kernels cannot take, a strain index past the queue, an epipolar search step above the search radius, and
(device-pointer forms with a cap) 2^31 POIs.  A refused call leaves the queue and the launch count as they were; n = 0 is
accepted without a launch; an accepted call makes the launches listed below.

The host refusals also run on a one-member group context (the group path of the host calls; a member's refusal is reported as
"device 0: ..."), and every device-pointer form is refused there.  The 2^31 case runs only on calls that refuse it before they
touch the queue."""
import ctypes

import numpy as np
import pytest
import torch

from opencorr_b200 import _capi, synth
from opencorr_b200.api import POI2D_FLOATS, POI2DS_FLOATS, POI3D_FLOATS

pytestmark = pytest.mark.gpu

OK, ARG, STATE, UNSUP = _capi.OCB_OK, _capi.OCB_ERR_ARG, _capi.OCB_ERR_STATE, _capi.OCB_ERR_UNSUPPORTED
CONV, STOP = 0.001, 10.0
W, H, D = 96, 80, 32
FUND = np.array([0, 0, 0, 0, 0, -1, 0, 1, 0], np.float32)  # a rectified pair
PAR = np.zeros(3, np.float32)
ST = (30.0, 4, 0.5, 1)  # strain: radius, min_neighbors, zncc_threshold, approximation


def vp(a):
    return ctypes.c_void_p(a.ctypes.data)


def queue_2d(r=None):
    q = np.zeros((12, POI2D_FLOATS), np.float32)
    q[:, :2] = synth.grid_2d(24, 24, 4, 3, 16, 16)
    return q


def queue_3d(r=None):
    q = np.zeros((8, POI3D_FLOATS), np.float32)
    q[:, :3] = synth.grid_3d(12, 12, 12, 2, 2, 2, 8, 8, 8)
    return q


def queue_2ds(r=None):
    q = np.zeros((12, POI2DS_FLOATS), np.float32)
    q[:, :2] = synth.grid_2d(24, 24, 4, 3, 16, 16)
    return q


def queue_adaptive(r):  # the self-adaptive call takes each POI's radius from its record
    q = queue_2d()
    q[:, 23] = q[:, 24] = r
    return q


def design(what, r, dims=2):
    return "%s: subset radius (%s) exceeds the shared-memory design limit" % (what, ",".join([str(r)] * dims))


class Entry:
    """One pair call.  host(lib, ctx, q, n, r) / dev(...) call it (None: no such form); what_host / what_dev name it in the host
    and device-pointer messages; queue(r): its records; dim: the pair it reads (0: none); unsupported: [(radius, message)];
    sharded: a group splits the queue between its members (strain: the first member runs it, and its refusals carry no device);
    extra: the call's own refusals, [(label, host(lib, ctx, q, n), dev(...) or None, code, message)]."""

    def __init__(self, name, host, dev, what_host, what_dev, queue, dim=2, prepared=True, r=8, unsupported=(), launches=1, cap=True,
                 radius_refused=True, extra=(), sharded=True):
        self.name, self.host, self.dev, self.what_host, self.what_dev = name, host, dev, what_host, what_dev
        self.queue, self.dim, self.prepared, self.r, self.unsupported = queue, dim, prepared, r, list(unsupported)
        self.launches, self.cap, self.radius_refused, self.extra = launches, cap, radius_refused, list(extra)
        self.sharded = sharded


ENTRIES = [
    Entry("fftcc2d", lambda l, c, q, n, r: l.ocb_fftcc2d(c, q, n, r, r), lambda l, c, q, n, r: l.ocb_fftcc2d_dev(c, q, n, r, r), "fftcc2d",
          "fftcc2d", queue_2d, prepared=False, unsupported=[(37, "fftcc2d: window size 74x74 has a prime factor > 31")]),
    Entry("fftcc3d", lambda l, c, q, n, r: l.ocb_fftcc3d(c, q, n, r, r, r), lambda l, c, q, n, r: l.ocb_fftcc3d_dev(c, q, n, r, r, r), "fftcc3d",
          "fftcc3d", queue_3d, dim=3, prepared=False, r=5, unsupported=[(37, "fftcc3d: window size has a prime factor > 31")]),
    Entry("icgn2d1", lambda l, c, q, n, r: l.ocb_icgn2d1(c, q, n, r, r, CONV, STOP), lambda l, c, q, n, r: l.ocb_icgn2d1_dev(c, q, n, r, r, CONV, STOP),
          "icgn2d", "icgn2d", queue_2d, unsupported=[(100, design("icgn2d", 100))]),
    Entry("icgn2d2", lambda l, c, q, n, r: l.ocb_icgn2d2(c, q, n, r, r, CONV, STOP), lambda l, c, q, n, r: l.ocb_icgn2d2_dev(c, q, n, r, r, CONV, STOP),
          "icgn2d", "icgn2d", queue_2d, unsupported=[(100, design("icgn2d", 100))]),
    Entry("icgn2d_ex", lambda l, c, q, n, r: l.ocb_icgn2d_ex(c, 2, q, n, r, r, CONV, STOP, None, 0),
          lambda l, c, q, n, r: l.ocb_icgn2d_ex_dev(c, 2, q, n, r, r, CONV, STOP, None), "icgn2d_ex", "icgn2d", queue_2d,
          unsupported=[(100, design("icgn2d", 100))]),
    Entry("icgn2d_ex_adaptive", lambda l, c, q, n, r: l.ocb_icgn2d_ex(c, 1, q, n, 8, 8, CONV, STOP, None, 1), None, "icgn2d_ex", "icgn2d",
          queue_adaptive, radius_refused=False,
          unsupported=[(100, "icgn2d_ex: subset radius (100,100) of a self-adaptive POI exceeds the shared-memory design limit")]),
    Entry("iclm2d", lambda l, c, q, n, r: l.ocb_iclm2d(c, 1, q, n, r, r, CONV, STOP, 10.0, 0.5, 4.0),
          lambda l, c, q, n, r: l.ocb_iclm2d_dev(c, 1, q, n, r, r, CONV, STOP, 10.0, 0.5, 4.0), "iclm2d", "icgn2d", queue_2d,
          unsupported=[(100, design("icgn2d", 100))]),
    Entry("nr2d1", lambda l, c, q, n, r: l.ocb_nr2d1(c, q, n, r, r, CONV, STOP), lambda l, c, q, n, r: l.ocb_nr2d1_dev(c, q, n, r, r, CONV, STOP),
          "nr2d1", "nr2d1", queue_2d, unsupported=[(100, design("nr2d1", 100))]),
    # candidates, IC-GN and selection of one block; an unsupported radius is refused by that IC-GN, after the candidates launch
    Entry("epipolar_search2d", lambda l, c, q, n, r: l.ocb_epipolar_search2d(c, q, n, vp(FUND), vp(PAR), vp(PAR), 4, 1, r, r, CONV, STOP),
          lambda l, c, q, n, r: l.ocb_epipolar_search2d_dev(c, q, n, vp(FUND), vp(PAR), vp(PAR), 4, 1, r, r, CONV, STOP), "epipolar_search2d",
          "epipolar_search2d", queue_2d, launches=3, cap=False,
          extra=[("step > radius", lambda l, c, q, n: l.ocb_epipolar_search2d(c, q, n, vp(FUND), vp(PAR), vp(PAR), 2, 3, 8, 8, CONV, STOP),
                  lambda l, c, q, n: l.ocb_epipolar_search2d_dev(c, q, n, vp(FUND), vp(PAR), vp(PAR), 2, 3, 8, 8, CONV, STOP),
                  ARG, "epipolar_search2d: search radius is less than search step")]),
    Entry("icgn3d1", lambda l, c, q, n, r: l.ocb_icgn3d1(c, q, n, r, r, r, CONV, 20.0), lambda l, c, q, n, r: l.ocb_icgn3d1_dev(c, q, n, r, r, r, CONV, 20.0),
          "icgn3d1", "icgn3d1", queue_3d, dim=3, r=5, unsupported=[(200, design("icgn3d1", 200, 3)), (600, "icgn3d1: subset too large")]),
]
# strain: bounding box, keys, sort, gather and the strain kernel
for _name, _q in (("strain2d", queue_2d), ("strain3d", queue_3d), ("strain2ds", queue_2ds)):
    ENTRIES.append(Entry(_name, (lambda f: lambda l, c, q, n, r: getattr(l, "ocb_" + f)(c, q, n, *ST))(_name),
                         (lambda f: lambda l, c, q, n, r: getattr(l, "ocb_" + f + "_dev")(c, q, n, *ST))(_name), "strain", "strain", _q, dim=0,
                         prepared=False, launches=5, radius_refused=False, sharded=False))
for _name, _q in (("strain2d_single", queue_2d), ("strain3d_single", queue_3d)):
    ENTRIES.append(Entry(_name, (lambda f: lambda l, c, q, n, r: getattr(l, "ocb_" + f)(c, q, n, n - 1 if n else 0, *ST))(_name), None, "strain",
                         "strain", _q, dim=0, prepared=False, launches=5, radius_refused=False, sharded=False,
                         extra=[("index >= n", (lambda f: lambda l, c, q, n: getattr(l, "ocb_" + f)(c, q, n, n, *ST))(_name), None, ARG,
                                 "strain: bad arguments")]))


class Contexts:
    """Contexts in three states: no images ("empty"), images without prepare ("unprepared"), images and every prepare ("ready"),
    each single-device and as a one-member group."""

    def __init__(self, lib):
        self.lib = lib
        self.ref, self.tar = synth.speckle_pair_2d(W, H)
        self.ref3, self.tar3 = synth.speckle_pair_3d(D, D, D)
        self.ctx = {}
        for group in (False, True):
            for state in ("empty", "unprepared", "ready"):
                c = lib.ocb_create_multi((ctypes.c_int * 1)(0), 1) if group else lib.ocb_create(0)
                assert c
                if state != "empty":
                    assert lib.ocb_set_images_2d(c, vp(self.ref), vp(self.tar), W, H, 0) == OK
                    assert lib.ocb_set_images_3d(c, vp(self.ref3), vp(self.tar3), D, D, D) == OK
                if state == "ready":
                    assert lib.ocb_icgn2d_prepare(c) == OK and lib.ocb_nr2d_prepare(c) == OK and lib.ocb_icgn3d_prepare(c) == OK
                self.ctx[group, state] = c

    def close(self):
        for c in self.ctx.values():
            self.lib.ocb_destroy(c)


@pytest.fixture(scope="module")
def ctxs():
    c = Contexts(_capi.load())
    yield c
    c.close()


def last_error(lib, ctx):
    return lib.ocb_last_error(ctx).decode()


def check_host(lib, ctx, call, queue, n, code, msg):
    """call(q, n) on a host queue returns code with msg and changes neither the queue nor the launch count"""
    before = lib.ocb_launch_count(ctx) if ctx else 0
    q0 = queue.copy()
    rc = call(vp(queue) if queue is not None else None, n)
    assert rc == code, (rc, last_error(lib, ctx))
    if code != OK:
        assert last_error(lib, ctx) == msg
    if ctx:
        assert lib.ocb_launch_count(ctx) == before
    assert np.array_equal(queue.view(np.uint32), q0.view(np.uint32))


def check_dev(lib, ctx, call, queue, n, code, msg):
    """the same for a device queue (n may exceed the buffer: a refused call does not touch it)"""
    t = torch.from_numpy(queue).cuda()
    torch.cuda.synchronize()
    before = lib.ocb_launch_count(ctx) if ctx else 0
    rc = call(ctypes.c_void_p(t.data_ptr()), n)
    assert rc == code, (rc, last_error(lib, ctx))
    if code != OK:
        assert last_error(lib, ctx) == msg
    if ctx:
        assert lib.ocb_launch_count(ctx) == before
    torch.cuda.synchronize()
    assert np.array_equal(t.cpu().numpy().view(np.uint32), queue.view(np.uint32))


def refusals(e, dev):
    """(state, radius, n, null queue, code, message) of every refusal of e's host (dev False) or device-pointer form, on a
    single-device context"""
    what = e.what_dev
    out = [("ready", e.r, 5, True, ARG, "%s: bad arguments" % (what if dev else e.what_host))]
    if e.radius_refused:
        out.append(("ready", 0, 5, False, ARG, "%s: bad arguments" % what))
    if e.dim:
        out.append(("empty", e.r, 5, False, STATE, "%s: images not set" % what))
    if e.prepared:
        out.append(("unprepared", e.r, 5, False, STATE, "%s: prepare() has not been called since setImages()" % what))
    out += [("ready", r, 5, False, UNSUP, m) for r, m in e.unsupported]
    return out


@pytest.mark.parametrize("e", ENTRIES, ids=lambda e: e.name)
def test_host_refusals(ctxs, e):
    lib = ctxs.lib
    # a null context: the message goes to the process-wide slot
    check_host(lib, None, lambda q, n: e.host(lib, None, q, n, e.r), e.queue(e.r), 5, ARG, "%s: bad arguments" % e.what_host)
    for group in (False, True):
        member = "device 0: " if group and e.sharded else ""  # refused by the member that runs the shard
        for state, r, n, null, code, msg in refusals(e, False):
            ctx = ctxs.ctx[group, state]
            check_host(lib, ctx, lambda q, n_: e.host(lib, ctx, None if null else q, n_, r), e.queue(r), n, code, (msg if null else member + msg))
        ctx = ctxs.ctx[group, "ready"]
        for _, host, _, code, msg in e.extra:
            check_host(lib, ctx, lambda q, n: host(lib, ctx, q, n), e.queue(e.r), len(e.queue(e.r)), code, member + msg)
        check_host(lib, ctx, lambda q, n: e.host(lib, ctx, q, n, e.r), e.queue(e.r), 0, OK, "")
        check_host(lib, ctx, lambda q, n: e.host(lib, ctx, None, n, e.r), e.queue(e.r), 0, OK, "")


@pytest.mark.parametrize("e", [e for e in ENTRIES if e.dev], ids=lambda e: e.name)
def test_dev_refusals(ctxs, e):
    lib = ctxs.lib
    check_dev(lib, None, lambda q, n: e.dev(lib, None, q, n, e.r), e.queue(e.r), 5, ARG, "%s: bad arguments" % e.what_dev)
    for state, r, n, null, code, msg in refusals(e, True):
        ctx = ctxs.ctx[False, state]
        check_dev(lib, ctx, lambda q, n_: e.dev(lib, ctx, None if null else q, n_, r), e.queue(r), n, code, msg)
    ctx = ctxs.ctx[False, "ready"]
    for _, _, dev, code, msg in e.extra:
        if dev:
            check_dev(lib, ctx, lambda q, n: dev(lib, ctx, q, n), e.queue(e.r), len(e.queue(e.r)), code, msg)
    if e.cap:
        check_dev(lib, ctx, lambda q, n: e.dev(lib, ctx, q, n, e.r), e.queue(e.r), 1 << 31, ARG, "%s: too many POIs in one call" % e.what_dev)
    check_dev(lib, ctx, lambda q, n: e.dev(lib, ctx, q, n, e.r), e.queue(e.r), 0, OK, "")
    # every device-pointer form is refused on a group context, first of all
    msg = "%s_dev: device-pointer / stream entry points need a single-device context (ocb_member)" % e.what_dev
    for state in ("empty", "ready"):
        g = ctxs.ctx[True, state]
        check_dev(lib, g, lambda q, n: e.dev(lib, g, q, n, 0), e.queue(e.r), 5, ARG, msg)


@pytest.mark.parametrize("e", ENTRIES, ids=lambda e: e.name)
def test_accepted_launches(ctxs, e):
    lib = ctxs.lib
    forms = [(False, e.host), (True, e.host)] + ([(False, e.dev)] if e.dev else [])
    for i, (group, call) in enumerate(forms):
        ctx = ctxs.ctx[group, "ready"]
        q = e.queue(e.r)
        before = lib.ocb_launch_count(ctx)
        if i == 2:
            t = torch.from_numpy(q).cuda()
            torch.cuda.synchronize()
            assert call(lib, ctx, ctypes.c_void_p(t.data_ptr()), len(q), e.r) == OK, last_error(lib, ctx)
            assert lib.ocb_sync(ctx) == OK
        else:
            assert call(lib, ctx, vp(q), len(q), e.r) == OK, last_error(lib, ctx)
        assert lib.ocb_launch_count(ctx) - before == e.launches, (group, i)


def _calibs(lib, ctx):
    intr = np.array([120, 120, 0, W / 2, H / 2] + [0] * 8, np.float32)
    out = []
    for _ in range(2):
        h = ctypes.c_void_p()
        assert lib.ocb_calib_prepare(ctx, vp(intr), H, W, 0.001, 5, ctypes.byref(h)) == OK, last_error(lib, ctx)
        out.append(h)
    p1 = np.array([120, 0, W / 2, 0, 0, 120, H / 2, 0, 0, 0, 1, 0], np.float32)
    p2 = p1.copy()
    p2[3] = -120 * 50.0
    return intr, out, p1, p2


def test_stereo_reconstruct(ctxs):
    lib = ctxs.lib
    pts = np.array([[40, 30], [50, 44], [60, 20], [30, 60]], np.float32)
    for group in (False, True):
        ctx = ctxs.ctx[group, "ready"]
        intr, (c1, c2), p1, p2 = _calibs(lib, ctx)
        try:
            def host(c, a, b, x, n, cal=c1):
                return lib.ocb_stereo_reconstruct(c, cal, vp(intr), vp(p1), c2, vp(intr), vp(p2), a, b, x, n)

            def dev(c, a, b, x, n, cal=c1):
                return lib.ocb_stereo_reconstruct_dev(c, cal, vp(intr), vp(p1), c2, vp(intr), vp(p2), a, b, x, n)

            a, b, x = pts.copy(), pts.copy(), np.zeros((4, 3), np.float32)
            snap = [v.copy() for v in (a, b, x)]
            cases = [(None, host, (vp(a), vp(b), vp(x), 4), ARG, "null context"),
                     (ctx, lambda c, *r: host(c, *r, cal=None), (vp(a), vp(b), vp(x), 4), ARG, "stereo_reconstruct: null calibration handle"),
                     (ctx, host, (None, vp(b), vp(x), 4), ARG, "stereo_reconstruct: bad arguments")]
            for c, call, args, code, msg in cases:
                before = lib.ocb_launch_count(ctx)
                assert call(c, *args) == code
                assert last_error(lib, c) == msg
                assert lib.ocb_launch_count(ctx) == before
                assert all(np.array_equal(v, s) for v, s in zip((a, b, x), snap))
            before = lib.ocb_launch_count(ctx)
            assert host(ctx, None, None, None, 0) == OK and lib.ocb_launch_count(ctx) == before
            assert host(ctx, vp(a), vp(b), vp(x), 4) == OK and lib.ocb_launch_count(ctx) - before == 1
            d = [torch.from_numpy(v).cuda() for v in (pts.copy(), pts.copy(), np.zeros((4, 3), np.float32))]
            torch.cuda.synchronize()
            ptrs = [ctypes.c_void_p(t.data_ptr()) for t in d]
            before = lib.ocb_launch_count(ctx)
            if group:
                assert dev(ctx, *ptrs, 4) == ARG
                assert last_error(lib, ctx) == ("stereo_reconstruct_dev: device-pointer / stream entry points need a single-device context "
                                                "(ocb_member)")
                assert lib.ocb_launch_count(ctx) == before
            else:
                assert dev(ctx, *ptrs, 0) == OK and lib.ocb_launch_count(ctx) == before
                assert dev(ctx, *ptrs, 4) == OK and lib.ocb_sync(ctx) == OK and lib.ocb_launch_count(ctx) - before == 1
        finally:
            lib.ocb_calib_destroy(c1)
            lib.ocb_calib_destroy(c2)
