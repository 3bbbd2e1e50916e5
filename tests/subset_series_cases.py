"""Shared cases of the IC-GN, IC-LM and NR2D1 image-series tests: the synthetic series; each method's pair call, series calls and
raw C series calls; the witness loops of pair calls the series calls must equal byte for byte; and the checks the three test
files run, each with its own methods."""
import ctypes

import numpy as np

import opencorr_b200 as ob
from opencorr_b200 import _capi, synth
from util import assert_same, compare_2d

CONV, STOP = 0.001, 10
DAMPING = (100.0, 0.1, 10.0)  # ocb_iclm2d's defaults (DampingParameter, src/oc_iclm.h)
OTHER_DAMPING = (30.0, 0.3, 4.0)


def render_series(width, height, n_frames, second_order=False, vy_step=0.0, jump=None, rho=2.0, seed=synth.REF_SEED):
    """ref and n_frames targets: the speckles of synth.speckle_pair_2d moved by (f + 1) / n_frames of its displacement field,
    so the last frame carries the full field.  vy_step adds a vertical stretch about the image centre of (f + 1) vy_step in
    frame f.  jump = (k, x0, y0, x1, y1, du, dv): from frame k on, the speckles whose reference centre lies in the box move by
    (du, dv) more."""
    rng = np.random.default_rng(seed)
    n = int(0.5 * width * height / (np.pi * rho * rho))
    cx = rng.uniform(-8, width + 8, n)
    cy = rng.uniform(-8, height + 8, n)
    amp = rng.uniform(0.4, 1.0, n)
    u, v = synth.displacement_2d(cx, cy, width, height, second_order)

    def image(f):  # f = -1: the reference
        s = (f + 1) / n_frames
        y, x = cy + s * v + (f + 1) * vy_step * (cy - height / 2), cx + s * u
        if jump is not None and f >= jump[0]:
            k, x0, y0, x1, y1, du, dv = jump
            inside = (cx >= x0) & (cx < x1) & (cy >= y0) & (cy < y1)
            y, x = y + np.where(inside, dv, 0.0), x + np.where(inside, du, 0.0)
        im = synth._render((height, width), np.stack([y, x], 1), amp, rho)
        return np.round(np.clip(synth.BACKGROUND + (255.0 - synth.BACKGROUND) * im, 0, 255)).astype(np.float32)

    return image(-1), np.stack([image(f) for f in range(n_frames)])


def true_displacement(xy, shape, n_frames, f, second_order=False, vy_step=0.0):
    """(u, v) of frame f of render_series at the reference points xy"""
    h, w = shape
    u, v = synth.displacement_2d(xy[:, 0], xy[:, 1], w, h, second_order)
    s = (f + 1) / n_frames
    return s * u, s * v + (f + 1) * vy_step * (xy[:, 1] - h / 2)


def fftcc_seeds(eng, ref, tar, xy, r):
    q = ob.make_poi2d(xy)
    eng.set_images_2d(ref, tar)
    eng.fftcc2d(q, r, r)
    return q


class Method:
    """A 2D subset method: "icgn" (IC-GN), "iclm" (IC-LM with damping), both of shape-function order 1 or 2, or "nr" (NR2D1)."""

    def __init__(self, kind, order=1, damping=DAMPING):
        self.kind, self.order, self.damping = kind, order, damping
        self.name = {"icgn": "icgn2d", "iclm": "iclm2d", "nr": "nr2d1"}[kind]  # of the engine's and the C ABI's series calls

    def __repr__(self):
        return "NR2D1" if self.kind == "nr" else "%s2D%d" % (self.kind.upper(), self.order)

    def pair(self, eng, q, r, stop=STOP, prepare=True):
        """prepare() (unless prepare is False) and compute(queue) on the pair set on eng"""
        if prepare:
            (eng.nr2d_prepare if self.kind == "nr" else eng.icgn2d_prepare)()
        if self.kind == "icgn":
            (eng.icgn2d1 if self.order == 1 else eng.icgn2d2)(q, r, r, CONV, stop)
        elif self.kind == "iclm":
            eng.iclm2d(self.order, q, r, r, CONV, stop, self.damping)
        else:
            eng.nr2d1(q, r, r, CONV, stop)

    def oracle(self, o, q, r, stop=STOP, exact=False):
        if self.kind == "icgn":
            (o.icgn2d1 if self.order == 1 else o.icgn2d2)(q, r, r, CONV, stop, exact=exact)
        elif self.kind == "iclm":
            o.iclm2d(self.order, q, r, r, CONV, stop, self.damping, exact=exact)
        else:
            o.nr2d1(q, r, r, CONV, stop, exact=exact)

    def _series_call(self, eng, suffix, *args):
        """eng.<name><suffix>([order,] *args[, damping=damping])"""
        lead = () if self.kind == "nr" else (self.order,)
        kw = dict(damping=self.damping) if self.kind == "iclm" else {}
        return getattr(eng, self.name + suffix)(*lead, *args, **kw)

    def series(self, eng, seeds, r, stop=STOP):
        return self._series_call(eng, "_series", seeds, r, r, CONV, stop)

    def series_reseed(self, eng, seeds, r, fr, zncc_min, stop=STOP):
        return self._series_call(eng, "_series_reseed", seeds, r, r, CONV, stop, fr, fr, zncc_min)

    def series_dev(self, eng, d_seeds, d_out, n, r):
        self._series_call(eng, "_series_dev", d_seeds, d_out, n, r, r, CONV, STOP)

    def series_reseed_dev(self, eng, d_seeds, d_out, n, r, fr, zncc_min):
        return self._series_call(eng, "_series_reseed_dev", d_seeds, d_out, n, r, r, CONV, STOP, fr, fr, zncc_min)

    def c_series(self, lib, ctx, suffix, order, seeds, out, n, r, *reseed):
        """The C ABI's ocb_<name>_series<suffix>(ctx, [order,] seeds, out, n, r, r, CONV, STOP, [damping,] *reseed) on raw
        pointers; order None: the method's."""
        lead = () if self.kind == "nr" else (self.order if order is None else order,)
        damping = tuple(self.damping) if self.kind == "iclm" else ()
        return getattr(lib, "ocb_%s_series%s" % (self.name, suffix))(ctx, *lead, seeds, out, n, r, r, CONV, STOP, *damping, *reseed)


def pair_loop(eng, method, ref, tars, seeds, r, stop=STOP):
    """for f: set_images_2d(ref, tars[f]); prepare(); compute(q), one queue carried from frame to frame"""
    q = seeds.copy()
    out = []
    for f in range(len(tars)):
        eng.set_images_2d(ref, tars[f])
        method.pair(eng, q, r, stop)
        out.append(q.copy())
    return np.stack(out)


def reseed_pair_loop(eng, method, ref, tars, seeds, r, fr, zncc_min):
    """pair_loop that re-seeds the POIs lost in frame f from their seeds at their latest good translation, then runs FFT-CC and
    the method on them against frame f (the rules of the ocb_*2d*_series_reseed calls)"""
    q = seeds.copy()
    anchor = seeds[:, [2, 8]].copy()
    out, counts = [], []
    for f in range(len(tars)):
        eng.set_images_2d(ref, tars[f])
        method.pair(eng, q, r)
        if f > 0:
            good = out[-1][:, 16] >= zncc_min
            anchor[good] = out[-1][good][:, [2, 8]]
        lost = np.nonzero(~(q[:, 16] >= zncc_min))[0]
        if len(lost):
            sub = np.zeros((len(lost), ob.POI2D_FLOATS), np.float32)
            for c in (0, 1, 23, 24):
                sub[:, c] = seeds[lost, c]
            sub[:, [2, 8]] = anchor[lost]
            eng.fftcc2d(sub, fr, fr)
            method.pair(eng, sub, r)
            q[lost] = sub
        out.append(q.copy())
        counts.append(len(lost))
    return np.stack(out), np.array(counts, np.int64)


def occlude(tars, k, box):
    """Cover box = (x0, y0, x1, y1) of frame k with speckles from elsewhere in the same frame (decorrelated from the subsets)."""
    x0, y0, x1, y1 = box
    out = tars.copy()
    out[k, y0:y1, x0:x1] = np.roll(tars[k], (tars.shape[1] // 2, tars.shape[2] // 2), (0, 1))[y0:y1, x0:x1]
    return out


def short_grid():
    return synth.grid_2d(60, 55, 6, 5, 48, 41)  # 30 POIs


def long_grid(r):
    return synth.grid_2d(r + 4, r + 4, 112, 70, 3, 4)  # 7840 POIs: more than the resident slots at these radii


# ---- the checks the test files run, each with its own methods ----------------------------------------------------------------

def check_equals_pair_loop(eng, method, ref, tars, xy, r, label, fft_r=None):
    """seeded by FFT-CC of radius fft_r (None: min(r, 16))"""
    seeds = fftcc_seeds(eng, ref, tars[0], xy, fft_r or min(r, 16))
    for n_frames in (1, len(tars)):
        expect = pair_loop(eng, method, ref, tars[:n_frames], seeds, r)
        eng.set_series_2d(ref, tars[:n_frames])
        got = method.series(eng, seeds, r)
        assert_same(got, expect, "%s %s F %d" % (method, label, n_frames))
        assert (got[-1][:, 16] >= 0).mean() > 0.8


def check_sentinels(eng, method, ref, tars, r):
    """Black frames, POIs at and past the image edge, NaN and negative seeds and the iteration limit give, frame after frame,
    exactly the codes and records of the pair loop."""
    h, w = ref.shape
    tars = tars.copy()
    tars[2:, 150:, :120] = 0.0  # a black background from frame 2 on under the lower-left POIs
    xy = np.array([[100, 100], [200, 150], [w - r - 1, 100], [w - 40, 200], [150, 160], [300, 250], [120, 260], [60, 220], [r, r],
                   [80, 250]], np.float32)
    seeds = fftcc_seeds(eng, ref, tars[0], xy, 16)
    seeds[2, 2] = 2.0          # the subset leaves the image as the series moves right
    seeds[3, 2] = w + 5.0      # |u| >= width: the guard rejects it
    seeds[4, 16] = -1.0        # arrives negative
    seeds[5, 2] += 7.5         # far from the optimum
    seeds[6, 8] = np.nan       # NaN guess
    for stop in (STOP, 2):
        expect = pair_loop(eng, method, ref, tars, seeds, r, stop)
        eng.set_series_2d(ref, tars)
        got = method.series(eng, seeds, r, stop)
        assert_same(got, expect, "%s stop %g" % (method, stop))
        assert (got[:, 3:5, 16] < 0).all() and (got[:, 6, 16] < 0).all()
        if stop == 2:
            assert (got[:, :, 16] == -4).any()


def check_chunks(eng, method, ref, tars, r):
    seeds = fftcc_seeds(eng, ref, tars[0], short_grid(), 16)
    eng.set_series_2d(ref, tars)
    whole = method.series(eng, seeds, r)
    eng.set_series_2d(ref, tars[:2])
    a = method.series(eng, seeds, r)
    eng.set_series_2d(ref, tars[2:])
    b = method.series(eng, a[-1].copy(), r)
    assert_same(np.concatenate([a, b]), whole, "%s in two chunks" % method)


def check_pair_state_undisturbed(eng, method, ref, tars, r, series_method=None):
    """method's pair call returns the same records after series calls of series_method (None: method) on another stack"""
    series_method = series_method or method
    seeds = fftcc_seeds(eng, ref, tars[-1], short_grid(), 16)
    before = seeds.copy()
    method.pair(eng, before, r)
    eng.set_series_2d(ref[::-1].copy(), tars[:, ::-1].copy())
    series_method.series(eng, seeds, r)
    series_method.series_reseed(eng, seeds, r, 16, 0.99)
    after = seeds.copy()
    method.pair(eng, after, r, prepare=False)  # the pair (ref, tars[-1]) is still set and prepared
    assert_same(after, before, "%s pair call after series calls" % method)


def check_dev_matches_host(eng, method, ref, tars, r):
    import torch
    xy = short_grid()
    seeds = fftcc_seeds(eng, ref, tars[0], xy, 16)
    seeds[[1, 8, 20], 16] = -1.0  # re-seeded in frame 0
    eng.set_series_2d(ref, tars)
    host = method.series(eng, seeds, r)
    host_re, host_counts = method.series_reseed(eng, seeds, r, 16, 0.99)
    assert host_counts.sum() > 0
    d_ref, d_tars, d_seeds = (torch.from_numpy(a).cuda() for a in (ref, tars, seeds))
    d_out = torch.empty((len(tars), len(seeds), 25), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    eng.set_series_2d_dev(d_ref.data_ptr(), d_tars.data_ptr(), len(tars), ref.shape[1], ref.shape[0])
    method.series_dev(eng, d_seeds.data_ptr(), d_out.data_ptr(), len(seeds), r)
    eng.sync()
    assert_same(d_out.cpu().numpy(), host, "%s device-pointer variant" % method)
    counts = method.series_reseed_dev(eng, d_seeds.data_ptr(), d_out.data_ptr(), len(seeds), r, 16, 0.99)
    assert_same(d_out.cpu().numpy(), host_re, "%s re-seeding device-pointer variant" % method)
    assert np.array_equal(counts, host_counts)
    assert_same(d_seeds.cpu().numpy(), seeds, "device seeds changed")


def check_group(method, ref, tars, r):
    single = ob.Engine(0)
    seeds = fftcc_seeds(single, ref, tars[0], short_grid(), 16)
    seeds[[1, 8, 20], 16] = -1.0  # re-seeded in frame 0
    single.set_series_2d(ref, tars)
    expect = method.series(single, seeds, r)
    expect_re, expect_counts = method.series_reseed(single, seeds, r, 16, 0.99)
    group = ob.Engine([0, 1])
    group.set_series_2d(ref, tars)
    assert_same(method.series(group, seeds, r), expect, "%s group context" % method)
    got_re, counts = method.series_reseed(group, seeds, r, 16, 0.99)
    assert_same(got_re, expect_re, "%s re-seeding, group context" % method)
    assert np.array_equal(counts, expect_counts)
    group.close()
    single.close()


def check_nothing_lost(eng, method, ref, tars, xy, r):
    seeds = fftcc_seeds(eng, ref, tars[0], xy, 16)
    seeds[::7, 16] = -1.0  # failed seeds stay failed: -10 is below every code
    eng.set_series_2d(ref, tars)
    expect = method.series(eng, seeds, r)
    got, counts = method.series_reseed(eng, seeds, r, 16, -10.0)
    assert_same(got, expect, "%s r %d, nothing lost" % (method, r))
    assert counts.shape == (len(tars),) and (counts == 0).all()


def lossy_series(width=387, height=320, n_frames=6):
    """(ref, tars, xy, [(frame, POIs occluded in it)]): frame 2 occludes a block of POIs.  check_reseed_equals_pair_loop fails
    three seeds (index 3, 17, 40)."""
    ref, tars = render_series(width, height, n_frames)
    xy = synth.grid_2d(50, 50, 8, 6, 40, 40)
    sel = (xy[:, 0] >= 130) & (xy[:, 0] < 210) & (xy[:, 1] >= 130) & (xy[:, 1] < 210)
    u, v = true_displacement(np.array([[150.0, 150.0]]), ref.shape, n_frames, 2)
    x0, y0 = xy[sel].min(0) + (u[0], v[0])
    x1, y1 = xy[sel].max(0) + (u[0], v[0])
    tars = occlude(tars, 2, (int(x0) - 24, int(y0) - 24, int(x1) + 25, int(y1) + 25))
    return ref, tars, xy, [(2, sel)]


def check_reseed_equals_pair_loop(eng, method, lossy, r, fr):
    ref, tars, xy, occluded = lossy
    seeds = fftcc_seeds(eng, ref, tars[0], xy, 16)
    seeds[[3, 17, 40], 16] = -1.0
    for n_frames in (1, len(tars)):
        expect, expect_counts = reseed_pair_loop(eng, method, ref, tars[:n_frames], seeds, r, fr, 0.9)
        eng.set_series_2d(ref, tars[:n_frames])
        got, counts = method.series_reseed(eng, seeds, r, fr, 0.9)
        assert_same(got, expect, "%s fft r %d F %d" % (method, fr, n_frames))
        assert np.array_equal(counts, expect_counts), (counts, expect_counts)
        assert counts[0] >= 3
        if n_frames == len(tars):
            for k, sel in occluded:  # the last frame is re-seeded too
                assert counts[k] >= sel.sum(), (k, counts)


def check_oracle_and_ground_truth(eng, method, ref, tars, r, second_order=False, vy_step=0.0, bound=0.05, fft_r=16, every_frame=False):
    """The last frame (every_frame: every frame, against the oracle's exact mode) matches the float64 oracle run from the GPU's
    records of the frame before, and the last frame the ground truth.  Seeded by FFT-CC of radius fft_r."""
    from oracle.oracle import Oracle2D
    xy = synth.grid_2d(40, 40, 12, 10, 27, 24)
    seeds = fftcc_seeds(eng, ref, tars[0], xy, fft_r)
    eng.set_series_2d(ref, tars)
    got = method.series(eng, seeds, r)
    last = len(tars) - 1
    for f in range(len(tars)) if every_frame else [last]:
        q = (seeds if f == 0 else got[f - 1]).copy()  # from the same records as the GPU's
        method.oracle(Oracle2D(ref, tars[f]), q, r, exact=every_frame)
        compare_2d(got[f], q, "%s frame %d" % (method, f), order=method.order)
    ok = got[last][:, 16] >= 0
    assert ok.mean() > 0.95
    u, v = true_displacement(xy, ref.shape, len(tars), last, second_order, vy_step)
    assert np.abs(got[last][ok, 2] - u[ok]).max() < bound and np.abs(got[last][ok, 8] - v[ok]).max() < bound


def check_errors_leave_out_untouched(method):
    """Refused series calls of the method, plain and re-seeding, with host and device pointers, leave out and the re-seed counts
    untouched; refused set_series_2d calls set nothing; the engine stays usable."""
    eng = ob.Engine(0)
    lib, ctx = eng._lib, eng._ctx
    ref, tars = render_series(96, 80, 2)
    seeds = ob.make_poi2d(synth.grid_2d(40, 40, 2, 2, 10, 10))
    n = len(seeds)
    out = np.full((2, n, 25), 7.0, np.float32)
    counts = np.full(2, 99, np.uint64)
    vp = lambda a: None if a is None else ctypes.c_void_p(a.ctypes.data)

    def call(order=None, r=8, s=seeds, o=out, count=n):
        return method.c_series(lib, ctx, "", order, vp(s), vp(o), count, r)

    def reseed(order=None, r=8, fr=8, zmin=0.5, s=seeds, o=out, count=n):
        return method.c_series(lib, ctx, "_reseed", order, vp(s), vp(o), count, r, fr, fr, zmin, vp(counts))

    assert call() == _capi.OCB_ERR_STATE and reseed() == _capi.OCB_ERR_STATE
    assert lib.ocb_set_series_2d(ctx, vp(ref), vp(tars), 0, 96, 80) == _capi.OCB_ERR_ARG
    assert lib.ocb_set_series_2d(ctx, vp(ref), None, 2, 96, 80) == _capi.OCB_ERR_ARG
    assert call() == _capi.OCB_ERR_STATE and reseed() == _capi.OCB_ERR_STATE  # the refused calls set nothing
    assert lib.ocb_set_series_2d(ctx, vp(ref), vp(tars), 2, 96, 80) == _capi.OCB_OK
    bad = [dict(r=0), dict(s=None), dict(o=None), dict(count=1 << 40)] + ([] if method.kind == "nr" else [dict(order=0), dict(order=3)])
    for kw in bad:
        assert call(**kw) == _capi.OCB_ERR_ARG and reseed(**kw) == _capi.OCB_ERR_ARG, kw
    too_large = "nr2d1: subset radius" if method.kind == "nr" else "exceeds the shared-memory design limit"
    for c in (call, reseed):
        assert c(r=200) == _capi.OCB_ERR_UNSUPPORTED and too_large in _capi.last_error(ctx)
    assert reseed(zmin=float("nan")) == _capi.OCB_ERR_ARG
    assert reseed(fr=0) == _capi.OCB_ERR_ARG
    assert reseed(fr=37) == _capi.OCB_ERR_UNSUPPORTED and "prime factor > 31" in _capi.last_error(ctx)
    assert method.c_series(lib, ctx, "_dev", None, None, None, 5, 8) == _capi.OCB_ERR_ARG
    assert method.c_series(lib, ctx, "_reseed_dev", None, None, None, 5, 8, 8, 8, 0.5, vp(counts)) == _capi.OCB_ERR_ARG
    assert (out == 7.0).all() and (counts == 99).all()
    assert call() == _capi.OCB_OK and not (out == 7.0).all()  # the engine is still usable
    out[:] = 7.0
    assert reseed() == _capi.OCB_OK and not (out == 7.0).all() and (counts < 99).all()
    eng.close()
