"""GPU: FFTCC2D on all three kernels and both window-load paths, at every window size and image edge, against two float64
witnesses.

ocb::fftcc2d_plan (opencorr_b200/csrc/ocb_kernels.h) sends r = 16 to fftcc2d_w32.cu (one warp per POI; the windows arrive as two
TMA boxes when POI and guess are whole pixels and the pitch allows it, by a per-lane gather otherwise), square windows of
2^a 3^b 5^c <= 64 points to fftcc2d_reg.cu (128 / N POIs per CTA) and everything else whose prime factors are <= 31 to the
shared-memory Stockham kernel of fftcc.cu; test_fftcc2d_plan_host.py checks on the CPU that every case below lands on the kernel
it names, that the generic cases reach every radix and the register cases every size and every POIs-per-CTA count.

Witnesses: (a) `witness` below, plain numpy in float64 (np.fft), which shares no code with the oracle; (b) Oracle2D.fftcc2d with
exact=True.  Pass rule (`_check`): u, v, u0, v0 are bit-identical to both witnesses on every POI whose float64 peak stands more
than 1e-5 (in ZNCC units) above the runner-up; a POI with a smaller gap may return any maximum within 1e-5 of the peak; ZNCC is
within 1e-5 of both; every other field, and every field of a skipped POI, keeps its bytes.  Each case prints one line: kernel, n,
compared, max |dZNCC|, non-decisive POIs."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

import opencorr_b200 as ob
from opencorr_b200 import _capi, synth
from oracle.oracle import Oracle2D

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
W, H = 640, 600
INT_COLS = [2, 8, 14, 15]
OTHER_COLS = np.delete(np.arange(25), INT_COLS + [16])
GAP = 1e-5

# ------------------------------------------------------------------------------------------------ the cases, by kernel
REG_R = (4, 5, 6, 8, 9, 10, 12, 15, 18, 20, 24, 25, 27, 30, 32)  # fftcc2d_reg.cu: every size it has
GENERIC_SQUARE = (7, 11, 13, 14, 17, 19, 21, 22, 23, 26, 29, 31, 33, 35, 36, 40, 45, 58)  # every odd radix 7 ... 31; > 64 points
GENERIC_NONSQUARE = ((12, 10), (16, 15), (15, 16), (31, 4), (4, 31), (100, 30), (9, 50))
FORCED_GENERIC = (16, 20, 15, 32)  # OCB_FFTCC2D_GENERIC against the kernel the window takes by default
EDGE_R = ((16, 16), (10, 10), (7, 7), (12, 10))  # W32, REG, GENERIC, GENERIC non-square
TIE_R = ((8, False), (16, False), (32, False), (10, False), (16, True))  # (r, forced generic)
REJECTED = ((59, 59, "prime factor"), (37, 37, "prime factor"), (60, 60, "shared memory"))  # at an H100's 227 KB opt-in limit


def sweep_n(rx, ry):
    """Queue length of a sweep case, 40 ... 64: never a multiple of the register kernel's POIs per CTA (128 // N), so that its
    last batch is partly filled."""
    n = 41 + (3 * rx + ry) % 20
    pp = 128 // (2 * rx)
    while pp > 1 and n % pp == 0:
        n += 1
    return n


SWEEP = [(r, r) for r in REG_R] + [(16, 16)] + [(r, r) for r in GENERIC_SQUARE] + list(GENERIC_NONSQUARE)
# (rx, ry, forced generic, kernel, queue length) of every case: what test_fftcc2d_plan_host.py checks against the plan
PLAN_CASES = ([(r, r, 0, "REG", sweep_n(r, r)) for r in REG_R] + [(16, 16, 0, "W32", sweep_n(16, 16))]
              + [(r, r, 0, "GENERIC", sweep_n(r, r)) for r in GENERIC_SQUARE]
              + [(rx, ry, 0, "GENERIC", sweep_n(rx, ry)) for rx, ry in GENERIC_NONSQUARE]
              + [(r, r, 1, "GENERIC", sweep_n(r, r)) for r in FORCED_GENERIC]
              + [(rx, ry, 0, k, 24) for (rx, ry), k in zip(EDGE_R, ("W32", "REG", "GENERIC", "GENERIC"))]
              + [(r, r, int(g), "GENERIC" if g else ("W32" if r == 16 else "REG"), 12) for r, g in TIE_R]
              + [(rx, ry, 0, "rejected (%s)" % why, 3) for rx, ry, why in REJECTED])


def build_plan_tool(out_dir):
    """Compiles tests/native/fftcc2d_plan_host_test.cpp (ocb::fftcc2d_plan of ocb_kernels.h, host only) into out_dir."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    exe = os.path.join(out_dir, "fftcc2d_plan_host_test")
    cmd = [nvcc, "-x", "cu", "-std=c++17", "-O1", "-Wno-deprecated-gpu-targets", "-I", os.path.join(ROOT, "opencorr_b200", "csrc"),
           "-o", exe, os.path.join(ROOT, "tests", "native", "fftcc2d_plan_host_test.cpp")]
    if os.path.exists("/usr/bin/g++"):
        cmd[1:1] = ["-ccbin", "/usr/bin/g++"]
    build = subprocess.run(cmd, capture_output=True, text=True)
    assert build.returncode == 0, "nvcc failed:\n" + build.stdout + build.stderr
    return exe


def run_plan_tool(exe, *args, cases=None):
    text = "".join("%d %d %d %d\n" % (rx, ry, g, n) for rx, ry, g, _, n in cases) if cases else None
    return subprocess.run([exe] + [str(a) for a in args], input=text, capture_output=True, text=True, timeout=60)


# ------------------------------------------------------------------------------------------------ witness (a)
def witness(ref, tar, q, rx, ry):
    """FFTCC2D::compute of the reference (src/oc_fftcc.cpp:177-275) in float64 on float32 inputs.  Returns the records, which
    POIs were computed, each one's gap between the peak and the runner-up (ZNCC units), and each one's (u, v) candidates: every
    maximum within GAP of the peak."""
    h, w = ref.shape
    f32 = np.float32
    sw, sh, m = 2 * rx, 2 * ry, 4 * rx * ry
    out, computed, gap, cands = q.copy(), np.zeros(len(q), bool), np.full(len(q), np.inf), [None] * len(q)
    cx, cy = np.arange(sw).astype(f32), np.arange(sh).astype(f32)
    for i, p in enumerate(q):
        px, py, u0, v0 = p[0], p[1], p[2], p[8]
        if not np.isfinite([px, py, u0, v0]).all():  # NaN, and (int)inf, leave the POI untouched
            continue
        with np.errstate(over="ignore"):
            tx, ty = px + u0, py + v0  # float32 sums
        if not (rx <= int(px) < w - rx and ry <= int(py) < h - ry and np.isfinite([tx, ty]).all()
                and rx <= int(tx) < w - rx and ry <= int(ty) < h - ry):
            continue
        # float32 coordinate arithmetic px + c - rx, then + u0, then truncation toward zero (:204-219)
        rpx, rpy = (px + cx) - f32(rx), (py + cy) - f32(ry)
        a = ref[np.ix_(rpy.astype(np.int64), rpx.astype(np.int64))].astype(np.float64)
        b = tar[np.ix_((rpy + v0).astype(np.int64), (rpx + u0).astype(np.int64))].astype(np.float64)
        a -= a.mean()
        b -= b.mean()
        corr = np.fft.ifft2(np.conj(np.fft.fft2(a)) * np.fft.fft2(b)).real.ravel() * m  # what the unnormalised inverse returns
        with np.errstate(invalid="ignore", divide="ignore"):
            zncc = corr / (np.sqrt((a * a).sum() * (b * b).sum()) * m)
        idx = int(np.argmax(corr))  # the first maximum in linear order
        near = np.flatnonzero(corr >= corr[idx] - GAP * np.sqrt((a * a).sum() * (b * b).sum()) * m)
        uv = set()
        for j in near:
            du, dv = int(j) % sw, int(j) // sw
            uv.add((f32(du - sw if du > rx else du) + u0, f32(dv - sh if dv > ry else dv) + v0))
        du, dv = idx % sw, idx // sw
        out[i, 2], out[i, 8] = f32(du - sw if du > rx else du) + u0, f32(dv - sh if dv > ry else dv) + v0
        out[i, 14], out[i, 15], out[i, 16] = u0, v0, zncc[idx]
        computed[i], cands[i] = True, uv
        rest = np.delete(zncc, idx)
        gap[i] = zncc[idx] - rest.max() if np.isfinite(zncc[idx]) else 0.0
    return out, computed, gap, cands


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _check(label, got, q, ref, tar, rx, ry, min_decisive=None, oracle_exact=True, expect_computed=None):
    """got: the GPU's records for the queue q.  Applies the pass rule of the module docstring against both witnesses."""
    wa, computed, gap, cands = witness(ref, tar, q, rx, ry)
    wb = Oracle2D(ref, tar).fftcc2d(q.copy(), rx, ry, exact=oracle_exact)
    if expect_computed is not None:
        assert np.array_equal(computed, expect_computed), "%s: computed POIs %s, expected %s" % (label, np.flatnonzero(computed), np.flatnonzero(expect_computed))
    skipped = ~computed
    assert np.array_equal(_bits(got[skipped]), _bits(q[skipped])), "%s: a skipped POI was written: %s" % (
        label, np.flatnonzero(skipped)[(_bits(got[skipped]) != _bits(q[skipped])).any(1)][:10])
    assert np.array_equal(_bits(wb[skipped]), _bits(q[skipped])), "%s: the oracle computed a POI the witness skips" % label
    assert np.array_equal(_bits(got[:, OTHER_COLS]), _bits(q[:, OTHER_COLS])), "%s: a field FFT-CC does not own changed" % label
    dec = computed & (gap > GAP)
    for name, w_ in (("numpy witness", wa), ("oracle", wb)):
        bad = np.flatnonzero(dec & (_bits(got[:, INT_COLS]) != _bits(w_[:, INT_COLS])).any(1))
        assert len(bad) == 0, "%s: u, v, u0, v0 differ from the %s at POIs %s: got %s, expected %s (gap %s)" % (
            label, name, bad[:8], got[bad[:4]][:, INT_COLS].tolist(), w_[bad[:4]][:, INT_COLS].tolist(), gap[bad[:4]])
    for i in np.flatnonzero(computed & ~dec):
        assert (got[i, 2], got[i, 8]) in cands[i], "%s: POI %d returned (%g, %g), not one of the tied maxima %s" % (
            label, i, got[i, 2], got[i, 8], sorted(cands[i]))
        assert got[i, 14] == q[i, 2] and got[i, 15] == q[i, 8], label
    dz = 0.0
    if computed.any():
        dz = max(np.abs(got[computed, 16] - wa[computed, 16]).max(), np.abs(got[computed, 16] - wb[computed, 16]).max())
        assert dz < GAP, "%s: max |dZNCC| = %.3g" % (label, dz)
    nd = int((computed & ~dec).sum())
    if min_decisive is not None:
        assert computed.sum() - nd >= min_decisive * len(q), "%s: only %d of %d POIs are decisive" % (label, computed.sum() - nd, len(q))
    print("%s: n=%d compared=%d max|dZNCC|=%.2e non-decisive=%d" % (label, len(q), computed.sum(), dz, nd))
    return computed


# ------------------------------------------------------------------------------------------------ images and queues
@pytest.fixture(scope="module")
def pair():
    return synth.speckle_pair_2d(W, H)


def sweep_queue(rx, ry, n, seed, w=W, h=H):
    """A third whole-pixel POIs with a zero guess, a third whole-pixel POIs with an integer guess of mixed sign (every residue
    mod 4), a third fractional POIs with a fractional guess; every window inside the image."""
    rng = np.random.default_rng(seed)
    x = rng.uniform(rx + 6, w - rx - 7, n)
    y = rng.uniform(ry + 6, h - ry - 7, n)
    q = ob.make_poi2d(np.stack([x, y], 1))
    kind = np.arange(n) % 3
    whole = kind < 2
    q[whole, 0], q[whole, 1] = np.floor(q[whole, 0]), np.floor(q[whole, 1])
    q[kind == 1, 2] = rng.integers(-3, 5, (kind == 1).sum(), endpoint=True)
    q[kind == 1, 8] = rng.integers(-5, 3, (kind == 1).sum(), endpoint=True)
    q[kind == 2, 2] = rng.uniform(-3, 5, (kind == 2).sum())
    q[kind == 2, 8] = rng.uniform(-5, 3, (kind == 2).sum())
    return q


def _kernel(rx, ry, generic=False):
    if generic:
        return "GENERIC (forced)"
    return "W32" if (rx, ry) == (16, 16) else ("REG" if rx == ry and rx in REG_R else "GENERIC")


def _label(rx, ry, what="", generic=False):
    return "FFTCC2D %s r=(%d,%d)%s" % (_kernel(rx, ry, generic), rx, ry, " " + what if what else "")


def _run(engine, ref, tar, q, rx, ry):
    engine.set_images_2d(ref, tar)
    got = q.copy()
    engine.fftcc2d(got, rx, ry)
    return got


def _mark(q):
    """Distinct values in every field FFT-CC does not read, u0, v0 and ZNCC included: they must survive on a skipped POI."""
    for c in range(3, 25):
        if c != 8:
            q[:, c] = 0.5 + c + 0.001 * np.arange(len(q))
    return q


# ------------------------------------------------------------------------------------------------ window sweep
@pytest.mark.parametrize("rx,ry", SWEEP, ids=["r=(%d,%d)" % r for r in SWEEP])
def test_window_sweep(engine, pair, rx, ry):
    ref, tar = pair
    q = sweep_queue(rx, ry, sweep_n(rx, ry), seed=100 * rx + ry)
    _check(_label(rx, ry), _run(engine, ref, tar, q, rx, ry), q, ref, tar, rx, ry, min_decisive=0.95)


@pytest.mark.parametrize("r", FORCED_GENERIC)
def test_forced_generic_equals_default(engine, pair, monkeypatch, r):
    ref, tar = pair
    q = sweep_queue(r, r, sweep_n(r, r), seed=7 * r)
    a = _run(engine, ref, tar, q, r, r)
    monkeypatch.setenv("OCB_FFTCC2D_GENERIC", "1")
    b = _run(engine, ref, tar, q, r, r)
    _check(_label(r, r, generic=True), b, q, ref, tar, r, r, min_decisive=0.95)
    assert np.array_equal(_bits(a[:, INT_COLS]), _bits(b[:, INT_COLS]))
    assert np.abs(a[:, 16] - b[:, 16]).max() < 2e-6


# ------------------------------------------------------------------------------------------------ w32 load paths
def _both_load_paths(engine, monkeypatch, ref, tar, q, label):
    monkeypatch.delenv("OCB_NO_TMA", raising=False)
    a = _run(engine, ref, tar, q, 16, 16)
    monkeypatch.setenv("OCB_NO_TMA", "1")
    b = _run(engine, ref, tar, q, 16, 16)
    monkeypatch.delenv("OCB_NO_TMA")
    assert np.array_equal(_bits(a), _bits(b)), "%s: TMA boxes and the per-lane gather deliver different windows at POIs %s" % (
        label, np.flatnonzero((_bits(a) != _bits(b)).any(1))[:10])
    return a


@pytest.mark.parametrize("width", [W, 333, 334, 335, 336])
def test_w32_tma_and_gather_agree(engine, pair, monkeypatch, width):
    """The TMA map needs a pitch that is a multiple of 4 floats: widths 333 ... 335 gather every window, 336 and 640 take boxes."""
    ref, tar = (np.ascontiguousarray(a[:300, :width]) for a in pair)
    q = sweep_queue(16, 16, 61, seed=width, w=width, h=300)
    label = _label(16, 16, "width %d" % width)
    _check(label, _both_load_paths(engine, monkeypatch, ref, tar, q, label), q, ref, tar, 16, 16, min_decisive=0.95)


def test_w32_every_box_alignment(engine, pair, monkeypatch):
    """Whole-pixel POIs whose reference and target windows start at every combination of x0 mod 4: the boxes start at the
    multiple of 4 below, each lane skips x0 mod 4 columns of its own box."""
    ref, tar = pair
    rows = []
    for a in range(4):
        for b in range(4):
            for k in range(3):
                x = 100 + 44 * k + a  # x0r = x - 16 = a (mod 4)
                u0 = (b - a) % 4 - 4 * ((a + k) % 2)  # x0t = x + u0 - 16 = b (mod 4), both signs
                rows.append((x, 60 + 30 * (4 * a + b), u0, (a + 2 * b) % 5 - 2))
    rows = np.array(rows, np.float32)
    q = ob.make_poi2d(rows[:, :2])
    q[:, 2], q[:, 8] = rows[:, 2], rows[:, 3]
    seen = {(int(x - 16) % 4, int(x + u - 16) % 4) for x, _, u, _ in rows}
    assert len(seen) == 16
    label = _label(16, 16, "16 box alignments")
    _check(label, _both_load_paths(engine, monkeypatch, ref, tar, q, label), q, ref, tar, 16, 16, min_decisive=0.95)


# ------------------------------------------------------------------------------------------------ warp reuse on w32
@pytest.fixture(scope="module")
def device():
    torch = pytest.importorskip("torch")
    p = torch.cuda.get_device_properties(0)
    return p.multi_processor_count, p.shared_memory_per_block_optin


def _pinned(lib, q):
    p = lib.ocb_host_alloc(q.nbytes)
    assert p
    a = np.frombuffer((ctypes.c_byte * q.nbytes).from_address(p), np.float32).reshape(q.shape)
    a[...] = q
    return p, a


@pytest.mark.parametrize("order", ["tma-skip-gather", "gather-tma-tma"])
def test_w32_warp_takes_several_pois(engine, pair, device, monkeypatch, order):
    """The grid is 16 x SMs CTAs of 4 warps, so a warp takes POIs i, i + 64 SMs, i + 128 SMs, ...: a queue of 3 x 64 x SMs + 5
    records in ONE launch makes every warp take three POIs (the first five a fourth), and the order of the thirds decides what
    each warp's tiles and mbarrier phase have seen before: a TMA load, a skipped POI, or a gather.  One launch means a queue
    that is not split: a pageable queue with OCB_NO_PIPELINE (queues of >= 16384 records are otherwise cut into four launches),
    or a page-locked queue, which the kernel reads and writes in place."""
    ref, tar = pair
    stride = 64 * device[0]
    n = 3 * stride + 5
    rng = np.random.default_rng(len(order))
    whole = sweep_queue(16, 16, 3 * n, seed=5)[0::3][:n]  # kind 0 and 1 alternate: whole pixels, zero and integer guesses
    whole[1::2] = sweep_queue(16, 16, 3 * n, seed=6)[1::3][:n][1::2]
    frac = sweep_queue(16, 16, 3 * n, seed=7)[2::3][:n]
    border = ob.make_poi2d(np.stack([rng.integers(0, 16, n), rng.integers(0, H, n)], 1))
    border[:, 16] = 0.375
    kinds = {"tma-skip-gather": (whole, border, frac), "gather-tma-tma": (frac, whole, whole)}[order]
    q = np.empty((n, 25), np.float32)
    for k in range(4):
        q[k * stride:(k + 1) * stride] = kinds[k % 3][k * stride:min(n, (k + 1) * stride)]
    label = _label(16, 16, order)
    monkeypatch.setenv("OCB_NO_PIPELINE", "1")
    got = _run(engine, ref, tar, q, 16, 16)
    computed = _check(label, got, q, ref, tar, 16, 16, min_decisive=0.6)
    assert computed[:stride].all() and computed[2 * stride:].all() and (computed[stride:2 * stride].all() or order == "tma-skip-gather")
    # each third alone, where no warp takes a second POI
    for k in range(4):
        part = q[k * stride:(k + 1) * stride].copy()
        engine.fftcc2d(part, 16, 16)
        assert np.array_equal(_bits(part), _bits(got[k * stride:(k + 1) * stride])), "%s: third %d differs when run alone" % (label, k)
    # the same queue page-locked: read and written in place
    lib = _capi.load()
    p, pinned = _pinned(lib, q)
    try:
        engine.fftcc2d(pinned, 16, 16)
        assert np.array_equal(_bits(pinned), _bits(got)), "%s: the page-locked queue differs at POIs %s" % (
            label, np.flatnonzero((_bits(pinned) != _bits(got)).any(1))[:10])
        del pinned
    finally:
        lib.ocb_host_free(p)


# ------------------------------------------------------------------------------------------------ image edges
@pytest.mark.parametrize("rx,ry", EDGE_R, ids=["r=(%d,%d)" % r for r in EDGE_R])
def test_windows_at_every_image_edge(engine, pair, rx, ry):
    w, h = 200, 180
    ref, tar = (np.ascontiguousarray(a[100:100 + h, 200:200 + w]) for a in pair)
    cx, cy = w // 2, h // 2
    lo_x, hi_x, lo_y, hi_y = rx, w - rx - 1, ry, h - ry - 1
    inside = [(lo_x, cy), (hi_x, cy), (cx, lo_y), (cx, hi_y), (lo_x, lo_y), (hi_x, lo_y), (lo_x, hi_y), (hi_x, hi_y)]
    outside = [(lo_x - 1, cy), (hi_x + 1, cy), (cx, lo_y - 1), (cx, hi_y + 1), (lo_x - 1, lo_y - 1), (hi_x + 1, lo_y - 1),
               (lo_x - 1, hi_y + 1), (hi_x + 1, hi_y + 1)]
    rows = [(x, y, 0, 0, True) for x, y in inside] + [(x, y, 0, 0, False) for x, y in outside]
    # the guess moves only the target window to each edge, and one pixel past it
    for tx, ok in ((lo_x, True), (lo_x - 1, False), (hi_x, True), (hi_x + 1, False)):
        rows.append((cx, cy, tx - cx, 0, ok))
    for ty, ok in ((lo_y, True), (lo_y - 1, False), (hi_y, True), (hi_y + 1, False)):
        rows.append((cx, cy, 0, ty - cy, ok))
    # fractional coordinates truncate toward zero: r - 0.25 is column r - 1 (outside), r + 0.75 column r (inside)
    rows += [(lo_x - 0.25, cy, 0, 0, False), (lo_x + 0.75, cy, 0, 0, True), (cx, lo_y - 0.25, 0, 0, False), (cx, lo_y + 0.75, 0, 0, True),
             (hi_x + 0.75, cy, 0, 0, True), (cx, hi_y + 1.0, 0, 0, False), (cx + 0.5, cy, lo_x - 0.75 - cx, 0, False),
             (cx + 0.5, cy, lo_x + 0.25 - cx, 0, True), (cx, cy + 0.5, 0, hi_y + 0.75 - cy, False), (cx, cy + 0.5, 0, -cy - 0.25, False)]
    rows = np.array(rows, np.float32)
    q = _mark(ob.make_poi2d(rows[:, :2]))
    q[:, 2], q[:, 8] = rows[:, 2], rows[:, 3]
    _check(_label(rx, ry, "image edges"), _run(engine, ref, tar, q, rx, ry), q, ref, tar, rx, ry, expect_computed=rows[:, 4] > 0)


@pytest.mark.parametrize("rx,ry", EDGE_R, ids=["r=(%d,%d)" % r for r in EDGE_R])
def test_smallest_images(engine, pair, rx, ry):
    """w = 2 rx + 1, h = 2 ry + 1 holds exactly one POI; 2 r + 4 holds a 4 x 4 block of them."""
    for extra in (1, 4):
        w, h = 2 * rx + extra, 2 * ry + extra
        ref, tar = (np.ascontiguousarray(a[300:300 + h, 300:300 + w]) for a in pair)
        xs, ys = np.meshgrid(np.arange(rx - 1, rx + extra + 1), np.arange(ry - 1, ry + extra + 1))
        q = _mark(ob.make_poi2d(np.stack([xs.ravel(), ys.ravel()], 1)))
        ok = (q[:, 0] >= rx) & (q[:, 0] < w - rx) & (q[:, 1] >= ry) & (q[:, 1] < h - ry)
        assert ok.sum() == extra * extra
        _check(_label(rx, ry, "image %dx%d" % (w, h)), _run(engine, ref, tar, q, rx, ry), q, ref, tar, rx, ry, expect_computed=ok)


# ------------------------------------------------------------------------------------------------ skips
@pytest.mark.parametrize("rx,ry", EDGE_R[:3], ids=["r=(%d,%d)" % r for r in EDGE_R[:3]])
def test_non_finite_fields_skip_the_poi(engine, pair, rx, ry):
    """NaN, +-inf and 1e30 in x, y, u0 or v0: the record keeps every byte, as in the float32 oracle (whose (int) conversions
    are the reference's own); good POIs between them are computed."""
    ref, tar = pair
    bad = [np.nan, np.inf, -np.inf, 1e30, -1e30]
    q = _mark(ob.make_poi2d(np.tile([[300.0, 280.0]], (5 * len(bad), 1))))
    q[:, 2], q[:, 8] = 1.0, -2.0
    expect = np.ones(len(q), bool)
    for j, col in enumerate((0, 1, 2, 8)):
        for k, v in enumerate(bad):
            q[j * len(bad) + k, col] = v
            expect[j * len(bad) + k] = False
    q[4 * len(bad):, 0] += np.arange(len(bad))  # the last five stay good
    _check(_label(rx, ry, "non-finite fields"), _run(engine, ref, tar, q, rx, ry), q, ref, tar, rx, ry, oracle_exact=False, expect_computed=expect)
    # a queue in which every POI is skipped, and queues of one POI
    q_all = q[~expect].copy()
    _check(_label(rx, ry, "all skipped"), _run(engine, ref, tar, q_all, rx, ry), q_all, ref, tar, rx, ry, oracle_exact=False,
           expect_computed=np.zeros(len(q_all), bool))
    for one, ok in ((q[-1:].copy(), True), (q[:1].copy(), False)):
        _check(_label(rx, ry, "one POI"), _run(engine, ref, tar, one, rx, ry), one, ref, tar, rx, ry, oracle_exact=False,
               expect_computed=np.array([ok]))


# ------------------------------------------------------------------------------------------------ degenerate windows
@pytest.mark.parametrize("rx,ry", EDGE_R, ids=["r=(%d,%d)" % r for r in EDGE_R])
@pytest.mark.parametrize("flat", ["reference", "target", "both"])
def test_constant_window(engine, pair, rx, ry, flat):
    """A window of constant grey has zero norm and a zero spectrum, so the reference's correlation surface is zero everywhere
    (src/oc_fftcc.cpp:239-255): its strict '>' scan keeps index 0 -- the displacement is the guess -- and ZNCC is 0 / 0 = NaN.
    The kernels and the oracle pack both windows into one transform, where Z(k) + conj Z(-k) only cancels up to rounding and
    noise would pick the displacement, so they apply the rule themselves when a norm is zero."""
    ref, tar = (a.copy() for a in pair)
    if flat in ("reference", "both"):
        ref[150:350, 150:450] = 128.0
    if flat in ("target", "both"):
        tar[150:350, 150:450] = 128.0
    xy = np.array([[300, 250], [280, 240], [310.5, 260.25], [290, 245], [305, 255]], np.float32)
    q = _mark(ob.make_poi2d(xy))
    q[:, 2] = [0, 2, 1.5, -3, 0]
    q[:, 8] = [0, -1, 0.25, 2, 4]
    got = _run(engine, ref, tar, q, rx, ry)
    wa, computed, _, _ = witness(ref, tar, q, rx, ry)
    wb = Oracle2D(ref, tar).fftcc2d(q.copy(), rx, ry, exact=True)
    assert computed.all()
    label = _label(rx, ry, "constant %s window" % flat)
    assert np.array_equal(got[:, [2, 8]], q[:, [2, 8]]) and np.array_equal(got[:, [14, 15]], q[:, [2, 8]]), "%s: displacement %s, guess %s" % (
        label, got[:, [2, 8]].tolist(), q[:, [2, 8]].tolist())
    assert np.isnan(wa[:, 16]).all() and np.isnan(got[:, 16]).all(), "%s: ZNCC %s" % (label, got[:, 16])
    assert np.array_equal(got, wb, equal_nan=True), "%s: differs from the oracle: %s vs %s" % (label, got[:, [2, 8, 16]].tolist(), wb[:, [2, 8, 16]].tolist())
    assert np.array_equal(got, wa, equal_nan=True), label
    print("%s: n=%d compared=%d index 0 won, ZNCC NaN" % (label, len(q), len(q)))


@pytest.mark.parametrize("r,generic", TIE_R, ids=["r=%d%s" % (r, " generic" if g else "") for r, g in TIE_R])
def test_near_exact_ties(engine, monkeypatch, r, generic):
    """Small integer intensities repeated with period r in x and y: the 2r x 2r window holds 2 x 2 periods, so the correlation has
    four equal maxima in exact arithmetic -- (0, 0), (r, 0), (0, r), (r, r) -- which float32 twiddles separate by rounding.  Each
    kernel must return one of them, with ZNCC = 1."""
    rng = np.random.default_rng(r)
    img = np.tile(rng.integers(0, 64, (r, r)).astype(np.float32), (12, 12))[:8 * r + 40, :8 * r + 44]
    img = np.ascontiguousarray(img)
    q = sweep_queue(r, r, 12, seed=r, w=img.shape[1], h=img.shape[0])
    q[:, [0, 1, 2, 8]] = np.floor(q[:, [0, 1, 2, 8]])
    if generic:
        monkeypatch.setenv("OCB_FFTCC2D_GENERIC", "1")
    got = _run(engine, img, img, q, r, r)
    wa, computed, gap, cands = witness(img, img, q, r, r)
    assert computed.all() and (gap < GAP).all() and all(len(c) == 4 for c in cands)
    for i in range(len(q)):
        assert (got[i, 2], got[i, 8]) in cands[i], "r=%d POI %d: (%g, %g) is not one of %s" % (r, i, got[i, 2], got[i, 8], sorted(cands[i]))
    assert np.array_equal(got[:, [14, 15]], q[:, [2, 8]])
    dz = np.abs(got[:, 16] - wa[:, 16]).max()
    assert dz < GAP
    assert np.array_equal(_bits(got[:, OTHER_COLS]), _bits(q[:, OTHER_COLS]))
    print("%s: n=%d compared=%d max|dZNCC|=%.2e non-decisive=%d" % (_label(r, r, "four-fold tie", generic), len(q), len(q), dz, len(q)))


# ------------------------------------------------------------------------------------------------ limits
def test_largest_window_and_rejections(engine, device, tmp_path):
    """The largest square window the shared-memory check accepts matches the witnesses (M = 13456 on an H100: the kernel's
    reciprocal-multiply index division far from small arguments); the first one it refuses, windows with a prime factor above 31
    and radii below 1 return an error that names the window, leave the queue untouched and leave the engine usable."""
    exe = build_plan_tool(str(tmp_path))
    out = run_plan_tool(exe, "limits", device[1])
    assert out.returncode == 0, out.stdout + out.stderr
    largest, first = (int(v) for v in out.stdout.replace("\n", " ").split() if v.isdigit())
    if device[1] == 227 * 1024:
        assert (largest, first) == (58, 60)
    rng = np.random.default_rng(3)
    ref, tar = synth.speckle_pair_2d(800, 800)
    xy = np.stack([rng.integers(largest + 8, 800 - largest - 8, 3), rng.integers(largest + 8, 800 - largest - 8, 3)], 1)
    q = ob.make_poi2d(xy)
    q[1, 2], q[2, 8] = 2.0, -1.5
    _check(_label(largest, largest, "largest"), _run(engine, ref, tar, q, largest, largest), q, ref, tar, largest, largest, min_decisive=1.0)
    refused = [(first, first, _capi.OCB_ERR_UNSUPPORTED, "%dx%d" % (2 * first, 2 * first)), (0, 8, _capi.OCB_ERR_ARG, "fftcc2d"),
               (8, -1, _capi.OCB_ERR_ARG, "fftcc2d")]
    refused += [(rx, ry, _capi.OCB_ERR_UNSUPPORTED, "%dx%d" % (2 * rx, 2 * ry)) for rx, ry, why in REJECTED if why == "prime factor"]
    for rx, ry, code, text in refused:
        bad = _mark(q.copy())
        before = bad.copy()
        with pytest.raises(_capi.OpenCorrB200Error) as e:
            engine.fftcc2d(bad, rx, ry)
        assert e.value.code == code and text in str(e.value), (rx, ry, str(e.value))
        assert np.array_equal(_bits(bad), _bits(before)), "a refused call wrote to the queue"
        again = q.copy()
        engine.fftcc2d(again, 10, 10)  # the engine is still usable
        assert (again[:, 16] > 0.5).all()
        print("FFTCC2D r=(%d,%d): refused, %s" % (rx, ry, e.value))
