"""GPU: FFTCC3D on all three kernels and both window-load paths, at every window size and volume face, against two float64
witnesses.

ocb::fftcc3d_plan (opencorr_b200/csrc/ocb_kernels.h) sends r = 16 to fftcc3d_w32.cu (one POI per CTA of 8 warps; each z-slice of
the windows arrives as two TMA boxes when POI and guess are whole voxels and the volume pitch is a multiple of 4 floats, by a
per-lane gather otherwise), cubic windows of N = 2^a 3^b 5^c <= 64 points to fftcc3d_reg.cu (one thread per 1D transform, 128 / N
z-slices per round) and everything else whose prime factors are <= 31 to the shared-memory Stockham kernel of fftcc.cu;
test_fftcc3d_plan_host.py checks on the CPU that every case below lands on the kernel it names, that the generic cases reach
every radix and the register cases every size and every slices-per-round count.

Witnesses: (a) `witness` below, plain numpy in float64 (np.fft), which shares no code with the oracle; (b) Oracle3D.fftcc3d with
exact=True.  Pass rule (`_check`): u, v, w, u0, v0, w0 are bit-identical to both witnesses on every POI whose float64 peak stands
more than 1e-5 (in ZNCC units) above the runner-up; a POI with a smaller gap may return any maximum within 1e-5 of the peak; ZNCC
is within 1e-5 of both; every other field, and every field of a skipped POI, keeps its bytes.  Each case prints one line:
kernel, n, compared, max |dZNCC|, non-decisive POIs.  The volume is not cubic (dx != dy != dz), so a swapped stride cannot pass."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import opencorr_b200 as ob
from opencorr_b200 import _capi, synth
from oracle.oracle import Oracle3D

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DX, DY, DZ = 140, 124, 108  # room for the largest accepted cube (84 points) plus guesses
INT_COLS = [3, 7, 11, 15, 16, 17]  # u, v, w, u0, v0, w0
ZNCC = 18
OTHER_COLS = np.delete(np.arange(31), INT_COLS + [ZNCC])
GAP = 1e-5

# ------------------------------------------------------------------------------------------------ the cases, by kernel
REG_R = (4, 5, 6, 8, 9, 10, 12, 15, 18, 20, 24, 25, 27, 30, 32)  # fftcc3d_reg.cu: every size it has
GENERIC_CUBIC = (7, 11, 13, 17, 19, 23, 29, 31, 33, 36, 42)  # every odd radix 7 ... 31; > 64 points, up to the largest accepted
GENERIC_NONCUBIC = ((16, 16, 15), (8, 8, 16), (32, 4, 4), (4, 31, 4), (12, 10, 14))  # axes of register sizes, a radix-5 axis
FORCED_GENERIC = (8, 16, 30)  # OCB_FFTCC3D_GENERIC against the kernel the window takes by default
EDGE_R = ((16, 16, 16), (10, 10, 10), (7, 7, 7), (12, 10, 14))  # W32, REG, GENERIC, GENERIC non-cubic
LONG_R = ((16, 16, 16), (4, 4, 4), (7, 7, 7))  # W32, REG, GENERIC at small windows
TIE_R = ((16, (0,), False), (8, (0, 1), False), (10, (0, 1, 2), False), (7, (1, 2), False), (16, (2,), True))  # (r, periodic axes, forced generic)
REJECTED = ((44, "shared memory"), (43, "prime factor"), (37, "prime factor"))  # at an H100's 227 KB opt-in limit


def _kernel_name(r, generic=False):
    if generic:
        return "GENERIC"
    rx, ry, rz = r
    if r == (16, 16, 16):
        return "W32"
    return "REG" if rx == ry == rz and rx in REG_R else "GENERIC"


def sweep_n(r):
    """Queue length of a sweep case: 20 ... 31, fewer where a window is large."""
    return 12 + sum(r) % 7 if max(r) > 32 else 20 + sum(r) % 12


SWEEP = [(r, r, r) for r in REG_R] + [(16, 16, 16)] + [(r, r, r) for r in GENERIC_CUBIC] + list(GENERIC_NONCUBIC)
# (rx, ry, rz, forced generic, kernel, queue length) of every case: what test_fftcc3d_plan_host.py checks against the plan
PLAN_CASES = ([r + (0, _kernel_name(r), sweep_n(r)) for r in SWEEP]
              + [(r, r, r, 1, "GENERIC", sweep_n((r, r, r))) for r in FORCED_GENERIC]
              + [r + (0, _kernel_name(r), 40) for r in EDGE_R]
              + [r + (0, _kernel_name(r), 60) for r in EDGE_R] + [(16, 16, 16, 1, "GENERIC", 60)]  # sentinels
              + [r + (0, _kernel_name(r), 1) for r in LONG_R]
              + [(r, r, r, int(g), _kernel_name((r, r, r), g), 12) for r, _, g in TIE_R]
              + [(r, r, r, 0, "rejected (%s)" % why, 3) for r, why in REJECTED])


def build_plan_tool(out_dir):
    """Compiles tests/native/fftcc3d_plan_host_test.cpp (ocb::fftcc3d_plan of ocb_kernels.h, host only) into out_dir."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    exe = os.path.join(out_dir, "fftcc3d_plan_host_test")
    cmd = [nvcc, "-x", "cu", "-std=c++17", "-O1", "-Wno-deprecated-gpu-targets", "-I", os.path.join(ROOT, "opencorr_b200", "csrc"),
           "-o", exe, os.path.join(ROOT, "tests", "native", "fftcc3d_plan_host_test.cpp")]
    if os.path.exists("/usr/bin/g++"):
        cmd[1:1] = ["-ccbin", "/usr/bin/g++"]
    build = subprocess.run(cmd, capture_output=True, text=True)
    assert build.returncode == 0, "nvcc failed:\n" + build.stdout + build.stderr
    return exe


def run_plan_tool(exe, *args, cases=None):
    text = "".join("%d %d %d %d %d\n" % (c[0], c[1], c[2], c[3], c[5]) for c in cases) if cases else None
    return subprocess.run([exe] + [str(a) for a in args], input=text, capture_output=True, text=True, timeout=60)


# ------------------------------------------------------------------------------------------------ witness (a)
def _c_int(v):
    """(int) of a float on the GPU (cvt.rzi.s32.f32): truncation toward zero, saturating at the int range."""
    v = float(v)
    return int(np.clip(np.trunc(v), -2 ** 31, 2 ** 31 - 1)) if np.isfinite(v) else (2 ** 31 - 1 if v > 0 else -2 ** 31)


def witness(ref, tar, q, rx, ry, rz):
    """FFTCC3D::compute of the reference (src/oc_fftcc.cpp:327-427) in float64 on float32 inputs, with the kernels' border, NaN
    and zero-norm rules.  Returns the records, which POIs were computed, each one's gap between the peak and the runner-up (ZNCC
    units), and each one's (u, v, w) candidates: every maximum within GAP of the peak."""
    dz, dy, dx = ref.shape
    f32 = np.float32
    rad, size = (rx, ry, rz), (2 * rx, 2 * ry, 2 * rz)
    dims = (dx, dy, dz)
    out, computed, gap, cands = q.copy(), np.zeros(len(q), bool), np.full(len(q), np.inf), [None] * len(q)
    for i, p in enumerate(q):
        pos, guess = p[0:3], p[[3, 7, 11]]
        if np.isnan(pos).any() or np.isnan(guess).any():
            continue
        inside = True
        with np.errstate(all="ignore"):
            for a in range(3):  # the kernels' guard, in their float32 arithmetic
                lo = pos[a] - f32(rad[a])
                hi = (pos[a] + f32(size[a] - 1)) - f32(rad[a])
                if (_c_int(lo) < 0 or _c_int(hi) >= dims[a] or _c_int(lo + guess[a]) < 0 or _c_int(hi + guess[a]) >= dims[a]
                        or lo < 0 or lo + guess[a] < 0):
                    inside = False
        if not inside:
            continue
        # float32 coordinate arithmetic (p + k) - r, then + u0, then truncation toward zero (:353-360)
        rc = [(pos[a] + np.arange(size[a], dtype=f32)) - f32(rad[a]) for a in range(3)]
        ia = [c.astype(np.int64) for c in rc]
        ib = [(rc[a] + guess[a]).astype(np.int64) for a in range(3)]
        va = ref[np.ix_(ia[2], ia[1], ia[0])].astype(np.float64)
        vb = tar[np.ix_(ib[2], ib[1], ib[0])].astype(np.float64)
        va -= va.mean()
        vb -= vb.mean()
        na, nb = (va * va).sum(), (vb * vb).sum()
        shape = va.shape
        corr = np.fft.irfftn(np.conj(np.fft.rfftn(va)) * np.fft.rfftn(vb), s=shape, axes=(0, 1, 2)).ravel()  # sum_x a(x) b(x + d)
        if na == 0 or nb == 0:  # constant grey: the reference's surface is zero everywhere
            corr[:] = 0.0
        with np.errstate(invalid="ignore", divide="ignore"):
            zncc = corr / np.sqrt(na * nb)
        idx = int(np.argmax(corr))  # the first maximum in (z, y, x) linear order

        def disp(j):
            d = [int(j) % size[0], (int(j) // size[0]) % size[1], int(j) // (size[0] * size[1])]
            return tuple(f32(d[a] - size[a] if d[a] > rad[a] else d[a]) + guess[a] for a in range(3))

        near = np.flatnonzero(corr >= corr[idx] - GAP * np.sqrt(na * nb)) if na * nb > 0 else [idx]
        out[i, [3, 7, 11]] = disp(idx)
        out[i, [15, 16, 17]] = guess
        out[i, ZNCC] = zncc[idx]
        computed[i], cands[i] = True, {disp(j) for j in near}
        gap[i] = zncc[idx] - np.delete(zncc, idx).max() if np.isfinite(zncc[idx]) else 0.0
    return out, computed, gap, cands


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _check(label, got, q, ref, tar, r, min_decisive=None, expect_computed=None, ztol=GAP):
    """got: the GPU's records for the queue q.  Applies the pass rule of the module docstring against both witnesses (ztol: the
    ZNCC tolerance, GAP unless a case says why not)."""
    wa, computed, gap, cands = witness(ref, tar, q, *r)
    wb = Oracle3D(ref, tar).fftcc3d(q.copy(), *r, exact=True)
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
        assert len(bad) == 0, "%s: u, v, w, u0, v0, w0 differ from the %s at POIs %s: got %s, expected %s (gap %s)" % (
            label, name, bad[:8], got[bad[:4]][:, INT_COLS].tolist(), w_[bad[:4]][:, INT_COLS].tolist(), gap[bad[:4]])
    for i in np.flatnonzero(computed & ~dec):
        assert tuple(got[i, [3, 7, 11]]) in cands[i], "%s: POI %d returned %s, not one of the tied maxima %s" % (
            label, i, got[i, [3, 7, 11]].tolist(), sorted(cands[i]))
        assert np.array_equal(got[i, [15, 16, 17]], q[i, [3, 7, 11]]), label
    # ZNCC is NaN exactly where a window is constant (0 / 0), finite elsewhere
    flat = computed & np.isnan(wa[:, ZNCC])
    for name, w_ in (("numpy witness", wa), ("oracle", wb)):
        assert np.array_equal(np.isnan(got[computed, ZNCC]), np.isnan(w_[computed, ZNCC])), "%s: ZNCC is NaN at POIs %s, the %s at %s" % (
            label, np.flatnonzero(computed & np.isnan(got[:, ZNCC])), name, np.flatnonzero(computed & np.isnan(w_[:, ZNCC])))
    dz = 0.0
    fin = computed & ~flat
    if fin.any():
        dz = max(np.abs(got[fin, ZNCC] - wa[fin, ZNCC]).max(), np.abs(got[fin, ZNCC] - wb[fin, ZNCC]).max())
        assert dz < ztol, "%s: max |dZNCC| = %.3g" % (label, dz)
    nd = int((computed & ~dec).sum())
    if min_decisive is not None:
        assert computed.sum() - nd >= min_decisive * len(q), "%s: only %d of %d POIs are decisive" % (label, computed.sum() - nd, len(q))
    print("%s: n=%d compared=%d max|dZNCC|=%.2e non-decisive=%d" % (label, len(q), computed.sum(), dz, nd))
    return computed


# ------------------------------------------------------------------------------------------------ volumes and queues
@pytest.fixture(scope="module")
def vol():
    return synth.speckle_pair_3d(DX, DY, DZ, device="cuda")  # rendered on the GPU: seconds instead of half a minute


@pytest.fixture(scope="module")
def device():
    torch = pytest.importorskip("torch")
    p = torch.cuda.get_device_properties(0)
    return p.multi_processor_count, p.shared_memory_per_block_optin


@pytest.fixture(scope="module")
def plan_tool(tmp_path_factory):
    return build_plan_tool(str(tmp_path_factory.mktemp("fftcc3d_plan")))


def sweep_queue(r, n, seed, dims=(DX, DY, DZ)):
    """A quarter whole-voxel POIs with a zero guess, a quarter whole-voxel POIs with an integer guess of mixed sign (every residue
    mod 4), a quarter whole-voxel POIs with a fractional guess (what a re-seed passes), a quarter fractional POIs with a fractional
    guess; every window inside the volume."""
    rng = np.random.default_rng(seed)
    xyz = np.stack([rng.uniform(r[a] + 6, dims[a] - r[a] - 7, n) for a in range(3)], 1)
    q = ob.make_poi3d(xyz)
    kind = np.arange(n) % 4
    whole = kind < 3
    q[whole, 0:3] = np.floor(q[whole, 0:3])
    for c, lo, hi in ((3, -3, 5), (7, -5, 3), (11, -4, 4)):
        q[kind == 1, c] = rng.integers(lo, hi, (kind == 1).sum(), endpoint=True)
        q[kind >= 2, c] = rng.uniform(lo, hi, (kind >= 2).sum())
    return q


def _label(r, what="", generic=False):
    return "FFTCC3D %s%s r=(%d,%d,%d)%s" % (_kernel_name(r, generic), " (forced)" if generic else "", *r, " " + what if what else "")


def _run(engine, ref, tar, q, r):
    engine.set_images_3d(ref, tar)
    got = q.copy()
    engine.fftcc3d(got, *r)
    return got


def _mark(q):
    """Distinct values in every field FFT-CC does not read, u0, v0, w0 and ZNCC included: they must survive on a skipped POI."""
    for c in range(3, 31):
        if c not in (3, 7, 11):
            q[:, c] = 0.5 + c + 0.001 * np.arange(len(q))
    return q


# ------------------------------------------------------------------------------------------------ window sweep
@pytest.mark.parametrize("r", SWEEP, ids=["r=(%d,%d,%d)" % r for r in SWEEP])
def test_window_sweep(engine, vol, r):
    ref, tar = vol
    q = sweep_queue(r, sweep_n(r), seed=sum(r) * 31 + r[0])
    _check(_label(r), _run(engine, ref, tar, q, r), q, ref, tar, r, min_decisive=0.9)


@pytest.mark.parametrize("rr", FORCED_GENERIC)
def test_forced_generic_equals_default(engine, vol, monkeypatch, rr):
    ref, tar = vol
    r = (rr, rr, rr)
    q = sweep_queue(r, sweep_n(r), seed=7 * rr)
    a = _run(engine, ref, tar, q, r)
    monkeypatch.setenv("OCB_FFTCC3D_GENERIC", "1")
    b = _run(engine, ref, tar, q, r)
    _check(_label(r, generic=True), b, q, ref, tar, r, min_decisive=0.9)
    assert np.array_equal(_bits(a[:, INT_COLS]), _bits(b[:, INT_COLS]))
    assert np.abs(a[:, ZNCC] - b[:, ZNCC]).max() < 2e-6


# ------------------------------------------------------------------------------------------------ w32 load paths
def _both_load_paths(engine, monkeypatch, ref, tar, q, label):
    monkeypatch.delenv("OCB_NO_TMA", raising=False)
    a = _run(engine, ref, tar, q, (16, 16, 16))
    monkeypatch.setenv("OCB_NO_TMA", "1")
    b = _run(engine, ref, tar, q, (16, 16, 16))
    monkeypatch.delenv("OCB_NO_TMA")
    assert np.array_equal(_bits(a), _bits(b)), "%s: TMA boxes and the per-lane gather deliver different windows at POIs %s" % (
        label, np.flatnonzero((_bits(a) != _bits(b)).any(1))[:10])
    return a


@pytest.mark.parametrize("width", [DX, 139, 138, 137])
def test_w32_tma_and_gather_agree(engine, vol, monkeypatch, width):
    """The TMA map needs a pitch that is a multiple of 4 floats: widths 137 ... 139 gather every window, 140 takes boxes for its
    whole-voxel POIs and gathers the fractional ones; OCB_NO_TMA gathers all of them, with the same bits."""
    ref, tar = (np.ascontiguousarray(a[:, :, :width]) for a in vol)
    q = sweep_queue((16, 16, 16), 30, seed=width, dims=(width, DY, DZ))
    label = _label((16, 16, 16), "width %d" % width)
    _check(label, _both_load_paths(engine, monkeypatch, ref, tar, q, label), q, ref, tar, (16, 16, 16), min_decisive=0.9)


def test_w32_every_box_alignment(engine, vol, monkeypatch):
    """Whole-voxel POIs whose reference and target windows start at every combination of x0 mod 4: the boxes start at the
    multiple of 4 below, each lane skips x0 mod 4 columns of its own box."""
    ref, tar = vol
    rows = []
    for a in range(4):
        for b in range(4):
            for k in range(2):
                x = 24 + 40 * k + a  # x0r = x - 16 = a (mod 4)
                u0 = (b - a) % 4 - 4 * ((a + k) % 2)  # x0t = x + u0 - 16 = b (mod 4), both signs
                rows.append((x, 24 + 5 * b + k, 30 + 3 * a, u0, (a + 2 * b) % 5 - 2, (a + b + k) % 3 - 1))
    rows = np.array(rows, np.float32)
    q = ob.make_poi3d(rows[:, :3])
    q[:, 3], q[:, 7], q[:, 11] = rows[:, 3], rows[:, 4], rows[:, 5]
    seen = {(int(x - 16) % 4, int(x + u - 16) % 4) for x, u in rows[:, [0, 3]]}
    assert len(seen) == 16
    label = _label((16, 16, 16), "16 box alignments")
    _check(label, _both_load_paths(engine, monkeypatch, ref, tar, q, label), q, ref, tar, (16, 16, 16), min_decisive=0.9)


# ------------------------------------------------------------------------------------------------ volume faces
def _face_rows(r, dims):
    """(x, y, z, u0, v0, w0, accepted) rows: the reference window and the guessed target window touching each of the six faces
    exactly, one voxel further, and fractional positions where truncation and the `p - r < 0` test disagree."""
    c = [d // 2 for d in dims]
    lo = list(r)
    hi = [dims[a] - r[a] for a in range(3)]  # window [p - r, p + r - 1]: its last voxel is dims - 1
    rows = []

    def row(pos, guess, ok):
        rows.append(tuple(pos) + tuple(guess) + (ok,))

    for a in range(3):
        for edge, past in ((lo[a], -1), (hi[a], 1)):
            p = list(c)
            p[a] = edge
            row(p, (0, 0, 0), True)  # the reference window on the face
            p[a] = edge + past
            row(p, (0, 0, 0), False)  # one voxel past it
            g = [0, 0, 0]  # the guess moves only the target window to the face, and one voxel past it
            g[a] = edge - c[a]
            row(c, g, True)
            g[a] = edge + past - c[a]
            row(c, g, False)
        # fractional coordinates truncate toward zero: r - 0.25 truncates to column 0 but p - r < 0 refuses it; r + 0.75 is
        # column r; dims - r + 0.75 still ends on the last voxel, dims - r + 1 does not
        for v, ok in ((lo[a] - 0.25, False), (lo[a] + 0.75, True), (hi[a] + 0.75, True), (hi[a] + 1.0, False)):
            p = list(map(float, c))
            p[a] = v
            row(p, (0, 0, 0), ok)
        for g_, ok in ((lo[a] - 0.75 - c[a], False), (lo[a] + 0.25 - c[a], True), (hi[a] + 0.25 - c[a], True)):
            p = list(map(float, c))
            p[a] += 0.5
            g = [0.0, 0.0, 0.0]
            g[a] = g_
            row(p, g, ok)
    return np.array(rows, np.float32)


@pytest.mark.parametrize("r", EDGE_R, ids=["r=(%d,%d,%d)" % r for r in EDGE_R])
def test_windows_at_every_volume_face(engine, vol, monkeypatch, r):
    dims = (76, 68, 60)
    ref, tar = (np.ascontiguousarray(a[20:20 + dims[2], 30:30 + dims[1], 40:40 + dims[0]]) for a in vol)
    rows = _face_rows(r, dims)
    q = _mark(ob.make_poi3d(rows[:, :3]))
    q[:, 3], q[:, 7], q[:, 11] = rows[:, 3], rows[:, 4], rows[:, 5]
    label = _label(r, "volume faces")
    got = _both_load_paths(engine, monkeypatch, ref, tar, q, label) if r == (16, 16, 16) else _run(engine, ref, tar, q, r)
    _check(label, got, q, ref, tar, r, expect_computed=rows[:, 6] > 0)


# ------------------------------------------------------------------------------------------------ skips
SENTINEL_CASES = [(r, False) for r in EDGE_R] + [((16, 16, 16), True)]


@pytest.mark.parametrize("r,generic", SENTINEL_CASES, ids=["r=(%d,%d,%d)%s" % (r + (" generic" if g else "",)) for r, g in SENTINEL_CASES])
def test_non_finite_fields_skip_the_poi(engine, vol, monkeypatch, r, generic):
    """NaN, +-inf and +-1e30 in x, y, z, u0, v0 or w0: the record keeps every byte, in the kernels and in both witnesses; good POIs
    between them are computed."""
    ref, tar = vol
    bad = [np.nan, np.inf, -np.inf, 1e30, -1e30]
    cols = (0, 1, 2, 3, 7, 11)
    q = _mark(ob.make_poi3d(np.tile([[70.0, 62.0, 54.0]], (2 * len(cols) * len(bad), 1))))
    q[:, 3], q[:, 7], q[:, 11] = 1.0, -2.0, 0.5
    expect = np.ones(len(q), bool)
    for j, col in enumerate(cols):
        for k, v in enumerate(bad):
            i = 2 * (j * len(bad) + k)  # every other POI is good: the bad ones are interleaved
            q[i, col] = v
            expect[i] = False
    q[1::2, 0] += np.arange(len(q) // 2) % 5
    if generic:
        monkeypatch.setenv("OCB_FFTCC3D_GENERIC", "1")
    _check(_label(r, "non-finite fields", generic), _run(engine, ref, tar, q, r), q, ref, tar, r, expect_computed=expect)
    q_all = q[~expect].copy()
    _check(_label(r, "all skipped", generic), _run(engine, ref, tar, q_all, r), q_all, ref, tar, r, expect_computed=np.zeros(len(q_all), bool))


# ------------------------------------------------------------------------------------------------ degenerate windows
CONST_BOX = (slice(24, 84), slice(32, 92), slice(40, 100))  # z, y, x: 60^3 voxels around the centre of the volume


def _const_queue(r):
    """POIs whose reference and target windows lie inside CONST_BOX, with whole and fractional guesses."""
    xyz = np.array([[70, 62, 54], [68, 60, 52], [71.5, 63.25, 55.75], [72, 61, 53], [69, 64, 56]], np.float32)
    q = _mark(ob.make_poi3d(xyz))
    q[:, 3] = [0, 2, 1.5, -3, 0]
    q[:, 7] = [0, -1, 0.25, 2, 3]
    q[:, 11] = [0, 1, -0.5, 0, -2]
    return q


CONST_CASES = [(r, False) for r in EDGE_R] + [((16, 16, 16), True), ((10, 10, 10), True)]


@pytest.mark.parametrize("r,generic", CONST_CASES, ids=["r=(%d,%d,%d)%s" % (r + (" generic" if g else "",)) for r, g in CONST_CASES])
@pytest.mark.parametrize("flat", ["reference", "target", "both"])
def test_constant_window(engine, vol, monkeypatch, r, generic, flat):
    """A window of constant grey has zero norm and a zero spectrum, so the reference's correlation surface is zero everywhere
    (src/oc_fftcc.cpp:378-402): its strict '>' scan keeps index 0 -- the displacement is the guess -- and ZNCC is 0 / 0 = NaN.
    The kernels and the oracle pack both windows into one transform, where Z(k) + conj Z(-k) only cancels up to rounding and
    noise would pick the displacement, so they apply the rule themselves when a norm is zero.  The grey is an integer
    (synth.BACKGROUND), so the float32 means are exact and the norm is exactly zero."""
    ref, tar = (a.copy() for a in vol)
    if flat in ("reference", "both"):
        ref[CONST_BOX] = synth.BACKGROUND
    if flat in ("target", "both"):
        tar[CONST_BOX] = synth.BACKGROUND
    q = _const_queue(r)
    if generic:
        monkeypatch.setenv("OCB_FFTCC3D_GENERIC", "1")
    got = _run(engine, ref, tar, q, r)
    wa, computed, _, _ = witness(ref, tar, q, *r)
    wb = Oracle3D(ref, tar).fftcc3d(q.copy(), *r, exact=True)
    assert computed.all()
    label = _label(r, "constant %s window" % flat, generic)
    assert np.array_equal(got[:, [3, 7, 11]], q[:, [3, 7, 11]]) and np.array_equal(got[:, [15, 16, 17]], q[:, [3, 7, 11]]), (
        "%s: displacement %s, guess %s" % (label, got[:, [3, 7, 11]].tolist(), q[:, [3, 7, 11]].tolist()))
    assert np.isnan(wa[:, ZNCC]).all() and np.isnan(got[:, ZNCC]).all(), "%s: ZNCC %s" % (label, got[:, ZNCC])
    assert np.array_equal(got, wb, equal_nan=True), "%s: differs from the oracle: %s vs %s" % (
        label, got[:, [3, 7, 11, ZNCC]].tolist(), wb[:, [3, 7, 11, ZNCC]].tolist())
    assert np.array_equal(got, wa, equal_nan=True), label
    print("%s: n=%d compared=%d index 0 won, ZNCC NaN" % (label, len(q), len(q)))


@pytest.mark.parametrize("r", EDGE_R, ids=["r=(%d,%d,%d)" % r for r in EDGE_R])
@pytest.mark.parametrize("step", [231.0, 1.0])
def test_constant_window_but_one_voxel(engine, vol, r, step):
    """The rule fires only at exactly zero norm: one voxel of a constant reference window raised by `step` gives a finite ZNCC and
    the speckle target decides the displacement (8-bit target values tie, which the gap rule allows).  The packed transform
    recovers the reference spectrum with an error of about eps |B|, so the ZNCC error grows as 1 / sqrt(na): a voxel of 255 in
    grey 24 keeps it below 1e-5, one of 25 (na ~ 1 against nb ~ 1e8 at r = 16) leaves about 1e-4."""
    ref, tar = (a.copy() for a in vol)
    ref[CONST_BOX] = synth.BACKGROUND
    ref[54, 62, 70] += step  # inside every window of the queue
    q = _const_queue(r)
    got = _run(engine, ref, tar, q, r)
    _check(_label(r, "constant window but one voxel of +%g" % step), got, q, ref, tar, r, expect_computed=np.ones(len(q), bool),
           ztol=GAP if step > 100 else 3e-4)
    assert np.isfinite(got[:, ZNCC]).all() and (got[:, ZNCC] > 0).all(), got[:, ZNCC]


# ------------------------------------------------------------------------------------------------ persistent CTAs
@pytest.mark.parametrize("r", LONG_R, ids=["r=(%d,%d,%d)" % r for r in LONG_R])
def test_cta_takes_several_pois(engine, vol, device, plan_tool, r):
    """3 x (the plan's CTAs) + 5 POIs: every CTA takes three POIs, the first five a fourth, and reuses its shared memory and its
    scratch volume; skipped POIs (past a face) and constant windows are interleaved.  A shuffled queue gives the permuted records
    and each third run alone the same bits."""
    out = run_plan_tool(plan_tool, device[1], device[0], cases=[r + (0, "", 1)])
    assert out.returncode == 0, out.stdout + out.stderr
    ctas = int(re.search(r"(\d+) CTA\(s\)", out.stdout).group(1))
    ref = vol[0].copy()
    ref[CONST_BOX] = synth.BACKGROUND
    tar = vol[1]
    n = 3 * ctas + 5
    q = _mark(sweep_queue(r, n, seed=n))
    kind = np.arange(n) % 7
    q[kind == 3, 0] = r[0] - 1  # past the x = 0 face: skipped
    const = kind == 5  # both windows inside the constant reference box
    q[const, 0:3] = np.array([70, 62, 54], np.float32) + (np.arange(const.sum()) % 5)[:, None]
    q[const, 3], q[const, 7], q[const, 11] = 1.0, -1.0, 0.0
    label = _label(r, "%d POIs on %d CTAs" % (n, ctas))
    got = _run(engine, ref, tar, q, r)
    computed = _check(label, got, q, ref, tar, r, expect_computed=kind != 3)
    assert np.isnan(got[const, ZNCC]).all()  # _check holds every other NaN to the witnesses
    perm = np.random.default_rng(1).permutation(n)
    shuffled = _run(engine, ref, tar, q[perm], r)
    assert np.array_equal(_bits(shuffled), _bits(got[perm])), "%s: the shuffled queue differs at POIs %s" % (
        label, perm[(_bits(shuffled) != _bits(got[perm])).any(1)][:10])
    for k in range(3):
        part = slice(k * n // 3, (k + 1) * n // 3)
        alone = _run(engine, ref, tar, q[part], r)
        assert np.array_equal(_bits(alone), _bits(got[part])), "%s: third %d differs when run alone" % (label, k)


# ------------------------------------------------------------------------------------------------ near-ties
@pytest.mark.parametrize("rr,axes,generic", TIE_R, ids=["r=%d periodic %s%s" % (r, "".join("xyz"[a] for a in ax), " generic" if g else "")
                                                        for r, ax, g in TIE_R])
def test_near_exact_ties(engine, monkeypatch, rr, axes, generic):
    """Small integer intensities repeated with period r = N / 2 along the given axes: the 2r window holds two periods there, so
    the correlation of a volume with itself has 2^(periodic axes) equal maxima in exact arithmetic, which float32 twiddles
    separate by rounding.  Each kernel must return one of them."""
    r = (rr, rr, rr)
    rng = np.random.default_rng(rr + 10 * len(axes))
    dims = (4 * rr + 32, 4 * rr + 26, 4 * rr + 22)  # x, y, z; a pitch of a multiple of 4 floats: W32 takes TMA boxes
    idx = np.ix_(*[np.arange(dims[a]) % rr if a in axes else np.arange(dims[a]) for a in (2, 1, 0)])
    base = rng.integers(0, 64, (dims[2], dims[1], dims[0])).astype(np.float32)
    img = np.ascontiguousarray(base[idx])
    q = sweep_queue(r, 12, seed=rr, dims=dims)
    q[:, [0, 1, 2, 3, 7, 11]] = np.floor(q[:, [0, 1, 2, 3, 7, 11]])
    q[:, [3, 7, 11]] = 0.0
    if generic:
        monkeypatch.setenv("OCB_FFTCC3D_GENERIC", "1")
    got = _run(engine, img, img, q, r)
    wa, computed, gap, cands = witness(img, img, q, *r)
    assert computed.all() and (gap < GAP).all() and all(len(c) == 2 ** len(axes) for c in cands), [len(c) for c in cands]
    _check(_label(r, "%d-fold tie" % 2 ** len(axes), generic), got, q, img, img, r, expect_computed=np.ones(len(q), bool))


# ------------------------------------------------------------------------------------------------ limits
def test_largest_window_and_rejections(engine, vol, device, plan_tool):
    """The largest cubic window the shared-memory check accepts is in GENERIC_CUBIC; the first one it refuses and windows with a
    prime factor above 31 return an error, leave the queue untouched and leave the engine usable."""
    out = run_plan_tool(plan_tool, "limits", device[1])
    assert out.returncode == 0, out.stdout + out.stderr
    largest, first = (int(v) for v in re.findall(r"\d+", out.stdout))
    if device[1] == 227 * 1024:
        assert (largest, first) == (42, 44) and largest in GENERIC_CUBIC
    ref, tar = vol
    q = _mark(sweep_queue((10, 10, 10), 3, seed=3))
    q[:, [3, 7, 11]] = 0.0
    engine.set_images_3d(ref, tar)
    refused = [(first, "shared memory")] + [(rr, "prime factor") for rr, why in REJECTED if why == "prime factor"]
    for rr, why in refused:
        bad = q.copy()
        with pytest.raises(_capi.OpenCorrB200Error) as e:
            engine.fftcc3d(bad, rr, rr, rr)
        assert e.value.code == _capi.OCB_ERR_UNSUPPORTED and why in str(e.value), (rr, str(e.value))
        assert np.array_equal(_bits(bad), _bits(q)), "a refused call wrote to the queue"
        again = q.copy()
        engine.fftcc3d(again, 10, 10, 10)  # the engine is still usable
        assert (again[:, ZNCC] > 0.5).all()
        print("FFTCC3D r=(%d,%d,%d): refused, %s" % (rr, rr, rr, e.value))
