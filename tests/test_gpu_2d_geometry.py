"""GPU: ICGN2D1/2, ICLM2D1/2 and NR2D1 at every launch geometry and sampling path they select, against the float64 oracle
(Oracle2D, exact=1).

ocb::icgn2d_plan (opencorr_b200/csrc/ocb_kernels.h) picks the pair kernel icgn2d_kernel<NP, RC, LM, WPP> and its grid from the
subset radii and the queue length, ocb::nr2d1_plan the warps per NR2D1 CTA; test_icgn2d_plan_host.py checks on the CPU that
every case below lands in the branch it is meant to cover (each of the twelve instantiations, idle lanes, tail columns, every
rolling-window remainder in both warps of a POI, NR2D1 CTAs of 4, 2 and 1 warps, rejection).  Inside a kernel a pass takes the
whole-pixel shortcut (a whole-pixel seed), the rolling 4x4 window (a fractional seed), the 12-parameter loop, or the checked loop
with its per-sample fallback to global memory (sheared targets, samples outside the image); the cases below reach each of them.
Warps per POI are forced with OCB_ICGN2D_WPP, so that no record depends on the SM count.

Tolerances (those of test_gpu_3d_geometry.py): 1e-4 px and 1e-5 ZNCC (all 6 or 12 parameters within 1e-4) on POIs whose
iteration counts agree; at most max(1, 2 %) POIs per case may take one iteration more or less (||dp|| within float noise of the
convergence criterion).  ICLM2D: the last step's `znssd < znssd0` test at convergence is decided by rounding (see
test_gpu_2d.py::_iclm_compare), so a POI whose accepted-step sequence differs counts against the same budget and is held to the
convergence criterion.  NR2D1: util.nr_compare.  The -3 decisions of ICGN2D (a sample outside the image, or below zero) follow the
reference's float arithmetic and are compared with the exact=0 oracle.  Each case prints one line with its largest deviations."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import opencorr_b200 as ob
from opencorr_b200 import synth
from oracle.oracle import Oracle2D
import util

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
W = H = 512
CONV, STOP = 0.001, 20


# ------------------------------------------------------------------------------------------------ the launch plans
def build_plan_tool(out_dir):
    """Compiles tests/native/icgn2d_plan_host_test.cpp (the plan functions of ocb_kernels.h, host only) into out_dir."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    exe = os.path.join(out_dir, "icgn2d_plan_host_test")
    cmd = [nvcc, "-x", "cu", "-std=c++17", "-O1", "-Wno-deprecated-gpu-targets", "-I", os.path.join(ROOT, "opencorr_b200", "csrc"),
           "-o", exe, os.path.join(ROOT, "tests", "native", "icgn2d_plan_host_test.cpp")]
    if os.path.exists("/usr/bin/g++"):
        cmd[1:1] = ["-ccbin", "/usr/bin/g++"]
    build = subprocess.run(cmd, capture_output=True, text=True)
    assert build.returncode == 0, "nvcc failed:\n" + build.stdout + build.stderr
    return exe


def run_plan_tool(exe, *args):
    return subprocess.run([exe] + [str(a) for a in args], capture_output=True, text=True, timeout=60)


# (kind, order, (rx, ry), POIs, warps per POI: 1 or 2 forced, 0 automatic)
SWEEP = ([("icgn", 1, r, n, w) for r, n in (((4, 4), 32), ((5, 6), 32), ((6, 7), 32), ((7, 5), 32), ((15, 15), 32), ((16, 16), 32),
                                             ((16, 15), 32), ((24, 9), 24), ((40, 40), 8)) for w in (1, 2)]
         + [("icgn", 1, (20, 2), 32, w) for w in (0, 2)]  # 5 rows: the automatic choice is one warp
         + [("icgn", 2, r, n, w) for r, n in (((20, 20), 24), ((20, 19), 24), ((11, 11), 32), ((33, 8), 16)) for w in (1, 2)]
         + [("lm", o, r, 32, w) for o in (1, 2) for r in ((12, 12), (17, 17)) for w in (1, 2)])
SHEAR = [("icgn", 1, (16, 16)), ("icgn", 1, (11, 11)), ("icgn", 2, (20, 20)), ("lm", 1, (12, 12))]
OFFSETS = [(1, (15, 15)), (2, (20, 20))]
EDGE_R = (14, 14)
NEGATIVE = [(1, (11, 11)), (2, (20, 20))]
LARGE_XY = [("icgn", 2, (18, 18)), ("lm", 1, (16, 16))]
AUTO_R = (40, 40)
NR_SWEEP = [(4, 4), (8, 8), (12, 12), (16, 16), (18, 18), (20, 20), (24, 9), (40, 40)]
NR_SHEAR_R = (14, 14)

# every (NP, rx, ry, LM, WPP) the cases run, and every NR2D1 radius; the largest accepted radii are derived from the plans at
# run time and checked against the H100 table by the plan test itself
ICGN2D_PLAN_CASES = sorted(set(
    [(6 * o, *r, int(k == "lm"), w) for k, o, r, _, w in SWEEP]
    + [(6 * o, *r, int(k == "lm"), w) for k, o, r in SHEAR for w in (1, 2)]
    + [(6 * o, *r, 0, w) for o, r in OFFSETS for w in (1, 2)]
    + [(6 * o, *EDGE_R, lm, 2) for o in (1, 2) for lm in (0, 1)]
    + [(6 * o, *r, 0, 2) for o, r in NEGATIVE]
    + [(6 * o, *r, int(k == "lm"), 2) for k, o, r in LARGE_XY]
    + [(6, *AUTO_R, 0, 0)]))
NR2D_PLAN_CASES = NR_SWEEP + [NR_SHEAR_R, EDGE_R]


@pytest.fixture(scope="module")
def device():
    torch = pytest.importorskip("torch")
    p = torch.cuda.get_device_properties(0)
    return p.multi_processor_count, p.shared_memory_per_block_optin


@pytest.fixture(scope="module")
def plan_tool(tmp_path_factory):
    return build_plan_tool(str(tmp_path_factory.mktemp("plan")))


def _query(plan_tool, device, r, lm):
    out = run_plan_tool(plan_tool, "query", device[1], r[0], r[1], int(lm))
    assert out.returncode == 0, out.stdout + out.stderr
    q = {m[0]: int(m[1]) for m in re.findall(r"^(.*): (\d+)$", out.stdout, re.M)}
    return q


# ------------------------------------------------------------------------------------------------ images and queues
@pytest.fixture(scope="module")
def pair1():
    return synth.speckle_pair_2d(W, H)


@pytest.fixture(scope="module")
def pair2():
    return synth.speckle_pair_2d(W, H, second_order=True)


def _pois(r, n, seed, margin=6, w=W, h=H):
    """n integer POIs whose subset (and its image under the synthetic displacement) is inside."""
    rng = np.random.default_rng(seed)
    x = rng.integers(r[0] + margin, w - 1 - r[0] - margin, n, endpoint=True)
    y = rng.integers(r[1] + margin, h - 1 - r[1] - margin, n, endpoint=True)
    return np.stack([x, y], 1).astype(np.float32)


def _seed(xy, order, w=W, h=H, x0=0, y0=0):
    """Even POIs: the whole-pixel seed FFT-CC returns (the rounded true displacement), whose first pass takes the whole-pixel
    shortcut.  Odd POIs: a fractional seed with small ux and vy, which takes the interpolating loops from the first pass."""
    q = ob.make_poi2d(xy)
    u, v = synth.displacement_2d(xy[:, 0] - x0, xy[:, 1] - y0, w, h, second_order=(order == 2))
    frac = np.arange(len(xy)) % 2 == 1
    q[:, 2], q[:, 8] = np.round(u), np.round(v)
    q[frac, 2], q[frac, 8] = u[frac] + 0.21, v[frac] - 0.17
    q[frac, 3], q[frac, 10] = 2e-3, -1e-3
    return q


def _set_wpp(monkeypatch, wpp):
    if wpp:
        monkeypatch.setenv("OCB_ICGN2D_WPP", str(wpp))
    else:
        monkeypatch.delenv("OCB_ICGN2D_WPP", raising=False)


def _gpu(engine, kind, order, ref, tar, q, r, offsets=None):
    engine.set_images_2d(ref, tar)
    if kind == "nr":
        engine.nr2d_prepare()
        engine.nr2d1(q, r[0], r[1], CONV, STOP)
        return q
    engine.icgn2d_prepare()
    if kind == "lm":
        engine.iclm2d(order, q, r[0], r[1], CONV, STOP)
    elif offsets is not None:
        engine.icgn2d_ex(order, q, r[0], r[1], CONV, STOP, center_offsets=offsets)
    else:
        (engine.icgn2d1 if order == 1 else engine.icgn2d2)(q, r[0], r[1], CONV, STOP)
    return q


def _oracle(o, kind, order, q, r, offsets=None, exact=True):
    if kind == "nr":
        return o.nr2d1(q, r[0], r[1], CONV, STOP, exact=exact)
    if kind == "lm":
        return o.iclm2d(order, q, r[0], r[1], CONV, STOP, exact=exact)
    if offsets is not None:
        return o.icgn2d_ex(order, q, r[0], r[1], CONV, STOP, center_offsets=offsets, exact=exact)
    return (o.icgn2d1 if order == 1 else o.icgn2d2)(q, r[0], r[1], CONV, STOP, exact=exact)


def _check(a, b, kind, order, label, min_valid=0.75, tol=1e-4):
    """a: GPU records, b: exact oracle records (POI2D [n, 25])."""
    n = len(a)
    if kind == "nr":
        d, dz = util.nr_compare(a, b, label, tol=tol)
        ok = (a[:, 17] == b[:, 17]) & (a[:, 16] >= 0) & (b[:, 16] >= 0)
        assert ok.sum() >= min_valid * n, "%s: only %d of %d POIs compared" % (label, ok.sum(), n)
        print("%s: n=%d compared=%d max|ddisp|=%.2e max|dZNCC|=%.2e" % (label, n, ok.sum(), d, dz))
        return
    budget = max(1.0, 0.02 * n)
    cols = [2, 3, 4, 8, 9, 10] if order == 1 else list(range(2, 14))
    same_it = a[:, 17] == b[:, 17]
    valid = (a[:, 16] >= 0) & (b[:, 16] >= 0)
    flips = int((~same_it).sum())
    accept_flips = 0
    if kind == "lm":
        # a different accept/reject sequence at convergence: same iteration count, displacement apart by up to the criterion
        far = same_it & valid & (np.abs(a[:, [2, 8]] - b[:, [2, 8]]).max(1) > tol)
        accept_flips = int(far.sum())
        if far.any():
            assert np.abs(a[far][:, [2, 8]] - b[far][:, [2, 8]]).max() < 1.5e-3, label
            assert np.abs(a[far, 16] - b[far, 16]).max() < 1e-4, label
        a, b = a[~far], b[~far]
        same_it, valid = same_it[~far], valid[~far]
    # the flip budget as a count (a fraction such as 1 - 35/36 can round above 1/36); compare_2d bounds each flip's deviation
    assert flips + accept_flips <= budget, "%s: %d iteration and %d acceptance flips in %d POIs" % (label, flips, accept_flips, n)
    stats = util.compare_2d(a, b, label, tol_disp=tol, max_iter_mismatch_frac=1.0, order=order)
    ok = valid & same_it
    dp = np.abs(a[ok][:, cols] - b[ok][:, cols]).max() if ok.any() else 0.0
    assert dp < tol, "%s: max |d parameter| = %.3g" % (label, dp)
    assert ok.sum() >= min_valid * n, "%s: only %d of %d POIs compared" % (label, ok.sum(), n)
    print("%s: n=%d compared=%d max|ddisp|=%.2e max|dparam|=%.2e max|dZNCC|=%.2e flips=%d%s"
          % (label, n, ok.sum(), stats["max_disp"], dp, stats["max_zncc"], flips, " acceptance flips=%d" % accept_flips if kind == "lm" else ""))


def _name(kind, order):
    return {"icgn": "ICGN2D%d" % order, "lm": "ICLM2D%d" % order, "nr": "NR2D1"}[kind]


def _label(kind, order, r, wpp=None):
    s = "%s r=(%d,%d)" % (_name(kind, order), r[0], r[1])
    return s if wpp is None else s + " wpp=%s" % (wpp or "auto")


# ------------------------------------------------------------------------------------------------ radius sweep
@pytest.mark.parametrize("kind,order,r,n,wpp", SWEEP, ids=[_label(k, o, r, w) for k, o, r, _, w in SWEEP])
def test_radius_sweep(engine, pair1, pair2, monkeypatch, kind, order, r, n, wpp):
    ref, tar = pair1 if order == 1 else pair2
    q = _seed(_pois(r, n, seed=31 * r[0] + r[1]), order)
    _set_wpp(monkeypatch, wpp)
    a = _gpu(engine, kind, order, ref, tar, q.copy(), r)
    b = _oracle(Oracle2D(ref, tar), kind, order, q.copy(), r)
    _check(a, b, kind, order, _label(kind, order, r, wpp))


@pytest.mark.parametrize("r", NR_SWEEP, ids=lambda r: "r=(%d,%d)" % r)
def test_nr2d1_radius_sweep(engine, pair1, r):
    ref, tar = pair1
    q = _seed(_pois(r, 64, seed=17 * r[0] + r[1]), 1)
    a = _gpu(engine, "nr", 1, ref, tar, q.copy(), r)
    b = _oracle(Oracle2D(ref, tar), "nr", 1, q.copy(), r)
    _check(a, b, "nr", 1, _label("nr", 1, r))


# ------------------------------------------------------------------------------------------------ largest and rejected subsets
def test_largest_accepted_and_first_rejected_subsets(engine, monkeypatch, plan_tool, device):
    """The largest square subsets the plans accept on this device run (2r + 1 = 117 on an H100: 85 tail columns); one pixel
    more raises without touching the queue."""
    ref, tar = synth.speckle_pair_2d(256, 256)
    xy = np.array([[128, 128], [126, 131], [131, 126]], np.float32)
    q = ob.make_poi2d(xy)
    u, v = synth.displacement_2d(xy[:, 0], xy[:, 1], 256, 256)
    q[:, 2], q[:, 8] = np.round(u), np.round(v)
    o = Oracle2D(ref, tar)
    for kind, order in (("icgn", 1), ("icgn", 2), ("lm", 1)):
        lm = kind == "lm"
        lim = _query(plan_tool, device, (1, 1), lm)
        for wpp in (1, 2):
            rr = lim["largest icgn2d lm=%d wpp=%d" % (lm, wpp)]
            assert rr >= 40
            _set_wpp(monkeypatch, wpp)
            a = _gpu(engine, kind, order, ref, tar, q.copy(), (rr, rr))
            b = _oracle(o, kind, order, q.copy(), (rr, rr))
            _check(a, b, kind, order, "largest " + _label(kind, order, (rr, rr), wpp), min_valid=1.0)
        _set_wpp(monkeypatch, 0)
        rr = lim["largest icgn2d lm=%d wpp=1" % lm] + 1
        q0 = q.copy()
        with pytest.raises(ob.OpenCorrB200Error, match="exceeds the shared-memory design limit"):
            _gpu(engine, kind, order, ref, tar, q0, (rr, rr))
        assert q0.tobytes() == q.tobytes()
    rr = _query(plan_tool, device, (1, 1), False)["largest nr2d1"]
    a = _gpu(engine, "nr", 1, ref, tar, q.copy(), (rr, rr))
    b = _oracle(o, "nr", 1, q.copy(), (rr, rr))
    _check(a, b, "nr", 1, "largest " + _label("nr", 1, (rr, rr)), min_valid=1.0)
    q0 = q.copy()
    with pytest.raises(ob.OpenCorrB200Error, match="exceeds the shared-memory design limit"):
        _gpu(engine, "nr", 1, ref, tar, q0, (rr + 1, rr + 1))
    assert q0.tobytes() == q.tobytes()


# ------------------------------------------------------------------------------------------------ automatic warps per POI
def test_automatic_warps_per_poi(engine, pair1, monkeypatch, plan_tool, device):
    """Two warps per POI only while the queue is shorter than the one-warp slots of the whole GPU (sm_count x slots(1))."""
    ref, tar = pair1
    full = device[0] * _query(plan_tool, device, AUTO_R, False)["slots r=(%d,%d) lm=0 wpp=1" % AUTO_R]
    for n, forced in ((full - 1, 2), (full, 1)):
        q = _seed(_pois(AUTO_R, n, seed=n), 1)
        _set_wpp(monkeypatch, 0)
        auto = _gpu(engine, "icgn", 1, ref, tar, q.copy(), AUTO_R)
        _set_wpp(monkeypatch, forced)
        same = _gpu(engine, "icgn", 1, ref, tar, q.copy(), AUTO_R)
        _set_wpp(monkeypatch, 3 - forced)
        other = _gpu(engine, "icgn", 1, ref, tar, q.copy(), AUTO_R)
        assert auto.tobytes() == same.tobytes(), "%d POIs: the automatic choice is not %d warp(s) per POI" % (n, forced)
        assert auto.tobytes() != other.tobytes()  # the records tell the two apart
        print("auto r=(%d,%d): %d POIs -> %d warp(s) per POI" % (AUTO_R + (n, forced)))


# ------------------------------------------------------------------------------------------------ shear
G_BASE = np.array([[0.03, -0.025], [0.02, 0.035]])
T_TRUE = np.array([1.4, -0.8])
SHEAR_REACH = 2.0  # px by which the shear moves a subset corner beyond the translated subset


def _shear_g(r):
    return G_BASE * SHEAR_REACH / (np.abs(G_BASE).sum(1).max() * r[0])


def _sheared_target(ref, g):
    """Target = reference resampled (oracle bicubic) under x' = c + t + (I + G)(x - c), all four gradients non-zero."""
    o = Oracle2D(ref, ref)
    o.prepare()
    h, w = ref.shape
    c = np.array([0.5 * (w - 1), 0.5 * (h - 1)])
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    dst = np.stack([xx.ravel(), yy.ravel()], 1)
    src = (dst - c - T_TRUE) @ np.linalg.inv(np.eye(2) + g).T + c
    tar = o.bicubic(src.astype(np.float32)).reshape(h, w)
    return np.where(tar < 0, synth.BACKGROUND, tar).astype(np.float32)  # -1: source point outside the reference


def _shear_queue(r, n, g, w, h):
    xy = _pois(r, n, seed=7 * r[0], margin=14, w=w, h=h)
    c = np.array([0.5 * (w - 1), 0.5 * (h - 1)])
    q = ob.make_poi2d(xy)
    disp = T_TRUE + (xy - c) @ g.T
    true_map = np.arange(n) % 2 == 0
    disp[~true_map] = np.round(disp[~true_map])  # an FFT-CC-like start
    q[:, 2], q[:, 8] = disp[:, 0], disp[:, 1]
    q[true_map, 3], q[true_map, 4], q[true_map, 9], q[true_map, 10] = g[0, 0], g[0, 1], g[1, 0], g[1, 1]
    return q


def _tile_replay(q, r, w, h, nr=False):
    """Replays the target-tile placement of icgn2d.cu (tx0, ty0, TW, TH, the warp-wide corner test) or nr2d.cu (the gradient
    tile's fast region) at the warp each POI starts from.  Returns the number of POIs that fail the corner test and the number
    of samples outside the tile's fast region but inside the image, which the kernels read from global memory."""
    rx, ry = r
    margin = 1  # ICGN2D_TILE_MARGIN, NR2D_TILE_MARGIN
    corner_fail = samples_out = 0
    yl, xl = np.mgrid[-ry:ry + 1, -rx:rx + 1].astype(np.float64)
    for p in q.astype(np.float64):
        px, py, u, ux, uy, v, vx, vy = p[0], p[1], p[2], p[3], p[4], p[8], p[9], p[10]
        if nr:
            tx0 = (int(np.floor(px + u)) - rx - 1 - margin - 2) & ~3
            ty0 = int(np.floor(py + v)) - ry - 1 - margin - 2
            tw, th = (2 * rx + 1 + 3 + 2 * margin + 4 + 3 + 3) & ~3, 2 * ry + 1 + 3 + 2 * margin + 4
            x0, y0, tw, th = tx0 + 2, ty0 + 2, tw - 4, th - 4  # the gradient tile
        else:
            x0 = (int(np.floor(px + u)) - rx - 1 - margin) & ~3
            y0 = int(np.floor(py + v)) - ry - 1 - margin
            tw, th = (2 * rx + 1 + 3 + 2 * margin + 3 + 3) & ~3, 2 * ry + 1 + 3 + 2 * margin
        xlo, xhi = max(1.0, x0 + 1.0), min(w - 2.0, x0 + tw - 2.0)
        ylo, yhi = max(1.0, y0 + 1.0), min(h - 2.0, y0 + th - 2.0)
        ex, ey = abs(1 + ux) * rx + abs(uy) * ry, abs(vx) * rx + abs(1 + vy) * ry
        if not (px + u - ex >= xlo and px + u + ex < xhi and py + v - ey >= ylo and py + v + ey < yhi):
            corner_fail += 1
        X = px + (1 + ux) * xl + uy * yl + u
        Y = py + vx * xl + (1 + vy) * yl + v
        fast = (X >= xlo) & (X < xhi) & (Y >= ylo) & (Y < yhi)
        inside = (X >= 1) & (Y >= 1) & (X < w - 2) & (Y < h - 2)
        samples_out += int((~fast & inside).sum())
    return corner_fail, samples_out


@pytest.fixture(scope="module")
def shear_targets(pair1):
    return {r[0]: _sheared_target(pair1[0], _shear_g(r)) for r in [r for _, _, r in SHEAR] + [NR_SHEAR_R]}


@pytest.mark.parametrize("wpp", [1, 2])
@pytest.mark.parametrize("kind,order,r", SHEAR, ids=[_label(k, o, r) for k, o, r in SHEAR])
def test_shear_tma_and_staged_loads(engine, pair1, shear_targets, monkeypatch, kind, order, r, wpp):
    """Off-diagonal gradients move samples out of the staged target tile (whose origin follows the translation only): the
    corner test fails and the checked loop reads those samples from global memory.  Half the POIs start at the true map, half
    at the rounded translation.  TMA and staged (OCB_NO_TMA) tile loads must give identical records."""
    ref, tar, g = pair1[0], shear_targets[r[0]], _shear_g(r)
    n = 16
    q = _shear_queue(r, n, g, W, H)
    corner_fail, samples_out = _tile_replay(q, r, W, H)
    assert corner_fail >= 1 and samples_out >= 1, (corner_fail, samples_out)
    _set_wpp(monkeypatch, wpp)
    a = _gpu(engine, kind, order, ref, tar, q.copy(), r)
    monkeypatch.setenv("OCB_NO_TMA", "1")
    s = _gpu(engine, kind, order, ref, tar, q.copy(), r)
    monkeypatch.delenv("OCB_NO_TMA")
    assert a.tobytes() == s.tobytes(), "TMA and staged tile loads differ"
    b = _oracle(Oracle2D(ref, tar), kind, order, q.copy(), r)
    label = "shear " + _label(kind, order, r, wpp)
    print("%s: %d POIs fail the corner test, %d samples outside the tile at the starting warps" % (label, corner_fail, samples_out))
    _check(a, b, kind, order, label, min_valid=0.5)
    ok = a[:, 16] > 0.9
    assert ok.sum() >= n // 2
    assert np.abs(a[ok][:, [3, 4, 9, 10]] - g.ravel()).max() < 2e-3  # the shear is recovered


def test_nr2d1_shear_tma_and_staged_loads(engine, pair1, shear_targets, monkeypatch):
    r = NR_SHEAR_R
    ref, tar, g = pair1[0], shear_targets[r[0]], _shear_g(r)
    n = 64
    q = _shear_queue(r, n, g, W, H)
    _, samples_out = _tile_replay(q, r, W, H, nr=True)
    assert samples_out >= 1, samples_out
    a = _gpu(engine, "nr", 1, ref, tar, q.copy(), r)
    monkeypatch.setenv("OCB_NO_TMA", "1")
    s = _gpu(engine, "nr", 1, ref, tar, q.copy(), r)
    monkeypatch.delenv("OCB_NO_TMA")
    assert a.tobytes() == s.tobytes(), "TMA and staged tile loads differ"
    b = _oracle(Oracle2D(ref, tar), "nr", 1, q.copy(), r)
    label = "shear " + _label("nr", 1, r)
    print("%s: %d samples outside the tile at the starting warps" % (label, samples_out))
    _check(a, b, "nr", 1, label, min_valid=0.5)
    ok = a[:, 16] > 0.9
    assert ok.sum() >= n // 2
    assert np.abs(a[ok][:, [3, 4, 9, 10]] - g.ravel()).max() < 2e-3


# ------------------------------------------------------------------------------------------------ centre offsets
@pytest.mark.parametrize("wpp", [1, 2])
@pytest.mark.parametrize("order,r", OFFSETS, ids=[_label("icgn", o, r) for o, r in OFFSETS])
def test_center_offsets(engine, pair1, pair2, monkeypatch, order, r, wpp):
    """compute(queue, center_offset_queue) with non-integral offsets: local coordinates (integer - offset), target subset centred
    at poi + offset."""
    ref, tar = pair1 if order == 1 else pair2
    xy = _pois(r, 32, seed=5 * r[0], margin=10)
    off = np.random.default_rng(r[0]).uniform(-3, 3, (len(xy), 2)).astype(np.float32)
    q = _seed(xy, order)
    _set_wpp(monkeypatch, wpp)
    a = _gpu(engine, "icgn", order, ref, tar, q.copy(), r, offsets=off)
    b = _oracle(Oracle2D(ref, tar), "icgn", order, q.copy(), r, offsets=off)
    _check(a, b, "icgn", order, "offsets " + _label("icgn", order, r, wpp))


# ------------------------------------------------------------------------------------------------ samples outside the image
MARGIN_EDGE = 0.15  # px: no sample of a designed border case lies closer than this to a validity boundary under the true map


def _edge_queue(r, order):
    """POIs along the right and top borders, where the true displacement (u ~ +2.4, v ~ -1.6 px) carries some subset columns or
    rows outside [1, w - 2) x [1, h - 2), and POIs just inside; every sample at least MARGIN_EDGE px from the boundaries, so
    that the reference's float arithmetic and the float64 oracle agree on which samples are outside."""
    rx, ry = r
    yl, xl = np.mgrid[-ry:ry + 1, -rx:rx + 1].astype(np.float64)
    cand = [(x, y) for x in range(W - 1 - rx - 8, W - rx) for y in (150, 260, 371)]
    cand += [(x, y) for y in range(ry, ry + 9) for x in (140, 255, 366)]
    keep = []
    for x, y in cand:
        u, v = synth.displacement_2d(x + xl, y + yl, W, H, second_order=(order == 2))
        X, Y = x + xl + u, y + yl + v
        dist = min(np.abs(X - 1).min(), np.abs(X - (W - 2)).min(), np.abs(Y - 1).min(), np.abs(Y - (H - 2)).min())
        if dist >= MARGIN_EDGE:
            keep.append((x, y, bool((X >= W - 2).any() or (Y < 1).any())))
    keep = np.array(keep)
    out, inside = keep[keep[:, 2] == 1][:, :2], keep[keep[:, 2] == 0][:, :2]
    assert len(out) >= 4 and len(inside) >= 2, (len(out), len(inside))
    xy = np.vstack([out[::max(1, len(out) // 12)], inside[::max(1, len(inside) // 6)], _pois(r, 8, seed=3)]).astype(np.float32)
    q = ob.make_poi2d(xy)
    u, v = synth.displacement_2d(xy[:, 0], xy[:, 1], W, H, second_order=(order == 2))
    q[:, 2], q[:, 8] = u, v
    q[:, 3], q[:, 4], q[:, 9], q[:, 10] = 1.5e-3, -0.8e-3, 0.6e-3, 2.1e-3
    return q, len(out[::max(1, len(out) // 12)])


@pytest.mark.parametrize("order", [1, 2])
def test_samples_outside_the_image(engine, pair1, pair2, monkeypatch, order):
    """ICGN2D rejects a POI with -3 as soon as a sample leaves the image (decided like the exact=0 oracle); ICLM2D uses the
    interpolant's -1 as the sample value and must match the oracle, as must NR2D1 (order 1)."""
    ref, tar = pair1 if order == 1 else pair2
    r = EDGE_R
    q, n_out = _edge_queue(r, order)
    o = Oracle2D(ref, tar)
    _set_wpp(monkeypatch, 2)
    a = _gpu(engine, "icgn", order, ref, tar, q.copy(), r)
    e0 = _oracle(o, "icgn", order, q.copy(), r, exact=False)
    rej = e0[:, 16] == -3
    assert np.array_equal(a[:, 16] == -3, rej), "-3 decided differently at POIs %s" % np.where((a[:, 16] == -3) != rej)[0]
    assert rej[:n_out].all() and rej.sum() == n_out
    assert np.array_equal(a[rej], e0[rej])  # rejected records are left untouched apart from the code
    b = _oracle(o, "icgn", order, q.copy(), r)
    _check(a[~rej], b[~rej], "icgn", order, "edges " + _label("icgn", order, r, 2), min_valid=0.9)
    kinds = [("lm", order)] + ([("nr", 1)] if order == 1 else [])
    for kind, k_order in kinds:
        a = _gpu(engine, kind, k_order, ref, tar, q.copy(), r)
        b = _oracle(o, kind, k_order, q.copy(), r)
        assert (a[:n_out, 16] >= 0).mean() >= 0.5  # the POIs that leave the image are kept and fitted with -1 samples
        _check(a, b, kind, k_order, "edges " + _label(kind, k_order, r, 2 if kind == "lm" else None), min_valid=0.75)


# ------------------------------------------------------------------------------------------------ the exact-negative rescan
@pytest.mark.parametrize("order,r", NEGATIVE, ids=[_label("icgn", o, r) for o, r in NEGATIVE])
def test_negative_sample_rule_away_from_r16(engine, monkeypatch, order, r):
    """Black regions: the `any interpolated sample < 0 -> -3` rule (re-decided in the reference's arithmetic by
    icgn2d_exact_negative when the smallest sample is borderline) must reject exactly the POIs the exact=0 oracle rejects."""
    from test_gpu_sentinel import patterns_2d
    _set_wpp(monkeypatch, 2)
    seen_rej = seen_kept = 0
    for name, ref, tar in patterns_2d():
        q = ob.make_poi2d(synth.grid_2d(40, 40, 20, 20, 22, 22))
        o = Oracle2D(ref, tar)
        o.fftcc2d(q, 16, 16)
        a = _gpu(engine, "icgn", order, ref, tar, q.copy(), r)
        e0 = _oracle(o, "icgn", order, q.copy(), r, exact=False)
        rej = e0[:, 16] == -3
        differ = np.where((a[:, 16] == -3) != rej)[0]
        assert len(differ) == 0, "%s %s: -3 decided differently at POIs %s" % (name, _label("icgn", order, r), differ[:10])
        assert np.array_equal(a[rej], e0[rej])
        seen_rej += int(rej.sum())
        seen_kept += int((~rej).sum())
    print("negative %s: %d rejected, %d kept" % (_label("icgn", order, r, 2), seen_rej, seen_kept))
    assert seen_rej >= 20 and seen_kept >= 20


# ------------------------------------------------------------------------------------------------ large coordinates
@pytest.fixture(scope="module")
def far_pair():
    """3080 x 3080 pixels: a 200 x 200 speckle block at x, y = 2880..3079 in a uniform background."""
    rb, tb = synth.speckle_pair_2d(200, 200)
    ref = np.full((3080, 3080), synth.BACKGROUND, np.float32)
    tar = ref.copy()
    ref[2880:, 2880:], tar[2880:, 2880:] = rb, tb
    return ref, tar


@pytest.mark.parametrize("kind,order,r", LARGE_XY, ids=[_label(k, o, r) for k, o, r in LARGE_XY])
def test_large_image_coordinates(engine, far_pair, monkeypatch, kind, order, r):
    """x, y ~ 3000: a float ulp is 2.4e-4 px there, so the order `centre + warped offset` matters."""
    ref, tar = far_pair
    k = 2880 + np.arange(30, 171, 28)
    xy = np.stack(np.meshgrid(k, k), -1).reshape(-1, 2).astype(np.float32)
    q = _seed(xy, 1, w=200, h=200, x0=2880, y0=2880)
    _set_wpp(monkeypatch, 2)
    a = _gpu(engine, kind, order, ref, tar, q.copy(), r)
    b = _oracle(Oracle2D(ref, tar), kind, order, q.copy(), r)
    _check(a, b, kind, order, "large xy " + _label(kind, order, r, 2), tol=1.5e-4)
