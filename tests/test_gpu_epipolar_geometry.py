"""GPU: EpipolarSearch (opencorr_b200/csrc/epipolar.cu, ocb_epipolar_search2d[_dev]) at every slot count, IC-GN geometry, tile load
and candidate-block boundary it meets, against the float64 witness of tests/epipolar_cases.py (pinned to the oracle by
test_epipolar_witness_host.py).

The candidate queue of a block of POIs reaches the ordinary ICGN2D1 launch, so its plan (icgn2d_plan: the RC = 16 kernel and its
whole-pixel first pass for rx = ry = 16, warps per POI from the candidate count or OCB_ICGN2D_WPP, TMA or the gather path) is the
plan of n * slots records.  Slots that fail the border test carry ZNCC = -inf, which the IC-GN guard leaves alone in every
kernel and which never wins the selection.

Pass rule (that of test_gpu_fftcc2d_geometry.py and util.compare_2d): u0, v0 are bit-identical to the witness on every POI whose
best ZNCC stands more than GAP = 1e-5 above the runner-up; a POI with a smaller gap may return any slot within GAP of the best
(two candidates that converge to the same point), and is then compared with the witness's record of that slot.  Parameters agree
within 1e-4 px and ZNCC within 1e-5 where the iteration counts agree, sentinel codes exactly, at most max(1, 2 %) POIs take one
iteration more or less; fields 0, 1 and 20-24 keep their bytes.  Each case prints one line: slots, IC-GN plan, POIs compared and
the worst deviations.

Vertical epipolar lines (e[1] == 0) are out of scope: the reference converts an infinite or NaN float to int there (undefined
behaviour), so there is nothing to match."""
import ctypes
import os

import numpy as np
import pytest

import opencorr_b200 as ob
from opencorr_b200 import _capi, synth
import epipolar_cases as ec
import util
from test_epipolar_witness_host import rig_fundamental

pytestmark = pytest.mark.gpu

W, H = 512, 384
CONV, STOP = 0.001, 10
KEEP = [0, 1, 20, 21, 22, 23, 24]


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _vp(a):
    return ctypes.c_void_p(a.ctypes.data) if a is not None else None


@pytest.fixture(scope="module")
def pair():
    return synth.speckle_pair_2d(W, H)


@pytest.fixture(scope="module")
def pair_odd():
    return synth.speckle_pair_2d(W - 2, H)  # width % 4 != 0: no tensor map, the gather path


@pytest.fixture(scope="module")
def rig():
    w, h = 448, 384
    xy = synth.grid_2d(60, 50, 8, 7, 45, 45)
    d = synth.speckle_stereo_series(w, h, 1, points=xy)
    return d, rig_fundamental(w, h), xy


@pytest.fixture(scope="module")
def sm_slots():
    """(SM count, ICGN2D one-warp slots per SM for a radius): what the unforced warps-per-POI choice depends on."""
    torch = pytest.importorskip("torch")
    p = torch.cuda.get_device_properties(0)
    from test_gpu_2d_geometry import build_plan_tool, run_plan_tool
    import tempfile
    exe = build_plan_tool(tempfile.mkdtemp())

    def slots(rx, ry):
        out = run_plan_tool(exe, "query", p.shared_memory_per_block_optin, rx, ry, 0)
        line = [ln for ln in out.stdout.splitlines() if ln.startswith("slots r=")][0]
        return int(line.rsplit(":", 1)[1])
    return p.multi_processor_count, slots


def _plan(sm_slots, n_cand, rx, ry, w):
    rc = 16 if (rx, ry) == (16, 16) else 0
    forced = os.environ.get("OCB_ICGN2D_WPP")
    if forced in ("1", "2"):
        wpp = int(forced)
    else:
        sm, slots = sm_slots
        wpp = 2 if n_cand < sm * slots(rx, ry) and 2 * ry + 1 >= 8 else 1
    load = "gather" if os.environ.get("OCB_NO_TMA") or (w * 4) % 16 else "TMA"
    return "RC=%d wpp=%d%s %s" % (rc, wpp, "" if forced else " (auto)", load)


def _search(engine, ref, tar, q, F, par_x, par_y, radius, step, rx, ry, conv=CONV, stop=STOP):
    engine.set_images_2d(ref, tar)
    engine.icgn2d_prepare()
    got = q.copy()
    engine.epipolar_search2d(got, F, par_x, par_y, radius, step, rx, ry, conv, stop)
    return got


def _check(label, got, q, ref, tar, F, par_x, par_y, radius, step, rx, ry, conv=CONV, stop=STOP, plan="", min_decisive=0.5, oracle=None):
    """Holds the GPU's records `got` for the queue q to the witness (module docstring).  Returns the witness's (out, gap, valid)."""
    out, gap, near, cand, valid = ec.witness(ref, tar, q, F, par_x, par_y, radius, step, rx, ry, conv, stop, oracle=oracle)
    assert np.array_equal(_bits(got[:, KEEP]), _bits(q[:, KEEP])), "%s: a field EpipolarSearch does not own changed" % label
    dec = gap > ec.GAP
    expect = out.copy()
    for i in np.flatnonzero(~dec):
        pick = [s for s in near[i] if got[i, 14] == cand[i, s, 14] and got[i, 15] == cand[i, s, 15]]
        assert pick, "%s: POI %d returned the slot seeded at (%g, %g), not one of the tied maxima %s" % (
            label, i, got[i, 14], got[i, 15], sorted(near[i]))
        expect[i, 2:20] = cand[i, pick[0], 2:20]
    bad = np.flatnonzero(dec & ((got[:, 14] != out[:, 14]) | (got[:, 15] != out[:, 15])))
    assert len(bad) == 0, "%s: another candidate won at POIs %s: seeds %s, expected %s (gap %s)" % (
        label, bad[:8], got[bad[:4]][:, 14:16].tolist(), out[bad[:4]][:, 14:16].tolist(), gap[bad[:4]])
    flips = max(1, int(0.02 * len(q))) / max(1, len(q))
    st = util.compare_2d(got, expect, label, max_iter_mismatch_frac=flips)
    assert dec.mean() >= min_decisive, "%s: only %d of %d POIs are decisive" % (label, dec.sum(), len(q))
    print("%s: slots=%d %s n=%d decisive=%d compared=%d valid slots=%d max|du,dv|=%.2e max|dZNCC|=%.2e flips=%.3f" % (
        label, ec.slot_count(radius, step), plan, len(q), dec.sum(), st["n_compared"], valid.sum(), st["max_disp"], st["max_zncc"],
        st["iter_mismatch_frac"]))
    return out, gap, valid


def _grid(n, r, seed, w=W, h=H, half=False, margin=4):
    rng = np.random.default_rng(seed)
    x = rng.integers(r[0] + margin, w - 1 - r[0] - margin, n, endpoint=True).astype(np.float32)
    y = rng.integers(r[1] + margin, h - 1 - r[1] - margin, n, endpoint=True).astype(np.float32)
    if half:
        x += 0.5
        y += 0.5
    return np.stack([x, y], 1)


PAR = ([0.002, 0, 2.0], [0, 0.001, 0.0])  # x_view2 = x + 2 + 0.002 (x - W/2): the match sits 0.3 ... 0.9 px off the slots


# ------------------------------------------------------------------------------------------------ slot counts
# (radius, step): 1, 3, 31, 33 (one slot past a warp), 65 and 301 slots; step 6 keeps one candidate per match
SLOTS = [(8, 8), (9, 8), (91, 6), (97, 6), (193, 6), (901, 6)]


@pytest.mark.parametrize("radius,step", SLOTS)
def test_slot_counts(engine, pair, sm_slots, radius, step):
    ref, tar = pair
    r = (16, 16)
    q = ob.make_poi2d(_grid(24, r, radius))
    got = _search(engine, ref, tar, q, ec.rectified_f(), *PAR, radius, step, *r)
    plan = _plan(sm_slots, len(q) * ec.slot_count(radius, step), *r, W)
    _check("slots r=%d s=%d" % (radius, step), got, q, ref, tar, ec.rectified_f(), *PAR, radius, step, *r, plan=plan)


# ------------------------------------------------------------------------------------------------ IC-GN geometry, warps per POI
GEOMETRY = [((16, 16), False), ((16, 16), True), ((20, 20), False), ((12, 10), False), ((20, 9), False)]


@pytest.mark.parametrize("wpp", ["1", "2"])
@pytest.mark.parametrize("r,half", GEOMETRY)
def test_icgn_geometry(engine, pair, sm_slots, monkeypatch, r, half, wpp):
    monkeypatch.setenv("OCB_ICGN2D_WPP", wpp)
    ref, tar = pair
    q = ob.make_poi2d(_grid(32, r, 7 + r[0] + r[1], half=half))
    args = (ec.rectified_f(), *PAR, 37, 6)
    got = _search(engine, ref, tar, q, *args, *r)
    plan = _plan(sm_slots, len(q) * ec.slot_count(37, 6), *r, W)
    _check("geometry r=%s %s" % (r, "x.5" if half else "integral"), got, q, ref, tar, *args, *r, plan=plan)


@pytest.mark.parametrize("n", [12, 600])
def test_unforced_warps_per_poi(engine, pair, sm_slots, monkeypatch, n):
    """12 POIs x 13 slots cannot fill the GPU (two warps per candidate), 600 x 13 can (one)."""
    monkeypatch.delenv("OCB_ICGN2D_WPP", raising=False)
    ref, tar = pair
    r = (16, 16)
    q = ob.make_poi2d(_grid(n, r, n))
    args = (ec.rectified_f(), *PAR, 37, 6)
    got = _search(engine, ref, tar, q, *args, *r)
    plan = _plan(sm_slots, n * 13, *r, W)
    assert ("wpp=2" in plan) == (n == 12), plan
    _check("unforced n=%d" % n, got, q, ref, tar, *args, *r, plan=plan)


# ------------------------------------------------------------------------------------------------ tile load
@pytest.mark.parametrize("load", ["tma", "no_tma", "odd_width"])
def test_tile_load(engine, pair, pair_odd, sm_slots, monkeypatch, load):
    if load == "no_tma":
        monkeypatch.setenv("OCB_NO_TMA", "1")
    ref, tar = pair_odd if load == "odd_width" else pair
    w = ref.shape[1]
    for r, half in (((16, 16), False), ((12, 10), True)):
        q = ob.make_poi2d(_grid(24, r, 3 + r[1], w=w, half=half))
        args = (ec.rectified_f(), *PAR, 31, 6)
        got = _search(engine, ref, tar, q, *args, *r)
        _check("load %s r=%s" % (load, r), got, q, ref, tar, *args, *r, plan=_plan(sm_slots, len(q) * 11, *r, w))


# ------------------------------------------------------------------------------------------------ line geometry
TRUE_UV = (2.37, -1.62)  # synth.displacement_2d at the image centre
LINE_SLOPES = {"steep+": 2.5, "steep-": -3.0, "negative": -0.4, "gentle": 0.15}


@pytest.mark.parametrize("name", sorted(LINE_SLOPES))
def test_line_geometry(engine, pair, sm_slots, name):
    """Lines of every slope through the match: the parallax puts x_view2 next to it, and the slots step |slope| * step in y."""
    s = LINE_SLOPES[name]
    F = ec.sloped_f(s, TRUE_UV[1] - s * TRUE_UV[0])
    par_x, par_y = (0, 0, TRUE_UV[0]), (0, 0, TRUE_UV[1])
    ref, tar = pair
    r = (14, 14)
    q = ob.make_poi2d(_grid(32, r, len(name), margin=30))
    got = _search(engine, ref, tar, q, F, par_x, par_y, 31, 6, *r)
    out, gap, valid = _check("line %s" % name, got, q, ref, tar, F, par_x, par_y, 31, 6, *r, plan=_plan(sm_slots, len(q) * 11, *r, W))
    assert (got[:, 16] > 0.9).mean() > 0.8


def test_stereo_rig_lines(engine, rig, sm_slots):
    d, F, xy = rig
    r = (16, 16)
    q = ob.make_poi2d(xy)
    args = (F, (0, 0, 4.0), (0, 0, 0), 25, 6)
    got = _search(engine, d["ref1"], d["r2"], q, *args, *r)
    _check("stereo rig", got, q, d["ref1"], d["r2"], *args, *r, plan=_plan(sm_slots, len(q) * 9, *r, d["ref1"].shape[1]))


def test_stereo_rig_ground_truth(engine, rig):
    """The winning candidate, refined by ICGN2D2 as the reference's 3D-DIC example does, lands on the true view-2 point."""
    d, F, xy = rig
    q = ob.make_poi2d(xy)
    engine.set_images_2d(d["ref1"], d["r2"])
    engine.icgn2d_prepare()
    engine.epipolar_search2d(q, F, (0, 0, 4.0), (0, 0, 0), 25, 6, 16, 16, CONV, STOP)
    engine.icgn2d2(q, 16, 16, 0.001, 20)
    ok = q[:, 16] > 0.9
    assert ok.mean() > 0.9, ok.mean()
    err = np.abs(np.c_[q[:, 0] + q[:, 2], q[:, 1] + q[:, 8]] - d["r2_true"])[ok].max()
    print("stereo rig ground truth: %d of %d POIs, max error %.3g px" % (ok.sum(), len(q), err))
    assert err < 0.05, err


# ------------------------------------------------------------------------------------------------ borders and inputs
def test_borders(engine, pair, sm_slots):
    """Slots fail the border test on each side; a POI whose slots all fail keeps the centre's record (-3 when the centre leaves
    the image); a parallax that puts x_view2 at -0.6 truncates it to 0."""
    ref, tar = pair
    r = (12, 12)
    cases = [
        ("left", [[16, 200], [20, 100], [30, 300]], ec.rectified_f(), (0, 0, -3.0)),
        ("right", [[W - 17, 200], [W - 21, 120], [W - 30, 250]], ec.rectified_f(), (0, 0, 3.0)),
        ("top", [[200, 14], [300, 16], [100, 20]], ec.sloped_f(0, -4.0), (0, 0, 0)),
        ("bottom", [[200, H - 15], [300, H - 17], [100, H - 21]], ec.sloped_f(0, 4.0), (0, 0, 0)),
        ("centre outside", [[300, 200], [250, 100], [200, 300]], ec.rectified_f(), (0, 0, float(W))),
        ("x_view2 < 0", [[40, 200], [41, 150], [40, 100]], ec.rectified_f(), (0, 0, -40.6)),
    ]
    for name, xy, F, par_x in cases:
        q = ob.make_poi2d(np.array(xy, np.float32))
        got = _search(engine, ref, tar, q, F, par_x, (0, 0, 0), 25, 6, *r)
        out, gap, valid = _check("border %s" % name, got, q, ref, tar, F, par_x, (0, 0, 0), 25, 6, *r, plan=_plan(sm_slots, len(q) * 9, *r, W),
                                 min_decisive=0)
        assert (~valid[:, 1:]).any(), name
        if name == "centre outside":
            assert not valid[:, 1:].any() and np.all(got[:, 16] == -3), got[:, 16]
        if name == "x_view2 < 0":  # x_view2 = 0, not -1: the slots at x = 18 and 24 pass the border test, not 17 and 23
            assert all(v.tolist() == [True, False, False, False, False, True, False, True, False] for v in valid)


def test_incoming_guess_and_negative_zncc(engine, pair, sm_slots):
    """The incoming u, v move the epipolar line's anchor (x + u, y + v); an incoming negative ZNCC does not stop the search (the
    reference builds every candidate from a cleared POI)."""
    ref, tar = pair
    r = (16, 16)
    q = ob.make_poi2d(_grid(24, r, 99, margin=20))
    q[:, 2] = np.float32(-3.0)
    q[:, 8] = np.float32(1.5)
    q[::3, 16] = -2.0
    q[1::3, 17] = 7.0
    got = _search(engine, ref, tar, q, ec.sloped_f(0, -2.0), (0, 0, 5.0), (0, 0, 0), 31, 6, *r)
    _check("incoming u, v, ZNCC", got, q, ref, tar, ec.sloped_f(0, -2.0), (0, 0, 5.0), (0, 0, 0), 31, 6, *r, plan=_plan(sm_slots, len(q) * 11, *r, W))
    assert (got[::3, 16] > 0.5).all()


def test_exact_ties_go_to_the_earlier_slot(engine, sm_slots):
    """Candidates whose results are computed from identical numbers tie exactly, and the earlier slot wins.

    The target repeats with a period of two steps and the reference matches it half a period off, so slots 1, 2, 3, ... (+-step,
    +-3 step, ...) see the same target pixels; with whole-pixel POIs and seeds and one iteration (RC = 16: the whole-pixel pass),
    their ZNCCs are bit-identical, and the rule gives slot 1: x_view2 + step."""
    step, r = 8, (16, 16)
    base, _ = synth.speckle_pair_2d(2 * step, 256)
    tar = np.tile(base, (1, 20))
    ref = np.roll(tar, -step, axis=1)
    h, w = tar.shape
    xy = np.array([[x, y] for y in (60, 128, 190) for x in (100, 150, 160, 200)], np.float32)
    for radius, expect_slot in ((33, 1), (260, 1)):
        q = ob.make_poi2d(xy)
        got = _search(engine, ref, tar, q, ec.rectified_f(), (0, 0, 0), (0, 0, 0), radius, step, *r, conv=0.001, stop=1)
        out, gap, valid = _check("tie r=%d" % radius, got, q, ref, tar, ec.rectified_f(), (0, 0, 0), (0, 0, 0), radius, step, *r, conv=0.001,
                                 stop=1, plan=_plan(sm_slots, len(q) * ec.slot_count(radius, step), *r, w), min_decisive=0)
        assert np.all(gap == 0) and np.all(got[:, 16] > 0.99)
        assert np.array_equal(got[:, 14], np.full(len(q), step, np.float32)), got[:, 14]
    # conv = 0: no slot converges, every one ends on a failure code (-4, or -3 where its one step leaves the image); equal codes
    # tie exactly, so the witness's first slot of the best code wins
    q = ob.make_poi2d(xy)
    got = _search(engine, ref, tar, q, ec.rectified_f(), (0, 0, 0), (0, 0, 0), 260, step, *r, conv=0.0, stop=1)
    out, gap, valid = _check("tie codes", got, q, ref, tar, ec.rectified_f(), (0, 0, 0), (0, 0, 0), 260, step, *r, conv=0.0, stop=1,
                             plan=_plan(sm_slots, len(q) * ec.slot_count(260, step), *r, w), min_decisive=0)
    assert np.all(got[:, 16] < 0) and np.array_equal(got[:, 14:17], out[:, 14:17])


# ------------------------------------------------------------------------------------------------ candidate blocks
def test_candidate_block_boundary(engine, sm_slots):
    """Blocks of 2^22 / slots POIs: 4095 slots -> 1024 POIs per block, 2300 POIs -> three blocks (9.4 M candidate records, ~0.5 M
    inside the image).  The witness runs on POIs around each boundary, the last one and a random sample; the whole queue must not
    depend on the POIs' order."""
    ref, tar = synth.speckle_pair_2d(256, 256)
    r, radius, step = (16, 16), 2048, 1
    slots = ec.slot_count(radius, step)
    block = (1 << 22) // slots
    assert slots == 4095 and block == 1024
    n = 2300
    xy = _grid(n, r, 4, w=256, h=256)
    q = ob.make_poi2d(xy)
    args = (ec.rectified_f(), (0, 0, 2.0), (0, 0, 0), radius, step)
    got = _search(engine, ref, tar, q, *args, *r)
    rng = np.random.default_rng(0)
    sample = sorted(set([block - 1, block, block + 1, 2 * block - 1, 2 * block, n - 1] + rng.integers(0, n, 40).tolist()))
    _check("blocks n=%d" % n, got[sample], q[sample], ref, tar, *args, *r, plan=_plan(sm_slots, block * slots, *r, 256), min_decisive=0)
    perm = rng.permutation(n)
    shuffled = q[perm].copy()
    engine.epipolar_search2d(shuffled, *args, *r, CONV, STOP)
    assert np.array_equal(_bits(shuffled), _bits(got[perm]))


# ------------------------------------------------------------------------------------------------ variants and errors
def test_device_pointer_variant(engine, pair):
    torch = pytest.importorskip("torch")
    ref, tar = pair
    r = (16, 16)
    q = ob.make_poi2d(_grid(40, r, 11))
    F = ec.rectified_f()
    host = _search(engine, ref, tar, q, F, PAR[0], PAR[1], 31, 6, *r)
    d = torch.from_numpy(q.copy()).cuda()
    torch.cuda.synchronize()
    f = np.ascontiguousarray(F.reshape(9))
    ax, ay = np.array(PAR[0], np.float32), np.array(PAR[1], np.float32)
    rc = engine._lib.ocb_epipolar_search2d_dev(engine._ctx, ctypes.c_void_p(d.data_ptr()), len(q), _vp(f), _vp(ax), _vp(ay), 31, 6, *r, CONV, STOP)
    assert rc == _capi.OCB_OK, _capi.last_error(engine._ctx)
    engine.sync()
    assert np.array_equal(_bits(d.cpu().numpy()), _bits(host))


def test_group_context(engine, pair):
    ref, tar = pair
    r = (16, 16)
    n_dev = _capi.load().ocb_device_count()
    q = ob.make_poi2d(_grid(256 * n_dev + 37, r, 12))
    single = _search(engine, ref, tar, q, ec.rectified_f(), *PAR, 31, 6, *r)
    grp = ob.Engine(list(range(n_dev)))
    assert grp.member_count == n_dev
    group = _search(grp, ref, tar, q, ec.rectified_f(), *PAR, 31, 6, *r)
    print("group context: %d member(s), %d POIs" % (n_dev, len(q)))
    assert np.array_equal(_bits(group), _bits(single))


def test_refused_calls_leave_the_queue_unchanged(engine, pair):
    ref, tar = pair
    q = ob.make_poi2d(_grid(8, (16, 16), 13))
    q[:, 16] = 0.25
    f = np.ascontiguousarray(ec.rectified_f().reshape(9))
    ax, ay = np.array(PAR[0], np.float32), np.array(PAR[1], np.float32)

    def call(eng, queue, n, radius=31, step=6, rx=16, ry=16):
        return eng._lib.ocb_epipolar_search2d(eng._ctx, _vp(queue), n, _vp(f), _vp(ax), _vp(ay), radius, step, rx, ry, CONV, STOP)

    fresh = ob.Engine(0)
    a = q.copy()
    assert call(fresh, a, len(a)) == _capi.OCB_ERR_STATE and "images not set" in _capi.last_error(fresh._ctx)
    fresh.set_images_2d(ref, tar)
    assert call(fresh, a, len(a)) == _capi.OCB_ERR_STATE and "prepare()" in _capi.last_error(fresh._ctx)
    fresh.icgn2d_prepare()
    assert call(fresh, a, len(a), radius=5, step=6) == _capi.OCB_ERR_ARG
    assert call(fresh, a, len(a), rx=0) == _capi.OCB_ERR_ARG
    assert call(fresh, a, len(a), ry=0) == _capi.OCB_ERR_ARG
    assert call(fresh, None, len(a)) == _capi.OCB_ERR_ARG
    assert np.array_equal(_bits(a), _bits(q))
    assert call(fresh, None, 0) == _capi.OCB_OK
    assert call(fresh, a, len(a)) == _capi.OCB_OK and not np.array_equal(_bits(a), _bits(q))
