"""CPU: the FFTCC3D routing (ocb::fftcc3d_plan, opencorr_b200/csrc/ocb_kernels.h) compiled for the host.  Every case of
test_gpu_fftcc3d_geometry.py must land on the kernel it names, and together the cases must reach every radix of the generic
kernel, every size of the register kernel and every slices-per-round count; run with -s to see the plan of each case.  Also here,
because it needs no GPU either: the GPU file's numpy witness against the float64 oracle."""
import re

import numpy as np
import pytest

from opencorr_b200 import synth
from oracle.oracle import Oracle3D
import test_gpu_fftcc3d_geometry as geometry

H100_SMEM_OPTIN = 227 * 1024  # cudaDevAttrMaxSharedMemoryPerBlockOptin of an H100
H100_SMS = 132


@pytest.fixture(scope="module")
def vol():
    return synth.speckle_pair_3d(geometry.DX, geometry.DY, geometry.DZ)


def test_fftcc3d_plan_covers_every_kernel(tmp_path):
    exe = geometry.build_plan_tool(str(tmp_path))
    out = geometry.run_plan_tool(exe, H100_SMEM_OPTIN, H100_SMS, cases=geometry.PLAN_CASES)
    print(out.stdout)
    assert out.returncode == 0, out.stdout + out.stderr
    planned = {}
    for m in re.finditer(r"^r=\((-?\d+),(-?\d+),(-?\d+)\) force=(\d) n=(\d+): (?:kernel (\w+)|(rejected \([a-z ]+\)))(.*)$", out.stdout, re.M):
        planned[tuple(int(v) for v in m.groups()[:5])] = (m.group(6) or m.group(7), m.group(8))
    # every case the GPU file runs is listed, on the kernel that file names
    for rx, ry, rz, generic, kernel, n in geometry.PLAN_CASES:
        key = (rx, ry, rz, generic, n)
        assert key in planned, "no plan for r=(%d,%d,%d) force=%d n=%d" % key
        assert planned[key][0] == kernel, "r=(%d,%d,%d) force=%d: %s, not %s" % (rx, ry, rz, generic, planned[key][0], kernel)
    for r in geometry.SWEEP:
        assert any(c[:4] == r + (0,) for c in geometry.PLAN_CASES)
    # the generic cases reach every butterfly: radix 4, 2, 3, 5 and the odd-radix loop at every prime 7 ... 31
    radices = set()
    for kernel, rest in planned.values():
        if kernel == "GENERIC":
            for axis in re.findall(r"[xyz]=\[([\d,]+)\]", rest):
                radices |= {int(v) for v in axis.split(",")}
    assert radices == {2, 3, 4, 5, 7, 11, 13, 17, 19, 23, 29, 31}, sorted(radices)
    # the register cases reach every size and every slices-per-round count, and the idle threads of N = 36, 40, 50, 54, 60
    reg = {tuple(int(v) for v in re.search(r"N=(\d+) G=(\d+), (\d+) idle", rest).groups()) for kernel, rest in planned.values() if kernel == "REG"}
    assert {g[0] for g in reg} == {8, 10, 12, 16, 18, 20, 24, 30, 36, 40, 48, 50, 54, 60, 64}
    assert {g[1] for g in reg} == {16, 12, 10, 8, 7, 6, 5, 4, 3, 2}
    assert {(40, 3, 8), (60, 2, 8), (54, 2, 20)} <= reg
    # windows above 64 points and non-cubic windows of register sizes run on the generic kernel; the sentinel and constant-window
    # cases force one W32 window onto it
    for key in [(r, r, r, 0, geometry.sweep_n((r, r, r))) for r in (33, 36, 42)] + [r + (0, geometry.sweep_n(r)) for r in geometry.GENERIC_NONCUBIC]:
        assert planned[key][0] == "GENERIC", key
    # the long queues give every CTA three POIs and the first five a fourth
    for r in geometry.LONG_R:
        ctas = int(re.search(r"(\d+) CTA\(s\)", planned[r + (0, 1)][1]).group(1))
        assert ctas >= H100_SMS
    # accept / reject boundary at an H100's opt-in limit: r = 42 is the largest cubic window, r = 44 the first refused for its
    # shared memory (43 is prime)
    lim = geometry.run_plan_tool(exe, "limits", H100_SMEM_OPTIN)
    assert lim.returncode == 0 and re.findall(r"\d+", lim.stdout) == ["42", "44"], lim.stdout
    assert 42 in geometry.GENERIC_CUBIC


@pytest.mark.parametrize("r", [(16, 16, 16), (7, 7, 7), (12, 10, 14), (29, 29, 29)])
def test_numpy_witness_matches_exact_oracle(vol, r):
    """The two witnesses of the GPU file agree with each other on its sweep queues: identical integers on decisive POIs, ZNCC
    within 1e-9 (plus one float32 rounding)."""
    ref, tar = vol
    q = geometry.sweep_queue(r, geometry.sweep_n(r), seed=sum(r) * 31 + r[0])
    wa, computed, gap, _ = geometry.witness(ref, tar, q, *r)
    wb = Oracle3D(ref, tar).fftcc3d(q.copy(), *r, exact=True)
    assert computed.all()
    dec = gap > geometry.GAP
    assert dec.sum() >= 0.9 * len(q)
    assert np.array_equal(wa[dec][:, geometry.INT_COLS], wb[dec][:, geometry.INT_COLS])
    assert np.abs(wa[:, geometry.ZNCC].astype(np.float64) - wb[:, geometry.ZNCC]).max() <= 1e-9 + 6e-8
    print("witness r=(%d,%d,%d): n=%d decisive=%d max|dZNCC|=%.2e" % (*r, len(q), dec.sum(), np.abs(wa[:, geometry.ZNCC] - wb[:, geometry.ZNCC]).max()))


def test_witness_and_oracle_agree_on_refusals_and_constant_windows(vol):
    """The guard (faces, fractional positions, NaN, +-inf, 1e30) and the zero-norm rule of the two witnesses, on the GPU file's own
    queues: the same POIs are refused, and a constant window returns the guess with ZNCC NaN in both."""
    ref, tar = vol
    dims = (76, 68, 60)
    fr, ft = (np.ascontiguousarray(a[20:20 + dims[2], 30:30 + dims[1], 40:40 + dims[0]]) for a in (ref, tar))
    for r in geometry.EDGE_R:
        rows = geometry._face_rows(r, dims)
        q = geometry._mark(geometry.ob.make_poi3d(rows[:, :3]))
        q[:, 3], q[:, 7], q[:, 11] = rows[:, 3], rows[:, 4], rows[:, 5]
        _, computed, _, _ = geometry.witness(fr, ft, q, *r)
        wb = Oracle3D(fr, ft).fftcc3d(q.copy(), *r, exact=True)
        assert np.array_equal(computed, rows[:, 6] > 0), (r, np.flatnonzero(computed != (rows[:, 6] > 0)))
        assert np.array_equal(geometry._bits(wb[~computed]), geometry._bits(q[~computed])) and (wb[computed, 18] != q[computed, 18]).all()
    bad = geometry._mark(geometry.ob.make_poi3d(np.tile([[70.0, 62.0, 54.0]], (30, 1))))
    for j, col in enumerate((0, 1, 2, 3, 7, 11)):
        for k, v in enumerate([np.nan, np.inf, -np.inf, 1e30, -1e30]):
            bad[5 * j + k, col] = v
    _, computed, _, _ = geometry.witness(ref, tar, bad, 7, 7, 7)
    wb = Oracle3D(ref, tar).fftcc3d(bad.copy(), 7, 7, 7, exact=True)
    assert not computed.any() and np.array_equal(geometry._bits(wb), geometry._bits(bad))
    flat = ref.copy()
    flat[geometry.CONST_BOX] = synth.BACKGROUND
    q = geometry._const_queue((10, 10, 10))
    wa, computed, _, _ = geometry.witness(flat, tar, q, 10, 10, 10)
    wb = Oracle3D(flat, tar).fftcc3d(q.copy(), 10, 10, 10, exact=True)
    assert computed.all() and np.array_equal(wa, wb, equal_nan=True) and np.isnan(wb[:, 18]).all()
    assert np.array_equal(wb[:, [3, 7, 11]], q[:, [3, 7, 11]])
