"""CPU: the FFTCC2D routing (ocb::fftcc2d_plan, opencorr_b200/csrc/ocb_kernels.h) compiled for the host.  Every case of
test_gpu_fftcc2d_geometry.py must land on the kernel it names, and together the cases must reach every radix of the generic
kernel, every size of the register kernel and every POIs-per-CTA count; run with -s to see the plan of each case.  Also here,
because it needs no GPU either: the GPU file's numpy witness against the float64 oracle."""
import re

import numpy as np
import pytest

from opencorr_b200 import synth
from oracle.oracle import Oracle2D
import test_gpu_fftcc2d_geometry as geometry

H100_SMEM_OPTIN = 227 * 1024  # cudaDevAttrMaxSharedMemoryPerBlockOptin of an H100


def test_fftcc2d_plan_covers_every_kernel(tmp_path):
    exe = geometry.build_plan_tool(str(tmp_path))
    out = geometry.run_plan_tool(exe, H100_SMEM_OPTIN, cases=geometry.PLAN_CASES)
    print(out.stdout)
    assert out.returncode == 0, out.stdout + out.stderr
    planned = {}
    for m in re.finditer(r"^r=\((-?\d+),(-?\d+)\) force=(\d) n=(\d+): (?:kernel (\w+)|(rejected \([a-z ]+\)))(.*)$", out.stdout, re.M):
        planned[tuple(int(v) for v in m.groups()[:4])] = (m.group(5) or m.group(6), m.group(7))
    # every case the GPU file runs is listed, on the kernel that file names
    for rx, ry, generic, kernel, n in geometry.PLAN_CASES:
        assert (rx, ry, generic, n) in planned, "no plan for r=(%d,%d) force=%d n=%d" % (rx, ry, generic, n)
        assert planned[(rx, ry, generic, n)][0] == kernel, "r=(%d,%d) force=%d: %s, not %s" % (rx, ry, generic, planned[(rx, ry, generic, n)][0], kernel)
    for rx, ry in geometry.SWEEP:
        assert any(c[:3] == (rx, ry, 0) for c in geometry.PLAN_CASES)
    # the generic cases reach every butterfly: radix 4, 2, 3, 5 and the odd-radix loop at every prime 7 ... 31
    radices = set()
    for kernel, rest in planned.values():
        if kernel == "GENERIC":
            for axis in re.findall(r"[xy]=\[([\d,]+)\]", rest):
                radices |= {int(v) for v in axis.split(",")}
    assert radices == {2, 3, 4, 5, 7, 11, 13, 17, 19, 23, 29, 31}, sorted(radices)
    # the register cases reach every size, every POIs-per-CTA count, the idle threads of N = 40, and always a partly filled last batch
    reg = [re.search(r"N=(\d+) PP=(\d+), (\d+) idle thread\(s\), (\d+) batch\(es\), (\d+) POI\(s\) in the last", rest).groups()
           for kernel, rest in planned.values() if kernel == "REG"]
    reg = [tuple(int(v) for v in g) for g in reg]
    assert {g[0] for g in reg} == {8, 10, 12, 16, 18, 20, 24, 30, 36, 40, 48, 50, 54, 60, 64}
    assert {g[1] for g in reg} == {16, 12, 10, 8, 7, 6, 5, 4, 3, 2}
    assert (40, 3, 8) in {g[:3] for g in reg}
    sweep_keys = {(r, r, 0, geometry.sweep_n(r, r)) for r in geometry.REG_R}
    for key in sweep_keys:
        g = tuple(int(v) for v in re.search(r"PP=(\d+), .*?(\d+) POI\(s\) in the last", planned[key][1]).groups())
        assert g[1] < g[0], "r=%d: the last batch of the sweep queue is full" % key[0]
    assert 40 <= min(k[3] for k in sweep_keys) and max(geometry.sweep_n(rx, ry) for rx, ry in geometry.SWEEP) <= 64
    # windows above 64 points and strongly non-square ones run on the generic kernel
    assert planned[(100, 30, 0, geometry.sweep_n(100, 30))][0] == "GENERIC" and planned[(58, 58, 0, geometry.sweep_n(58, 58))][0] == "GENERIC"
    # accept / reject boundary at an H100's opt-in limit: r = 58 is the largest square window, r = 60 the first refused for its
    # shared memory (59 is prime)
    lim = geometry.run_plan_tool(exe, "limits", H100_SMEM_OPTIN)
    assert lim.returncode == 0 and re.findall(r"\d+", lim.stdout) == ["58", "60"], lim.stdout


@pytest.mark.parametrize("rx,ry", [(16, 16), (7, 7), (29, 29), (100, 30)])
def test_numpy_witness_matches_exact_oracle(rx, ry):
    """The two witnesses of the GPU file agree with each other on its sweep queues: identical integers on decisive POIs, ZNCC
    within 1e-9."""
    ref, tar = synth.speckle_pair_2d(geometry.W, geometry.H)
    q = geometry.sweep_queue(rx, ry, geometry.sweep_n(rx, ry), seed=100 * rx + ry)
    wa, computed, gap, _ = geometry.witness(ref, tar, q, rx, ry)
    wb = Oracle2D(ref, tar).fftcc2d(q.copy(), rx, ry, exact=True)
    assert computed.all()
    dec = gap > geometry.GAP
    assert dec.sum() >= 0.95 * len(q)
    assert np.array_equal(wa[dec][:, geometry.INT_COLS], wb[dec][:, geometry.INT_COLS])
    # both store ZNCC as float32: equal up to one rounding of a float64 difference below 1e-9
    assert np.abs(wa[:, 16].astype(np.float64) - wb[:, 16]).max() <= 1e-9 + 6e-8
    print("witness r=(%d,%d): n=%d decisive=%d max|dZNCC|=%.2e" % (rx, ry, len(q), dec.sum(), np.abs(wa[:, 16] - wb[:, 16]).max()))
