"""CPU: the Strain cell grid (ocb::strain_grid_plan, opencorr_b200/csrc/ocb_kernels.h) compiled for the host, on the bounding box
and radius of every grid case of strain_cases.py: the cell is at least |radius| for a finite non-zero radius, a non-finite radius
takes one cell over the bbox, the grid stays below 2^30 cells, and the growth cases grow their cell but for the two whose grid
of |radius| cells already fits (growth_none_2d_x: 100 009 x 9 cells, growth_3d_r4: 752^3).  Run with -s to see the plan of each
case."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import strain_cases as sc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = np.float32
NO_GROWTH = ("growth_none_2d_x", "growth_3d_r4")


def build_tool(out_dir):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    exe = os.path.join(out_dir, "strain_grid_host_test")
    cmd = [nvcc, "-x", "cu", "-std=c++17", "-O1", "-Wno-deprecated-gpu-targets", "-I", os.path.join(ROOT, "opencorr_b200", "csrc"),
           "-o", exe, os.path.join(ROOT, "tests", "native", "strain_grid_host_test.cpp")]
    if os.path.exists("/usr/bin/g++"):
        cmd[1:1] = ["-ccbin", "/usr/bin/g++"]
    build = subprocess.run(cmd, capture_output=True, text=True)
    assert build.returncode == 0, "nvcc failed:\n" + build.stdout + build.stderr
    return exe


def case_line(c):
    """name, search dims, the float32 bbox of the finite positions (as the bbox kernel reduces it), radius"""
    sd = sc.layout(c.q)["sd"]
    pos = c.q[:, :sd]
    pos = pos[np.isfinite(pos).all(1)]
    lo, hi = np.zeros(3, F), np.zeros(3, F)
    lo[:sd], hi[:sd] = pos.min(0), pos.max(0)
    vals = [repr(float(v)) for v in (*lo, *hi, F(c.radius))]
    return "%s %d %s" % (c.name, sd, " ".join(vals)), sd, lo, hi


def test_strain_grid_plan(tmp_path):
    cases = sc.small_cases()
    growth = {c.name for c in sc.growth_cases()}
    lines, info = [], {}
    for c in cases:
        line, sd, lo, hi = case_line(c)
        lines.append(line)
        info[c.name] = (c, sd, lo, hi)
    out = subprocess.run([build_tool(str(tmp_path))], input="\n".join(lines) + "\n", capture_output=True, text=True, timeout=60)
    print(out.stdout)
    assert out.returncode == 0, out.stdout + out.stderr
    plans = {m[0]: m[1:] for m in re.findall(r"^(\S+): cell=(\S+) nc=(\d+),(\d+),(\d+) cells=(\d+) top=(\d+),(\d+),(\d+)$", out.stdout, re.M)}
    assert set(plans) == set(info), "cases without a plan: %s" % sorted(set(info) - set(plans))
    seen = {"finite": 0, "non-finite": 0}
    for name, (c, sd, lo, hi) in info.items():
        cell, cells = float(plans[name][0]), int(plans[name][4])
        nc = [int(v) for v in plans[name][1:4]]
        top = [int(v) for v in plans[name][5:8]]
        r = abs(float(F(c.radius)))
        assert cells < 2 ** 30 and cells == nc[0] * nc[1] * nc[2], (name, nc, cells)
        assert nc[sd:] == [1] * (3 - sd), (name, nc)
        if np.isfinite(r) and r > 0:
            seen["finite"] += 1
            assert cell >= r, (name, cell, r)
        elif not np.isfinite(r):
            seen["non-finite"] += 1
            assert top == [0, 0, 0], (name, top)  # every finite position lies in cell 0
        if name in growth:
            assert (cell > r) == (name not in NO_GROWTH), (name, cell, r)
    assert seen["finite"] > 50 and seen["non-finite"] >= 9, seen
    assert {"growth_2d_wrap", "outlier_1e30_2", "outlier_1e30_3", "growth_none_2d_x"} <= growth
