"""CPU: the ICGN3D1 launch plan (ocb::icgn3d1_plan, opencorr_b200/csrc/ocb_kernels.h) compiled for the host.  Every subvolume
radius set of test_gpu_3d_geometry.py must land in the kernel variant and slab layout its case is meant to cover; run with -s
to see the plan of each case."""
import os
import re
import shutil
import subprocess

import pytest

import test_gpu_3d_geometry as geometry

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(shutil.which("nvcc") is None and not os.path.exists("/usr/local/cuda/bin/nvcc"), reason="nvcc not available")
def test_icgn3d_plan_covers_every_branch(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    exe = str(tmp_path / "icgn3d_plan_host_test")
    cmd = [nvcc, "-x", "cu", "-std=c++17", "-O1", "-Wno-deprecated-gpu-targets", "-I", os.path.join(ROOT, "opencorr_b200", "csrc"),
           "-o", exe, os.path.join(ROOT, "tests", "native", "icgn3d_plan_host_test.cpp")]
    if os.path.exists("/usr/bin/g++"):
        cmd[1:1] = ["-ccbin", "/usr/bin/g++"]
    build = subprocess.run(cmd, capture_output=True, text=True)
    assert build.returncode == 0, "nvcc failed:\n" + build.stdout + build.stderr
    out = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    print(out.stdout)
    assert out.returncode == 0, out.stdout
    planned = {tuple(int(v) for v in m) for m in re.findall(r"r=\((\d+),(\d+),(\d+)\)", out.stdout)}
    # every radius set the GPU cases run is in the checked table
    missing = [r for r in geometry.ICGN3D_RADII if tuple(r) not in planned]
    assert not missing, "radius sets of test_gpu_3d_geometry.py without a checked plan: %s" % missing
    # the shear case replays the kernel's tile placement with these slab thicknesses
    slab_k = {int(m[0]): int(m[1]) for m in re.findall(r"r=\((\d+),\1,\1\): .*? slab\(s\) x (\d+) layers", out.stdout)}
    for r, k in geometry.SHEAR_SLAB_K.items():
        assert slab_k[r] == k, (r, slab_k.get(r), k)
    kernels = set(re.findall(r"kernel (<\d+,\d+>)", out.stdout))
    assert {"<0,256>", "<0,512>", "<16,256>", "<30,512>"} <= kernels
    assert "rejected" in out.stdout
