"""CPU: the SIFT3D pyramid plan (ocb::sift3d_plan, opencorr_b200/csrc/ocb_kernels.h) compiled for the host.  On every case of
sift3d_cases.py the octave count, the octaves' dimensions and units and the layers' scales and sigmas equal a float32 restatement
of createGaussianPyramid (src/oc_sift.cpp:676-739), and every blurred layer's radii and weights are the oracle's blur_kernel at
that layer's sigma and units, bit for bit.  The refusals sit exactly at their bounds: n_octave_layers 13 / 14, the unit ratio
whose blur radius first exceeds 64 voxels, and n_octave_layers x voxels = 2^62."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import sift3d_cases as sc
from oracle import sift3d as s3

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = np.float32
REJECT = {"OCTAVE_LAYERS": 1, "VOLUME_SIZE": 2, "BLUR_RADIUS": 3}  # ocb::Sift3dReject


def build_tool(out_dir):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    exe = os.path.join(out_dir, "sift3d_plan_host_test")
    cmd = [nvcc, "-x", "cu", "-std=c++17", "-O1", "-Wno-deprecated-gpu-targets", "-I", os.path.join(ROOT, "opencorr_b200", "csrc"),
           "-o", exe, os.path.join(ROOT, "tests", "native", "sift3d_plan_host_test.cpp")]
    if os.path.exists("/usr/bin/g++"):
        cmd[1:1] = ["-ccbin", "/usr/bin/g++"]
    build = subprocess.run(cmd, capture_output=True, text=True)
    assert build.returncode == 0, "nvcc failed:\n" + build.stdout + build.stderr
    return exe


def _f(hexbits):
    return np.array([int(hexbits, 16)], np.uint32).view(F)[0]


def plans(tmp_path, cases):
    """cases: name -> (dims, unit, config floats).  Returns name -> reject code, or the plan as a dict."""
    lines = ["%s %d %d %d %s %s" % (name, *dims, " ".join(repr(float(u)) for u in F(unit)), " ".join(repr(float(c)) for c in F(cfg)))
             for name, (dims, unit, cfg) in cases.items()]
    out = subprocess.run([build_tool(str(tmp_path))], input="\n".join(lines) + "\n", capture_output=True, text=True, timeout=60)
    assert out.returncode == 0, out.stdout + out.stderr
    got = {}
    for line in out.stdout.splitlines():
        name, rest = line.split(": ", 1)
        kind, *v = rest.split()
        if kind == "reject":
            got[name] = int(v[0])
        elif kind == "plan":
            got[name] = dict(n_octave=int(v[0]), L=int(v[1]), kappa=_f(v[2]), octave=[], layer={})
        elif kind == "octave":
            got[name]["octave"].append(([int(x) for x in v[1:4]], np.array([_f(x) for x in v[4:7]], F)))
        else:
            o, l, r = int(v[0]), int(v[1]), [int(x) for x in v[4:7]]
            w, k = [], 7
            for a in range(3):
                w.append(np.array([_f(x) for x in v[k:k + r[a] + 1]], F))
                k += r[a] + 1
            got[name]["layer"][o, l] = (_f(v[2]), _f(v[3]), r, w)
    assert set(got) == set(cases), sorted(set(cases) - set(got))
    return got


def restate(dims, unit, cfg, kappa):
    """createGaussianPyramid in float32: n_octave, per octave (dims, unit), per layer (scale, sigma); kappa = pow(2.f, 1.f / nol)"""
    nol, L = int(cfg[0]), int(cfg[0]) + 3
    n_octave = max(int(np.floor(np.log2(F(min(dims))) - np.log2(F(int(cfg[2]))))) + 1, 1)
    octaves = [(list(dims), F(unit))]
    for o in range(1, n_octave):
        d, u = octaves[-1]
        octaves.append(([x // 2 for x in d], u * F(2)))
    scale, sigma = np.zeros(n_octave * L, F), np.zeros(n_octave * L, F)
    scale[0] = F(1) / kappa * F(cfg[7])
    with np.errstate(invalid="ignore"):  # NaN when scale[0] < sigma_source (n_octave_layers = 2): blurred with radius 1, as there
        sigma[0] = np.sqrt(scale[0] * scale[0] - F(cfg[6]) * F(cfg[6]))
    for i in range(1, n_octave * L):
        o, lio = divmod(i, L)
        if lio == 0:
            scale[i] = scale[(o - 1) * L + nol]
        else:
            scale[i] = kappa * scale[i - 1]
            sigma[i] = np.sqrt(kappa * kappa - F(1)) * scale[lio - 1]
    return n_octave, octaves, scale, sigma


def _bits(x):
    return np.asarray(x, F).view(np.uint32).tolist()


def test_sift3d_plan_cases(tmp_path):
    assert np.load(os.path.join(ROOT, sc.CROP))["ref"].shape == sc.CASES["al_foam4_crop"][0][::-1]
    cases = {name: (dims, unit, sc.cfg(**kw)) for name, (dims, unit, kw) in sc.CASES.items()}
    got = plans(tmp_path, cases)
    for name, (dims, unit, cfg) in cases.items():
        p = got[name]
        assert isinstance(p, dict), (name, p)
        L = int(cfg[0]) + 3
        n_octave, octaves, scale, sigma = restate(dims, unit, cfg, p["kappa"])
        assert (p["n_octave"], p["L"]) == (n_octave, L), name
        for o in range(n_octave):
            assert p["octave"][o][0] == octaves[o][0] and _bits(p["octave"][o][1]) == _bits(octaves[o][1]), (name, o)
            for l in range(L):
                s, sg, r, w = p["layer"][o, l]
                assert _bits(s) == _bits(scale[o * L + l]) and _bits(sg) == _bits(sigma[o * L + l]), (name, o, l)
                if o > 0 and l == 0:  # downsampled, not blurred
                    assert r == [0, 0, 0], (name, o)
                    continue
                r_o, w_o = s3.blur_kernel(sg, octaves[o][1])
                assert r == r_o.tolist() and all(_bits(w[a]) == _bits(w_o[a]) for a in range(3)), (name, o, l)
        print("%s: %d octaves, radii of octave 0: %s" % (name, n_octave, [p["layer"][0, l][2] for l in range(L)]))


def test_sift3d_plan_refusals(tmp_path):
    d = sc.cfg()
    # default config: the widest blur has ceil(3 sigma) = 8, times the unit ratio rounded to an integer: 64 below 8.5, 72 at it
    below = float(np.nextafter(F(8.5), F(0)))
    cases = {
        "layers_13": ((64, 64, 64), (1.0, 1.0, 1.0), sc.cfg(n_octave_layers=13)),
        "layers_14": ((64, 64, 64), (1.0, 1.0, 1.0), sc.cfg(n_octave_layers=14)),
        "ratio_below": ((100, 100, 100), (1.0, 1.0, below), d),
        "ratio_8.5": ((100, 100, 100), (1.0, 1.0, 8.5), d),
        "ratio_8.5_x": ((100, 100, 100), (8.5, 1.0, 1.0), d),
        "voxels_2^62": ((1 << 21, 1 << 21, 1 << 20), (1.0, 1.0, 1.0), sc.cfg(n_octave_layers=1)),
        "voxels_2^62+": ((1 << 21, 1 << 21, (1 << 20) + 1), (1.0, 1.0, 1.0), sc.cfg(n_octave_layers=1)),
        "layers_4_2^60": ((1 << 20, 1 << 20, 1 << 20), (1.0, 1.0, 1.0), sc.cfg(n_octave_layers=4)),
        "layers_4_2^60+": (((1 << 20) + 1, 1 << 20, 1 << 20), (1.0, 1.0, 1.0), sc.cfg(n_octave_layers=4)),
    }
    got = plans(tmp_path, cases)
    for name in ("layers_13", "ratio_below", "voxels_2^62", "layers_4_2^60"):
        assert isinstance(got[name], dict), (name, got[name])
    assert got["layers_14"] == REJECT["OCTAVE_LAYERS"]
    assert got["ratio_8.5"] == got["ratio_8.5_x"] == REJECT["BLUR_RADIUS"]
    assert got["voxels_2^62+"] == got["layers_4_2^60+"] == REJECT["VOLUME_SIZE"]
    # the accepted ratio is the boundary: its widest blur is exactly 64 voxels, along the axes of the smaller unit
    p = got["ratio_below"]
    widest = max(max(r) for (_, _, r, _) in p["layer"].values())
    assert widest == 64, widest
    r, _ = s3.blur_kernel(p["layer"][0, p["L"] - 1][1], (1.0, 1.0, 8.5))
    assert r.max() > 64, r
