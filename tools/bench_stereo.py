"""Stereo-reconstruction timings at the geometry of the reference's test_3d_reconstruction_epipolar.cpp: Calibration::prepare of
both cameras (two 2448x2048 maps) and Stereovision::reconstruct of the 313x313 POI grid (97 969 pairs).  Prints one JSON line;
`python tools/bench_stereo.py [--steps K] [--warmup W]`.  Writes nothing.  Not the headline benchmark (that is bench.py).

The calibration is that example's; the view-2 points are the grid moved by the shipped table's mean parallax (-121, -98) px plus
seeded +-2 px noise.
  map_build_ms      : device time of both prepare() calls (CUDA events, 256 MiB L2 flush before each step)
  reconstruct_ms    : device time of one reconstruct of all pairs on device-resident points (ocb_stereo_reconstruct_dev)
  e2e_reconstruct_ms: host clock around reconstruct() from host arrays (H2D, kernel, D2H, synchronise)
  cpu_oracle        : the faithful float32 oracle (oracle/oc_stereo.cpp) on nproc-1 threads, host clock
The reference's own figures for this program (examples/3d_dic/..._reconstruction_epipolar_time.csv) are quoted beside:
0.0086 s for reconstruction and 0.18 s of "Initialization", which includes both prepare() maps."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

STEP18_SIZE = (2048, 2448)
STEP18_INTRINSICS = [[10664.80664, 10643.88965, 0, 1176.03418, 914.7337036, 0.030823536, -1.350255132, 74.21749878, 0, 0, 0, 0, 0],
                     [10749.53223, 10726.52441, 0, 1034.707886, 1062.162842, 0.070953421, -4.101067066, 74.21749878, 0, 0, 0, 0, 0]]
STEP18_EXTRINSICS = [[0, 0, 0, 0, 0, 0], [250.881488962793, -1.15469183120196, 37.4849858174401, 0.01450813, -0.39152833, 0.01064092]]


def gpu_power_limit():
    """(name, power limit) of GPU 0 as nvidia-smi reports them (a read-only query), or (None, None)."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        name, limit = [s.strip() for s in out.split(",")]
        return name, limit
    except Exception:
        return None, None


def cpu_model():
    try:
        for line in open("/proc/cpuinfo"):
            if line.lower().startswith("model name"):
                return line.split(":", 1)[1].strip()
    except Exception:
        pass
    return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()

    import torch
    import opencorr_b200 as ob
    from oracle import stereo as so

    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device; opencorr_b200 has no CPU fallback"}))
        return 1
    h, w = STEP18_SIZE
    names = ("tx", "ty", "tz", "rx", "ry", "rz")
    eng = ob.Engine(0)
    cams = [ob.Calibration(engine=eng, **dict(zip(ob.api.INTRINSIC_NAMES, STEP18_INTRINSICS[i])), **dict(zip(names, STEP18_EXTRINSICS[i])))
            for i in range(2)]
    gy, gx = np.meshgrid(np.arange(313), np.arange(313), indexing="ij")
    pts1 = np.stack([420 + 5 * gx.ravel(), 250 + 5 * gy.ravel()], axis=1).astype(np.float32)
    rng = np.random.default_rng(18)
    pts2 = (pts1 + np.array([-121.0, -98.0], np.float32) + rng.uniform(-2, 2, pts1.shape)).astype(np.float32)
    n = len(pts1)
    dev = torch.device("cuda", 0)
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)  # 256 MiB > the 50 MB L2
    stream = torch.cuda.current_stream(dev)
    eng.set_stream(stream.cuda_stream)

    def timed(fn):
        times = []
        for i in range(args.warmup + args.steps):
            flush.zero_()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            fn()
            b.record(stream)
            torch.cuda.synchronize(dev)
            if i >= args.warmup:
                times.append(a.elapsed_time(b))
        return times

    def build_maps():
        for c in cams:
            c.prepare(h, w)

    t_map = timed(build_maps)
    sv = ob.Stereovision(cams[0], cams[1], 0, eng)
    sv.prepare()
    d1, d2 = torch.from_numpy(pts1).to(dev), torch.from_numpy(pts2).to(dev)
    d3 = torch.empty((n, 3), dtype=torch.float32, device=dev)
    t_rec = timed(lambda: sv.reconstruct_dev(d1.data_ptr(), d2.data_ptr(), d3.data_ptr(), n))
    eng.use_own_stream()
    t_e2e = []
    for i in range(args.warmup + args.steps):
        a1, a2 = pts1.copy(), pts2.copy()
        t0 = time.perf_counter()
        out = sv.reconstruct(a1, a2)
        if i >= args.warmup:
            t_e2e.append((time.perf_counter() - t0) * 1e3)
    assert np.array_equal(out, d3.cpu().numpy()), "device and host reconstructions differ"

    threads = max(1, (os.cpu_count() or 2) - 1)
    t0 = time.perf_counter()
    o = [so.CalibOracle(c.intrinsic_vector(), h, w, threads=threads) for c in cams]
    cpu_map = time.perf_counter() - t0
    t0 = time.perf_counter()
    oc = so.reconstruct(o[0], cams[0].projection_vector(), o[1], cams[1].projection_vector(), pts1.copy(), pts2.copy())
    cpu_rec = time.perf_counter() - t0
    gpu_name, power = gpu_power_limit()
    line = {
        "metric": "stereo reconstruction at Step18 geometry (2 x 2448x2048 maps, %d pairs)" % n,
        "gpu": gpu_name or torch.cuda.get_device_name(dev), "power_limit": power,
        "steps": args.steps, "warmup": args.warmup,
        "map_build_ms": {"median": statistics.median(t_map), "min": min(t_map)},
        "reconstruct_ms": {"median": statistics.median(t_rec), "min": min(t_rec)},
        "e2e_reconstruct_ms": {"median": statistics.median(t_e2e), "min": min(t_e2e)},
        "reconstruct_pairs_per_s": n / (statistics.median(t_rec) * 1e-3),
        "cpu_oracle": {"threads": threads, "cpu": cpu_model(), "map_build_ms": cpu_map * 1e3, "reconstruct_ms": cpu_rec * 1e3,
                       "max_abs_diff_vs_gpu_mm": float(np.abs(oc - out).max())},
        "reference_shipped_s": {"reconstruction": 0.0085629, "initialization_incl_both_maps": 0.183311,
                                "source": "examples/3d_dic/Step18 00,00-0005_1_reconstruction_epipolar_time.csv"},
        "timing": "device legs: CUDA events around the calls, 256 MiB L2 flush before each step; e2e and CPU: host clock",
    }
    eng.close()
    print(json.dumps(line))
    return 0


if __name__ == "__main__":
    sys.exit(main())
