"""SIFT3D benchmark: per-stage CUDA-event times, keypoint and match counts, end-to-end time from host volumes, and the CPU
oracle's time on the same pair.  Prints one JSON record (and writes it to --out).

Workloads: the 100^3 al_foam4 crop (tests/golden), and a synthetic speckle pair covering the extent of the keypoints of the
reference's shipped DVC example (Torus: x <= 959, y <= 286, z <= 588), 960 x 288 x 592 by default.

    python tools/bench_sift3d.py --repeat 2 --oracle crop --out profiles/h100_bench_sift3d.json

The oracle is timed on the crop only by default: on the large pair its brute-force matching alone is N x M x 768 x 3 ~ 8.5e14
float operations for the ~6e5 keypoints per volume of the synthetic speckle, hours on one host.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import opencorr_b200 as ob  # noqa: E402
from opencorr_b200 import synth  # noqa: E402


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in q.split(",")]
        return dict(name=name, power_limit_w=float(power), max_sm_clock_mhz=float(clock))
    except Exception as e:  # the record still says what could not be read
        return dict(error=str(e))


def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _workload(name, dims):
    if name == "al_foam4_crop":
        z = np.load(os.path.join(ROOT, "tests", "golden", "al_foam4_crop.npz"))
        return z["ref"].astype(np.float32), z["tar"].astype(np.float32)
    dx, dy, dz = dims
    ref, tar = synth.speckle_pair_3d(dx, dy, dz, device="cuda")
    return np.ascontiguousarray(ref, np.float32), np.ascontiguousarray(tar, np.float32)


def run(name, ref, tar, eng, repeat, card, sm_count, oracle):
    rec = dict(workload=name, shape_zyx=list(ref.shape))
    eng.set_images_3d(ref, tar)
    eng.sift3d()  # warm-up: module load, buffer growth, every kernel shape
    e2e, stages = [], []
    for _ in range(repeat):
        t0 = time.perf_counter()
        eng.set_images_3d(ref, tar)
        a, b, n_oct = eng.sift3d()
        e2e.append((time.perf_counter() - t0) * 1e3)
        stages.append(eng.sift3d_stage_times())
    n1, n2 = eng.sift3d_inspect_counts(0), eng.sift3d_inspect_counts(1)
    rec.update(n_octave=n_oct, ref_keypoints=n1, tar_keypoints=n2, matches=len(a),
               ref_candidates=int(eng.sift3d_inspect(0)["cand"].shape[0]), tar_candidates=int(eng.sift3d_inspect(1)["cand"].shape[0]))
    rec["end_to_end_ms"] = e2e
    rec["stage_ms"] = {k: [s[k] for s in stages] for k in ob.api.SIFT3D_STAGES}
    # the distance pass issues one FSUB, one FMUL and one FADD per pair and component (no FMA: the sums are the reference's)
    instr = float(n1) * n2 * 768 * 3
    t_match = min(rec["stage_ms"]["matching"]) * 1e-3
    rec["matching_instructions"] = instr
    if t_match > 0 and "max_sm_clock_mhz" in card:
        issue = sm_count * 128 * card["max_sm_clock_mhz"] * 1e6  # FP32 lanes x clock: non-FMA instructions per second
        rec["matching_instr_per_s"] = instr / t_match
        rec["matching_fp32_issue_rate_per_s"] = issue
        rec["matching_share_of_fp32_issue"] = instr / t_match / issue
    if oracle:
        from oracle import sift3d as s3
        threads = max(1, (os.cpu_count() or 2) - 1)
        t0 = time.perf_counter()
        s3.sift3d(ref, tar, threads=threads)
        rec["oracle_cpu_s"] = time.perf_counter() - t0
        rec["oracle_threads"] = threads
    else:
        rec["oracle_cpu_s"] = "not measured"
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--large", default="960,288,592", help="x,y,z of the synthetic pair")
    ap.add_argument("--oracle", default="crop", choices=["none", "crop", "all"], help="workloads on which the CPU oracle is timed")
    ap.add_argument("--only", default="", help="run only this workload")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    card = _card()
    sm_count = _sm_count()
    eng = ob.Engine(0)
    dims = tuple(int(v) for v in args.large.split(","))
    out = dict(card=card, sm_count=sm_count, nproc=os.cpu_count(), workloads=[])
    for name in ("al_foam4_crop", "synthetic_%dx%dx%d" % dims):
        if args.only and args.only != name:
            continue
        ref, tar = _workload(name, dims)
        oracle = args.oracle == "all" or (args.oracle == "crop" and name == "al_foam4_crop")
        out["workloads"].append(run(name, ref, tar, eng, args.repeat, card, sm_count, oracle))
        if args.out:  # rewritten after every workload
            os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
            with open(args.out, "w") as f:
                f.write(json.dumps(out, indent=1) + "\n")
    eng.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
