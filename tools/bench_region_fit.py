"""RegionFit2D / RegionFit3D: three arms on the same synthetic records, alternated over rounds in one process.

  host:   ocb_region_fit2d / 3d on numpy records (both sets up, the queue back), host clock around the call;
  dev:    ocb_region_fit*_dev on device records, CUDA events;
  oracle: the CPU oracle (oracle/oc_region_fit.cpp, the reference's float32 arithmetic on a uniform grid) on all the host's threads,
          the CPU reference arm.

Workloads: 2D at the geometry of the reference's SIFT -> ICGN2 -> RegionFit example, 521 x 521 POIs at a 3 px pitch
(271 441 POIs), radius 12, 9 neighbours at least, with 1 % of the POIs unreliable (scattered) and 10 % (discs of 5 to 15 px);
3D at config D's POI grid (20 000 POIs at 4 x 7 x 8 voxels), radius 20, 12 neighbours at least, 10 % unreliable in balls.  The
reliable records carry an affine displacement field plus noise; the unreliable ones garbage.  Each arm's records are compared
with the float64 witness of tests/region_fit_cases.py, and the launches per call are read with ocb_launch_count.

    python tools/bench_region_fit.py --out profiles/h100_bench_region_fit.json
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import opencorr_b200 as ob  # noqa: E402
from opencorr_b200 import synth  # noqa: E402
from bench_series import _card  # noqa: E402
from oracle import region_fit as oracle  # noqa: E402
import region_fit_cases as rc  # noqa: E402


def _blobs(pos, frac, radii, rng):
    """A mask of the POIs inside random discs / balls, grown until it holds frac of them."""
    bad = np.zeros(len(pos), bool)
    lo, hi = pos.min(0), pos.max(0)
    while bad.mean() < frac:
        c = rng.uniform(lo, hi)
        bad |= ((pos - c) ** 2).sum(1) < rng.uniform(*radii) ** 2
    return bad


def workload(name, seed=0):
    rng = np.random.default_rng(seed)
    if name.startswith("2d"):
        pos = synth.grid_2d(20, 20, 521, 521, 3, 3)
        radius, k_min = 12.0, 9
        bad = rng.uniform(size=len(pos)) < 0.01 if name == "2d_scattered_1pct" else _blobs(pos, 0.10, (5.0, 15.0), rng)
    else:
        pos = synth.grid_3d(*synth.CONFIGS["D"]["grid"])
        radius, k_min = 20.0, 12
        bad = _blobs(pos, 0.10, (8.0, 20.0), rng)
    rel = rc.reliable_set(pos[~bad], rng, noise=0.05)
    q = rc.queue_set(pos[bad], rng)
    return rel, q, radius, k_min


def run(name, rounds, reps, eng):
    import torch
    rel, q, radius, k_min = workload(name)
    kind = "2d" if q.shape[1] == 25 else "3d"
    w = rc.witness(rel, q, radius, k_min)
    d_rel = torch.from_numpy(rel).cuda()
    d_q = torch.from_numpy(q.copy()).cuda()
    stream = torch.cuda.current_stream()
    eng.set_stream(stream.cuda_stream)
    threads = oracle.max_threads()

    def host():
        out = q.copy()
        t0 = time.perf_counter()
        eng.region_fit(rel, out, radius, k_min)
        return (time.perf_counter() - t0) * 1e3, out

    def dev():
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(reps):
            eng.region_fit_dev(kind, d_rel.data_ptr(), len(rel), d_q.data_ptr(), len(q), radius, k_min)
        e1.record(stream)
        e1.synchronize()
        return e0.elapsed_time(e1) / reps

    def cpu():
        out = q.copy()
        t0 = time.perf_counter()
        oracle.region_fit(rel, out, radius, k_min, threads=threads)
        return (time.perf_counter() - t0) * 1e3, out

    before = eng.launch_count()
    _, out_host = host()  # also the warm-up
    launches = eng.launch_count() - before
    dev()
    ms_host, ms_dev, ms_cpu = [], [], []
    for _ in range(rounds):
        ms_host.append(min(host()[0] for _ in range(reps)))
        ms_dev.append(dev())
        t, out_cpu = cpu()
        ms_cpu.append(t)
    torch.cuda.synchronize()
    out_dev = d_q.cpu().numpy()
    eng.use_own_stream()
    checks = {}
    for arm, out, tol in (("host", out_host, rc.TOL), ("dev", out_dev, rc.TOL), ("oracle", out_cpu, 1e-2)):
        n, d = rc.compare(out, q, w, tol, "%s %s" % (name, arm))
        checks[arm] = dict(written=n, max_rel_diff_vs_witness=float("%.3g" % d))
    return dict(workload=name, n_reliable=len(rel), n_queue=len(q), radius=radius, min_neighbors=k_min,
                fallback_pois=int((w.computed & w.fallback).sum()), reps_per_round=reps, launches_per_call=launches,
                host_ms=[round(x, 3) for x in ms_host], dev_ms=[round(x, 4) for x in ms_dev], oracle_ms=[round(x, 2) for x in ms_cpu],
                oracle_threads=threads, oracle_over_dev=[round(c / d, 1) for c, d in zip(ms_cpu, ms_dev)], records_vs_witness=checks)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="2d_scattered_1pct,2d_blobs_10pct,3d_blobs_10pct")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    eng = ob.Engine(0)
    rec = dict(card=_card(), runs=[run(w, args.rounds, args.reps, eng) for w in args.workloads.split(",")])
    eng.close()
    print(json.dumps(rec))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
