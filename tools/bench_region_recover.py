"""Recovery of unreliable POIs (ocb_icgn2d_recover / ocb_icgn3d_recover): three arms on the same registered queue, alternated
over rounds in one process.

  call:    the one call on device records (ocb_icgn*_recover_dev), CUDA events around it;
  witness: the same loop written with ocb_region_fit*_dev, the _dev pair calls and torch bookkeeping on device records
           (tests/region_recover_cases.py witness), CUDA events around it;
  host:    the one call on a numpy queue (ocb_icgn*_recover), host clock around it.

Workloads: config B's geometry (2048^2, 250 x 200 POIs, r = 16) with 10 % of the POIs seeded with garbage in discs, ICGN2D1 and
ICGN2D2; config D's geometry (256^3, 40 x 25 x 20 POIs, r = 16) with 10 % in balls, ICGN3D1; the reference's oht_cfrp pair and
grid (FFTCC2D -> ICGN2D1, then 0.9 / 0.5, radius 12, 9 neighbours, 20 rounds).  The three arms' records must be byte-identical.
A separate pass times each round's RegionFit call (ocb_region_fit*_dev on the round's working records) to report the share of a
call that the fit takes, and how many of its POIs take the k-nearest fallback.

    python tools/bench_region_recover.py --out profiles/h100_bench_region_recover.json
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
import region_recover_cases as rr  # noqa: E402


def config_d_balls(eng):
    cfg = synth.CONFIGS["D"]
    r = cfg["r"]
    ref, tar = synth.speckle_pair_3d(*cfg["size"])
    xyz = synth.grid_3d(*cfg["grid"])
    eng.set_images_3d(ref, tar)
    eng.icgn3d_prepare()
    q = ob.make_poi3d(xyz)
    eng.fftcc3d(q, r, r, r)
    eng.icgn3d1(q, r, r, r, cfg["conv"], cfg["stop"])
    bad = np.flatnonzero(rr.discs(xyz, 0.10, (15.0, 40.0), np.random.default_rng(3)))
    q[bad, 3:15] = 0
    q[bad, 3], q[bad, 7], q[bad, 11] = 11.0, -9.0, 13.0
    sub = np.ascontiguousarray(q[bad])
    eng.icgn3d1(sub, r, r, r, cfg["conv"], cfg["stop"])
    q[bad] = sub
    return rr.Case("config_d_balls", 3, ref, tar, q, (r, r, r), cfg["conv"], cfg["stop"], 30.0, 12, 0.9, 0.5, 20, None, bad)


def build(name, eng):
    if name == "configB_icgn2d1":
        return rr.config_b_discs(eng, 1), 1
    if name == "configB_icgn2d2":
        return rr.config_b_discs(eng, 2), 2
    if name == "configD_icgn3d1":
        return config_d_balls(eng), 1
    return rr.oht_cfrp(eng), 1


def fit_share(eng, c, order, torch):
    """The witness loop again with each RegionFit call timed by CUDA events: total fit ms, and its k-nearest fallback POIs."""
    kind = "2d" if c.dim == 2 else "3d"
    ms = []

    def fit(rel, work):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        eng.set_stream(torch.cuda.current_stream().cuda_stream)
        e0.record()
        eng.region_fit_dev(kind, rel.data_ptr() if len(rel) else 0, len(rel), work.data_ptr(), len(work), c.radius, c.k_min)
        e1.record()
        e1.synchronize()
        eng.use_own_stream()
        ms.append(e0.elapsed_time(e1))

    def register(work):
        torch.cuda.synchronize()
        if c.dim == 3:
            eng.icgn3d1_dev(work.data_ptr(), len(work), *c.r, c.conv, c.stop)
        else:
            (eng.icgn2d1_dev if order == 1 else eng.icgn2d2_dev)(work.data_ptr(), len(work), *c.r, c.conv, c.stop)
        eng.sync()

    d_q = torch.from_numpy(c.q.copy()).cuda()
    rr.witness_loop(d_q, fit, register, c.conv, c.zncc_high, c.zncc_low, c.max_rounds)
    return ms


def run(name, rounds, eng):
    import torch
    c, order = build(name, eng)
    rr.set_pair(eng, c)
    stream = torch.cuda.current_stream()
    n = len(c.q)
    zc, cc = rr.COLS[c.q.shape[1]]
    args = (c.conv, c.stop, c.radius, c.k_min, c.zncc_high, c.zncc_low, c.max_rounds)

    def call():
        d = torch.from_numpy(c.q.copy()).cuda()
        eng.set_stream(stream.cuda_stream)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        before = eng.launch_count()
        if c.dim == 2:
            rec, left = eng.icgn2d_recover_dev(order, d.data_ptr(), n, *c.r, *args)
        else:
            rec, left = eng.icgn3d_recover_dev(d.data_ptr(), n, *c.r, *args)
        launches = eng.launch_count() - before
        e1.record(stream)
        e1.synchronize()
        eng.use_own_stream()
        return e0.elapsed_time(e1), d.cpu().numpy(), rec, left, launches

    def witness():
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        out = rr.witness(eng, c, order=order)
        e1.record(stream)
        e1.synchronize()
        return e0.elapsed_time(e1), out

    def host():
        q = c.q.copy()
        t0 = time.perf_counter()
        if c.dim == 2:
            rec, left = eng.icgn2d_recover(order, q, *c.r, *args)
        else:
            rec, left = eng.icgn3d_recover(q, *c.r, *args)
        return (time.perf_counter() - t0) * 1e3, q, rec, left

    call(), witness(), host()  # warm-up
    ms_call, ms_wit, ms_host = [], [], []
    for _ in range(rounds):
        t, out_call, rec, left, launches = call()
        ms_call.append(t)
        t, w = witness()
        ms_wit.append(t)
        t, out_host, rec_host, left_host = host()
        ms_host.append(t)
    bits = lambda a: np.ascontiguousarray(a).view(np.uint32)
    identical = bool(np.array_equal(bits(out_call), bits(w[0])) and np.array_equal(bits(out_host), bits(w[0]))
                     and np.array_equal(rec, w[1]) and np.array_equal(rec_host, w[1]) and left == w[2] == left_host)
    fit_ms = fit_share(eng, c, order, torch)
    unreliable = int(((c.q[:, zc] < c.zncc_low) | (c.q[:, cc] > c.conv)).sum())
    reliable0 = int((~((c.q[:, zc] < c.zncc_low) | (c.q[:, cc] > c.conv)) & (c.q[:, zc] >= c.zncc_high)).sum())
    return dict(workload=name, n=n, reliable_at_start=reliable0, unreliable_at_start=unreliable, rounds_run=w[3],
                recovered_per_round=w[1][:w[3]].tolist(), remaining=int(w[2]), launches_per_call=launches,
                call_ms=[round(x, 3) for x in ms_call], witness_ms=[round(x, 3) for x in ms_wit], host_ms=[round(x, 3) for x in ms_host],
                witness_over_call=[round(a / b, 2) for a, b in zip(ms_wit, ms_call)],
                region_fit_ms_per_round=[round(x, 3) for x in fit_ms],
                region_fit_share_of_call=round(sum(fit_ms) / float(np.median(ms_call)), 3),
                records_identical_across_arms=identical)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="configB_icgn2d1,configB_icgn2d2,configD_icgn3d1,oht_cfrp")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    eng = ob.Engine(0)
    rec = dict(card=_card(), runs=[run(w, args.rounds, eng) for w in args.workloads.split(",")])
    eng.close()
    print(json.dumps(rec))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rec, f, indent=1)
    if not all(r["records_identical_across_arms"] for r in rec["runs"]):
        sys.exit("the arms' records differ")


if __name__ == "__main__":
    main()
