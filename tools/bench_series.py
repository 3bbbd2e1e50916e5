"""Image- and volume-series IC-GN benchmark: one reference against F targets, two arms on the same synthetic series, alternated
over rounds in one process and timed with CUDA events.

  (a) the device-resident loop of pair calls: per frame set_images_2d_dev / set_images_3d_dev + icgn2d_prepare /
      icgn3d_prepare + icgn2d1/2_dev / icgn3d1_dev on one carried queue, and a device copy of the frame's records;
  (b) one icgn2d_series_dev / icgn3d_series_dev call.

Geometries: bench.py's config B (2048^2, 50 k POIs, r = 16, ICGN2D1) and C (r = 20, ICGN2D2), and for volumes config D
(256^3, 20 k POIs, r = 16) and F (288^3, 1728 POIs, r = 30); F = 8 frames whose displacement is (f + 1) / F of synth's field.
Both arms' records are compared as uint32 in the same run.

    python tools/bench_series.py --out profiles/h100_bench_series.json
    python tools/bench_series.py --configs D,F --out profiles/h100_bench_series_3d.json
"""
import argparse
import json
import os
import subprocess
import sys

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


def render_series(width, height, n_frames, second_order, rho=2.0, seed=synth.REF_SEED):
    rng = np.random.default_rng(seed)
    n = int(0.5 * width * height / (np.pi * rho * rho))
    cx = rng.uniform(-8, width + 8, n)
    cy = rng.uniform(-8, height + 8, n)
    amp = rng.uniform(0.4, 1.0, n)
    u, v = synth.displacement_2d(cx, cy, width, height, second_order)

    def image(s):
        im = synth._render((height, width), np.stack([cy + s * v, cx + s * u], 1), amp, rho, "cuda")
        return np.round(np.clip(synth.BACKGROUND + (255.0 - synth.BACKGROUND) * im, 0, 255)).astype(np.float32)

    return image(0.0), np.stack([image((f + 1) / n_frames) for f in range(n_frames)])


def run(config, n_frames, rounds, reps, eng):
    if synth.CONFIGS[config]["kind"] == "3d":
        return run_3d(config, n_frames, rounds, reps, eng)
    import torch
    cfg = synth.CONFIGS[config]
    w, h = cfg["size"]
    r, order, conv, stop = cfg["r"], cfg["order"], cfg["conv"], cfg["stop"]
    ref, tars = render_series(w, h, n_frames, order == 2)
    xy = synth.grid_2d(*cfg["grid"])
    n = len(xy)
    seeds = ob.make_poi2d(xy)
    eng.set_images_2d(ref, tars[0])
    eng.fftcc2d(seeds, r, r)
    dev = torch.device("cuda")
    d_ref, d_tars, d_seeds = (torch.from_numpy(a).to(dev) for a in (ref, tars, seeds))
    d_q = torch.empty_like(d_seeds)
    out_a = torch.empty((n_frames, n, ob.POI2D_FLOATS), dtype=torch.float32, device=dev)
    out_b = torch.empty_like(out_a)
    stream = torch.cuda.current_stream()
    eng.set_stream(stream.cuda_stream)
    icgn_dev = eng.icgn2d1_dev if order == 1 else eng.icgn2d2_dev

    def loop():
        d_q.copy_(d_seeds)
        for f in range(n_frames):
            eng.set_images_2d_dev(d_ref.data_ptr(), d_tars[f].data_ptr(), w, h)
            eng.icgn2d_prepare()
            icgn_dev(d_q.data_ptr(), n, r, r, conv, stop)
            out_a[f].copy_(d_q)

    def series():
        eng.set_series_2d_dev(d_ref.data_ptr(), d_tars.data_ptr(), n_frames, w, h)
        eng.icgn2d_series_dev(order, d_seeds.data_ptr(), out_b.data_ptr(), n, r, r, conv, stop)

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(reps):
            fn()
        e1.record(stream)
        e1.synchronize()
        return e0.elapsed_time(e1) / reps

    loop()
    series()  # warm-up: module load, buffers, both kernels
    torch.cuda.synchronize()
    identical = torch.equal(out_a.view(torch.int32), out_b.view(torch.int32))
    ms_a, ms_b = [], []
    for _ in range(rounds):
        ms_a.append(timed(loop))
        ms_b.append(timed(series))
    identical = identical and torch.equal(out_a.view(torch.int32), out_b.view(torch.int32))
    eng.use_own_stream()
    last = out_b[-1].cpu().numpy()
    return dict(config=config, size=[w, h], n_poi=n, r=r, order=order, n_frames=n_frames, reps_per_round=reps,
                loop_ms=[round(x, 4) for x in ms_a], series_ms=[round(x, 4) for x in ms_b],
                loop_over_series=[round(a / b, 4) for a, b in zip(ms_a, ms_b)],
                records_identical=bool(identical), last_frame_valid_frac=float((last[:, 16] >= 0).mean()))


def run_3d(config, n_frames, rounds, reps, eng):
    import torch
    cfg = synth.CONFIGS[config]
    dx, dy, dz = cfg["size"]
    r, conv, stop = cfg["r"], cfg["conv"], cfg["stop"]
    ref, tars = synth.speckle_series_3d(dx, dy, dz, n_frames, device="cuda")
    xyz = synth.grid_3d(*cfg["grid"])
    n = len(xyz)
    seeds = ob.make_poi3d(xyz)
    eng.set_images_3d(ref, tars[0])
    eng.fftcc3d(seeds, r, r, r)
    dev = torch.device("cuda")
    d_ref, d_tars, d_seeds = (torch.from_numpy(a).to(dev) for a in (ref, tars, seeds))
    d_q = torch.empty_like(d_seeds)
    out_a = torch.empty((n_frames, n, ob.POI3D_FLOATS), dtype=torch.float32, device=dev)
    out_b = torch.empty_like(out_a)
    stream = torch.cuda.current_stream()
    eng.set_stream(stream.cuda_stream)

    def loop():
        d_q.copy_(d_seeds)
        for f in range(n_frames):
            eng.set_images_3d_dev(d_ref.data_ptr(), d_tars[f].data_ptr(), dx, dy, dz)
            eng.icgn3d_prepare()
            eng.icgn3d1_dev(d_q.data_ptr(), n, r, r, r, conv, stop)
            out_a[f].copy_(d_q)

    def series():
        eng.set_series_3d_dev(d_ref.data_ptr(), d_tars.data_ptr(), n_frames, dx, dy, dz)
        eng.icgn3d_series_dev(d_seeds.data_ptr(), out_b.data_ptr(), n, r, r, r, conv, stop)

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(reps):
            fn()
        e1.record(stream)
        e1.synchronize()
        return e0.elapsed_time(e1) / reps

    loop()
    series()  # warm-up: module load, buffers, every kernel
    torch.cuda.synchronize()
    identical = torch.equal(out_a.view(torch.int32), out_b.view(torch.int32))
    ms_a, ms_b = [], []
    for _ in range(rounds):
        ms_a.append(timed(loop))
        ms_b.append(timed(series))
    identical = identical and torch.equal(out_a.view(torch.int32), out_b.view(torch.int32))
    eng.use_own_stream()
    last = out_b[-1].cpu().numpy()
    return dict(config=config, size=[dx, dy, dz], n_poi=n, r=r, order=1, n_frames=n_frames, reps_per_round=reps,
                loop_ms=[round(x, 4) for x in ms_a], series_ms=[round(x, 4) for x in ms_b],
                loop_over_series=[round(a / b, 4) for a, b in zip(ms_a, ms_b)],
                records_identical=bool(identical), last_frame_valid_frac=float((last[:, 18] >= 0).mean()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="B,C")
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    eng = ob.Engine(0)
    rec = dict(card=_card(), runs=[run(c, args.frames, args.rounds, args.reps, eng) for c in args.configs.split(",")])
    eng.close()
    line = json.dumps(rec)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rec, f, indent=1)
    if not all(x["records_identical"] for x in rec["runs"]):
        sys.exit("series records differ from the loop of pair calls")


if __name__ == "__main__":
    main()
