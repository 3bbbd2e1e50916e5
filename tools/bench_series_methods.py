"""Image-series benchmark of the IC-LM and NR2D1 series calls: one reference against F targets, two arms on the same synthetic
series, alternated over rounds in one process and timed with CUDA events.

  (a) the device-resident loop of pair calls: per frame set_images_2d_dev + prepare (icgn2d_prepare / nr2d_prepare) + the
      method's _dev pair call (ocb_iclm2d_dev / ocb_nr2d1_dev) on one carried queue, and a device copy of the frame's records;
  (b) one iclm2d_series_dev / nr2d1_series_dev call.

Methods and geometries: ICLM2D1 and NR2D1 at bench.py's config B (2048^2, 50 k POIs, r = 16) and ICLM2D2 at config C's r = 20,
F = 8 frames whose displacement is (f + 1) / F of synth's field.  IC-LM runs with the default damping (100, 0.1, 10).  Both
arms' records are compared as uint32 in the same run.

    python tools/bench_series_methods.py --out profiles/h100_bench_series_methods.json
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import opencorr_b200 as ob  # noqa: E402
from opencorr_b200 import synth  # noqa: E402
from bench_series import _card, render_series  # noqa: E402

DAMPING = (100.0, 0.1, 10.0)
METHODS = {"ICLM2D1": ("B", "iclm", 1), "NR2D1": ("B", "nr", 1), "ICLM2D2": ("C", "iclm", 2)}


def run(name, n_frames, rounds, reps, eng):
    import torch
    config, kind, order = METHODS[name]
    cfg = synth.CONFIGS[config]
    w, h = cfg["size"]
    r, conv, stop = cfg["r"], cfg["conv"], cfg["stop"]
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
    lib, ctx = eng._lib, eng._ctx

    def pair():
        if kind == "iclm":
            eng.icgn2d_prepare()
            eng._ck(lib.ocb_iclm2d_dev(ctx, order, d_q.data_ptr(), n, r, r, conv, stop, *DAMPING))
        else:
            eng.nr2d_prepare()
            eng._ck(lib.ocb_nr2d1_dev(ctx, d_q.data_ptr(), n, r, r, conv, stop))

    def loop():
        d_q.copy_(d_seeds)
        for f in range(n_frames):
            eng.set_images_2d_dev(d_ref.data_ptr(), d_tars[f].data_ptr(), w, h)
            pair()
            out_a[f].copy_(d_q)

    def series():
        eng.set_series_2d_dev(d_ref.data_ptr(), d_tars.data_ptr(), n_frames, w, h)
        if kind == "iclm":
            eng.iclm2d_series_dev(order, d_seeds.data_ptr(), out_b.data_ptr(), n, r, r, conv, stop, DAMPING)
        else:
            eng.nr2d1_series_dev(d_seeds.data_ptr(), out_b.data_ptr(), n, r, r, conv, stop)

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
    return dict(method=name, config=config, size=[w, h], n_poi=n, r=r, n_frames=n_frames, reps_per_round=reps,
                loop_ms=[round(x, 4) for x in ms_a], series_ms=[round(x, 4) for x in ms_b],
                loop_over_series=[round(a / b, 4) for a, b in zip(ms_a, ms_b)],
                records_identical=bool(identical), last_frame_valid_frac=float((last[:, 16] >= 0).mean()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--methods", default="ICLM2D1,NR2D1,ICLM2D2")
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    eng = ob.Engine(0)
    rec = dict(card=_card(), runs=[run(m, args.frames, args.rounds, args.reps, eng) for m in args.methods.split(",")])
    eng.close()
    print(json.dumps(rec))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rec, f, indent=1)
    if not all(x["records_identical"] for x in rec["runs"]):
        sys.exit("series records differ from the loop of pair calls")


if __name__ == "__main__":
    main()
