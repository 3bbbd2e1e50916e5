"""Series calls that recover unreliable POIs: what recovery costs, timed with CUDA events, arms alternated over rounds in one process.

Two comparisons per geometry, on synthetic series of F = 8 frames whose displacement is (f + 1) / F of synth's field:
  clean: the plain series call (icgn2d_series_dev / icgn3d_series_dev) against the recovering call on the same series, where
         (almost) nothing is unreliable: the overhead of the scan and the classification;
  lossy: frame 3 covers the subsets of a box of POIs with speckles from elsewhere in the frame.  The recovering call against the
         device-resident loop of existing calls that does the same: per frame set_images_*_dev + prepare + IC-GN on every POI,
         then icgn*_recover_dev on the queue.
The records of the two arms of the lossy comparison, and the per-frame counts, are compared in the same run; the clean arms are
compared when the recovering call recovers nothing.  2D runs with OCB_ICGN2D_WPP=1 (the choice a 50 k POI launch makes anyway).

Geometries: bench.py's config B (2048^2, 50 k POIs, r = 16, ICGN2D1) and D (256^3, 20 k POIs, r = 16, ICGN3D1).  Recovery:
radius 20, 9 (2D) / 12 (3D) neighbours, zncc_high 0.9, zncc_low 0.5, at most 20 rounds.

    python tools/bench_series_recover.py --out profiles/h100_bench_series_recover.json
"""
import argparse
import json
import os
import sys

os.environ.setdefault("OCB_ICGN2D_WPP", "1")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402

import opencorr_b200 as ob  # noqa: E402
from opencorr_b200 import synth  # noqa: E402
from bench_series import _card, render_series  # noqa: E402
from bench_series_reseed import _occlude, _timed  # noqa: E402

LOSSY_FRAME = 3
RADIUS, HIGH, LOW, ROUNDS = 20.0, 0.9, 0.5, 20


def _compare(name, arm_a, arm_b, out_a, out_b, counts_a, counts_b, rounds, timed, check_records=True):
    import torch
    arm_a()
    arm_b()  # warm-up: module load, buffers, every kernel
    torch.cuda.synchronize()
    identical = torch.equal(out_a.view(torch.int32), out_b.view(torch.int32))
    ms_a, ms_b = [], []
    for _ in range(rounds):
        ms_a.append(timed(arm_a))
        ms_b.append(timed(arm_b))
    identical = identical and torch.equal(out_a.view(torch.int32), out_b.view(torch.int32))
    same_counts = counts_a is None or all(np.array_equal(a, b) for a, b in zip(counts_a, counts_b))
    return dict(comparison=name, a_ms=[round(x, 4) for x in ms_a], b_ms=[round(x, 4) for x in ms_b],
                b_over_a=[round(b / a, 4) for a, b in zip(ms_a, ms_b)], records_identical=bool(identical) if check_records else None,
                counts_identical=bool(same_counts), recovered_per_frame=counts_b[0].sum(1).tolist(), remaining=counts_b[1].tolist())


def run(config, n_frames, rounds, reps, eng):
    import torch
    cfg = synth.CONFIGS[config]
    three = cfg["kind"] == "3d"
    r, conv, stop = cfg["r"], cfg["conv"], cfg["stop"]
    k_min = 12 if three else 9
    if three:
        dx, dy, dz = cfg["size"]
        ref, clean = synth.speckle_series_3d(dx, dy, dz, n_frames, device="cuda")
        pts = synth.grid_3d(*cfg["grid"])
        seeds = ob.make_poi3d(pts)
        eng.set_images_3d(ref, clean[0])
        eng.fftcc3d(seeds, r, r, r)
        rec = ob.POI3D_FLOATS
        lo_p, hi_p = pts.min(0), pts.max(0)
        box_lo, box_hi = lo_p + 0.2 * (hi_p - lo_p), lo_p + 0.33 * (hi_p - lo_p)
    else:
        w, h = cfg["size"]
        ref, clean = render_series(w, h, n_frames, cfg["order"] == 2)
        pts = synth.grid_2d(*cfg["grid"])
        seeds = ob.make_poi2d(pts)
        eng.set_images_2d(ref, clean[0])
        eng.fftcc2d(seeds, r, r)
        rec = ob.POI2D_FLOATS
        lo_p, hi_p = pts.min(0), pts.max(0)
        box_lo, box_hi = lo_p + 0.3 * (hi_p - lo_p), lo_p + 0.5 * (hi_p - lo_p)
    block = np.all((pts >= box_lo) & (pts <= box_hi), 1)
    xyz_lo = np.floor(box_lo - r - 4 - 3).astype(int)
    xyz_hi = np.ceil(box_hi + r + 4 + 3).astype(int)
    lossy = _occlude(clean, LOSSY_FRAME, (xyz_lo[::-1], xyz_hi[::-1]))  # array axes are (z,) y, x
    n = len(pts)
    dev = torch.device("cuda")
    d_ref, d_clean, d_lossy, d_seeds = (torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (ref, clean, lossy, seeds))
    out_a = torch.empty((n_frames, n, rec), dtype=torch.float32, device=dev)
    out_b = torch.empty_like(out_a)
    d_q = torch.empty_like(d_seeds)
    stream = torch.cuda.current_stream()
    eng.set_stream(stream.cuda_stream)
    timed = _timed(stream, reps)
    dims = (dx, dy, dz) if three else (w, h)
    radii = (r, r, r) if three else (r, r)
    args = (conv, stop, RADIUS, k_min, HIGH, LOW, ROUNDS)
    set_series = eng.set_series_3d_dev if three else eng.set_series_2d_dev
    counts_a = [np.zeros((n_frames, ROUNDS), np.int64), np.zeros(n_frames, np.int64)]
    counts_b = [np.zeros((n_frames, ROUNDS), np.int64), np.zeros(n_frames, np.int64)]

    def plain(tars):
        def call():
            set_series(d_ref.data_ptr(), tars.data_ptr(), n_frames, *dims)
            if three:
                eng.icgn3d_series_dev(d_seeds.data_ptr(), out_a.data_ptr(), n, r, r, r, conv, stop)
            else:
                eng.icgn2d_series_dev(cfg["order"], d_seeds.data_ptr(), out_a.data_ptr(), n, r, r, conv, stop)
        return call

    def recover(tars):
        def call():
            set_series(d_ref.data_ptr(), tars.data_ptr(), n_frames, *dims)
            if three:
                c = eng.icgn3d_series_recover_dev(d_seeds.data_ptr(), out_b.data_ptr(), n, *radii, *args)
            else:
                c = eng.icgn2d_series_recover_dev(cfg["order"], d_seeds.data_ptr(), out_b.data_ptr(), n, *radii, *args)
            counts_b[0][:], counts_b[1][:] = c
        return call

    def loop(tars):
        def call():
            d_q.copy_(d_seeds)
            for f in range(n_frames):
                if three:
                    eng.set_images_3d_dev(d_ref.data_ptr(), tars[f].data_ptr(), *dims)
                    eng.icgn3d_prepare()
                    eng.icgn3d1_dev(d_q.data_ptr(), n, r, r, r, conv, stop)
                    c = eng.icgn3d_recover_dev(d_q.data_ptr(), n, *radii, *args)
                else:
                    eng.set_images_2d_dev(d_ref.data_ptr(), tars[f].data_ptr(), *dims)
                    eng.icgn2d_prepare()
                    (eng.icgn2d1_dev if cfg["order"] == 1 else eng.icgn2d2_dev)(d_q.data_ptr(), n, r, r, conv, stop)
                    c = eng.icgn2d_recover_dev(cfg["order"], d_q.data_ptr(), n, *radii, *args)
                counts_a[0][f], counts_a[1][f] = c
                out_a[f].copy_(d_q)
        return call

    runs = [_compare("clean: plain series (a) vs recovering call (b)", plain(d_clean), recover(d_clean), out_a, out_b, None, counts_b, rounds,
                     timed)]
    runs[-1]["records_identical"] = bool(torch.equal(out_a.view(torch.int32), out_b.view(torch.int32))) if counts_b[0].sum() == 0 else None
    runs.append(_compare("lossy: loop of existing calls (a) vs recovering call (b)", loop(d_lossy), recover(d_lossy), out_a, out_b, counts_a,
                         counts_b, rounds, timed))
    eng.use_own_stream()
    return dict(config=config, size=list(cfg["size"]), n_poi=n, r=r, order=cfg["order"], n_frames=n_frames, occluded_frame=LOSSY_FRAME,
                pois_centred_in_box=int(block.sum()), radius=RADIUS, min_neighbors=k_min, zncc_high=HIGH, zncc_low=LOW, max_rounds=ROUNDS,
                reps_per_round=reps, comparisons=runs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="B,D")
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    eng = ob.Engine(0)
    rec = dict(card=_card(), icgn2d_wpp=os.environ.get("OCB_ICGN2D_WPP"),
               runs=[run(c, args.frames, args.rounds, args.reps, eng) for c in args.configs.split(",")])
    eng.close()
    print(json.dumps(rec))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rec, f, indent=1)
    bad = [c for x in rec["runs"] for c in x["comparisons"] if c["records_identical"] is False or not c["counts_identical"]]
    if bad:
        sys.exit("records or counts differ between the arms of a comparison")


if __name__ == "__main__":
    main()
