"""Series calls that re-seed lost POIs: what re-seeding costs, timed with CUDA events, arms alternated over rounds in one process.

Two comparisons per geometry, on synthetic series of F = 8 frames whose displacement is (f + 1) / F of synth's field:
  clean: the plain series call (icgn2d_series_dev / icgn3d_series_dev) against the re-seeding call with zncc_min = 0.5 on the
         same series, where nothing is lost: the overhead of a call that loses nothing;
  lossy: frame 3 covers the subsets of a box of POIs with speckles from elsewhere in the frame (`reseeded` in the record
         gives the POIs re-seeded per frame).  The re-seeding call against the device-resident loop of pair calls that does
         the same: per frame set_images_*_dev + prepare + IC-GN on every POI, the
         lost POIs found and rebuilt with torch, FFT-CC + IC-GN on them, scattered back.
The records of the two arms of each comparison are compared as uint32 in the same run.  2D runs with OCB_ICGN2D_WPP=1 (the
choice a 50 k POI launch makes anyway), so that the pair loop's sub-queue launches take the same warps per POI as the call's.

Geometries: bench.py's config B (2048^2, 50 k POIs, r = 16, ICGN2D1) and D (256^3, 20 k POIs, r = 16, ICGN3D1); FFT-CC r = 16.

    python tools/bench_series_reseed.py --out profiles/h100_bench_series_reseed.json
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

ZNCC_MIN = 0.5
LOSSY_FRAME = 3


def _timed(stream, reps):
    import torch

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(reps):
            fn()
        e1.record(stream)
        e1.synchronize()
        return e0.elapsed_time(e1) / reps
    return timed


def _occlude(tars, k, box):
    """box: (lo, hi) corner arrays in array-axis order; the box of frame k gets the frame's content from half a frame away."""
    lo, hi = box
    sl = tuple(slice(a, b) for a, b in zip(lo, hi))
    out = tars.copy()
    shifts = tuple(s // 2 for s in tars.shape[1:])
    out[(k,) + sl] = np.roll(tars[k], shifts, tuple(range(tars.ndim - 1)))[sl]
    return out


def _compare(name, arm_a, arm_b, out_a, out_b, rounds, timed):
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
    return dict(comparison=name, a_ms=[round(x, 4) for x in ms_a], b_ms=[round(x, 4) for x in ms_b],
                b_over_a=[round(b / a, 4) for a, b in zip(ms_a, ms_b)], records_identical=bool(identical))


def run(config, n_frames, rounds, reps, eng):
    import torch
    cfg = synth.CONFIGS[config]
    three = cfg["kind"] == "3d"
    r, conv, stop = cfg["r"], cfg["conv"], cfg["stop"]
    fr = 16
    if three:
        dx, dy, dz = cfg["size"]
        ref, clean = synth.speckle_series_3d(dx, dy, dz, n_frames, device="cuda")
        pts = synth.grid_3d(*cfg["grid"])
        seeds = ob.make_poi3d(pts)
        eng.set_images_3d(ref, clean[0])
        eng.fftcc3d(seeds, r, r, r)
        rec, zc, disp, keep = ob.POI3D_FLOATS, 18, [3, 7, 11], [0, 1, 2, 28, 29, 30]
        # the POIs whose subvolume meets a box of 0.13 of the grid's extent per axis (plus the subvolume and a margin)
        lo_p, hi_p = pts.min(0), pts.max(0)
        box_lo, box_hi = lo_p + 0.2 * (hi_p - lo_p), lo_p + 0.33 * (hi_p - lo_p)
    else:
        w, h = cfg["size"]
        ref, clean = render_series(w, h, n_frames, cfg["order"] == 2)
        pts = synth.grid_2d(*cfg["grid"])
        seeds = ob.make_poi2d(pts)
        eng.set_images_2d(ref, clean[0])
        eng.fftcc2d(seeds, r, r)
        rec, zc, disp, keep = ob.POI2D_FLOATS, 16, [2, 8], [0, 1, 23, 24]
        # the POIs whose subset meets a box of 0.2 of the grid's extent per axis (plus the subset and a margin)
        lo_p, hi_p = pts.min(0), pts.max(0)
        box_lo, box_hi = lo_p + 0.3 * (hi_p - lo_p), lo_p + 0.5 * (hi_p - lo_p)
    block = np.all((pts >= box_lo) & (pts <= box_hi), 1)
    xyz_lo = np.floor(box_lo - r - 4 - 3).astype(int)  # 3: room for the displacement
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
    set_series = eng.set_series_3d_dev if three else eng.set_series_2d_dev
    keep_t = torch.tensor(keep, device=dev)
    disp_t = torch.tensor(disp, device=dev)

    def plain(tars):
        def call():
            set_series(d_ref.data_ptr(), tars.data_ptr(), n_frames, *dims)
            if three:
                eng.icgn3d_series_dev(d_seeds.data_ptr(), out_a.data_ptr(), n, r, r, r, conv, stop)
            else:
                eng.icgn2d_series_dev(cfg["order"], d_seeds.data_ptr(), out_a.data_ptr(), n, r, r, conv, stop)
        return call

    def reseed(tars, counts):
        def call():
            set_series(d_ref.data_ptr(), tars.data_ptr(), n_frames, *dims)
            if three:
                c = eng.icgn3d_series_reseed_dev(d_seeds.data_ptr(), out_b.data_ptr(), n, r, r, r, conv, stop, fr, fr, fr, ZNCC_MIN)
            else:
                c = eng.icgn2d_series_reseed_dev(cfg["order"], d_seeds.data_ptr(), out_b.data_ptr(), n, r, r, conv, stop, fr, fr, ZNCC_MIN)
            counts[:] = c
        return call

    def pair_loop(tars):
        def call():
            d_q.copy_(d_seeds)
            anchor = d_seeds[:, disp_t].clone()
            for f in range(n_frames):
                if three:
                    eng.set_images_3d_dev(d_ref.data_ptr(), tars[f].data_ptr(), *dims)
                    eng.icgn3d_prepare()
                    eng.icgn3d1_dev(d_q.data_ptr(), n, r, r, r, conv, stop)
                else:
                    eng.set_images_2d_dev(d_ref.data_ptr(), tars[f].data_ptr(), *dims)
                    eng.icgn2d_prepare()
                    (eng.icgn2d1_dev if cfg["order"] == 1 else eng.icgn2d2_dev)(d_q.data_ptr(), n, r, r, conv, stop)
                if f > 0:
                    good = out_a[f - 1][:, zc] >= ZNCC_MIN
                    anchor[good] = out_a[f - 1][good][:, disp_t]
                lost = torch.nonzero(~(d_q[:, zc] >= ZNCC_MIN)).flatten()
                m = int(lost.numel())
                if m:
                    sub = torch.zeros((m, rec), dtype=torch.float32, device=dev)
                    sub[:, keep_t] = d_seeds[lost][:, keep_t]
                    sub[:, disp_t] = anchor[lost]
                    if three:
                        eng.fftcc3d_dev(sub.data_ptr(), m, fr, fr, fr)
                        eng.icgn3d1_dev(sub.data_ptr(), m, r, r, r, conv, stop)
                    else:
                        eng.fftcc2d_dev(sub.data_ptr(), m, fr, fr)
                        (eng.icgn2d1_dev if cfg["order"] == 1 else eng.icgn2d2_dev)(sub.data_ptr(), m, r, r, conv, stop)
                    d_q[lost] = sub
                out_a[f].copy_(d_q)
        return call

    counts_clean = np.zeros(n_frames, np.int64)
    counts_lossy = np.zeros(n_frames, np.int64)
    runs = [_compare("clean: plain series (a) vs re-seeding call (b)", plain(d_clean), reseed(d_clean, counts_clean), out_a, out_b, rounds, timed)]
    runs[-1]["reseeded"] = counts_clean.tolist()
    runs.append(_compare("lossy: pair-call loop (a) vs re-seeding call (b)", pair_loop(d_lossy), reseed(d_lossy, counts_lossy), out_a, out_b, rounds,
                         timed))
    runs[-1]["reseeded"] = counts_lossy.tolist()
    eng.use_own_stream()
    return dict(config=config, size=list(cfg["size"]), n_poi=n, r=r, fft_r=fr, order=cfg["order"], n_frames=n_frames, zncc_min=ZNCC_MIN,
                occluded_frame=LOSSY_FRAME, pois_centred_in_box=int(block.sum()), reps_per_round=reps, comparisons=runs)


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
    if not all(c["records_identical"] for x in rec["runs"] for c in x["comparisons"]):
        sys.exit("records differ between the arms of a comparison")


if __name__ == "__main__":
    main()
