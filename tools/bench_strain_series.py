"""Strain over a series: two arms on the same synthetic records, alternated over rounds in one process and timed with CUDA events.

  (a) the loop of n_frames pair calls ocb_strain*_dev on the frame slices of one device buffer;
  (b) one ocb_strain*_series_dev call on a copy of that buffer.

Geometries (the reference's strain examples): 2D at bench.py's config B grid (50 000 POIs at 7 x 9 px, about 20 neighbours each)
with radius 20 (test_2d_dic_strain.cpp); 3D at config D's grid (20 000 POIs at 4 x 7 x 8 voxels, about 500 neighbours each) with
radius 30 (test_dvc_strain.cpp); stereo POI2DS records at the Step18 grid of tools/bench_stereo_series.py (97 969 POIs) with
radius 20 (test_3d_dic_strain.cpp).  Records: fixed positions, per frame an affine displacement field growing with the frame
plus noise, and ZNCCs with about 10 % below 0.9, drawn again in every frame.  Both arms' records are compared as uint32 in the
same run, and each arm's launches per call are read with ocb_launch_count.  "list_overflow_pois" counts the POIs whose
neighbour lists outgrow what the series kernel keeps (strain.cu STRAIN_LIST) and that search again in every frame.

    python tools/bench_strain_series.py --out profiles/h100_bench_strain_series.json
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import opencorr_b200 as ob  # noqa: E402
from opencorr_b200 import synth  # noqa: E402
from bench_series import _card  # noqa: E402

STRAIN_LIST = 32  # strain.cu: indices kept per lane
K_MIN = 5
# name -> record floats, positions, radius
GEOMETRIES = {
    "2d": (ob.POI2D_FLOATS, lambda: synth.grid_2d(*synth.CONFIGS["B"]["grid"]), 20.0),
    "3d": (ob.POI3D_FLOATS, lambda: synth.grid_3d(*synth.CONFIGS["D"]["grid"]), 30.0),
    "2ds": (28, lambda: synth.grid_2d(420, 250, 313, 313, 5, 5), 20.0),
}
# record floats -> displacement fields, ZNCC fields, fit coordinates (POI2DS ref_coor)
LAYOUT = {25: ((2, 8), (16,), None), 31: ((3, 7, 11), (18,), None), 28: ((2, 3, 4), (5, 6, 7), 14)}


def records(floats, pos, n_frames, seed=0):
    rng = np.random.default_rng(seed)
    disp, zncc, fc = LAYOUT[floats]
    n = len(pos)
    q = np.zeros((n_frames, n, floats), np.float32)
    q[:, :, :pos.shape[1]] = pos
    fit = pos.astype(np.float64)
    for f in range(n_frames):
        qf = q[f]
        if fc is not None:  # a curved surface over the image plane
            x, y = fit[:, 0], fit[:, 1]
            qf[:, fc:fc + 3] = np.stack([x - 40, y + 25, 400 + 2 * np.sin(x / 90.0) * np.cos(y / 70.0) + rng.normal(0, 0.05, n)], 1)
        coords = qf[:, fc:fc + 3].astype(np.float64) if fc is not None else fit
        G = (f + 1) / n_frames * rng.normal(0, 0.01, (coords.shape[1], len(disp)))
        d = (coords - coords.min(0)) @ G + rng.normal(0, 0.1, (n, len(disp)))
        qf[:, list(disp)] = d
        qf[:, list(zncc)] = rng.uniform(0.91, 1.0, (n, len(zncc)))
        low = rng.uniform(size=n) < 0.1
        qf[low, zncc[0]] = rng.uniform(0.3, 0.89, low.sum())
    return q


def list_overflow(pos, radius, k_min):
    """The POIs whose radius search keeps more than STRAIN_LIST indices on some lane: strain.cu's grid (a finite radius, no
    growth), stable sort, cell runs and lane assignment replayed in numpy."""
    from scipy.spatial import cKDTree
    P = np.asarray(pos, np.float32)
    D = P.shape[1]
    lo, hi = P.min(0), P.max(0)
    cell = float(abs(np.float32(radius)))
    inv = np.float32(np.float32(1.0 / cell) * np.float32(0.999))
    nc = (np.floor((hi.astype(np.float64) - lo.astype(np.float64)) / cell) + 2).astype(np.int64)
    c = np.clip(np.floor((P - lo) * inv).astype(np.int64), 0, nc - 1)
    key = c[:, 0] + nc[0] * (c[:, 1] + (nc[1] * c[:, 2] if D == 3 else 0))
    order = np.argsort(key, kind="stable")
    skey, rank = key[order], np.empty(len(P), np.int64)
    rank[order] = np.arange(len(P))
    lists = cKDTree(P.astype(np.float64)).query_ball_point(P.astype(np.float64), radius * 1.001)
    owner = np.repeat(np.arange(len(P)), [len(x) for x in lists])
    other = np.concatenate([np.asarray(x, np.int64) for x in lists])
    diff = P[other] - P[owner]
    d2 = diff[:, 0] * diff[:, 0]
    for k in range(1, D):
        d2 = d2 + diff[:, k] * diff[:, k]
    keep = d2 < np.float32(np.float32(radius) * np.float32(radius))
    owner, other = owner[keep], other[keep]
    found = np.bincount(owner, minlength=len(P))
    run_lo = np.searchsorted(skey, key[other] - c[other, 0] + np.maximum(c[owner, 0] - 1, 0), "left")
    per_lane = np.bincount(owner * 32 + (rank[other] - run_lo) % 32, minlength=32 * len(P)).reshape(-1, 32)
    return int(((per_lane.max(1) > STRAIN_LIST) & (found >= k_min)).sum())


def run(name, n_frames, rounds, reps, eng):
    import torch
    floats, make_pos, radius = GEOMETRIES[name]
    pos = make_pos()
    n = len(pos)
    q = records(floats, pos, n_frames)
    dev = torch.device("cuda")
    d_a = torch.from_numpy(q).to(dev)
    d_b = d_a.clone()
    stream = torch.cuda.current_stream()
    eng.set_stream(stream.cuda_stream)
    lib, ctx = eng._lib, eng._ctx
    pair = getattr(lib, "ocb_strain%s_dev" % name)
    rec_bytes = n * floats * 4

    def loop():
        for f in range(n_frames):
            eng._ck(pair(ctx, d_a.data_ptr() + f * rec_bytes, n, radius, K_MIN, 0.9, 1))

    def series():
        eng.strain_series_dev(name, d_b.data_ptr(), n_frames, n, radius, K_MIN, 0.9, 1)

    def launches(fn):
        before = eng.launch_count()
        fn()
        return eng.launch_count() - before

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(reps):
            fn()
        e1.record(stream)
        e1.synchronize()
        return e0.elapsed_time(e1) / reps

    launches_a, launches_b = launches(loop), launches(series)  # also the warm-up
    torch.cuda.synchronize()
    identical = torch.equal(d_a.view(torch.int32), d_b.view(torch.int32))
    ms_a, ms_b = [], []
    for _ in range(rounds):
        ms_a.append(timed(loop))
        ms_b.append(timed(series))
    torch.cuda.synchronize()
    identical = identical and torch.equal(d_a.view(torch.int32), d_b.view(torch.int32))
    eng.use_own_stream()
    out = d_b.cpu().numpy()
    fitted = float((out[..., {25: 20, 31: 22, 28: 20}[floats]] != 0).mean())
    return dict(geometry=name, n_poi=n, radius=radius, min_neighbors=K_MIN, n_frames=n_frames, reps_per_round=reps,
                loop_ms=[round(x, 4) for x in ms_a], series_ms=[round(x, 4) for x in ms_b],
                loop_over_series=[round(a / b, 4) for a, b in zip(ms_a, ms_b)], launches_per_call=dict(loop=launches_a, series=launches_b),
                list_overflow_pois=list_overflow(pos, radius, K_MIN), fitted_frac=round(fitted, 4), records_identical=bool(identical))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--geometries", default="2d,3d,2ds")
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    eng = ob.Engine(0)
    rec = dict(card=_card(), runs=[run(g, args.frames, args.rounds, args.reps, eng) for g in args.geometries.split(",")])
    eng.close()
    print(json.dumps(rec))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rec, f, indent=1)
    if not all(x["records_identical"] for x in rec["runs"]):
        sys.exit("series records differ from the loop of pair calls")


if __name__ == "__main__":
    main()
