"""Stereo series (ocb_stereo_series): one call against the device-resident loop of pair calls it replaces, timed with CUDA events,
arms alternated over rounds in one process.

Geometry: the reference's Step18 stereo example (2448 x 2048, its 313 x 313 POI grid at 5 px from (420, 250): 97 969 POIs), r = 16,
ICGN2D1 for the temporal match r1 -> t1 and ICGN2D2 for the cross match r1 -> t2 as in examples/test_3d_dic_epipolar_sift.cpp, on
a synthetic stereo series of F = 8 frames (synth.speckle_stereo_series, rendered on the GPU).
  a: set_stereo_series_dev + one stereo_series_dev call;
  b: per frame set_images_2d_dev + icgn2d_prepare + icgn2d1_dev for view 1, the same with icgn2d2_dev for view 2, then
     stereo_reconstruct_dev of (t1, t2) and the POI2DS records assembled with torch (ref_coor triangulated once per call).
The records of both arms (out1, out2, out2ds) are compared as uint32 in the same run.  The r1 -> r2 match and the frame-0 seeds
are computed once, outside the timed window, with the pair calls (INTEGRATION.md "Stereo series").

    python tools/bench_stereo_series.py --out profiles/h100_bench_stereo_series.json
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402

import opencorr_b200 as ob  # noqa: E402
from opencorr_b200 import synth  # noqa: E402
from bench_series import _card  # noqa: E402

W, H, R, CONV, STOP = 2448, 2048, 16, 0.001, 10


def _rig(eng):
    intr, extr = synth.stereo_rig(W, H)
    cams = []
    for i in range(2):
        kw = {k: float(v) for k, v in zip(ob.api.INTRINSIC_NAMES, intr[i])}
        kw.update({k: float(v) for k, v in zip(("tx", "ty", "tz", "rx", "ry", "rz"), extr[i])})
        c = ob.Calibration(engine=eng, **kw)
        c.prepare(H, W)
        cams.append(c)
    rig = ob.Stereovision(cams[0], cams[1], 0, eng)
    rig.prepare()
    return rig


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    F = args.frames
    dev = torch.device("cuda")
    xy = synth.grid_2d(420, 250, 313, 313, 5, 5)
    n = len(xy)
    d = synth.speckle_stereo_series(W, H, F, points=xy, device="cuda")
    eng = ob.Engine(0)
    rig = _rig(eng)
    # the r1 -> r2 match (ICGN2D2 from the true r2 rounded) and the recipe's frame-0 seeds, with the pair calls
    stereo = ob.make_poi2d(xy)
    g = np.round(d["r2_true"]) - xy
    stereo[:, 2], stereo[:, 8] = g[:, 0], g[:, 1]
    eng.set_images_2d(d["ref1"], d["r2"])
    eng.icgn2d_prepare()
    eng.icgn2d2(stereo, R, R, CONV, STOP)
    seeds1 = ob.make_poi2d(xy)
    eng.set_images_2d(d["ref1"], d["tars1"][0])
    eng.fftcc2d(seeds1, R, R)
    seeds2 = seeds1.copy()
    seeds2[:, 2] += stereo[:, 2]
    seeds2[:, 8] += stereo[:, 8]

    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    d_ref, d_tars1, d_tars2, d_stereo, d_s1, d_s2 = (t(a) for a in (d["ref1"], d["tars1"], d["tars2"], stereo, seeds1, seeds2))
    outs = {arm: [torch.empty((F, n, k), dtype=torch.float32, device=dev) for k in (25, 25, 28)] for arm in "ab"}
    stream = torch.cuda.current_stream()
    eng.set_stream(stream.cuda_stream)

    def arm_a():
        o1, o2, ods = outs["a"]
        eng.set_stereo_series_dev(d_ref.data_ptr(), d_tars1.data_ptr(), d_tars2.data_ptr(), F, W, H)
        eng.stereo_series_dev(rig, d_stereo.data_ptr(), d_s1.data_ptr(), d_s2.data_ptr(), o1.data_ptr(), o2.data_ptr(), ods.data_ptr(), n, 1, 2,
                              R, R, CONV, STOP)

    q1, q2 = torch.empty_like(d_s1), torch.empty_like(d_s2)
    pts = lambda o: torch.stack([o[:, 0] + o[:, 2], o[:, 1] + o[:, 8]], 1).contiguous()  # noqa: E731
    ref3 = torch.empty((n, 3), dtype=torch.float32, device=dev)
    tar3 = torch.empty((n, 3), dtype=torch.float32, device=dev)

    def arm_b():
        o1, o2, ods = outs["b"]
        q1.copy_(d_s1)
        q2.copy_(d_s2)
        r2 = pts(d_stereo)
        c1, c2 = d_s1[:, 0:2].contiguous(), r2.clone()  # copies for the in-place clamp, alive until the launch is enqueued
        rig.reconstruct_dev(c1.data_ptr(), c2.data_ptr(), ref3.data_ptr(), n)
        for f in range(F):
            eng.set_images_2d_dev(d_ref.data_ptr(), d_tars1[f].data_ptr(), W, H)
            eng.icgn2d_prepare()
            eng.icgn2d1_dev(q1.data_ptr(), n, R, R, CONV, STOP)
            eng.set_images_2d_dev(d_ref.data_ptr(), d_tars2[f].data_ptr(), W, H)
            eng.icgn2d_prepare()
            eng.icgn2d2_dev(q2.data_ptr(), n, R, R, CONV, STOP)
            o1[f].copy_(q1)
            o2[f].copy_(q2)
            t1, t2 = pts(q1), pts(q2)
            rec = ods[f]
            rec.zero_()
            rec[:, 0:2] = d_s1[:, 0:2]
            rec[:, 5], rec[:, 6], rec[:, 7] = d_stereo[:, 16], q1[:, 16], q2[:, 16]
            rec[:, 8:10], rec[:, 10:12], rec[:, 12:14] = r2, t1, t2
            c1, c2 = t1.clone(), t2.clone()
            rig.reconstruct_dev(c1.data_ptr(), c2.data_ptr(), tar3.data_ptr(), n)
            rec[:, 14:17], rec[:, 17:20] = ref3, tar3
            rec[:, 2:5] = tar3 - ref3

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(args.reps):
            fn()
        e1.record(stream)
        e1.synchronize()
        return e0.elapsed_time(e1) / args.reps

    arm_a()
    arm_b()  # warm-up: module load, buffers, every kernel
    torch.cuda.synchronize()

    def same():
        return all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(outs["a"], outs["b"]))

    identical = same()
    ms_a, ms_b = [], []
    for _ in range(args.rounds):
        ms_a.append(timed(arm_a))
        ms_b.append(timed(arm_b))
    identical = identical and same()
    # per output, the record fields in which the arms differ and how many records differ there
    diff = {}
    for name, a, b in zip(("out1", "out2", "out2ds"), outs["a"], outs["b"]):
        bad = (a.view(torch.int32) != b.view(torch.int32)).sum((0, 1)).cpu().numpy()
        diff[name] = {int(k): int(bad[k]) for k in np.flatnonzero(bad)}
    o1, o2, ods = (o.cpu().numpy() for o in outs["a"])
    eng.use_own_stream()
    true = d["displaced"][-1] - d["material"]
    ok = (ods[-1][:, 6] >= 0) & (ods[-1][:, 7] >= 0)
    rec = dict(card=_card(), size=[W, H], n_poi=n, r=R, order1=1, order2=2, conv=CONV, stop=STOP, n_frames=F, reps_per_round=args.reps,
               call_ms=[round(x, 3) for x in ms_a], loop_ms=[round(x, 3) for x in ms_b], loop_over_call=[round(b / a, 4) for a, b in zip(ms_a, ms_b)],
               records_identical=bool(identical), differing_fields=diff, last_frame_ok_fraction=round(float(ok.mean()), 5),
               last_frame_max_abs_disp_error_mm=[round(float(v), 5) for v in np.abs(ods[-1][ok, 2:5] - true[ok]).max(0)])
    del rig
    eng.close()
    print(json.dumps(rec))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
