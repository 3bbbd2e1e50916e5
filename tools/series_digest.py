"""What every series entry point computes, as digests: one line per call on fixed seeded inputs, with the SHA-256 of each output
buffer, the reseeded counts and the launches the call made (launch_count() delta).  Two builds of the library (selected with
OCB_LIB_PATH) that compute the same and do the same work print the same lines.

Calls: the image series (ICGN2D1, ICGN2D2 and NR2D1), the volume series (float and 8-bit stacks) and the stereo series, each with host
buffers and with device pointers, plain and re-seeding (2D and 3D) at three zncc_min.

    python tools/series_digest.py > a.txt; OCB_LIB_PATH=other.so python tools/series_digest.py > b.txt; diff a.txt b.txt
"""
import hashlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(ROOT))
sys.path.insert(0, ROOT)

import opencorr_b200 as ob  # noqa: E402
from opencorr_b200 import synth  # noqa: E402
from bench_series import render_series  # noqa: E402

CONV, STOP, F = 0.001, 10, 4
ZMINS = (0.9, 0.999, 1.0)  # nothing lost; some POIs lost in 2D; every POI lost in every frame


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()[:16]


def report(name, eng, before, outs, counts=None):
    fields = [name, "launches=%d" % (eng.launch_count() - before)]
    if counts is not None:
        fields.append("reseeded=" + ",".join(str(int(c)) for c in counts))
    fields += [sha(o) for o in outs]
    print(" ".join(fields), flush=True)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host_of(t):
    torch.cuda.synchronize()
    return t.cpu().numpy()


def run_2d(eng):
    ref, tars = render_series(512, 384, F, second_order=True)
    xy = synth.grid_2d(40, 40, 22, 16, 20, 19)
    seeds = ob.make_poi2d(xy)
    eng.set_images_2d(ref, tars[0])
    eng.fftcc2d(seeds, 16, 16)
    eng.set_series_2d(ref, tars)
    for order in (1, 2):
        b = eng.launch_count()
        report("icgn2d_series order=%d" % order, eng, b, [eng.icgn2d_series(order, seeds, 16, 16, CONV, STOP)])
        for zmin in ZMINS:
            b = eng.launch_count()
            out, counts = eng.icgn2d_series_reseed(order, seeds, 16, 16, CONV, STOP, 16, 16, zmin)
            report("icgn2d_series_reseed order=%d zmin=%g" % (order, zmin), eng, b, [out], counts)
    d_ref, d_tars, d_seeds = dev(ref), dev(tars), dev(seeds)
    d_out = torch.empty((F,) + seeds.shape, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    eng.set_series_2d_dev(d_ref.data_ptr(), d_tars.data_ptr(), F, ref.shape[1], ref.shape[0])
    for order in (1, 2):
        b = eng.launch_count()
        eng.icgn2d_series_dev(order, d_seeds.data_ptr(), d_out.data_ptr(), len(seeds), 16, 16, CONV, STOP)
        eng.sync()
        report("icgn2d_series_dev order=%d" % order, eng, b, [host_of(d_out)])
        for zmin in ZMINS:
            b = eng.launch_count()
            counts = eng.icgn2d_series_reseed_dev(order, d_seeds.data_ptr(), d_out.data_ptr(), len(seeds), 16, 16, CONV, STOP, 16, 16, zmin)
            report("icgn2d_series_reseed_dev order=%d zmin=%g" % (order, zmin), eng, b, [host_of(d_out)], counts)
    eng.set_series_2d(ref, tars)
    b = eng.launch_count()
    report("nr2d1_series", eng, b, [eng.nr2d1_series(seeds, 16, 16, CONV, STOP)])
    for zmin in ZMINS:
        b = eng.launch_count()
        out, counts = eng.nr2d1_series_reseed(seeds, 16, 16, CONV, STOP, 16, 16, zmin)
        report("nr2d1_series_reseed zmin=%g" % zmin, eng, b, [out], counts)


def run_3d(eng):
    ref, tars = synth.speckle_series_3d(64, 64, 64, F)
    xyz = synth.grid_3d(16, 16, 16, 5, 5, 5, 8, 8, 8)
    seeds = ob.make_poi3d(xyz)
    eng.set_images_3d(ref, tars[0])
    eng.fftcc3d(seeds, 8, 8, 8)
    for kind, (r, t) in (("f32", (ref, tars)), ("u8", (ref.astype(np.uint8), tars.astype(np.uint8)))):
        eng.set_series_3d(r, t)
        b = eng.launch_count()
        report("icgn3d_series %s" % kind, eng, b, [eng.icgn3d_series(seeds, 8, 8, 8, CONV, 20)])
        for zmin in ZMINS:
            b = eng.launch_count()
            out, counts = eng.icgn3d_series_reseed(seeds, 8, 8, 8, CONV, 20, 8, 8, 8, zmin)
            report("icgn3d_series_reseed %s zmin=%g" % (kind, zmin), eng, b, [out], counts)
    d_ref, d_tars, d_seeds = dev(ref), dev(tars), dev(seeds)
    d_out = torch.empty((F,) + seeds.shape, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    eng.set_series_3d_dev(d_ref.data_ptr(), d_tars.data_ptr(), F, 64, 64, 64)
    b = eng.launch_count()
    eng.icgn3d_series_dev(d_seeds.data_ptr(), d_out.data_ptr(), len(seeds), 8, 8, 8, CONV, 20)
    eng.sync()
    report("icgn3d_series_dev", eng, b, [host_of(d_out)])
    for zmin in ZMINS:
        b = eng.launch_count()
        counts = eng.icgn3d_series_reseed_dev(d_seeds.data_ptr(), d_out.data_ptr(), len(seeds), 8, 8, 8, CONV, 20, 8, 8, 8, zmin)
        report("icgn3d_series_reseed_dev zmin=%g" % zmin, eng, b, [host_of(d_out)], counts)


def run_stereo(eng):
    w, h = 384, 320
    xy = synth.grid_2d(40, 40, 13, 11, 25, 22)
    d = synth.speckle_stereo_series(w, h, F, points=xy)
    stereo = ob.make_poi2d(xy)
    eng.set_images_2d(d["ref1"], d["r2"])
    eng.fftcc2d(stereo, 16, 16)
    eng.icgn2d_prepare()
    eng.icgn2d2(stereo, 16, 16, CONV, STOP)
    s1 = ob.make_poi2d(xy)
    eng.set_images_2d(d["ref1"], d["tars1"][0])
    eng.fftcc2d(s1, 16, 16)
    s2 = s1.copy()
    s2[:, 2] += stereo[:, 2]
    s2[:, 8] += stereo[:, 8]
    rig = _rig_at(eng, w, h)
    eng.set_stereo_series(d["ref1"], d["tars1"], d["tars2"])
    b = eng.launch_count()
    report("stereo_series", eng, b, eng.stereo_series(rig, stereo, s1, s2, 1, 2, 16, 16, CONV, STOP))
    dr, dt1, dt2 = dev(d["ref1"]), dev(d["tars1"]), dev(d["tars2"])
    ds, d1, d2 = dev(stereo), dev(s1), dev(s2)
    n = len(xy)
    o1 = torch.empty((F, n, ob.POI2D_FLOATS), dtype=torch.float32, device="cuda")
    o2 = torch.empty_like(o1)
    o3 = torch.empty((F, n, ob.api.POI2DS_FLOATS), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    eng.set_stereo_series_dev(dr.data_ptr(), dt1.data_ptr(), dt2.data_ptr(), F, w, h)
    b = eng.launch_count()
    eng.stereo_series_dev(rig, ds.data_ptr(), d1.data_ptr(), d2.data_ptr(), o1.data_ptr(), o2.data_ptr(), o3.data_ptr(), n, 1, 2, 16, 16, CONV, STOP)
    eng.sync()
    report("stereo_series_dev", eng, b, [host_of(o1), host_of(o2), host_of(o3)])


def _rig_at(eng, w, h):
    """The cameras of synth.speckle_stereo_series, prepared on eng"""
    intr, extr = synth.stereo_rig(w, h)
    cams = []
    for i in range(2):
        kw = {k: float(v) for k, v in zip(ob.api.INTRINSIC_NAMES, intr[i])}
        kw.update({k: float(v) for k, v in zip(("tx", "ty", "tz", "rx", "ry", "rz"), extr[i])})
        cams.append(ob.Calibration(engine=eng, **kw))
        cams[-1].prepare(h, w)
    rig = ob.Stereovision(cams[0], cams[1], 0, eng)
    rig.prepare()
    return rig


def main():
    eng = ob.Engine(0)
    run_2d(eng)
    run_3d(eng)
    run_stereo(eng)
    eng.close()


if __name__ == "__main__":
    main()
