"""Shared data of the stereo-series tests (test_stereo_series_host.py, test_gpu_stereo_series.py): the synthetic stereo load
series of synth.speckle_stereo_series, the GT4 crop of the reference's 3D-DIC example (tests/golden/gt4_stereo_dic_crop.npz)
pasted into full-size canvases, the frame-0 seeding recipe, the host assembly of POI2DS records, and the bounds the CPU
oracle achieves on both, which the GPU tests reuse."""
import functools
import os

import numpy as np

import opencorr_b200 as ob
import stereo_cases as sc
from opencorr_b200 import synth

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gt4_stereo_dic_crop.npz")
CONV = 0.001

# Synthetic series: 384 x 320, 4 frames, r = 16, ICGN2D1 temporal and ICGN2D2 cross as in the reference's example.  Over the
# 13 x 11 grid the float32 oracle's t1 and t2 stay within 0.016 px of the true projections and its 3D displacements within
# (0.0011, 0.0019, 0.016) mm of the true ones (x, y, z; the rig is 600 mm away, z is along the line of sight).
SYN_W, SYN_H, SYN_F, SYN_R, SYN_STOP = 384, 320, 4, 16, 10
SYN_PX_BOUND = 0.025
SYN_DISP_BOUND = np.array([0.003, 0.003, 0.025])

# GT4, one frame (frame 273 of the reference's series): with the recipe's seed, ICGN2D2 r1 -> t2 reaches the table in 167 of 169
# POIs at stop = 20 (34 stop at 10 iterations: the frame lies 100 px from the reference, far beyond a load-series step); the
# other two end at the iteration limit (-4).  On the converged POIs r2, t1, t2 agree with the table within 1.9e-4 px, the
# ZNCCs within 6e-6 and ref_coor, tar_coor, u, v, w within 1.9e-4 mm.
GT4_R, GT4_STOP = 16, 20
GT4_PX_BOUND, GT4_ZNCC_BOUND, GT4_XYZ_BOUND, GT4_MAX_CAPPED = 3e-4, 1e-5, 3e-4, 2


@functools.lru_cache(maxsize=1)
def synthetic():
    """(series dict of synth.speckle_stereo_series with ground truth, grid points [n, 2] float32)."""
    xy = synth.grid_2d(40, 40, 13, 11, 25, 22)
    return synth.speckle_stereo_series(SYN_W, SYN_H, SYN_F, points=xy), xy


def synthetic_rig(engine=None):
    """(cam1, cam2) Calibration objects of the synthetic rig (not prepared)."""
    intr, extr = synth.stereo_rig(SYN_W, SYN_H)
    return sc.camera(intr[0], extr[0], engine), sc.camera(intr[1], extr[1], engine)


def translation_seeds(xy, targets):
    """POI2D records at xy with (u, v) = round(targets) - xy."""
    q = ob.make_poi2d(xy)
    d = np.round(np.asarray(targets, np.float64)) - xy
    q[:, 2], q[:, 8] = d[:, 0], d[:, 1]
    return q


def recipe_seeds2(seeds1, stereo):
    """The frame-0 seed of view 2: seeds1 with the r1 -> r2 match's u, v added."""
    s2 = seeds1.copy()
    s2[:, 2] += stereo[:, 2]
    s2[:, 8] += stereo[:, 8]
    return s2


@functools.lru_cache(maxsize=1)
def gt4():
    """dict: r1, r2, t1, t2 (1200 x 1920 float32 canvases holding the crops), table [169, 26], xy [169, 2] float32, and the
    GT4 intrinsics / extrinsics."""
    d, s = np.load(GOLDEN), sc.load()
    x0, y0 = (int(v) for v in d["origin"])
    h, w = (int(v) for v in d["size"])
    out = dict(table=d["table"], xy=np.ascontiguousarray(d["table"][:, 0:2], np.float32), intrinsics=s["gt4_intrinsics"],
               extrinsics=s["gt4_extrinsics"], size=(h, w))
    for name, im in zip(("r1", "r2", "t1", "t2"), d["images"]):
        c = np.zeros((h, w), np.float32)
        c[y0:y0 + im.shape[0], x0:x0 + im.shape[1]] = im
        out[name] = c
    return out


def points(q):
    """Location + (u, v) of POI2D records [..., 25], float32 [..., 2], one float32 addition per axis."""
    return np.ascontiguousarray(np.stack([q[..., 0] + q[..., 2], q[..., 1] + q[..., 8]], -1), np.float32)


def assemble(reconstruct, stereo, seeds1, out1, out2):
    """POI2DS records [F, n, 28] of a stereo series, built on the host from its registrations: reconstruct(pts1, pts2) -> [n, 3]
    triangulates (and may clamp) float32 [n, 2] point arrays; it is given copies."""
    f32 = np.float32
    F, n = out1.shape[0], out1.shape[1]
    xy = np.ascontiguousarray(seeds1[:, 0:2])
    r2 = points(stereo)
    ref = reconstruct(xy.copy(), r2.copy())
    rec = np.zeros((F, n, 28), f32)
    for f in range(F):
        t1, t2 = points(out1[f]), points(out2[f])
        tar = reconstruct(t1.copy(), t2.copy())
        r = rec[f]
        r[:, 0:2] = xy
        r[:, 2:5] = (tar - ref).astype(f32)
        r[:, 5], r[:, 6], r[:, 7] = stereo[:, 16], out1[f][:, 16], out2[f][:, 16]
        r[:, 8:10], r[:, 10:12], r[:, 12:14] = r2, t1, t2
        r[:, 14:17], r[:, 17:20] = ref, tar
    return rec
