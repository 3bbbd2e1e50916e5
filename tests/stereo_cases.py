"""Shared data of the stereo-reconstruction tests: the committed fixture tests/golden/stereo_reconstruction.npz (the reference's
Step18 and GT4 stereo tables, their calibrations and image sizes), the cameras built from it, synthetic calibrations that
exercise every term of the distortion model, and a NumPy float32 restatement of Calibration::prepare
(reference src/oc_calibration.cpp:161-219)."""
import os

import numpy as np

import opencorr_b200 as ob

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "stereo_reconstruction.npz")
NAMES = ob.api.INTRINSIC_NAMES


def load():
    return np.load(GOLDEN)


def camera(intrinsics, extrinsics, engine=None):
    """api.Calibration from 13 intrinsics and 6 extrinsics (tx ty tz rx ry rz)."""
    kw = {k: float(v) for k, v in zip(NAMES, intrinsics)}
    kw.update({k: float(v) for k, v in zip(("tx", "ty", "tz", "rx", "ry", "rz"), extrinsics)})
    return ob.Calibration(engine=engine, **kw)


def rig(d, name, engine=None):
    """(cam1, cam2, (height, width)) of the Step18 ('step18') or GT4 ('gt4') example."""
    h, w = (int(v) for v in d[name + "_size"])
    cams = [camera(d[name + "_intrinsics"][i], d[name + "_extrinsics"][i], engine) for i in range(2)]
    return cams[0], cams[1], (h, w)


def step18_points(d):
    """(pts1, pts2, ref) of the Step18 fixture rows: the POI grid position (420 + 5 (r mod 313), 250 + 5 (r div 313)) and r2."""
    r = d["step18_rows"].astype(np.int64)
    pts1 = np.stack([420 + 5 * (r % 313), 250 + 5 * (r // 313)], axis=1).astype(np.float32)
    return pts1, np.ascontiguousarray(d["step18_r2"], np.float32), d["step18_ref"]


def gt4_points(d):
    """(r1, r2, t1, t2, ref, tar) of all GT4 rows."""
    t = d["gt4_table"]
    c = lambda a: np.ascontiguousarray(a, np.float32)  # noqa: E731
    return c(t[:, 0:2]), c(t[:, 2:4]), c(t[:, 4:6]), c(t[:, 6:8]), t[:, 8:11], t[:, 11:14]


# Synthetic intrinsics: (name, intrinsics, height, width, convergence, iteration)
SYNTHETIC = [
    # skew, tangential and rational terms together
    ("full_model", [2400.0, 2380.0, 3.5, 330.0, 250.0, 0.12, -0.35, 0.9, 0.05, -0.08, 0.2, 0.0021, -0.0017], 480, 640, 0.001, 40),
    # k3 r^6 overflows float32 towards the corners: an infinite deviation and the reset of :198-203
    ("isinf_reset", [120.0, 118.0, 0.0, 320.0, 240.0, 0.0, 0.0, 1.0e36, 0.0, 0.0, 0.0, 0.0, 0.0], 480, 640, 0.001, 40),
    # setUndistortion(1e-6, 2): every pixel stops at the iteration cap
    ("iteration_cap", [1800.0, 1790.0, 0.8, 300.0, 260.0, 0.3, -1.2, 6.0, 0.0, 0.0, 0.0, 0.001, 0.0005], 512, 600, 1e-6, 2),
]


def numpy_map(intrinsics, height, width, convergence=0.001, iteration=40):
    """Calibration::prepare (:161-219) restated with NumPy float32 arrays: every operation rounds once, in the reference's order."""
    f = np.float32
    fx, fy, fs, cx, cy, k1, k2, k3, k4, k5, k6, p1, p2 = (f(v) for v in intrinsics)
    conv = f(convergence)
    r, c = np.meshgrid(np.arange(height, dtype=np.float32), np.arange(width, dtype=np.float32), indexing="ij")
    with np.errstate(all="ignore"):
        y0 = (r - cy) / fy
        x0 = (c - cx - fs * y0) / fx
        ix, iy = x0.copy(), y0.copy()
        active = np.ones_like(ix, dtype=bool)
        for _ in range(int(iteration)):
            if not active.any():
                break
            xx, yy, xy = ix * ix, iy * iy, ix * iy
            r2 = xx + yy
            r4 = r2 * r2
            r6 = r2 * r4
            radial = (f(1) + k1 * r2 + k2 * r4 + k3 * r6) / (f(1) + k4 * r2 + k5 * r4 + k6 * r6)
            dy = iy * radial
            dx = ix * radial
            dy = dy + (p1 * (r2 + f(2) * yy) + f(2) * p2 * xy)
            dx = dx + (f(2) * p1 * xy + p2 * (r2 + f(2) * xx))
            sy = dy * fy + cy
            sx = dx * fx + dy * fs + cx
            dev_y = r - sy
            dev_x = c - sx
            inf = active & (np.isinf(dev_x) | np.isinf(dev_y))
            iy = np.where(inf, y0, iy)
            ix = np.where(inf, x0, ix)
            move = active & ((np.abs(dev_x) > conv) | (np.abs(dev_y) > conv))
            dev_y = dev_y / fy
            ny = iy + dev_y
            nx = ix + (dev_x - dev_y * fs) / fx
            iy = np.where(move, ny, iy)
            ix = np.where(move, nx, ix)
            active = move & ~inf
    return ix.astype(np.float32), iy.astype(np.float32)
