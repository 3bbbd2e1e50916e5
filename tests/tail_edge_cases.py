"""Cases of the r = 16 tail test (tests/test_gpu_icgn2d_tail_edge.py) and of the script that records their expected records
(tests/golden/make_icgn2d_tail_edge_golden.py).

A 33 x 33 subset has one column beyond the 32 lanes, the tail.  When a pass's corner test (icgn2d.cu's iter_fast) holds, the
r = 16 kernel samples that column from the staged target tile without per-sample tests.  The tail is the subset's rightmost
column, so a stretch in x puts its samples next to the tile's right edge first.  These guesses choose, POI by POI, a
fractional u and a stretch ux such that the first pass still passes the corner test while every tail sample's 4x4 support
reaches the tile's last column.  The images are those of the whole-pixel fixture (tests/golden/icgn2d_whole_pixel_parent.npz).
"""
import numpy as np

import opencorr_b200 as ob
import whole_pixel_cases as wp

R = 16
CONV = 0.001
STOP = 10
TW = (2 * R + 1 + 3 + 2 + 3 + 3) // 4 * 4  # icgn2d_tar_w(16)
XY = wp.grid(R, 9)


def tile_x(cx, size=wp.SIZE):
    """(xlo, xhi) of the target tile staged for a warped centre cx (icgn2d.cu: x of the fast-sample window)."""
    tx0 = (int(np.floor(cx)) - R - 2) // 4 * 4
    return max(1, tx0 + 1), min(size - 2, tx0 + TW - 2)


def guess(seeds, size=wp.SIZE):
    """Per POI: u + du and ux such that the tail's X lies in [xhi - 0.3, xhi - 0.2] (floor X = xhi - 1, so the support's last
    column is the tile's last) while the leftmost column stays 0.05 px inside the window.  POIs without such a du keep the
    seed and are left out of `edge`."""
    q = seeds.copy()
    edge = np.zeros(len(q), bool)
    for k in range(len(q)):
        px, u = float(q[k, 0]), float(q[k, 2])
        for du in np.arange(-3.75, 3.8, 0.125):
            cx = px + u + du
            xlo, xhi = tile_x(cx, size)
            s = (xhi - 0.25 - cx) / R  # 1 + ux
            if 1.0 <= s < 1.25 and cx - s * R >= xlo + 0.05:
                q[k, 2] = u + du
                q[k, 3] = s - 1.0
                edge[k] = True
                break
    return q, edge


def run(engine, d):
    """(FFT-CC seed, IC-GN records, edge mask) on the speckle pair."""
    engine.set_images_2d(*wp.pair(d, "speckle"))
    q = ob.make_poi2d(XY)
    engine.fftcc2d(q, R, R)
    s = q.copy()
    q, edge = guess(q)
    engine.icgn2d_prepare()
    with wp.warps_per_poi(1):
        engine.icgn2d1(q, R, R, CONV, STOP)
    return s, q, edge
