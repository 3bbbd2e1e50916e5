"""Cases of the rolling-window IC-GN test (tests/test_gpu_icgn2d_rolling_window.py) and of the script that records their
expected records (tests/golden/make_icgn2d_rolling_window_golden.py).

icgn2d.cu's branch-free sampling loop keeps each lane's 4x4 pixel block in registers and, when a row's block is the previous
row's moved down by one pixel row (floor X unchanged, floor Y + 1), reads only the new bottom row.  Any other step reloads
the whole block.  The FFT-CC seeds of the speckle pairs are nearly pure translations, so their passes are regular on almost
every row.  The guesses here add shear and stretch or compression: X moves by uy per row and Y by 1 + vy, so floor X changes
and floor Y rises by 0 or 2 on some rows, at a different row in each lane.  Most batches of four rows then reload.  The guesses
are kept small enough that the warped subset stays inside the staged target tile (|vx| + |1 + vy| <= 1 + 1/r, and the same
in x).  Larger ones, such as 1 + vy = 1.3, send the whole pass to the general loop, which reads each sample on its own.

The 6-parameter cases cover the compiled-in radius 16 and generic ones (7: idle lanes; 19: a tail; 13 with two warps per POI:
batches with one to three remaining rows), one and two warps per POI, centre offsets and ICLM2D1 with one and two warps per
POI.  The 12-parameter kernels keep the full block load; their cases (radius 20, generic 11, each with one and two warps per
POI, ICLM2D2) guard that loop on the same guesses.
The images are those of the whole-pixel fixture (tests/golden/icgn2d_whole_pixel_parent.npz)."""
import numpy as np

import opencorr_b200 as ob
import whole_pixel_cases as wp

CONV = 0.001
STOP = 10

# (ux, uy, vx, vy, du) by POI index mod 6; du is added to the FFT-CC u (a non-integral translation)
GUESSES = np.array([
    (0.00, 0.04, 0.00, -0.04, 0.00),    # shear in x, compression in y
    (-0.04, 0.00, 0.04, 0.00, 0.00),    # compression in x, shear in y
    (0.02, -0.02, -0.02, 0.02, 0.37),   # stretch and shear both ways
    (0.00, -0.03, 0.03, -0.03, -0.21),
    (0.00, 0.00, 0.00, 0.04, 0.00),     # stretch in y only: floor Y rises by 2 every ~25 rows
    (0.00, 0.00, 0.00, 0.00, 0.00),     # the FFT-CC seed itself
], np.float32)


def guess(q):
    """Shear and stretch/compression guesses, POI by POI (index mod 6)."""
    g = GUESSES[np.arange(len(q)) % len(GUESSES)]
    q[:, 3], q[:, 4], q[:, 9], q[:, 10] = g[:, 0], g[:, 1], g[:, 2], g[:, 3]
    q[:, 2] += g[:, 4]
    return q


def offsets(q):
    """Centre offsets (index mod 3): none, integral, non-integral."""
    k = np.arange(len(q)) % 3
    off = np.zeros((len(q), 2), np.float32)
    off[k == 1] = (1.0, -2.0)
    off[k == 2] = (0.5, -0.25)
    return off


# name: (pair, operator, order, radius, warps per POI, POIs)
#   operator: "icgn" (ICGN2D1/2), "iclm" (ICLM2D1/2), "ex" (ocb_icgn2d_ex with centre offsets)
CASES = {
    "icgn1_r16": ("speckle", "icgn", 1, 16, 1, wp.grid(16, 9)),
    "icgn1_r16_wpp2": ("speckle", "icgn", 1, 16, 2, wp.grid(16, 9)),
    "icgn1_r7": ("speckle", "icgn", 1, 7, 1, wp.grid(7, 9)),
    "icgn1_r19": ("speckle", "icgn", 1, 19, 1, wp.grid(19, 9)),
    "icgn1_r13_wpp2": ("speckle", "icgn", 1, 13, 2, wp.grid(13, 9)),
    "icgn2_r20": ("speckle2", "icgn", 2, 20, 1, wp.grid(20, 9)),
    "icgn2_r20_wpp2": ("speckle2", "icgn", 2, 20, 2, wp.grid(20, 9)),
    "icgn2_r11": ("speckle2", "icgn", 2, 11, 1, wp.grid(11, 9)),
    "icgn2_r11_wpp2": ("speckle2", "icgn", 2, 11, 2, wp.grid(11, 9)),
    "iclm1_r16": ("speckle", "iclm", 1, 16, 1, wp.grid(16, 9)),
    "iclm1_r13_wpp2": ("speckle", "iclm", 1, 13, 2, wp.grid(13, 9)),
    "iclm2_r20": ("speckle2", "iclm", 2, 20, 2, wp.grid(20, 9)),
    "offsets1_r16": ("speckle", "ex", 1, 16, 1, wp.grid(16, 9)),
    "offsets2_r20": ("speckle2", "ex", 2, 20, 1, wp.grid(20, 9)),
}


def seed(engine, d, name):
    """The FFT-CC-seeded queue of a case, before its guess."""
    pair_name, _, _, r, _, xy = CASES[name]
    engine.set_images_2d(*wp.pair(d, pair_name))
    q = ob.make_poi2d(xy)
    engine.fftcc2d(q, r, r)
    return q


def run(engine, d, name):
    """(FFT-CC seed, IC-GN records) of one case.  d: the whole-pixel fixture (images)."""
    pair_name, op, order, r, wpp, _ = CASES[name]
    q = seed(engine, d, name)
    s = q.copy()
    q = guess(q)
    engine.icgn2d_prepare()
    with wp.warps_per_poi(wpp):
        if op == "icgn":
            (engine.icgn2d1 if order == 1 else engine.icgn2d2)(q, r, r, CONV, STOP)
        elif op == "iclm":
            engine.iclm2d(order, q, r, r, CONV, STOP)
        else:
            engine.icgn2d_ex(order, q, r, r, CONV, STOP, center_offsets=offsets(q))
    return s, q


def first_pass_steps(seeds, name, size=wp.SIZE):
    """Replay of the first pass's sampling positions in float64, for the POIs whose warped subset fits the staged target tile
    (icgn2d.cu's iter_fast, with a 0.1-pixel safety margin): per POI, (rows after a batch's first whose step is not regular in
    some lane, batches of four rows with such a step in some lane, batches).  Only approximate; it shows which path the first
    pass takes, not its exact samples."""
    q = guess(seeds.copy())
    r = CASES[name][3]
    off = offsets(q) if CASES[name][1] == "ex" else np.zeros((len(q), 2), np.float32)
    out = []
    for k in range(len(q)):
        px, py, u, ux, uy, v, vx, vy = (float(q[k, i]) for i in (0, 1, 2, 3, 4, 8, 9, 10))
        ox, oy = float(off[k, 0]), float(off[k, 1])
        pcx, pcy = px + ox, py + oy
        tx0 = (int(np.floor(pcx + u)) - r - 2) // 4 * 4
        ty0 = int(np.floor(pcy + v)) - r - 2
        tw, th = (2 * r + 9 + 3) // 4 * 4, 2 * r + 6
        fx, fy = r + abs(ox), r + abs(oy)
        ex, ey = abs(1 + ux) * fx + abs(uy) * fy, abs(vx) * fx + abs(1 + vy) * fy
        cx, cy = pcx + u, pcy + v
        if not (cx - ex >= max(1, tx0 + 1) + 0.1 and cx + ex < min(size - 2, tx0 + tw - 2) - 0.1
                and cy - ey >= max(1, ty0 + 1) + 0.1 and cy + ey < min(size - 2, ty0 + th - 2) - 0.1):
            continue
        xl = np.minimum(np.arange(32), 2 * r)[None, :] - r - ox
        yl = (np.arange(2 * r + 1) - r - oy)[:, None]
        xf = np.floor(pcx + (1 + ux) * xl + uy * yl + u)
        yf = np.floor(pcy + vx * xl + (1 + vy) * yl + v)
        irregular = ((xf[1:] != xf[:-1]) | (yf[1:] != yf[:-1] + 1)).any(1)  # row r + 1 against row r, any lane
        batches = [irregular[i:i + 4].any() for i in range(0, len(irregular), 4)]
        out.append((int(irregular.sum()), int(np.sum(batches)), len(batches)))
    return np.array(out, int).reshape(-1, 3)
