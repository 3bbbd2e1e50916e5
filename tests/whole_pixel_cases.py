"""Cases of the whole-pixel IC-GN pass test (tests/test_gpu_icgn2d_whole_pixel.py) and of the script that records their
expected records (tests/golden/make_icgn2d_whole_pixel_golden.py).

Pass 1 of a POI seeded by FFT-CC samples the target at whole pixels, and icgn2d.cu reads those samples straight from the
target pixels.  The records must be byte-identical to those of the full bicubic evaluation, so the fixture holds the records of
a library without the shortcut, and every case here runs FFT-CC on the 8-bit pair and then IC-GN on the seeded queue.

The cases cover both shape-function orders, the compiled-in radii (16 for ICGN2D1, 20 for ICGN2D2) and generic ones (7: fewer
than 32 columns, idle lanes; 19: a 7-column tail), one and two warps per POI (chosen with the library's OCB_ICGN2D_WPP knob,
so that the records do not depend on how many SMs the GPU has), stop = 1 (only the whole-pixel pass runs), the ICLM siblings, guesses and centre offsets that do not
sample at whole pixels, POIs whose shifted subset leaves the image, a black-background pattern (borderline min(t) re-decided in
the reference's arithmetic) and a float target with NaN and +-Inf pixels, both at sampled pixels and at pixels that only lie
in the 4x4 support of a subset's edge samples."""
import contextlib
import os

import numpy as np

import opencorr_b200 as ob
from opencorr_b200 import synth

SIZE = 192        # speckle pairs
BLACK_SIZE = 160  # black-background pair
CONV = 0.001


def make_images():
    """The 8-bit images stored in the fixture: a speckle reference with first- and second-order targets, and a
    black-background pair."""
    ref, tar = synth.speckle_pair_2d(SIZE, SIZE)
    _, tar2 = synth.speckle_pair_2d(SIZE, SIZE, second_order=True)  # same reference
    bref, btar = synth.speckle_pair_2d(BLACK_SIZE, BLACK_SIZE, background=0.0, rho=3.5, seed=7)
    return {k: v.astype(np.uint8) for k, v in (("speckle_ref", ref), ("speckle_tar", tar), ("speckle2_tar", tar2),
                                                ("black_ref", bref), ("black_tar", btar))}


def pair(d, name):
    """(ref, tar) of a pair of the fixture: "speckle", "speckle2" or "black"."""
    return d[("speckle" if name == "speckle2" else name) + "_ref"], d[name + "_tar"]


def grid(r, step, size=SIZE):
    """Every POI whose subset lies inside the image (the ICGN guard), on a square grid."""
    n = (size - 2 * r - 1) // step + 1
    return synth.grid_2d(r, r, n, n, step, step)


SPARSE = synth.grid_2d(24, 24, 4, 4, 40, 40)  # 16 POIs 40 px apart: a subset's support ring is no other subset's pixel


def place_edits(seeds, r):
    """(row, column, value) of the float target's non-finite pixels, placed with the FFT-CC seeds of the SPARSE queue:
    NaN at a sampled pixel of POI 5, +Inf two columns right of POI 10's subset and -Inf one row above POI 15's subset (both in
    the 4x4 support of the subset's edge samples only)."""
    def at(k, dy, dx):
        return float(seeds[k, 1] + seeds[k, 8] + dy), float(seeds[k, 0] + seeds[k, 2] + dx)
    return np.array([at(5, -3, 5) + (np.nan,), at(10, 2, r + 2) + (np.inf,), at(15, -r - 1, -4) + (-np.inf,)], np.float32)


def _guesses(q):
    """Guesses that are not whole-pixel translations, POI by POI (index mod 6): unchanged, ux, uy, non-integer u,
    non-integer POI coordinates, vy."""
    k = np.arange(len(q)) % 6
    q[k == 1, 3] = 0.01
    q[k == 2, 4] = -0.01
    q[k == 3, 2] += 0.25
    q[k == 4, 0:2] += 0.5
    q[k == 5, 10] = 0.01
    return q


def _offsets(q):
    """Centre offsets (index mod 4): none, integral, non-integral, and a half-pixel POI with a half-pixel offset, whose centre
    pcx = x + ox is integral although the subset's local coordinates are not."""
    k = np.arange(len(q)) % 4
    off = np.zeros((len(q), 2), np.float32)
    off[k == 1] = (1.0, -2.0)
    off[k == 2] = (0.5, -0.25)
    off[k == 3] = (0.5, 0.5)
    q[k == 3, 0:2] += 0.5
    return q, off


# name: (pair, target, operator, order, radius, stop, warps per POI, POIs, guess edit)
#   target "u8": the 8-bit pair; "float": the first-order pair as float32 with the non-finite pixels of place_edits
#   operator: "icgn" (ICGN2D1/2), "iclm" (ICLM2D1/2), "ex" (ocb_icgn2d_ex with centre offsets)
CASES = {
    "icgn1_r16": ("speckle", "u8", "icgn", 1, 16, 10, 1, grid(16, 9), None),
    "icgn1_r16_stop1": ("speckle", "u8", "icgn", 1, 16, 1, 1, grid(16, 9), None),
    "icgn1_r16_wpp2": ("speckle", "u8", "icgn", 1, 16, 10, 2, grid(16, 9), None),
    "icgn1_r7": ("speckle", "u8", "icgn", 1, 7, 10, 1, grid(7, 9), None),
    "icgn1_r19": ("speckle", "u8", "icgn", 1, 19, 10, 1, grid(19, 9), None),
    "icgn2_r20": ("speckle2", "u8", "icgn", 2, 20, 10, 1, grid(20, 9), None),
    "icgn2_r20_stop1": ("speckle2", "u8", "icgn", 2, 20, 1, 1, grid(20, 9), None),
    "icgn2_r20_wpp2": ("speckle2", "u8", "icgn", 2, 20, 10, 2, grid(20, 9), None),
    "iclm1_r16": ("speckle", "u8", "iclm", 1, 16, 10, 1, grid(16, 9), None),
    "iclm2_r20": ("speckle2", "u8", "iclm", 2, 20, 10, 1, grid(20, 9), None),
    "guesses1_r16": ("speckle", "u8", "icgn", 1, 16, 10, 1, grid(16, 9), _guesses),
    "guesses2_r20": ("speckle2", "u8", "icgn", 2, 20, 10, 1, grid(20, 9), _guesses),
    "offsets1_r16": ("speckle", "u8", "ex", 1, 16, 10, 1, grid(16, 9), _offsets),
    "offsets2_r16": ("speckle2", "u8", "ex", 2, 16, 10, 2, grid(16, 9), _offsets),
    "black1_r16": ("black", "u8", "icgn", 1, 16, 10, 1, grid(16, 6, BLACK_SIZE), None),
    "black2_r20": ("black", "u8", "icgn", 2, 20, 10, 2, grid(20, 6, BLACK_SIZE), None),
    "float_sparse_r16": ("speckle", "float", "icgn", 1, 16, 10, 2, SPARSE, None),
    "float_dense_r16": ("speckle", "float", "icgn", 1, 16, 10, 1, grid(16, 9), None),
}


@contextlib.contextmanager
def warps_per_poi(wpp):
    """Run the IC-GN launches inside with `wpp` warps per POI (the library reads OCB_ICGN2D_WPP at every launch)."""
    old = os.environ.get("OCB_ICGN2D_WPP")
    os.environ["OCB_ICGN2D_WPP"] = str(wpp)
    try:
        yield
    finally:
        if old is None:
            del os.environ["OCB_ICGN2D_WPP"]
        else:
            os.environ["OCB_ICGN2D_WPP"] = old


def seed(engine, d, name):
    """The FFT-CC-seeded queue of a case (before its guess edit), on the case's 8-bit pair."""
    pair_name, r, xy = CASES[name][0], CASES[name][4], CASES[name][7]
    engine.set_images_2d(*pair(d, pair_name))
    q = ob.make_poi2d(xy)
    engine.fftcc2d(q, r, r)
    return q


def run(engine, d, name):
    """(FFT-CC seed, IC-GN records) of one case.  d: the fixture (images and edits)."""
    pair_name, target, op, order, r, stop, wpp, _, edit = CASES[name]
    q = seed(engine, d, name)
    s = q.copy()
    off = None
    if edit is _offsets:
        q, off = _offsets(q)
    elif edit is not None:
        q = edit(q)
    ref, tar = pair(d, pair_name)
    if target == "float":
        ref, tar = ref.astype(np.float32), tar.astype(np.float32)
        for y, x, v in d["float_edits"]:
            tar[int(y), int(x)] = v
    engine.set_images_2d(ref, tar)
    engine.icgn2d_prepare()
    with warps_per_poi(wpp):
        if op == "icgn":
            (engine.icgn2d1 if order == 1 else engine.icgn2d2)(q, r, r, CONV, stop)
        elif op == "iclm":
            engine.iclm2d(order, q, r, r, CONV, stop)
        else:
            engine.icgn2d_ex(order, q, r, r, CONV, stop, center_offsets=off)
    return s, q
