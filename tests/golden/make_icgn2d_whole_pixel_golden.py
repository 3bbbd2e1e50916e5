"""Records tests/golden/icgn2d_whole_pixel_parent.npz: the IC-GN records of every case in tests/whole_pixel_cases.py, made by
a library whose sampling loops evaluate the bicubic interpolant at every sample (no whole-pixel shortcut), and the inputs they
came from.  Needs a GPU.

  OCB_LIB_PATH=<library without the shortcut> python tests/golden/make_icgn2d_whole_pixel_golden.py [OUT.npz]

The fixture holds the 8-bit images (whole_pixel_cases.make_images), the float target's non-finite pixels (row, column,
value), and per case the FFT-CC seed (u, v) and the records after IC-GN (float32 [n, 25]).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

import opencorr_b200 as ob  # noqa: E402
import whole_pixel_cases as wp  # noqa: E402


def main(out):
    engine = ob.Engine(0)
    d = wp.make_images()
    d["float_edits"] = wp.place_edits(wp.seed(engine, d, "float_sparse_r16"), wp.CASES["float_sparse_r16"][4])
    rec = {}
    for name in wp.CASES:
        s, q = wp.run(engine, d, name)
        uv = s[:, [2, 8]]
        assert np.array_equal(uv, np.round(uv)), name + ": FFT-CC seed is not integral"
        rec[name + "_seed_uv"] = uv.astype(np.int16)
        rec[name] = q
        z = q[:, 16]
        print("%-18s %5d POIs  kept %5d  -3 %4d  -4 %3d  -5 %3d  iterations %s" % (
            name, len(q), int((z >= 0).sum()), int((z == -3).sum()), int((z == -4).sum()), int((z == -5).sum()),
            np.bincount(q[z >= 0, 17].astype(int), minlength=4)[:8].tolist()))
    engine.close()
    np.savez_compressed(out, **d, **rec)
    print("wrote %s (%d bytes)" % (out, os.path.getsize(out)))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "icgn2d_whole_pixel_parent.npz"))
