"""Records tests/golden/icgn2d_rolling_window_parent.npz: the IC-GN records of every case in tests/rolling_window_cases.py,
made by a library whose sampling loop reads the full 4x4 pixel block at every sample (no rolling window).  The cases
icgn2_r11 and iclm1_r13_wpp2 were added later and recorded by the rolling-window library, after checking that it reproduces
every array already in the fixture byte for byte.  Needs a GPU and the whole-pixel fixture, whose images the cases use.

  OCB_LIB_PATH=<library without the rolling window> python tests/golden/make_icgn2d_rolling_window_golden.py [OUT.npz]

The fixture holds, per case, the FFT-CC seed (u, v) and the records after IC-GN (float32 [n, 25]).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

import opencorr_b200 as ob  # noqa: E402
import rolling_window_cases as rw  # noqa: E402


def main(out):
    engine = ob.Engine(0)
    d = dict(np.load(os.path.join(HERE, "icgn2d_whole_pixel_parent.npz")))
    rec = {}
    for name in rw.CASES:
        s, q = rw.run(engine, d, name)
        uv = s[:, [2, 8]]
        assert np.array_equal(uv, np.round(uv)), name + ": FFT-CC seed is not integral"
        rec[name + "_seed_uv"] = uv.astype(np.int16)
        rec[name] = q
        z = q[:, 16]
        print("%-16s %5d POIs  kept %5d  -3 %4d  -4 %3d  -5 %3d  iterations %s" % (
            name, len(q), int((z >= 0).sum()), int((z == -3).sum()), int((z == -4).sum()), int((z == -5).sum()),
            np.bincount(q[z >= 0, 17].astype(int), minlength=11)[:11].tolist()))
    engine.close()
    np.savez_compressed(out, **rec)
    print("wrote %s (%d bytes)" % (out, os.path.getsize(out)))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "icgn2d_rolling_window_parent.npz"))
