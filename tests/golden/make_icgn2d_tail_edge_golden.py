"""Records tests/golden/icgn2d_tail_edge_parent.npz: the IC-GN records of tests/tail_edge_cases.py, made by a library whose
r = 16 kernel tests every tail sample and falls back to global memory when its support leaves the tile.  Needs a GPU and the
whole-pixel fixture, whose images the cases use.

  OCB_LIB_PATH=<library without the lean tail> python tests/golden/make_icgn2d_tail_edge_golden.py [OUT.npz]

The fixture holds the FFT-CC seed (u, v) and the records after IC-GN (float32 [n, 25]).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

import opencorr_b200 as ob  # noqa: E402
import tail_edge_cases as te  # noqa: E402


def main(out):
    engine = ob.Engine(0)
    d = dict(np.load(os.path.join(HERE, "icgn2d_whole_pixel_parent.npz")))
    s, q, edge = te.run(engine, d)
    engine.close()
    uv = s[:, [2, 8]]
    assert np.array_equal(uv, np.round(uv)), "FFT-CC seed is not integral"
    z = q[:, 16]
    print("%d POIs  at the edge %d  kept %d  -3 %d  -4 %d  -5 %d" % (len(q), int(edge.sum()), int((z >= 0).sum()),
                                                                    int((z == -3).sum()), int((z == -4).sum()), int((z == -5).sum())))
    np.savez_compressed(out, seed_uv=uv.astype(np.int16), records=q)
    print("wrote %s (%d bytes)" % (out, os.path.getsize(out)))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "icgn2d_tail_edge_parent.npz"))
