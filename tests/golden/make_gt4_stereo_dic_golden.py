"""Regenerates tests/golden/gt4_stereo_dic_crop.npz from the reference checkout.

Run in the build container (the GPU box has no /root/reference):  python tests/golden/make_gt4_stereo_dic_golden.py
Only DATA is taken from the reference's 3D-DIC example (examples/test_3d_dic_epipolar_sift.cpp, 1920x1200, r = 16):

  table    the 13 x 13 central POI block of examples/3d_dic/GT4-0273_0_epipolar_sift_r16.csv (169 rows, all 26 columns as
           printed: x y u v w r1r2 r1t1 r1t2 r2_x r2_y t1_x t1_y t2_x t2_y ref_x ref_y ref_z tar_x tar_y tar_z e[6]); every
           row has all three ZNCCs >= 0.98.
  images   one common crop of GT4-0000_0 (r1), GT4-0000_1 (r2), GT4-0273_0 (t1) and GT4-0273_1 (t2), uint8 [4, h, w], that holds
           every r = 16 subset of the block at r1, r2, t1 and t2 with MARGIN pixels to spare; origin = (x0, y0) of the crop.
The cameras are in stereo_reconstruction.npz (gt4_*).  Tests paste the crops into 1920 x 1200 canvases at the origin, so that
coordinates and distortion maps are the cameras' own.
"""
import os

import numpy as np

REF = "/root/reference/examples/3d_dic"
OUT = os.path.dirname(os.path.abspath(__file__))
W, H, R, MARGIN = 1920, 1200, 16, 6


def load_tif(name):  # uncompressed 8-bit single-strip TIFF, pixel data at offset 8
    b = open(os.path.join(REF, name), "rb").read()
    return np.frombuffer(b[8:8 + W * H], np.uint8).reshape(H, W)


def main():
    path = os.path.join(REF, "GT4-0273_0_epipolar_sift_r16.csv")
    columns = open(path).readline().strip().split(",")
    t = np.genfromtxt(path, delimiter=",", skip_header=1)
    xs, ys = np.unique(t[:, 0]), np.unique(t[:, 1])
    bx, by = xs[len(xs) // 2 - 6:len(xs) // 2 + 7], ys[len(ys) // 2 - 6:len(ys) // 2 + 7]
    block = t[np.isin(t[:, 0], bx) & np.isin(t[:, 1], by)]
    assert len(block) == 169 and (block[:, 5:8] >= 0.98).all()
    pts = np.concatenate([block[:, 0:2], block[:, 8:10], block[:, 10:12], block[:, 12:14]])
    x0, y0 = (np.floor(pts.min(0)) - R - MARGIN).astype(int)
    x1, y1 = (np.ceil(pts.max(0)) + R + MARGIN + 1).astype(int)
    imgs = np.stack([load_tif(n)[y0:y1, x0:x1] for n in ("GT4-0000_0.tif", "GT4-0000_1.tif", "GT4-0273_0.tif", "GT4-0273_1.tif")])
    np.savez_compressed(os.path.join(OUT, "gt4_stereo_dic_crop.npz"), table=block, columns=np.array(columns), images=imgs,
                        origin=np.array([x0, y0]), size=np.array([H, W]))
    print("gt4_stereo_dic_crop.npz: %d rows, crop %d x %d at (%d, %d)" % (len(block), x1 - x0, y1 - y0, x0, y0))


if __name__ == "__main__":
    main()
