"""Regenerates tests/golden/stereo_reconstruction.npz from the reference checkout (the other fixtures come from make_golden.py
and are left as they are).

Run in the build container (the GPU box has no /root/reference):  python tests/golden/make_stereo_golden.py
Only DATA is taken (the two stereo result tables the reference ships in examples/3d_dic); the calibrations are the constants
hard-coded in the example programs.

  step18_*  examples/3d_dic/"Step18 00,00-0005_1_reconstruction_epipolar.csv" (test_3d_reconstruction_epipolar.cpp:46-88,
            2448x2048): every 4th row plus every row whose r2 lies outside [0, W-2] x [0, H-2] (undistort's clamp).  The row
            index r gives x = 420 + 5 (r mod 313), y = 250 + 5 (r div 313); r2 and ref_xyz as float32.
  gt4_*     examples/3d_dic/GT4-0273_0_epipolar_sift_r16.csv (test_3d_dic_epipolar_sift.cpp:58-100, 1920x1200): all rows,
            x, y, r2, t1, t2, ref_xyz, tar_xyz as float32 (ref = reconstruct(r1, r2), tar = reconstruct(t1, t2)).
Intrinsics are the 13 floats of CameraIntrinsics (fx fy fs cx cy k1..k6 p1 p2), extrinsics tx ty tz rx ry rz; the float32
rounding of the printed columns is below 6e-8 mm.
"""
import os

import numpy as np

REF = "/root/reference/examples"
OUT = os.path.dirname(os.path.abspath(__file__))


def make_stereo_fixture():
    f32 = np.float32
    s18 = np.genfromtxt(os.path.join(REF, "3d_dic", "Step18 00,00-0005_1_reconstruction_epipolar.csv"), delimiter=",", skip_header=1)
    assert s18.shape == (313 * 313, 8)
    idx = np.arange(s18.shape[0])
    assert np.array_equal(s18[:, 0], 420 + 5 * (idx % 313)) and np.array_equal(s18[:, 1], 250 + 5 * (idx // 313))
    h18, w18 = 2048, 2448
    out = (s18[:, 3] < 0) | (s18[:, 4] < 0) | (s18[:, 3] > w18 - 2) | (s18[:, 4] > h18 - 2)
    rows = np.flatnonzero((idx % 4 == 0) | out)
    step18_intr = np.array([[10664.80664, 10643.88965, 0, 1176.03418, 914.7337036, 0.030823536, -1.350255132, 74.21749878, 0, 0, 0, 0, 0],
                            [10749.53223, 10726.52441, 0, 1034.707886, 1062.162842, 0.070953421, -4.101067066, 74.21749878, 0, 0, 0, 0, 0]], f32)
    step18_extr = np.array([[0, 0, 0, 0, 0, 0],
                            [250.881488962793, -1.15469183120196, 37.4849858174401, 0.01450813, -0.39152833, 0.01064092]], f32)
    gt = np.genfromtxt(os.path.join(REF, "3d_dic", "GT4-0273_0_epipolar_sift_r16.csv"), delimiter=",", skip_header=1)
    # x y | r2_x r2_y t1_x t1_y t2_x t2_y | ref_x ref_y ref_z tar_x tar_y tar_z
    gt4 = gt[:, [0, 1, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18, 19]].astype(f32)
    gt4_intr = np.array([[6673.315918, 6669.302734, 0, 872.15778, 579.95532, 0.032258954, -1.01141417, 29.78838921, 0, 0, 0, 0, 0],
                         [6607.618164, 6602.857422, 0, 917.9733887, 531.6352539, 0.064598486, -4.531373978, 29.78838921, 0, 0, 0, 0, 0]], f32)
    gt4_extr = np.array([[0, 0, 0, 0, 0, 0], [122.24886, 1.8488892, 17.624638, 0.00307711, -0.33278773, 0.00524556]], f32)
    np.savez_compressed(os.path.join(OUT, "stereo_reconstruction.npz"),
                        step18_size=np.array([h18, w18]), step18_intrinsics=step18_intr, step18_extrinsics=step18_extr,
                        step18_rows=rows.astype(np.int32), step18_r2=s18[rows, 3:5].astype(f32), step18_ref=s18[rows, 5:8].astype(f32),
                        gt4_size=np.array([1200, 1920]), gt4_intrinsics=gt4_intr, gt4_extrinsics=gt4_extr,
                        gt4_columns=np.array("x,y,r2_x,r2_y,t1_x,t1_y,t2_x,t2_y,ref_x,ref_y,ref_z,tar_x,tar_y,tar_z".split(",")), gt4_table=gt4)
    print("stereo_reconstruction.npz: %d Step18 rows (%d outside the image), %d GT4 rows" % (len(rows), int(out.sum()), len(gt4)))


if __name__ == "__main__":
    make_stereo_fixture()
