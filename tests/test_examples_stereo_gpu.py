"""Acceptance: the reference's test_3d_reconstruction_epipolar.cpp (EpipolarSearch -> ICGN2D2 -> Calibration::prepare ->
Stereovision::reconstruct), compiled UNCHANGED against the C++ shim (examples/Makefile with OPENCORR_SRC), run on the GPU.
Without an upstream checkout the program is not built and the test skips (the upstream source may not be copied here).

The program reads d:/dic_tests/3d_dic/"Step18 00,00-0005_{0,1}.tif"; the committed crop of that pair (step18_epipolar_crop.npz) is
pasted into zero 2448x2048 images, so only its 60 POIs are matched on real texture.  Every row's 3D point is checked against the
exact (float64) oracle's reconstruction of that row's own x, y and r2, and the 60 POIs' r2 against the library's own
EpipolarSearch -> ICGN2D2 path."""
import os
import subprocess

import numpy as np
import pytest

import opencorr_b200 as ob
import stereo_cases as sc
import util
from oracle import stereo as so
from test_examples_gpu import _read_table, _write_tiff_stack

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROGRAM = os.path.join(ROOT, "examples", "bin", "test_3d_reconstruction_epipolar")


@pytest.mark.skipif(not os.path.exists(PROGRAM), reason="upstream example not built (needs OPENCORR_SRC)")
def test_reference_reconstruction_example_runs_unchanged(tmp_path, engine):
    v1, v2, _, tab = util.step18_epipolar_fixture()
    data = tmp_path / "d:" / "dic_tests" / "3d_dic"
    data.mkdir(parents=True)
    _write_tiff_stack(str(data / "Step18 00,00-0005_0.tif"), v1[None])
    _write_tiff_stack(str(data / "Step18 00,00-0005_1.tif"), v2[None])
    out = subprocess.run([PROGRAM], cwd=tmp_path, stdin=subprocess.DEVNULL, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout + out.stderr
    header, table = _read_table(str(data / "Step18 00,00-0005_1_reconstruction_epipolar.csv"))
    # IO2D::saveTable2DS of the current reference source writes every POI2DS column (the shipped table predates that)
    assert header == ("x,y,u,v,w,r1r2 ZNCC,r1t1 ZNCC,r1t2 ZNCC,r2_x,r2_y,t1_x,t1_y,t2_x,t2_y,ref_x,ref_y,ref_z,tar_x,tar_y,tar_z,"
                      "exx,eyy,ezz,exy,eyz,ezx,subset_rx,subset_ry").split(",")
    rows = table[:, [header.index(c) for c in ("x", "y", "r1r2 ZNCC", "r2_x", "r2_y", "ref_x", "ref_y", "ref_z")]]
    with open(data / "Step18 00,00-0005_1_reconstruction_epipolar_time.csv") as f:
        assert f.readline().strip() == "POI number,Initialization,Epipolar constraint aided matching,reconstruction"
        assert f.readline().split(",")[0] == "97969"
    assert rows.shape == (97969, 8)
    idx = np.arange(97969)
    assert np.array_equal(rows[:, 0], 420 + 5 * (idx % 313)) and np.array_equal(rows[:, 1], 250 + 5 * (idx // 313))

    # every row: the exact oracle on that row's own x, y, r2 (rows whose ZNCC was NaN store r2 = 0 instead of the point used)
    d = sc.load()
    c1, c2, (h, w) = sc.rig(d, "step18")
    o1 = so.CalibOracle(c1.intrinsic_vector(), h, w, exact=True)
    o2 = so.CalibOracle(c2.intrinsic_vector(), h, w, exact=True)
    use = rows[:, 2] != -2
    assert use.mean() > 0.5
    p1 = np.ascontiguousarray(rows[use, 0:2], np.float32)
    p2 = np.ascontiguousarray(rows[use, 3:5], np.float32)
    ref = so.reconstruct(o1, c1.projection_vector(), o2, c2.projection_vector(), p1, p2).astype(np.float64)
    assert np.abs(ref - rows[use, 5:8]).max() <= 5e-4

    # the 60 textured POIs: r2 as the library's EpipolarSearch -> ICGN2D2 finds it
    p = util.STEP18_EPIPOLAR
    es = ob.EpipolarSearch(c1, c2, engine=engine)
    es.set_images(v1, v2)
    es.set_parallax((-30, -40))
    es.set_search(p["search_radius"], p["search_step"])
    es.create_icgn(p["rx"], p["ry"], p["conv"], p["stop"])
    es.prepare()
    q = ob.make_poi2d(tab[:, 0:2])
    es.compute(q)
    icgn2 = ob.ICGN2D2(9, 9, 0.001, 10, engine=engine)
    icgn2.set_images(v1, v2)
    icgn2.prepare()
    icgn2.compute(q)
    # within 3e-4 px (2.5 float32 ulps at ~1100 px, the tolerance of test_gpu_nr_strain.py's golden crop test): the shim
    # (double cofactor inverse) and the Python mirror (NumPy inverse) round the fundamental matrix's last bit differently
    at = ((tab[:, 1] - 250) / 5 * 313 + (tab[:, 0] - 420) / 5).astype(np.int64)
    assert np.abs(rows[at, 3] - (q[:, 0] + q[:, 2])).max() < 3e-4
    assert np.abs(rows[at, 4] - (q[:, 1] + q[:, 8])).max() < 3e-4
