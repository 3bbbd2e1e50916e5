"""Shared helpers for the test-suite (not product code)."""
import os
import struct

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def read_bmp8(path):
    """8-bit palettised BMP with identity grey palette -> float32 [h, w] (== cv::imread GRAYSCALE
    for the reference's example images, SURVEY.md section 8(b))."""
    b = open(path, "rb").read()
    assert b[:2] == b"BM"
    off = struct.unpack("<I", b[10:14])[0]
    w, h = struct.unpack("<ii", b[18:26])
    bpp = struct.unpack("<H", b[28:30])[0]
    assert bpp == 8
    stride = (w + 3) // 4 * 4
    a = np.frombuffer(b, dtype=np.uint8, count=stride * abs(h), offset=off).reshape(abs(h), stride)[:, :w]
    if h > 0:
        a = a[::-1]
    return np.ascontiguousarray(a).astype(np.float32)


def oht_cfrp_pair():
    return read_bmp8(os.path.join(GOLDEN, "oht_cfrp_0.bmp")), read_bmp8(os.path.join(GOLDEN, "oht_cfrp_4.bmp"))


def oht_cfrp_golden():
    return np.load(os.path.join(GOLDEN, "oht_cfrp_4_fftcc_icgn1_r16.npz"))


def al_foam_crop():
    d = np.load(os.path.join(GOLDEN, "al_foam4_crop.npz"))
    return d["ref"].astype(np.float32), d["tar"].astype(np.float32), int(d["z_offset"]), d["cpu_table"], d["gpu_table"]


def assert_same(a, b, label):
    """a and b hold the same float32 bits (a NaN equals only the same NaN)"""
    assert a.shape == b.shape, label
    bad = a.view(np.uint32) != b.view(np.uint32)
    assert not bad.any(), "%s: %d floats differ, first at %s" % (label, bad.sum(), np.argwhere(bad)[:5].tolist())


def compare_2d(a, b, label="", tol_disp=1e-4, tol_zncc=1e-5, max_iter_mismatch_frac=0.01, order=1, flip_tol_disp=1e-3, flip_tol_zncc=1e-4):
    """a, b: POI2D arrays [n,25].  Sentinel codes and integer outputs must agree exactly on every POI;
    displacement/ZNCC tolerances (north_star: 1e-4 px, 1e-5) apply to POIs whose iteration counts
    agree; POIs whose ||dp|| sits within float noise of the convergence threshold may differ by ONE
    iteration: they are counted (bounded by max_iter_mismatch_frac, SURVEY.md section 7 'Iteration-count parity') and held
    to flip_tol_disp (the convergence criterion, 1e-3 px) / flip_tol_zncc (1e-4)."""
    assert a.shape == b.shape
    za, zb = a[:, 16], b[:, 16]
    neg_a, neg_b = za < 0, zb < 0
    it_same = a[:, 17] == b[:, 17]
    # sentinel parity: same failure code, except -4 flips that come with an iteration flip at `stop`
    code_mismatch = (neg_a | neg_b) & (za != zb) & ~(((za == -4) | (zb == -4)) & ~it_same)
    assert not code_mismatch.any(), "%s sentinel mismatch at %s: %s vs %s" % (
        label, np.where(code_mismatch)[0][:10], za[code_mismatch][:10], zb[code_mismatch][:10])
    assert np.array_equal(a[:, 14:16], b[:, 14:16]), label + " u0/v0 differ"
    ok = ~neg_a & ~neg_b & it_same
    frac = 1.0 - it_same.mean() if len(a) else 0.0
    assert frac <= max_iter_mismatch_frac, "%s iteration mismatch fraction %.4f" % (label, frac)
    cols = [2, 8]
    d = np.abs(a[ok][:, cols] - b[ok][:, cols]).max() if ok.any() else 0.0
    dz = np.abs(za[ok] - zb[ok]).max() if ok.any() else 0.0
    assert d <= tol_disp, "%s max |du,dv| = %.3g > %.3g" % (label, d, tol_disp)
    assert dz <= tol_zncc, "%s max |dZNCC| = %.3g > %.3g" % (label, dz, tol_zncc)
    _check_iteration_flips(a, b, ~neg_a & ~neg_b & ~it_same, cols, 16, 17, label, flip_tol_disp, flip_tol_zncc)
    return dict(n=len(a), n_compared=int(ok.sum()), iter_mismatch_frac=float(frac), max_disp=float(d), max_zncc=float(dz))


def _check_iteration_flips(a, b, flip, cols, zc, ic, label, tol_disp, tol_zncc):
    """POIs whose iteration counts differ (||dp|| within float noise of the convergence threshold on one side) are NOT exempt:
    the counts may differ by one only, and the extra Gauss-Newton step moves the result by less than the convergence
    criterion, so displacement and ZNCC stay within (looser) bounds."""
    if not flip.any():
        return
    it_gap = np.abs(a[flip, ic] - b[flip, ic]).max()
    assert it_gap <= 1, "%s iteration counts differ by %d" % (label, it_gap)
    d = np.abs(a[flip][:, cols] - b[flip][:, cols]).max()
    dz = np.abs(a[flip, zc] - b[flip, zc]).max()
    assert d <= tol_disp, "%s one-iteration flips: max |du,dv| = %.3g > %.3g" % (label, d, tol_disp)
    assert dz <= tol_zncc, "%s one-iteration flips: max |dZNCC| = %.3g > %.3g" % (label, dz, tol_zncc)


def nr_compare(a, b, label, tol=1e-4, tol_z=1e-5):
    """NR2D1 parity.  NR2D1 converges linearly, so POIs that stop within float noise of the threshold flip by one iteration
    more often than IC-GN; the displacement bound applies to POIs with equal iteration counts."""
    assert np.array_equal(a[:, 14:16], b[:, 14:16]), label
    za, zb = a[:, 16], b[:, 16]
    it_same = a[:, 17] == b[:, 17]
    code_mismatch = ((za < 0) | (zb < 0)) & (za != zb) & ~(((za == -4) | (zb == -4)) & ~it_same)
    assert not code_mismatch.any(), (label, np.where(code_mismatch)[0][:10], za[code_mismatch][:10], zb[code_mismatch][:10])
    assert it_same.mean() > 0.98, (label, it_same.mean())
    ok = it_same & (za >= 0) & (zb >= 0)
    d = np.abs(a[ok][:, [2, 8]] - b[ok][:, [2, 8]]).max()
    dz = np.abs(za[ok] - zb[ok]).max()
    dg = np.abs(a[ok][:, [3, 4, 9, 10]] - b[ok][:, [3, 4, 9, 10]]).max()
    assert d < tol and dz < tol_z and dg < 2e-5, (label, d, dz, dg)
    return d, dz


def compare_3d(a, b, label="", tol_disp=1e-4, tol_zncc=1e-5, max_iter_mismatch_frac=0.01, flip_tol_disp=1e-3, flip_tol_zncc=1e-4):
    assert a.shape == b.shape
    za, zb = a[:, 18], b[:, 18]
    neg_a, neg_b = za < 0, zb < 0
    it_same = a[:, 19] == b[:, 19]
    code_mismatch = (neg_a | neg_b) & (za != zb) & ~(((za == -4) | (zb == -4)) & ~it_same)
    assert not code_mismatch.any(), "%s sentinel mismatch at %s" % (label, np.where(code_mismatch)[0][:10])
    assert np.array_equal(a[:, 15:18], b[:, 15:18]), label + " u0/v0/w0 differ"
    ok = ~neg_a & ~neg_b & it_same
    frac = 1.0 - it_same.mean() if len(a) else 0.0
    assert frac <= max_iter_mismatch_frac, "%s iteration mismatch fraction %.4f" % (label, frac)
    d = np.abs(a[ok][:, [3, 7, 11]] - b[ok][:, [3, 7, 11]]).max() if ok.any() else 0.0
    dz = np.abs(za[ok] - zb[ok]).max() if ok.any() else 0.0
    assert d <= tol_disp, "%s max |du,dv,dw| = %.3g > %.3g" % (label, d, tol_disp)
    assert dz <= tol_zncc, "%s max |dZNCC| = %.3g > %.3g" % (label, dz, tol_zncc)
    _check_iteration_flips(a, b, ~neg_a & ~neg_b & ~it_same, [3, 7, 11], 18, 19, label, flip_tol_disp, flip_tol_zncc)
    return dict(n=len(a), n_compared=int(ok.sum()), iter_mismatch_frac=float(frac), max_disp=float(d), max_zncc=float(dz))


def oht_cfrp_iclm_golden():
    return np.load(os.path.join(GOLDEN, "oht_cfrp_4_fftcc_iclm1_r16.npz"))


def oht_cfrp_nr_golden():
    return np.load(os.path.join(GOLDEN, "oht_cfrp_4_fftcc_nr1_r16.npz"))


def torus_strain_crop():
    return np.load(os.path.join(GOLDEN, "torus_strain_crop.npz"))


def strain_band_queue():
    """POI2D queue of the 96-row band of the shipped NR2D1 + Strain table, golden strains, and the mask of rows whose
    20-px neighbourhood lies inside the band."""
    g = oht_cfrp_nr_golden()
    b = g["band"]
    q = np.zeros((b.shape[0], 25), np.float32)
    q[:, 0:2] = b[:, 0:2]
    q[:, 2] = b[:, 2]
    q[:, 8] = b[:, 3]
    q[:, 16] = b[:, 4]
    return q, b[:, 5:8], g["band_check"]


def torus_queue():
    g = torus_strain_crop()
    t = g["table"]
    q = np.zeros((t.shape[0], 31), np.float32)
    q[:, 0:3] = t[:, 0:3]
    q[:, 3] = t[:, 3]
    q[:, 7] = t[:, 4]
    q[:, 11] = t[:, 5]
    q[:, 18] = t[:, 6]
    return q, t[:, 7:13], g["check"]


def step18_epipolar_fixture():
    """Stereo pair of the reference's test_3d_reconstruction_epipolar.cpp cut down to what 60 POIs touch (pasted into
    zero images of the full 2448x2048 size), the example's fundamental matrix, and the shipped rows x,y,ZNCC,r2_x,r2_y."""
    g = np.load(os.path.join(GOLDEN, "step18_epipolar_crop.npz"))
    h, w = (int(v) for v in g["shape"])
    views = []
    for k in ("view1", "view2"):
        img = np.zeros((h, w), np.float32)
        a, o = g[k], g[k + "_origin"]
        img[o[0]:o[0] + a.shape[0], o[1]:o[1] + a.shape[1]] = a
        views.append(img)
    return views[0], views[1], g["fundamental"], g["table"]


# parameters of examples/test_3d_reconstruction_epipolar.cpp:137-150
STEP18_EPIPOLAR = dict(parallax_x=[0, 0, -30], parallax_y=[0, 0, -40], search_radius=150, search_step=4, rx=20, ry=20, conv=0.05, stop=5)


def gt4_stereo_queue():
    """POI2DS queue (28 floats per record) of the cropped stereo-DIC table, its shipped strains, and the interior mask."""
    g = np.load(os.path.join(GOLDEN, "gt4_stereo_strain_crop.npz"))
    t = g["table"]
    q = np.zeros((t.shape[0], 28), np.float32)
    q[:, 0:20] = t[:, 0:20]
    return q, t[:, 20:26], g["check"]


def oht_cfrp_icgn2_golden():
    return np.load(os.path.join(GOLDEN, "oht_cfrp_4_sift_icgn2_gpu_r16.npz"))


def utn_self_adaptive_fixture():
    """(ref, tar, table): the cropped self-adaptive-subset example (pasted into zero images of the full size) and the shipped rows."""
    g = np.load(os.path.join(GOLDEN, "utn_30_self_adaptive_crop.npz"))
    h, w = (int(v) for v in g["shape"])
    imgs = []
    for k in ("ref", "tar"):
        img = np.zeros((h, w), np.float32)
        a, o = g[k], g[k + "_origin"]
        img[o[0]:o[0] + a.shape[0], o[1]:o[1] + a.shape[1]] = a
        imgs.append(img)
    return imgs[0], imgs[1], g["table"]


def utn_self_adaptive_queue(tab):
    """POI2D queue seeded like the example: u0, v0 of the table, the affine part from its strains, per-POI radii."""
    q = np.zeros((tab.shape[0], 25), np.float32)
    q[:, 0:2] = tab[:, 0:2]
    q[:, 2], q[:, 8], q[:, 3], q[:, 10] = tab[:, 4], tab[:, 5], tab[:, 10], tab[:, 11]
    q[:, 23], q[:, 24] = tab[:, 13], tab[:, 14]
    return q
