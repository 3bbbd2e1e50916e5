"""GPU parity for the section-8(f) rows N2 (NR2D1) and N4 (Strain): the CUDA path through the C ABI vs the
CPU oracle and vs the result tables the reference ships."""
import numpy as np
import pytest

import opencorr_b200 as ob
from opencorr_b200 import synth
from oracle import oracle
from oracle.oracle import Oracle2D
import util

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("r", [16, 10, 20])
def test_nr2d1_matches_oracle(engine, r):
    ref, tar = synth.speckle_pair_2d(512, 512)
    xy = synth.grid_2d(64, 64, 16, 12, 24, 31)
    q = ob.make_poi2d(xy)
    o = Oracle2D(ref, tar)
    o.fftcc2d(q, 16, 16)
    q_gpu, q_cpu = q.copy(), q.copy()
    nr = ob.NR2D1(r, r, 0.001, 10, engine=engine)
    nr.set_images(ref, tar)
    nr.prepare()
    nr.compute(q_gpu)
    o.nr2d1(q_cpu, r, r, 0.001, 10)
    util.nr_compare(q_gpu, q_cpu, "nr2d1 r=%d" % r)
    assert (q_gpu[:, 16] > 0.9).mean() > 0.9


def test_nr2d1_nonsquare_and_sentinels(engine):
    ref, tar = util.oht_cfrp_pair()
    h, w = ref.shape
    xy = np.array([[5, 5], [w - 3, 100], [100, 100], [120, 120], [140, 140], [60, 700], [200, 450]], np.float32)
    q = ob.make_poi2d(xy)
    q[3, 16] = -2.0
    q[4, 2] = np.nan
    q[4, 14] = 1.5
    q[5, 8] = -4.0
    q[6, 8] = -5.0
    a, b = q.copy(), q.copy()
    nr = ob.NR2D1(14, 11, 0.001, 10, engine=engine)
    nr.set_images(ref, tar)
    nr.prepare()
    nr.compute(a)
    Oracle2D(ref, tar).nr2d1(b, 14, 11, 0.001, 10)
    assert a[0, 16] == -1 and a[1, 16] == -1 and a[3, 16] == -2 and a[4, 16] == -5 and a[4, 2] == 1.5
    assert np.array_equal(a[:, 16] < 0, b[:, 16] < 0)
    util.nr_compare(a, b, "nr2d1 sentinels")
    with pytest.raises(ob.OpenCorrB200Error):
        nr2 = ob.NR2D1(16, 16, 0.001, 10, engine=engine)
        nr2.set_images(ref, tar)
        nr2.compute(q.copy())  # prepare() not called since setImages()


def test_nr2d1_golden_table(engine):
    """FFTCC2D -> NR2D1 vs the reference's shipped examples/2d_dic/oht_cfrp_4_fftcc_nr1_r16.csv."""
    ref, tar = util.oht_cfrp_pair()
    tab = util.oht_cfrp_nr_golden()["table"]
    q = ob.make_poi2d(tab[:, 0:2])
    f = ob.FFTCC2D(16, 16, engine=engine)
    f.set_images(ref, tar)
    f.compute(q)
    nr = ob.NR2D1(16, 16, 0.001, 10, engine=engine)
    nr.set_images(ref, tar)
    nr.prepare()
    nr.compute(q)
    assert np.array_equal(q[:, 14:16], tab[:, 4:6])
    conv = tab[:, 7] < 10
    ok = conv & (q[:, 17] == tab[:, 7])
    assert ok.sum() > 0.9 * len(tab)
    good = ok & (tab[:, 6] >= 0.9)
    d = np.abs(q[:, [2, 8]] - tab[:, [2, 3]]).max(1)
    assert d[good].max() < 1e-4, d[good].max()
    assert np.abs(q[good, 16] - tab[good, 6]).max() < 1e-5


def test_nr2d1_large_image_coordinates(engine):
    """x, y ~ 3000: a float ulp is 2.4e-4 px there, so the order `centre + warped offset` matters."""
    ref, tar = synth.speckle_pair_2d(3200, 3200)
    xy = synth.grid_2d(2900, 2900, 12, 12, 20, 20)
    q = ob.make_poi2d(xy)
    o = Oracle2D(ref, tar)
    o.fftcc2d(q, 16, 16)
    a, b = q.copy(), q.copy()
    nr = ob.NR2D1(16, 16, 0.001, 10, engine=engine)
    nr.set_images(ref, tar)
    nr.prepare()
    nr.compute(a)
    o.nr2d1(b, 16, 16, 0.001, 10, exact=True)
    util.nr_compare(a, b, "nr2d1 large coords", tol=1.5e-4)


# ------------------------------------------------------------------------------------------------ Strain
def test_strain2d_golden_band(engine):
    q, gold, check = util.strain_band_queue()
    cpu = q.copy()
    s = ob.Strain(20.0, 5, engine=engine)
    s.prepare(q)
    s.compute(q)
    oracle.strain(cpu, 20.0, 5, 0.9, 1, exact=True)
    good = check & (q[:, 16] >= 0.9)
    assert np.abs(q[good, 20:23] - gold[good]).max() < 3e-7
    assert np.abs(q[:, 20:23] - cpu[:, 20:23]).max() < 1e-7          # every POI of the band, also next to its edges
    assert np.array_equal(q[:, 20:23] == 0, cpu[:, 20:23] == 0)      # the same POIs are skipped
    untouched = np.delete(np.arange(25), [20, 21, 22])
    assert np.array_equal(q[:, untouched], cpu[:, untouched])


def test_strain3d_golden_crop(engine):
    q, gold, check = util.torus_queue()
    cpu = q.copy()
    s = ob.Strain(30.0, 5, engine=engine)
    s.compute(q)
    oracle.strain(cpu, 30.0, 5, 0.9, 1, exact=True)
    good = check & (q[:, 18] >= 0.9)
    assert np.abs(q[good, 22:28] - gold[good]).max() < 2e-6
    assert np.abs(q[:, 22:28] - cpu[:, 22:28]).max() < 2e-7
    assert np.array_equal(q[:, 22:28] == 0, cpu[:, 22:28] == 0)


@pytest.mark.parametrize("approximation", [1, 2])
def test_strain2d_random_sparse_knn_fallback(engine, approximation):
    rng = np.random.default_rng(11)
    n = 3000
    xy = rng.uniform(0, 2000, (n, 2)).astype(np.float32)   # mean spacing ~36 px: radius search usually finds < 5
    q = ob.make_poi2d(xy)
    q[:, 2] = 0.01 * xy[:, 0] + 0.002 * xy[:, 1] + rng.normal(0, 0.01, n)
    q[:, 8] = -0.003 * xy[:, 0] + 0.02 * xy[:, 1] + rng.normal(0, 0.01, n)
    q[:, 16] = rng.uniform(0.85, 1.0, n)                   # a third of the POIs fall below the 0.9 threshold
    q[5, 0] = np.nan                                       # a POI with a non-finite position is ignored
    a, b = q.copy(), q.copy()
    s = ob.Strain(20.0, 5, engine=engine)
    s.set_approximation(approximation)
    a = q.copy()
    s.compute(a)
    bq = np.delete(b, 5, axis=0)
    oracle.strain(bq, 20.0, 5, 0.9, approximation, exact=True)
    aq = np.delete(a, 5, axis=0)
    assert np.array_equal(aq[:, 20:23] == 0, bq[:, 20:23] == 0)
    assert (bq[:, 20] != 0).sum() > 20
    assert np.abs(aq[:, 20:23] - bq[:, 20:23]).max() < 1e-6
    assert np.all(a[5, 20:23] == 0)


def test_strain2d_dense_radius_sweep(engine):
    xy = synth.grid_2d(10, 10, 3, 3, 120, 90)
    rng = np.random.default_rng(2)
    q = ob.make_poi2d(xy)
    q[:, 2] = 1e-3 * xy[:, 0] ** 1.5 + rng.normal(0, 0.005, len(xy))
    q[:, 8] = 0.5 * np.sin(xy[:, 1] / 40.0) + rng.normal(0, 0.005, len(xy))
    q[:, 16] = np.where(rng.uniform(size=len(xy)) < 0.1, 0.3, 0.97)
    for radius, k in ((3.0, 5), (9.0, 5), (31.5, 12), (2.0, 5)):   # 3.0: neighbours at distance exactly 3 are excluded (strict <)
        a, b = q.copy(), q.copy()
        s = ob.Strain(radius, k, engine=engine)
        s.set_zncc_threshold(0.9)
        s.compute(a)
        oracle.strain(b, radius, k, 0.9, 1, exact=True)
        assert np.array_equal(a[:, 20:23] == 0, b[:, 20:23] == 0), radius
        assert np.abs(a[:, 20:23] - b[:, 20:23]).max() < 2e-6, radius


def test_strain3d_random(engine):
    rng = np.random.default_rng(3)
    n = 6000
    xyz = rng.uniform(0, 300, (n, 3)).astype(np.float32)
    q = ob.make_poi3d(xyz)
    G = rng.normal(0, 0.01, (3, 3))
    disp = xyz @ G.T + rng.normal(0, 0.01, (n, 3))
    q[:, 3], q[:, 7], q[:, 11] = disp[:, 0], disp[:, 1], disp[:, 2]
    q[:, 18] = rng.uniform(0.8, 1.0, n)
    for radius, k, approx in ((30.0, 5, 1), (12.0, 6, 2)):
        a, b = q.copy(), q.copy()
        s = ob.Strain(radius, k, engine=engine)
        s.set_approximation(approx)
        s.compute(a)
        oracle.strain(b, radius, k, 0.9, approx, exact=True)
        assert np.array_equal(a[:, 22:28] == 0, b[:, 22:28] == 0)
        assert (b[:, 22] != 0).sum() > (1000 if radius > 20 else 50)
        assert np.abs(a[:, 22:28] - b[:, 22:28]).max() < 2e-6


def test_strain_empty_and_tiny_queues(engine):
    s = ob.Strain(20.0, 5, engine=engine)
    q = ob.make_poi2d(np.zeros((0, 2), np.float32))
    s.compute(q)
    q = ob.make_poi2d(np.array([[10, 10], [12, 10], [10, 12]], np.float32))
    q[:, 16] = 1.0
    s.compute(q)                      # 3 POIs < 5 neighbours: nothing is fitted
    assert np.all(q[:, 20:23] == 0)


# ------------------------------------------------------------------------------------------------ EpipolarSearch
def _step18_calibrations():
    """examples/test_3d_reconstruction_epipolar.cpp:46-88"""
    c1 = ob.Calibration(10664.80664, 10643.88965, 0.0, 1176.03418, 914.7337036)
    c2 = ob.Calibration(10749.53223, 10726.52441, 0.0, 1034.707886, 1062.162842, tx=250.881488962793, ty=-1.15469183120196,
                        tz=37.4849858174401, rx=0.01450813, ry=-0.39152833, rz=0.01064092)
    return c1, c2


def test_epipolar_search_golden_crop(engine):
    v1, v2, fm, tab = util.step18_epipolar_fixture()
    p = util.STEP18_EPIPOLAR
    es = ob.EpipolarSearch(*_step18_calibrations(), engine=engine)
    es.set_images(v1, v2)
    es.set_parallax((-30, -40))
    es.set_search(p["search_radius"], p["search_step"])
    es.create_icgn(p["rx"], p["ry"], p["conv"], p["stop"])
    es.prepare()
    assert np.abs(es.fundamental_matrix - fm).max() <= 1e-6 * np.abs(fm).max()
    es.fundamental_matrix = fm.copy()   # the fixture's float32 matrix, so candidate positions are identical by construction
    q = ob.make_poi2d(tab[:, 0:2])
    cpu = q.copy()
    es.compute(q)
    Oracle2D(v1, v2).epipolar_search(cpu, fm, p["parallax_x"], p["parallax_y"], p["search_radius"], p["search_step"], p["rx"], p["ry"],
                                     p["conv"], p["stop"])
    assert np.array_equal(q[:, 14:16], cpu[:, 14:16])      # the same candidate wins (its integer offset is kept in u0, v0)
    same_it = q[:, 17] == cpu[:, 17]
    assert same_it.mean() > 0.9
    assert np.abs(q[same_it][:, [2, 8]] - cpu[same_it][:, [2, 8]]).max() < 1e-4
    assert np.abs(q[same_it, 16] - cpu[same_it, 16]).max() < 1e-5
    # refine like the example does and compare with the shipped table
    icgn2 = ob.ICGN2D2(9, 9, 0.001, 10, engine=engine)
    icgn2.set_images(v1, v2)
    icgn2.prepare()
    icgn2.compute(q)
    assert np.abs(q[:, 0] + q[:, 2] - tab[:, 3]).max() < 3e-4
    assert np.abs(q[:, 1] + q[:, 8] - tab[:, 4]).max() < 3e-4
    conv = q[:, 16] != -4
    assert conv.mean() > 0.9
    assert np.abs(q[conv, 16] - tab[conv, 2]).max() < 1e-5


def test_epipolar_search_synthetic_borders_and_errors(engine):
    """A pure translation between the views; POIs near the border lose candidates to the border test, POIs whose every
    candidate fails keep the best sentinel code."""
    ref, tar = synth.speckle_pair_2d(512, 512)
    # epipolar lines y' = y (rectified pair): F = [[0,0,0],[0,0,-1],[0,1,0]]
    fm = np.array([[0, 0, 0], [0, 0, -1], [0, 1, 0]], np.float32)
    xy = np.array([[x, y] for y in (40, 200, 256, 470) for x in (30, 100, 256, 400, 490)], np.float32)
    q = ob.make_poi2d(xy)
    cpu = q.copy()
    args = dict(search_radius=24, search_step=3, rx=12, ry=10, conv=0.05, stop=5)
    engine.set_images_2d(ref, tar)
    engine.icgn2d_prepare()
    engine.epipolar_search2d(q, fm, [0.001, 0, 1.5], [0, 0.002, 0.5], **args)
    Oracle2D(ref, tar).epipolar_search(cpu, fm, [0.001, 0, 1.5], [0, 0.002, 0.5], args["search_radius"], args["search_step"], args["rx"],
                                       args["ry"], args["conv"], args["stop"])
    assert np.array_equal(q[:, 16] < 0, cpu[:, 16] < 0)
    neg = q[:, 16] < 0
    assert np.array_equal(q[neg, 16], cpu[neg, 16]) and np.array_equal(q[neg, 14:16], cpu[neg, 14:16])
    # two candidates equally far from the match (step 3, parallax x.5) converge to the same point and tie in ZNCC to
    # ~1e-7: which of them wins is decided by rounding, so the winner's seed (u0, v0) may differ while its result does not
    same_seed = np.all(q[:, 14:16] == cpu[:, 14:16], axis=1)
    assert same_seed.mean() > 0.7
    ok = ~neg & same_seed & (q[:, 17] == cpu[:, 17])
    assert ok.sum() >= 8
    assert np.abs(q[ok][:, [2, 8]] - cpu[ok][:, [2, 8]]).max() < 1e-4
    assert np.abs(q[ok, 16] - cpu[ok, 16]).max() < 1e-5
    conv = ~neg
    assert np.abs(q[conv][:, [2, 8]] - cpu[conv][:, [2, 8]]).max() < 0.05   # conv_criterion of the sweep
    assert np.abs(q[conv, 16] - cpu[conv, 16]).max() < 1e-3
    untouched = [0, 1, 20, 21, 22, 23, 24]
    assert np.array_equal(q[:, untouched], cpu[:, untouched])
    with pytest.raises(ob.OpenCorrB200Error):
        engine.epipolar_search2d(q, fm, [0, 0, 0], [0, 0, 0], search_radius=2, search_step=4, rx=12, ry=10, conv=0.05, stop=5)


def test_strain_stereo_poi2ds(engine):
    """Strain on POI2DS records (neighbours in the image plane, plane fit over the reconstructed 3D coordinates, three
    ZNCCs tested): GPU vs the double-precision oracle and vs the strains shipped in the reference's stereo table."""
    q, gold, check = util.gt4_stereo_queue()
    s = ob.Strain(20.0, 5, engine=engine)
    g = q.copy()
    s.compute(g)
    good = check & np.all(g[:, 5:8] >= 0.9, axis=1)
    d = np.abs(g[good, 20:26] - gold[good]).max(1)
    assert np.median(d) < 2e-5 and d.max() < 1e-3       # the shipped strains (see tests/test_oracle_nr_strain.py for the bound)
    q[7, 6] = 0.5      # r1t1 ZNCC below the threshold: POI skipped and not a neighbour
    q[11, 7] = 0.2     # r1t2 ZNCC likewise
    cpu = q.copy()
    s.compute(q)
    oracle.strain(cpu, 20.0, 5, 0.9, 1, exact=True)
    assert np.array_equal(q[:, 20:26] == 0, cpu[:, 20:26] == 0)
    assert np.all(q[[7, 11], 20:26] == 0)
    # normal equations in FP64 vs Householder QR in FP64 on a poorly conditioned fit (coordinates ~400 mm, spread ~3 mm)
    assert np.abs(q[:, 20:26] - cpu[:, 20:26]).max() < 1e-5
    untouched = np.delete(np.arange(28), np.arange(20, 26))
    assert np.array_equal(q[:, untouched], cpu[:, untouched])
    # Green strain
    a, b = cpu.copy(), cpu.copy()
    a[:, 20:26] = 0
    b[:, 20:26] = 0
    s.set_approximation(2)
    s.compute(a)
    oracle.strain(b, 20.0, 5, 0.9, 2, exact=True)
    assert np.abs(a[:, 20:26] - b[:, 20:26]).max() < 1e-5
