"""CPU checks behind the stereo series (ocb_stereo_series): the synthetic stereo load series is consistent with its ground truth,
and the CPU oracle plus the host assembly of POI2DS records reproduces the reference's GT4 3D-DIC table.  The bounds measured
here are the ones test_gpu_stereo_series.py holds the GPU to (stereo_series_cases.py)."""
import numpy as np

import opencorr_b200 as ob
import stereo_series_cases as ssc
from oracle import stereo as so
from oracle.oracle import Oracle2D


def _oracle_icgn(ref, tar, order, q, r, stop):
    o = Oracle2D(ref, tar)
    (o.icgn2d1 if order == 1 else o.icgn2d2)(q, r, r, ssc.CONV, stop)


def _reconstructor(intrinsics, extrinsics, h, w):
    cams = [so.CalibOracle(intrinsics[k], h, w) for k in range(2)]
    proj = [ob.Calibration(**{k: float(v) for k, v in zip(ob.api.INTRINSIC_NAMES, intrinsics[i])},
                           **{k: float(v) for k, v in zip(("tx", "ty", "tz", "rx", "ry", "rz"), extrinsics[i])}).projection_vector()
            for i in range(2)]
    return lambda p1, p2: so.reconstruct(cams[0], proj[0], cams[1], proj[1], p1, p2)


def test_synthetic_series_matches_ground_truth():
    """The oracle, run frame by frame as the series runs (ICGN2D1 r1 -> t1, ICGN2D2 r1 -> t2, each frame from the previous
    one's records, frame 0 from the true t1 rounded and the recipe), recovers the true projections in both views and the true
    3D displacements."""
    d, xy = ssc.synthetic()
    r = ssc.SYN_R
    assert d["ref1"].shape == (ssc.SYN_H, ssc.SYN_W) and d["tars1"].shape == d["tars2"].shape == (ssc.SYN_F, ssc.SYN_H, ssc.SYN_W)
    assert d["ref1"].std() > 40 and d["r2"].std() > 40 and (d["tars2"] == np.round(d["tars2"])).all()
    stereo = ssc.translation_seeds(xy, d["r2_true"])
    _oracle_icgn(d["ref1"], d["r2"], 2, stereo, r, ssc.SYN_STOP)
    assert (stereo[:, 16] > 0.99).all()
    assert np.abs(ssc.points(stereo) - d["r2_true"]).max() < ssc.SYN_PX_BOUND
    seeds1 = ssc.translation_seeds(xy, d["t1_true"][0])
    q1, q2 = seeds1.copy(), ssc.recipe_seeds2(seeds1, stereo)
    out1, out2 = [], []
    for f in range(ssc.SYN_F):
        _oracle_icgn(d["ref1"], d["tars1"][f], 1, q1, r, ssc.SYN_STOP)
        _oracle_icgn(d["ref1"], d["tars2"][f], 2, q2, r, ssc.SYN_STOP)
        out1.append(q1.copy())
        out2.append(q2.copy())
        assert (q1[:, 16] > 0.99).all() and (q2[:, 16] > 0.99).all()
        assert np.abs(ssc.points(q1) - d["t1_true"][f]).max() < ssc.SYN_PX_BOUND, f
        assert np.abs(ssc.points(q2) - d["t2_true"][f]).max() < ssc.SYN_PX_BOUND, f
    rec = ssc.assemble(_reconstructor(d["intrinsics"], d["extrinsics"], ssc.SYN_H, ssc.SYN_W), stereo, seeds1, np.stack(out1), np.stack(out2))
    for f in range(ssc.SYN_F):
        true = d["displaced"][f] - d["material"]
        assert (np.abs(rec[f, :, 2:5] - true).max(0) < ssc.SYN_DISP_BOUND).all(), f
    # the field grows with the load: frame 3 moves every point by more than 2.5 mm out of plane
    assert (rec[-1, :, 4] > 2.5).all()


def test_gt4_table_reproduced():
    """The reference's GT4 example, frame 273, on the 13 x 13 central POI block: ICGN2D2 r1 -> r2 from the table's r2 rounded,
    ICGN2D1 r1 -> t1 from the table's t1 rounded, ICGN2D2 r1 -> t2 from the recipe (the t1 seed plus the stereo match's u, v),
    then the host assembly with the CPU triangulation, against the shipped table."""
    g = ssc.gt4()
    t, xy = g["table"], g["xy"]
    r, stop = ssc.GT4_R, ssc.GT4_STOP
    stereo = ssc.translation_seeds(xy, t[:, 8:10])
    _oracle_icgn(g["r1"], g["r2"], 2, stereo, r, stop)
    seeds1 = ssc.translation_seeds(xy, t[:, 10:12])
    seeds2 = ssc.recipe_seeds2(seeds1, stereo)
    # the recipe's seed is within 1.3 px of the converged t2 (GT4's frame lies 100 px from the reference)
    assert np.abs(ssc.points(seeds2) - t[:, 12:14]).max() < 1.3
    out1, out2 = seeds1.copy(), seeds2.copy()
    _oracle_icgn(g["r1"], g["t1"], 1, out1, r, stop)
    _oracle_icgn(g["r1"], g["t2"], 2, out2, r, stop)
    rec = ssc.assemble(_reconstructor(g["intrinsics"], g["extrinsics"], *g["size"]), stereo, seeds1, out1[None], out2[None])[0]
    ok = rec[:, 7] >= 0
    assert (~ok).sum() <= ssc.GT4_MAX_CAPPED and (rec[~ok, 7] == -4).all()
    assert (rec[:, 5] >= 0).all() and (rec[:, 6] >= 0).all()
    px = ssc.GT4_PX_BOUND
    assert np.abs(rec[:, 0:2] - t[:, 0:2]).max() == 0
    assert np.abs(rec[:, 8:12] - t[:, 8:12]).max() < px
    assert np.abs(rec[ok, 12:14] - t[ok, 12:14]).max() < px
    assert np.abs(rec[:, 5:7] - t[:, 5:7]).max() < ssc.GT4_ZNCC_BOUND
    assert np.abs(rec[ok, 7] - t[ok, 7]).max() < ssc.GT4_ZNCC_BOUND
    xyz = ssc.GT4_XYZ_BOUND
    assert np.abs(rec[:, 14:17] - t[:, 14:17]).max() < xyz
    assert np.abs(rec[ok, 17:20] - t[ok, 17:20]).max() < xyz
    assert np.abs(rec[ok, 2:5] - t[ok, 2:5]).max() < xyz
    assert (rec[:, 20:] == 0).all()
