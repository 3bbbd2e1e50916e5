"""The reference's `any interpolated sample < 0 -> ZNCC = -3` rule (src/oc_icgn.cpp:251-255, :792-796, :1378-1390) on images
with truly black regions: the CUDA path and the oracle must return the SAME code for EVERY POI.

B-spline overshoot next to black pixels produces samples a hair below (or above) zero, so the rule is sensitive to the
evaluation order of the interpolant; the kernels re-make borderline decisions in the reference's own arithmetic
(icgn2d_exact_negative / icgn3d_exact_negative).  Patterns: a shifted and rescaled speckle (non-integral grey levels), SURVEY.md's
zero-background speckle, hard thresholding, a bright pattern with black discs (a specimen with holes)."""
import numpy as np
import pytest

import opencorr_b200 as ob
from opencorr_b200 import synth
from oracle.oracle import Oracle2D, Oracle3D

pytestmark = pytest.mark.gpu


def _discs(shape, n, rmin, rmax, seed):
    rng = np.random.default_rng(seed)
    grids = np.meshgrid(*[np.arange(s, dtype=np.float32) for s in shape], indexing="ij")
    mask = np.zeros(shape, bool)
    for _ in range(n):
        c = [rng.uniform(0, s) for s in shape]
        r = rng.uniform(rmin, rmax)
        mask |= sum((g - ci) ** 2 for g, ci in zip(grids, c)) < r * r
    return mask


def patterns_2d():
    ref, tar = synth.speckle_pair_2d(512, 512)
    yield "shift24x1.1", np.clip(ref - 24.0, 0, 255).astype(np.float32) * 1.1, np.clip(tar - 24.0, 0, 255).astype(np.float32) * 1.1
    r1, t1 = synth.speckle_pair_2d(512, 512, background=0.0, rho=3.5, seed=7)
    yield "background0_rho3.5", r1, t1
    yield "threshold60", np.where(ref < 60, 0, ref).astype(np.float32), np.where(tar < 60, 0, tar).astype(np.float32)
    holes = _discs((512, 512), 40, 4, 14, 3)
    yield "black_discs", np.where(holes, 0, ref).astype(np.float32), np.where(holes, 0, tar).astype(np.float32)


@pytest.mark.parametrize("order", [1, 2])
def test_negative_interpolated_sample_rule_2d(engine, order):
    seen_rejected = seen_kept = 0
    for name, ref, tar in patterns_2d():
        xy = synth.grid_2d(40, 40, 48, 48, 9, 9)
        q = ob.make_poi2d(xy)
        o = Oracle2D(ref, tar)
        o.fftcc2d(q, 16, 16)
        q_gpu, q_cpu = q.copy(), q.copy()
        engine.set_images_2d(ref, tar)
        engine.icgn2d_prepare()
        (engine.icgn2d1 if order == 1 else engine.icgn2d2)(q_gpu, 16, 16, 0.001, 10)
        (o.icgn2d1 if order == 1 else o.icgn2d2)(q_cpu, 16, 16, 0.001, 10)
        a, b = q_gpu[:, 16], q_cpu[:, 16]
        differ = np.where((a == -3) != (b == -3))[0]
        assert len(differ) == 0, "%s order %d: -3 decided differently at POIs %s" % (name, order, differ[:10])
        # rejected records are left untouched apart from the code
        rej = b == -3
        assert np.array_equal(q_gpu[rej], q_cpu[rej])
        seen_rejected += int(rej.sum())
        seen_kept += int((~rej).sum())
    assert seen_rejected > 1000 and seen_kept > 1000  # both outcomes are exercised


def test_negative_interpolated_sample_rule_3d(engine):
    seen_rejected = seen_kept = 0
    base_ref, base_tar = synth.speckle_pair_3d(96, 88, 80)
    voids = _discs((80, 88, 96), 25, 3, 7, 5)
    cases = [("background0",) + tuple(synth.speckle_pair_3d(96, 88, 80, background=0.0)),
             ("threshold50", np.where(base_ref < 50, 0, base_ref).astype(np.float32), np.where(base_tar < 50, 0, base_tar).astype(np.float32)),
             ("black_voids", np.where(voids, 0, base_ref).astype(np.float32), np.where(voids, 0, base_tar).astype(np.float32))]
    for name, ref, tar in cases:
        xyz = synth.grid_3d(24, 24, 24, 8, 7, 6, 6, 6, 6)
        q = ob.make_poi3d(xyz)
        o = Oracle3D(ref, tar)
        o.fftcc3d(q, 8, 8, 8)
        q_gpu, q_cpu = q.copy(), q.copy()
        engine.set_images_3d(ref, tar)
        engine.icgn3d_prepare()
        engine.icgn3d1(q_gpu, 8, 8, 8, 0.001, 20)
        o.icgn3d1(q_cpu, 8, 8, 8, 0.001, 20)
        a, b = q_gpu[:, 18], q_cpu[:, 18]
        differ = np.where((a == -3) != (b == -3))[0]
        assert len(differ) == 0, "%s: -3 decided differently at POIs %s" % (name, differ[:10])
        rej = b == -3
        assert np.array_equal(q_gpu[rej], q_cpu[rej])
        seen_rejected += int(rej.sum())
        seen_kept += int((~rej).sum())
    assert seen_rejected > 300 and seen_kept > 50


def test_negative_interpolated_sample_rule_long_queue(engine):
    """The same rule on a queue long enough (4 900 POIs) to fill every SM with one-warp-per-POI CTAs of the ICGN2D1 kernel."""
    ref, tar = synth.speckle_pair_2d(704, 704)
    holes = _discs((704, 704), 60, 4, 14, 3)
    ref, tar = np.where(holes, 0, ref).astype(np.float32), np.where(holes, 0, tar).astype(np.float32)
    xy = synth.grid_2d(40, 40, 70, 70, 9, 9)
    q = ob.make_poi2d(xy)
    o = Oracle2D(ref, tar)
    o.fftcc2d(q, 16, 16)
    q_gpu, q_cpu = q.copy(), q.copy()
    engine.set_images_2d(ref, tar)
    engine.icgn2d_prepare()
    engine.icgn2d1(q_gpu, 16, 16, 0.001, 10)
    o.icgn2d1(q_cpu, 16, 16, 0.001, 10)
    a, b = q_gpu[:, 16], q_cpu[:, 16]
    assert (b == -3).sum() > 500 and (b >= 0).sum() > 2000
    differ = np.where((a == -3) != (b == -3))[0]
    assert len(differ) == 0, "-3 decided differently at POIs %s" % differ[:10]
    assert np.array_equal(q_gpu[b == -3], q_cpu[b == -3])
    ok = (a >= 0) & (b >= 0) & (q_gpu[:, 17] == q_cpu[:, 17])
    assert np.abs(q_gpu[ok][:, [2, 8]] - q_cpu[ok][:, [2, 8]]).max() < 1e-4 and np.abs(a[ok] - b[ok]).max() < 1e-5
