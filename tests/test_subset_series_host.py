"""The float64 oracle's IC-LM and NR2D1 loops over the synthetic series of the IC-LM / NR2D1 series tests reach the ground truth
within the bounds those tests hold the GPU to: a check of the test data and the bounds that needs no GPU."""
import numpy as np
import pytest

import opencorr_b200 as ob
from opencorr_b200 import synth
from oracle.oracle import Oracle2D
import subset_series_cases as sc

CASES = [(sc.Method("iclm", 1), {}, 0.05), (sc.Method("iclm", 2), dict(second_order=True), 0.05), (sc.Method("nr"), {}, 0.05),
         (sc.Method("nr"), dict(vy_step=0.03), 0.1)]


@pytest.mark.parametrize("method,kw,bound", CASES, ids=["iclm1", "iclm2", "nr", "nr_stretch"])
def test_oracle_loop_reaches_ground_truth(method, kw, bound):
    ref, tars = sc.render_series(384, 320, 5, **kw)
    r = 20 if method.order == 2 else 16
    xy = synth.grid_2d(40, 40, 12, 10, 27, 24)
    q = ob.make_poi2d(xy)
    Oracle2D(ref, tars[0]).fftcc2d(q, 16, 16)
    for f in range(len(tars)):
        method.oracle(Oracle2D(ref, tars[f]), q, r)
        ok = q[:, 16] >= 0
        assert ok.mean() > 0.95, "frame %d" % f
        u, v = sc.true_displacement(xy, ref.shape, len(tars), f, **kw)
        assert np.abs(q[ok, 2] - u[ok]).max() < bound and np.abs(q[ok, 8] - v[ok]).max() < bound, "frame %d" % f
