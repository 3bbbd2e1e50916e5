"""SIFT3D on the GPU at every physical unit, threshold, matching ratio and match split of sift3d_cases.SWEEP, against the float32
oracle (oracle/oc_sift3d.cpp) bit for bit, by test_gpu_sift3d.py's rule; and the GPU's own matches against the float64 witness
tests/sift3d_match_witness.py, on its own descriptors, for every SWEEP case and every case of sift3d_cases.CASES.  Each case first
asserts that it reaches its branch (sift3d_cases.reach), with the match split evaluated for this device's SM count."""
import numpy as np
import pytest

import sift3d_cases as sc
import sift3d_match_witness as wit
from test_gpu_sift3d import _check_image, _expected_launches, _same_bits

pytestmark = pytest.mark.gpu

LAUNCH_CHECKED = ("flat_tar", "one_tar", "ratio_0.95")


def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _witness(label, a, b, g, ratio):
    """The GPU's matched coordinates against the witness on the GPU's descriptors.  At most max(1, 1 %) of the reference rows may
    be marginal, not counting near-copy rows (the tie fixture's: their nearest targets are descriptors of keypoints one period
    apart whose windows the border clips by a few low-weight voxels, within ~1e-6 of each other); a near-copy row's pair may only
    differ from the witness's by naming another of its near-copies.  Returns (marginal rows, near-copy rows)."""
    pairs, info = wit.match(g[0]["desc"], g[1]["desc"], ratio)
    only_gpu, only_wit, marginal, bad = wit.compare(a, b, g[0]["kp"], g[1]["kp"], pairs, info)
    n1 = len(g[0]["kp"])
    counted = [r for r in marginal if not info["near_copy"][r]]
    for r in counted:
        print("%s: witness marginal row %d: d0 %.9g d1 %.9g index0 %d" % (label, r, info["d0"][r], info["d1"][r], info["index0"][r]))
    if only_gpu or only_wit:
        print("%s: pairs only on the GPU %s, only in the witness %s" % (label, only_gpu[:5], only_wit[:5]))
    assert not bad, "%s: GPU and witness pairs differ away from marginal rows: %s" % (label, bad[:5])
    assert len(counted) <= max(1, 0.01 * n1), "%s: %d marginal rows of %d" % (label, len(counted), n1)
    return len(counted), len(marginal) - len(counted)


def _first_of_ties(label, b, g):
    """Every matched target whose descriptor the GPU produced more than once is the first of its copies (the scan's strict '<'
    over ascending j), checked on the GPU's own descriptors and matches"""
    _, first, group = np.unique(g[1]["desc"].view(np.uint32), axis=0, return_index=True, return_inverse=True)
    group = group.ravel()
    at = {}
    for i, c in enumerate(np.ascontiguousarray(g[1]["kp"][:, 3:6])):
        at.setdefault(c.tobytes(), []).append(i)
    tied = 0
    for c in np.ascontiguousarray(b):
        idx = at[c.tobytes()]
        copies = [i for i in idx if (group == group[i]).sum() > 1]
        tied += bool(copies)
        assert not copies or any(first[group[i]] == i for i in idx), "%s: matched target %s is not the first of its copies" % (label, idx)
    return tied


@pytest.mark.parametrize("name", list(sc.SWEEP))
def test_sift3d_sweep_matches_oracle(engine, name):
    print(sc.reach(name, _sm_count()))
    _, unit, kw, ratio, _ = sc.SWEEP[name]
    cfg = sc.cfg(**kw)
    ref, tar = sc.sweep_volumes(name)
    engine.set_images_3d(ref, tar)
    before = engine.launch_count()
    a, b, n_octave = engine.sift3d(cfg, unit, ratio)
    launches = engine.launch_count() - before
    g = [engine.sift3d_inspect(i) for i in (0, 1)]
    p = sc.products(name)
    fr, ft = p.fr, p.ft
    assert n_octave == fr.n_octave
    exceptions = _check_image(g[0], fr, name + "/ref") + _check_image(g[1], ft, name + "/tar")
    if exceptions == 0:
        assert _same_bits(a, fr.kp[p.pairs[:, 0], 3:6]) and _same_bits(b, ft.kp[p.pairs[:, 1], 3:6]), "%s: matches differ" % name
    else:
        assert abs(len(a) - len(p.pairs)) <= exceptions
    marginal, near_copy = _witness(name, a, b, g, ratio)
    if name == "ties":
        tied = _first_of_ties(name, b, g)
        assert tied > 0
        print("%s: %d matches on a duplicated target, each the first of its copies" % (name, tied))
    if name in LAUNCH_CHECKED:
        expected = _expected_launches(fr, ft, int(cfg[0]))
        assert launches == expected, (launches, expected)
    print("%s: %d octaves, %d / %d candidates, %d / %d keypoints, %d matches, %d exceptions, %d witness marginal rows (+ %d near-copy), "
          "%d launches" % (name, n_octave, len(fr.cand), len(ft.cand), len(fr.kp), len(ft.kp), len(a), exceptions, marginal, near_copy,
                           launches))


@pytest.mark.parametrize("name", list(sc.CASES))
def test_sift3d_cases_match_witness(engine, name):
    _, unit, kw = sc.CASES[name]
    ref, tar = sc.volumes(name)
    engine.set_images_3d(ref, tar)
    a, b, _ = engine.sift3d(sc.cfg(**kw), unit)
    g = [engine.sift3d_inspect(i) for i in (0, 1)]
    marginal, near_copy = _witness(name, a, b, g, 0.85)
    print("%s: %d / %d keypoints, %d matches, %d witness marginal rows (+ %d near-copy)" % (name, len(g[0]["kp"]), len(g[1]["kp"]),
                                                                                          len(a), marginal, near_copy))
    assert len(a) > 0
