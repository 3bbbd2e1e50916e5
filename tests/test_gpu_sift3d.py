"""SIFT3D on the GPU against the float32 oracle (oracle/oc_sift3d.cpp): candidates, max|DoG|, keypoints, descriptors and
matches are compared bit for bit.  A keypoint may differ only where the oracle's float64 margin of its orientation decision
is below MARGIN (none is expected: the kernels and the oracle perform the same float operations in the same order)."""
import numpy as np
import pytest

import opencorr_b200 as ob
from opencorr_b200 import _capi
from oracle import sift3d as s3
from sift3d_cases import CASES, cfg as _cfg, crop as _crop, volumes

pytestmark = pytest.mark.gpu

MARGIN = 1e-5


def _same_bits(a, b):
    return a.shape == b.shape and np.array_equal(np.ascontiguousarray(a).view(np.uint32), np.ascontiguousarray(b).view(np.uint32))


def _check_image(gpu, ora, label):
    assert np.array_equal(gpu["cand"], ora.cand), "%s: candidate lists differ" % label
    assert _same_bits(gpu["max_abs"], ora.max_abs), "%s: max|DoG| differs" % label
    if gpu["kp"].shape == ora.kp.shape and _same_bits(gpu["kp"], ora.kp):
        assert _same_bits(gpu["desc"], ora.desc), "%s: descriptors differ (max %.3g)" % (label, np.abs(gpu["desc"] - ora.desc).max())
        return 0
    # list the keypoint differences: each must be a decision the oracle calls marginal
    kept_o = {tuple(c) for c, k in zip(ora.cand.tolist(), ora.kept) if k}
    kept_g = {tuple(map(int, (r[6], r[7], r[2], r[1], r[0]))) for r in gpu["kp"]}
    diff = kept_o ^ kept_g
    idx = {tuple(c): i for i, c in enumerate(ora.cand.tolist())}
    bad = [(c, ora.margin[idx[c]]) for c in diff if ora.margin[idx[c]] >= MARGIN]
    print("%s: %d keypoint decisions differ, margins %s" % (label, len(diff), sorted(ora.margin[idx[c]] for c in diff)))
    assert not bad, "%s: keypoints differ at decisions with margin >= %g: %s" % (label, MARGIN, bad[:5])
    return len(diff)


@pytest.mark.parametrize("name", list(CASES))
def test_sift3d_matches_oracle(engine, name):
    _, unit, kw = CASES[name]
    ref, tar = volumes(name)
    cfg = _cfg(**kw)
    engine.set_images_3d(ref, tar)
    a, b, n_octave = engine.sift3d(cfg, unit)
    g = [engine.sift3d_inspect(i) for i in (0, 1)]
    fr, ft = s3.Features(ref, cfg, unit), s3.Features(tar, cfg, unit)
    assert n_octave == fr.n_octave
    exceptions = _check_image(g[0], fr, name + "/ref") + _check_image(g[1], ft, name + "/tar")
    pairs, _, rmargin = s3.match(fr.desc, ft.desc)
    print("%s: %d octaves, %d / %d candidates, %d / %d keypoints, %d matches, %d exceptions"
          % (name, n_octave, len(fr.cand), len(ft.cand), len(fr.kp), len(ft.kp), len(pairs), exceptions))
    if exceptions == 0:
        assert _same_bits(a, fr.kp[pairs[:, 0], 3:6]) and _same_bits(b, ft.kp[pairs[:, 1], 3:6]), "%s: matches differ" % name
    else:
        assert abs(len(a) - len(pairs)) <= exceptions
    assert len(a) > 0


def test_sift3d_repeatable(engine):
    ref, tar = _crop()
    engine.set_images_3d(ref, tar)
    first = engine.sift3d()
    g1 = [engine.sift3d_inspect(i) for i in (0, 1)]
    second = engine.sift3d()
    g2 = [engine.sift3d_inspect(i) for i in (0, 1)]
    assert _same_bits(first[0], second[0]) and _same_bits(first[1], second[1])
    for x, y in zip(g1, g2):
        assert np.array_equal(x["cand"], y["cand"]) and _same_bits(x["kp"], y["kp"]) and _same_bits(x["desc"], y["desc"])


def test_sift3d_constant_volume(engine):
    vol = np.full((40, 48, 56), 7.0, np.float32)
    engine.set_images_3d(vol, vol)
    a, b, _ = engine.sift3d()
    assert a.shape == (0, 3) and b.shape == (0, 3)
    assert engine.sift3d_inspect(0)["kp"].shape[0] == 0


def test_sift3d_group_matches_single_device(engine):
    ref, tar = _crop()
    engine.set_images_3d(ref, tar)
    a, b, n = engine.sift3d()
    grp = ob.Engine(list(range(_capi.load().ocb_device_count())))
    try:
        grp.set_images_3d(ref, tar)
        ga, gb, gn = grp.sift3d()
        assert gn == n and _same_bits(a, ga) and _same_bits(b, gb)
        assert _same_bits(grp.sift3d_inspect(1)["desc"], engine.sift3d_inspect(1)["desc"])
    finally:
        grp.close()


def test_sift3d_class_mirror(engine, capsys):
    ref, tar = _crop()
    op = ob.SIFT3D(engine=engine)
    op.setImages(ref, tar)
    op.prepare()
    op.compute()
    out = capsys.readouterr().out
    assert "features are extracted from the reference image." in out and "features are extracted from the target image." in out
    assert op.getSiftConfig()["n_octave"] == 4
    assert op.ref_matched_kp.dtype == np.float32 and op.ref_matched_kp.shape == op.tar_matched_kp.shape
    a, b, _ = engine.sift3d()
    assert _same_bits(op.ref_matched_kp, a) and _same_bits(op.tar_matched_kp, b)


def test_sift3d_rejects_bad_arguments(engine):
    ref, tar = _crop()
    engine.set_images_3d(ref, tar)
    with pytest.raises(_capi.OpenCorrB200Error):
        engine.sift3d(unit=(1.0, 0.0, 1.0))
    with pytest.raises(_capi.OpenCorrB200Error):
        engine.sift3d(_cfg(n_octave_layers=0))


def _expected_launches(fr, ft, n_octave_layers):
    """Launches of one call, from the oracle's products: per octave of each image the blurs (three passes each; octave > 0
    downsamples its bottom layer), the max|DoG| kernels and the extrema selection, then orientation and its selection where the
    octave has candidates, gather and descriptors where it keeps keypoints; matching where the reference image has keypoints."""
    L = n_octave_layers + 3
    n = 0
    for f in (fr, ft):
        for o in range(f.n_octave):
            n += (3 * L if o == 0 else 1 + 3 * (L - 1)) + (L - 1) + 1
            n += 2 * bool((f.cand[:, 0] == o).any()) + 2 * bool((f.kp[:, 6] == o).any())
    return n + (1 + bool(len(ft.kp)) if len(fr.kp) else 0)


def test_sift3d_launch_count(engine):
    """Two identical calls each add the same number of launches, the number the oracle's products imply."""
    ref, tar = _crop()
    engine.set_images_3d(ref, tar)
    added = []
    for _ in range(2):
        before = engine.launch_count()
        engine.sift3d()
        added.append(engine.launch_count() - before)
    expected = _expected_launches(s3.Features(ref), s3.Features(tar), 3)
    print("launches per call:", added, "expected", expected)
    assert added == [expected, expected]


def _matches(engine, n):
    a, b = np.empty((n, 3), np.float32), np.empty((n, 3), np.float32)
    engine._ck(engine._lib.ocb_sift3d_get_matches(engine._ctx, a.ctypes.data, b.ctypes.data))
    return a, b


def test_sift3d_refusal_keeps_results(engine):
    """A call refused before any device work (a blur radius above 64 voxels, n_octave_layers = 14) leaves the previous call's
    matches, image products and stage times readable, bit for bit."""
    ref, tar = _crop()
    engine.set_images_3d(ref, tar)
    a, b, _ = engine.sift3d()
    products = [engine.sift3d_inspect(i) for i in (0, 1)]
    times = engine.sift3d_stage_times()
    for kw in ({"unit": (1.0, 1.0, 8.5)}, {"config": _cfg(n_octave_layers=14)}):
        with pytest.raises(_capi.OpenCorrB200Error) as err:
            engine.sift3d(**kw)
        assert err.value.code == _capi.OCB_ERR_ARG, (kw, str(err.value))
        ga, gb = _matches(engine, len(a))
        assert _same_bits(ga, a) and _same_bits(gb, b), kw
        for i in (0, 1):
            now = engine.sift3d_inspect(i)
            assert all(_same_bits(now[k], products[i][k]) for k in products[i]), (kw, i)
        assert engine.sift3d_stage_times() == times, kw


def test_sift3d_shim_program(engine, tmp_path):
    """tests/native/sift3d_shim_test.cpp (the SIFT3D half of the reference's test_dvc_sift_icgn1.cpp) writes the same matches
    as the Python mirror."""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = tmp_path / "sift3d_shim_test"
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    lib = os.path.join(root, "opencorr_b200", "lib")
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-fopenmp", "-I" + os.path.join(root, "include", "opencorr"), "-o", str(exe),
                           os.path.join(root, "tests", "native", "sift3d_shim_test.cpp"), "-L" + lib, "-lopencorr_b200", "-Wl,-rpath," + lib])
    ref, tar = _crop()
    for name, vol in (("ref", ref), ("tar", tar)):  # int32[3] (x, y, z) header + float32 payload (src/oc_image.cpp:76-110)
        with open(tmp_path / (name + ".bin"), "wb") as f:
            f.write(np.array(vol.shape[::-1], np.int32).tobytes())
            f.write(vol.tobytes())
    out = subprocess.run([str(exe), str(tmp_path / "ref.bin"), str(tmp_path / "tar.bin")], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr
    assert "features are extracted from the reference image." in out.stdout
    rows = (tmp_path / "tar_matched_kp.csv").read_text().splitlines()
    assert rows[0] == "x_ref,y_ref,z_ref,x_tar,y_tar,z_tar"
    got = np.array([[float(v) for v in r.split(",")] for r in rows[1:]], np.float32)
    engine.set_images_3d(ref, tar)
    a, b, _ = engine.sift3d()
    assert got.shape == (len(a), 6) and np.array_equal(got[:, :3], a) and np.array_equal(got[:, 3:], b)
