"""SIFT3D oracle (oracle/oc_sift3d.cpp) checked on the CPU: its building blocks against independent computations, and its
whole pipeline against geometric transformations of a volume whose answer is known."""
import numpy as np
import scipy.ndimage as ndi

from opencorr_b200 import synth
from oracle import sift3d as s3


def test_blur_matches_scipy_mirror():
    rng = np.random.default_rng(1)
    vol = rng.random((23, 31, 40), dtype=np.float32) * 200
    for sigma, unit in ((1.23, (1, 1, 1)), (1.95, (1, 1, 1)), (0.97, (1, 1, 2))):
        radius, w = s3.blur_kernel(sigma, unit)
        ref = vol.astype(np.float64)
        for axis, a in ((2, 0), (1, 1), (0, 2)):  # x, then y, then z
            k = np.concatenate([w[a][:0:-1], w[a]]).astype(np.float64)
            ref = ndi.correlate1d(ref, k, axis=axis, mode="mirror")
        got = s3.blur(vol, sigma, unit)
        assert np.max(np.abs(got - ref) / np.maximum(np.abs(ref), 1.0)) <= 1e-6
        if unit[2] == 2:
            assert radius[0] == radius[1] == 2 * radius[2]


def test_exp_is_within_an_ulp_of_libm():
    x = np.linspace(-100, 5, 20001, dtype=np.float32)
    got = np.array([s3.lib().os3_exp(float(v)) for v in x], np.float32)
    ref = np.exp(x.astype(np.float64)).astype(np.float32)
    ulp = np.abs(got.view(np.int32).astype(np.int64) - ref.view(np.int32).astype(np.int64))
    assert ulp.max() <= 1


def test_eigen_routine_matches_eigh():
    rng = np.random.default_rng(2)
    for _ in range(500):
        a = rng.standard_normal((3, 3))
        m = (a @ a.T + 1e-3 * np.eye(3)).astype(np.float32)
        val, vec = s3.eig3(m)
        ref_val, ref_vec = np.linalg.eigh(m.astype(np.float64))
        ref_val, ref_vec = ref_val[::-1], ref_vec[:, ::-1]
        assert np.all(np.diff(val) <= 0)
        np.testing.assert_allclose(val, ref_val, rtol=1e-5, atol=1e-5 * ref_val[0])
        np.testing.assert_allclose(np.linalg.norm(vec, axis=1), 1.0, atol=1e-6)
        gap = np.min(np.abs(np.diff(ref_val))) / ref_val[0]
        if gap > 1e-3:  # well-separated eigenvalues: vectors agree up to sign
            dots = np.abs(np.sum(vec * ref_vec.T, axis=1))
            assert np.all(dots > 1 - 1e-4), dots


def test_every_direction_hits_an_icosahedron_face():
    rng = np.random.default_rng(3)
    g = rng.standard_normal((100000, 3))
    g /= np.linalg.norm(g, axis=1, keepdims=True)
    misses = 0
    for v in g.astype(np.float32):
        f, b = s3.ico_face(v)
        misses += f < 0
    assert misses == 0


def _desc(rows):
    d = np.zeros((len(rows), 768), np.float32)
    for i, r in enumerate(rows):
        d[i, :len(r)] = r
    return d


def test_match_post_pass_all_matched_returns_nothing():
    # every reference keypoint passes the ratio test -> matched_amount stays 0 (src/oc_sift.cpp:1309-1317)
    ref = _desc([[1, 0, 0], [0, 1, 0]])
    tar = _desc([[1, 0, 0], [0, 1, 0], [0, 0, 5]])
    pairs, top2, _ = s3.match(ref, tar)
    assert len(pairs) == 0
    assert list(top2[:, 1].astype(int)) == [0, 1]


def test_match_post_pass_trailing_many_to_one_run_and_ties():
    # ref 0 -> tar 2 (unique); ref 1, ref 2 -> tar 0 (a run that ends the tar-descending list); ref 3 fails the ratio test
    tar = _desc([[1, 0, 0, 0], [0, 0, 0, 9], [0, 1, 0, 0]])
    ref = _desc([[0, 1, 0, 0], [1, 0.1, 0, 0], [1, 0.3, 0, 0], [0.5, 0.5, 0, 0]])
    pairs, _, _ = s3.match(ref, tar)
    # tar-descending order: (0, 2) first, then the run on tar 0 resolved to its nearer reference keypoint 1
    assert pairs.tolist() == [[0, 2], [1, 0]]
    # an exact tie in the run: d0 == d1 fails the strict ratio test and drops the whole run
    ref_tie = _desc([[0, 1, 0, 0], [1, 0.2, 0, 0], [1, -0.2, 0, 0], [0.5, 0.5, 0, 0]])
    pairs, top2, _ = s3.match(ref_tie, tar)
    assert pairs.tolist() == [[0, 2]]
    # ties in the scan: the first index wins
    tar_dup = _desc([[1, 0], [1, 0], [0, 1]])
    _, top2, _ = s3.match(_desc([[1, 0], [0, 1]]), tar_dup)
    assert top2[0, 1] == 0 and top2[0, 0] == top2[0, 2] == 0


def _pair(shape, seed):
    ref, _ = synth.speckle_pair_3d(shape[2], shape[1], shape[0], seed=seed)
    return ref.astype(np.float32)


def test_integer_translation():
    big = _pair((88, 96, 104), 7)
    t = (8, -8, 8)  # (x, y, z), multiples of 2^(n_octave - 1) = 8 for 72^3 volumes (4 octaves)
    x0, y0, z0 = 16, 8, 8
    ref = big[z0:z0 + 72, y0:y0 + 72, x0:x0 + 72]
    tar = big[z0 - t[2]:z0 - t[2] + 72, y0 - t[1]:y0 - t[1] + 72, x0 - t[0]:x0 - t[0] + 72]  # the same voxels, moved by +t
    fr, ft, pairs, a, b = s3.sift3d(ref, tar)
    assert fr.n_octave == 4
    inner = np.all((a >= 12) & (a <= 60), axis=1)
    ok = np.all(b[inner] == a[inner] + np.array(t, np.float32), axis=1)
    frac = ok.mean()
    print("translation: %d matches, %d away from the borders, %.4f exact" % (len(pairs), inner.sum(), frac))
    assert len(pairs) >= 200
    assert frac >= 0.99


def test_rot90_about_z():
    ref = _pair((64, 72, 72), 11)
    tar = np.ascontiguousarray(np.rot90(ref, 1, axes=(1, 2)))  # (y, x) -> quarter turn in the xy plane
    fr, ft, pairs, a, b = s3.sift3d(ref, tar)
    # np.rot90 over axes (1, 2) moves the reference voxel (x, y, z) to the target voxel (y, W - 1 - x, z)
    W = ref.shape[2]
    kr = {tuple(p) for p in fr.kp[:, 3:6].tolist()}
    mapped = {(y, W - 1 - x, z) for (x, y, z) in kr}
    kt = {tuple(p) for p in ft.kp[:, 3:6].tolist()}
    common = len(mapped & kt) / max(len(kr), 1)
    expect = np.stack([a[:, 1], W - 1 - a[:, 0], a[:, 2]], 1)
    consistent = np.all(np.abs(expect - b) <= 1, axis=1).mean() if len(a) else 0.0
    print("rot90: %d / %d keypoints map one-to-one (%.3f), %d matches, %.3f consistent" % (len(mapped & kt), len(kr), common, len(a), consistent))
    assert common >= 0.95
    assert len(a) >= 500 and consistent >= 0.99
