"""The SIFT3D cases of tests/test_gpu_sift3d.py (checked against the oracle on the GPU) and tests/test_sift3d_plan_host.py (their
pyramid plans, on the host): name -> (dims (x, y, z), physical unit, config fields that differ from the defaults).

SWEEP holds the cases of tests/test_gpu_sift3d_sweep.py (GPU against the oracle, and the GPU's descriptors against the float64
matching witness tests/sift3d_match_witness.py) and tests/test_sift3d_sweep_host.py (their branches, on the oracle alone):
name -> (dims, unit, config overrides, matching ratio, volumes), volumes a key of VOLUMES.  Every case reaches a path of
opencorr_b200/csrc/sift3d.cu that the CASES leave alone, and reach() proves it from the oracle's products:
  - unit_*: x or y units other than 1.  Candidates whose orientation window has y_max = ceil(cly + R * uy) (the reference's
    :870, reproduced) different from ceil(cly + R / uy), neither clamped to ny - 1, in both images.  Where uy < 1 the first bound
    drops rows of the window's sphere, so only unit_y0.5 (octave 0) makes the quirk change a result; uy > 1 adds rows outside it.
  - alpha_*, beta_*, gamma_*, gradient_*, truncate_*, sigma_*, min_dimension_*: one threshold or scale off its default on the
    48^3 speckle reference, each changing the outcome against the default run on the same volume (candidate count; keypoints
    newly rejected or kept by the eigenvalue, cosine or gradient test; >= 10 % of descriptor bins exactly at the truncation
    threshold; octave count or layer sigmas).
  - layers_1, layers_13: n_octave_layers at both ends of what the plan accepts; 13 fills the 16 Gaussian layers of OctaveView.
  - ratio_*: matching ratios 0.5, 0.95 (many-to-one runs resolved by the post pass), 1.0 and 1.2 (every reference keypoint passes,
    so nothing is returned, :1309-1317) and NaN (no keypoint passes).
  - few_ref, few_tar, flat_tar, one_tar: a speckled 24^3 block in a constant volume against a speckled one (n1 <= 64: one row
    block, one segment per tile), the reverse (n2 <= 64: one segment), a speckled reference against a constant target (n2 = 0),
    and against a 10^3 block that keeps one keypoint (n2 = 1: the scan must stop at n2, or the 63 zero-padded columns of the
    tile, at distance |a|^2 from every row, replace d1 = FLT_MAX and change the pairs).
  - ties: an exactly periodic target (period 16, mirror-symmetric, so the mirrored borders keep it periodic) against the same
    pattern with a noisy slab.  Interior target keypoints one period apart have bit-identical descriptors, so rows tie exactly:
    d0 = d1 = 0 away from the slab, d0 = d1 > 0 next to it; at ratio 1.2 the latter pass and the first tied index is kept.  The
    ties span 4-column thread groups, 64-column tiles and segments, and the last segment of the split is partial."""
import functools

import numpy as np

import opencorr_b200 as ob
from opencorr_b200 import synth

CROP = "tests/golden/al_foam4_crop.npz"

CASES = {
    "al_foam4_crop": ((100, 100, 100), (1.0, 1.0, 1.0), {}),  # CROP
    "synthetic_120": ((120, 120, 120), (1.0, 1.0, 1.0), {}),
    "odd_101x77x130": ((101, 77, 130), (1.0, 1.0, 1.0), {}),
    "anisotropic_112x104x60": ((112, 104, 60), (1.0, 1.0, 2.0), {}),
    "two_octave_layers": ((96, 90, 84), (1.0, 1.0, 1.0), {"n_octave_layers": 2}),
    "mirror_clamp_128": ((128, 128, 128), (1.0, 1.0, 1.0), {}),  # top octave 8^3: blur radius 8 >= side
}

S64, S48, U1 = (64, 64, 64), (48, 48, 48), (1.0, 1.0, 1.0)
SWEEP = {
    "unit_y1.6": (S64, (1.0, 1.6, 1.0), {}, 0.85, "speckle"),
    "unit_0.7_1_1.3": (S64, (0.7, 1.0, 1.3), {}, 0.85, "speckle"),
    "unit_x2": (S64, (2.0, 1.0, 1.0), {}, 0.85, "speckle"),
    "unit_y0.5": (S64, (1.0, 0.5, 1.0), {}, 0.85, "speckle"),
    "alpha_0.2": (S48, U1, {"alpha": 0.2}, 0.85, "speckle"),
    "alpha_0.05": (S48, U1, {"alpha": 0.05}, 0.85, "speckle"),
    "beta_0.7": (S48, U1, {"beta": 0.7}, 0.85, "speckle"),
    "gamma_0.25": (S48, U1, {"gamma": 0.25}, 0.85, "speckle"),
    "gradient_1e6": (S48, U1, {"gradient_threshold": 1e6}, 0.85, "speckle"),
    "truncate_0.015": (S48, U1, {"truncate_threshold": 0.015}, 0.85, "speckle"),
    "sigma_source_0.5": (S48, U1, {"sigma_source": 0.5}, 0.85, "speckle"),
    "sigma_base_2.0": (S48, U1, {"sigma_base": 2.0}, 0.85, "speckle"),
    "min_dimension_16": (S48, U1, {"min_dimension": 16}, 0.85, "speckle"),
    "layers_1": (S48, U1, {"n_octave_layers": 1}, 0.85, "speckle"),
    "layers_13": (S48, U1, {"n_octave_layers": 13}, 0.85, "speckle"),
    "ratio_0.5": (S48, U1, {}, 0.5, "speckle"),
    "ratio_0.95": (S48, U1, {}, 0.95, "speckle"),
    "ratio_1.0": (S48, U1, {}, 1.0, "speckle"),
    "ratio_1.2": (S48, U1, {}, 1.2, "speckle"),
    "ratio_nan": (S48, U1, {}, float("nan"), "speckle"),
    "few_ref": (S48, U1, {}, 0.85, "block_ref"),
    "few_tar": (S48, U1, {}, 0.85, "block_tar"),
    "flat_tar": (S48, U1, {}, 0.85, "flat_tar"),
    "one_tar": (S48, U1, {}, 0.85, "one_tar"),
    "ties": ((97, 97, 97), U1, {"gamma": 0.1}, 1.2, "ties"),
}
SPLIT_SM = 132  # H100 SXM: the SM count the host test evaluates the match split for


def crop():
    z = np.load(CROP)
    return z["ref"].astype(np.float32), z["tar"].astype(np.float32)


def volumes(name):
    """(ref, tar) float32 [z, y, x] of a case: the crop, or a synthetic pair whose target is displaced by synth.displacement_3d"""
    if name == "al_foam4_crop":
        return crop()
    ref, tar = synth.speckle_pair_3d(*CASES[name][0])
    return ref.astype(np.float32), tar.astype(np.float32)


def cfg(**kw):
    c = ob.SIFT3D_DEFAULT_CONFIG.copy()
    for k, v in kw.items():
        c[ob.api.SIFT3D_CONFIG_FIELDS.index(k)] = v
    return c


# ---- SWEEP volumes ---------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _speckle(dims):
    ref, tar = synth.speckle_pair_3d(*dims)
    return ref.astype(np.float32), tar.astype(np.float32)


def _block(vol, side=24):
    """vol's speckle in a centred side^3 block, the background level everywhere else"""
    out = np.full_like(vol, synth.BACKGROUND)
    s = tuple(slice((n - side) // 2, (n - side) // 2 + side) for n in vol.shape)
    out[s] = vol[s]
    return out


def periodic(n, period=16, seed=5):
    """n^3 volume, exactly periodic with `period` along every axis and even about 0: a speckle block of (period/2 + 1)^3 voxels
    reflected into one period.  With n - 1 a multiple of period / 2 the mirrored borders (s3::mirror_lower/upper) continue the
    pattern, so every Gaussian layer of octave 0 is periodic too, bit for bit."""
    h = period // 2
    assert (n - 1) % h == 0
    a, _ = synth.speckle_pair_3d(h + 17, h + 17, h + 17, seed=seed)
    a = a[8:9 + h, 8:9 + h, 8:9 + h]
    t = np.arange(n) % period
    fold = np.where(t <= h, t, period - t)
    return np.ascontiguousarray(a[np.ix_(fold, fold, fold)], dtype=np.float32)


def _ties(dims):
    tar = periodic(dims[0])
    ref = tar.copy()
    rng = np.random.default_rng(7)
    ref[:, :, :30] += (0.5 * rng.standard_normal(ref[:, :, :30].shape)).astype(np.float32)
    return ref, tar


VOLUMES = {
    "speckle": lambda d: _speckle(d),
    "block_ref": lambda d: (_block(_speckle(d)[0]), _speckle(d)[1]),
    "block_tar": lambda d: (_speckle(d)[0], _block(_speckle(d)[1])),
    "flat_tar": lambda d: (_speckle(d)[0], np.full(d[::-1], synth.BACKGROUND, np.float32)),
    "one_tar": lambda d: (_speckle(d)[0], _block(_speckle(d)[1], 10)),
    "ties": _ties,
}


def sweep_volumes(name):
    dims, _, _, _, key = SWEEP[name]
    return VOLUMES[key](dims)


# ---- the match split of sift3d_run (opencorr_b200/csrc/sift3d.cu, the three lines after "split the target rows") ----------
def split(n1, n2, sm_count):
    """(row_blocks, col_tiles, segs, tiles_per_seg) of the matching grid: 64-row blocks of reference descriptors against segs
    segments of tiles_per_seg 64-column target tiles."""
    row_blocks, col_tiles = -(-n1 // 64), -(-n2 // 64)
    segs = max(1, min(col_tiles, -(-2 * sm_count // row_blocks)))
    tiles_per_seg = max(1, -(-col_tiles // segs))
    segs = max(1, -(-col_tiles // tiles_per_seg))
    return row_blocks, col_tiles, segs, tiles_per_seg


def split_branch(n1, n2, sm_count):
    if n2 == 0:
        return "n2 = 0"
    _, col_tiles, segs, tps = split(n1, n2, sm_count)
    if segs == 1:
        return "one segment"
    if segs == col_tiles:
        return "one tile per segment"
    return "partial last segment" if col_tiles % tps else "full segments"


# ---- oracle products of a case, and the branch it reaches -------------------------------------------------------------------
class Products:
    """The oracle's features of both volumes, its top-2 and pairs at the case's ratio."""

    def __init__(self, name):
        self.name = name
        self.dims, self.unit, self.kw, self.ratio, _ = SWEEP[name]
        self.cfg = cfg(**self.kw)

    fr = functools.cached_property(lambda self: features(self.name, 0))
    ft = functools.cached_property(lambda self: features(self.name, 1))

    @functools.cached_property
    def _match(self):
        from oracle import sift3d as s3
        return s3.match(self.fr.desc, self.ft.desc, self.ratio)

    pairs = property(lambda self: self._match[0])
    top2 = property(lambda self: self._match[1])


@functools.lru_cache(maxsize=None)
def features(name, image, default=False):
    """Oracle Features of image 0 / 1 of a SWEEP case (default: with the default config), shared by the cases on one volume"""
    dims, unit, kw, _, key = SWEEP[name]
    if (key, image) in (("block_ref", 1), ("block_tar", 0), ("flat_tar", 0), ("one_tar", 0)):
        key = "speckle"  # the unchanged image of the pair
    return _features(key, dims, unit, () if default else tuple(sorted(kw.items())), image)


@functools.lru_cache(maxsize=None)
def _features(key, dims, unit, kw, image):
    from oracle import sift3d as s3
    return s3.Features(VOLUMES[key](dims)[image], cfg(**dict(kw)), unit)


@functools.lru_cache(maxsize=None)
def products(name):
    return Products(name)


def layer_scales(c, n_octave):
    """(scale, sigma) float32 [n_octave * L] of createGaussianPyramid (src/oc_sift.cpp:705-729)"""
    F = np.float32
    nol = int(c[0])
    L = nol + 3
    kappa = F(np.power(F(2), F(1) / F(nol)))
    scale, sigma = np.zeros(n_octave * L, F), np.zeros(n_octave * L, F)
    scale[0] = F(1) / kappa * F(c[7])
    with np.errstate(invalid="ignore"):
        sigma[0] = np.sqrt(scale[0] * scale[0] - F(c[6]) * F(c[6]))
    for i in range(1, n_octave * L):
        o, lio = divmod(i, L)
        if lio == 0:
            scale[i] = scale[(o - 1) * L + nol]
        else:
            scale[i] = kappa * scale[i - 1]
            sigma[i] = np.sqrt(kappa * kappa - F(1)) * scale[lio - 1]
    return scale, sigma


def y_max_quirk(f, dims, unit, c):
    """Candidates of Features f whose orientation window bounds ceil(cly + R * uy) and ceil(cly + R / uy) differ, neither
    clamped to ny - 1 (R = 3 * 1.5 * scale, uy the octave's unit, as orientation_kernel computes them)"""
    F = np.float32
    L = int(c[0]) + 3
    scale, _ = layer_scales(c, f.n_octave)
    hits = 0
    for o, n, _, y, _ in f.cand.tolist():
        uy = F(unit[1]) * F(1 << o)
        ny = dims[1] >> o
        R = F(3) * (F(1.5) * scale[o * L + n])
        a, b = int(np.ceil(F(y) + R * uy)), int(np.ceil(F(y) + R / uy))
        hits += a != b and max(a, b) <= ny - 1
    return hits


def _kept(f):
    return {tuple(c) for c, k in zip(f.cand.tolist(), f.kept) if k}


def _runs(top2, ratio):
    """index0 of the rows that pass the ratio test, and how many target keypoints more than one of them points to"""
    r2 = np.float32(ratio) * np.float32(ratio)
    ok = top2[:, 0] < r2 * top2[:, 2]
    _, cnt = np.unique(top2[ok, 1], return_counts=True)
    return int(ok.sum()), int((cnt > 1).sum())


def tie_spread(p, sm_count):
    """For the rows with d0 = d1 > 0: pairs (index0, j) of target keypoints with bit-identical descriptors, j > index0, counted by
    where the split puts them: different tiles, different segments, one tile but different 4-column thread groups, and one
    segment, different tiles, with index0's thread group after j's (the order the warp merge must undo)."""
    _, _, _, tps = split(len(p.fr.kp), len(p.ft.kp), sm_count)
    _, group = np.unique(p.ft.desc.view(np.uint32), axis=0, return_inverse=True)
    group = group.ravel()
    d0, i0, d1 = p.top2[:, 0], p.top2[:, 1].astype(np.int64), p.top2[:, 2]
    out = dict(rows=0, tiles=0, segments=0, thread_groups=0, lane_order=0)
    for r in np.nonzero((d0 == d1) & (d0 > 0))[0]:
        j = i0[r]
        others = np.nonzero(group == group[j])[0]
        assert len(others) > 1 and others[0] == j, (r, j, others[:4])  # a tie is a duplicate, and the first index is kept
        out["rows"] += 1
        for k in others[1:]:
            out["tiles"] += j // 64 != k // 64
            out["segments"] += j // 64 // tps != k // 64 // tps
            out["thread_groups"] += j // 64 == k // 64 and j // 4 != k // 4
            out["lane_order"] += j // 64 // tps == k // 64 // tps and j // 64 != k // 64 and j % 64 // 4 > k % 64 // 4
    return out


def reach(name, sm_count):
    """Assert that SWEEP case `name` reaches its branch, from the oracle's products (and the match split for sm_count SMs).
    Returns a one-line description."""
    p = products(name)
    kind = name.split("_")[0]
    if kind in ("alpha", "beta", "gamma", "gradient", "truncate", "sigma", "min"):  # the reference image tells
        n1 = len(p.fr.kp)
        split_txt = "%d reference keypoints" % n1
    else:
        n1, n2 = len(p.fr.kp), len(p.ft.kp)
        split_txt = "split %s (%d x %d keypoints, %d SMs: %s)" % (split_branch(n1, n2, sm_count), n1, n2, sm_count, split(n1, n2, sm_count))
    what = ""
    if kind == "unit":
        hits = [y_max_quirk(f, p.dims, p.unit, p.cfg) for f in (p.fr, p.ft)]
        assert min(hits) > 0, (name, hits)
        if name == "unit_y0.5":  # uy < 1 at octave 0: the quirk drops rows inside the sphere, so it changes keypoints
            assert any(o == 0 for o in p.fr.cand[:, 0]), name
        what = "y_max quirk at %s candidates" % hits
    elif kind in ("alpha", "beta", "gamma", "gradient", "truncate", "sigma", "min"):
        base = features(name, 0, default=True)
        f = p.fr
        if kind == "alpha":
            assert (len(f.cand) < len(base.cand)) == (p.cfg[3] > 0.1) and len(f.cand) != len(base.cand), (len(f.cand), len(base.cand))
            what = "%d candidates against %d at the default alpha" % (len(f.cand), len(base.cand))
        elif kind in ("beta", "gamma", "gradient"):
            # same candidates, one orientation test moved: every changed decision is that test's
            assert np.array_equal(f.cand, base.cand)
            k, kb = _kept(f), _kept(base)
            if kind == "gamma" and p.cfg[5] < 0.4:
                assert kb < k, (len(k), len(kb))
            else:
                assert k < kb, (len(k), len(kb))
            what = "%d keypoints kept against %d at the default %s" % (len(k), len(kb), kind)
        elif kind == "truncate":
            assert np.array_equal(f.kp, base.kp)
            d = f.desc
            capped = (d == d.max(axis=1, keepdims=True)) & (d > 0)  # the first pass's threshold, scaled by the second
            frac = capped.sum() / d.size
            assert frac >= 0.10, frac
            what = "%.1f %% of descriptor bins at the truncation threshold" % (100 * frac)
        else:
            s, sg = layer_scales(p.cfg, f.n_octave)
            sb, sgb = layer_scales(cfg(), base.n_octave)
            if name.startswith("min_dimension"):
                assert f.n_octave != base.n_octave, f.n_octave
            elif name.startswith("sigma_base"):
                assert len(s) == len(sb) and not np.array_equal(s, sb)
            else:
                assert np.array_equal(s, sb) and not np.array_equal(sg, sgb)
            assert not np.array_equal(f.max_abs, base.max_abs) or f.n_octave != base.n_octave
            what = "%d octaves (default %d), layer 0 sigma %.4g (default %.4g), scale 0 %.4g (default %.4g)" % (
                f.n_octave, base.n_octave, sg[0], sgb[0], s[0], sb[0])
    elif kind == "layers":
        nol = int(p.cfg[0])
        assert len(p.fr.max_abs) == p.fr.n_octave * (nol + 2)
        assert (p.fr.cand[:, 1] == nol).any() and n1 > 0 and n2 > 0  # the top DoG layer detects: g[nol + 2], thr[nol]
        what = "L = %d, candidates on DoG layers %s" % (nol + 3, sorted(set(p.fr.cand[:, 1].tolist())))
    elif kind == "ratio":
        passed, runs = _runs(p.top2, p.ratio)
        if np.isnan(p.ratio):
            assert passed == 0 and len(p.pairs) == 0
        elif p.ratio >= 1:
            assert (p.top2[:, 0] > 0).all() and passed == n1 and len(p.pairs) == 0  # every keypoint passed: nothing returned
        else:
            base_pairs = len(_runs_at(name, 0.85))
            assert 0 < len(p.pairs) and (len(p.pairs) < base_pairs) == (p.ratio < 0.85)
            if p.ratio > 0.85:
                assert runs > 0 and len(p.pairs) < passed  # many-to-one runs, resolved
        what = "%d of %d rows pass, %d many-to-one runs, %d pairs" % (passed, n1, runs, len(p.pairs))
    elif name == "few_ref":
        assert 0 < n1 <= 64 and split_branch(n1, n2, sm_count) == "one tile per segment"
    elif name == "few_tar":
        assert 0 < n2 <= 64 and split_branch(n1, n2, sm_count) == "one segment"
    elif name == "flat_tar":
        assert n1 > 0 and n2 == 0 and len(p.pairs) == 0
    elif name == "one_tar":
        # n2 = 1: the 63 other columns of the only tile are zero padding, at distance |a|^2 (~1) from every row.  match_kernel
        # must stop at n2; a padded column in the scan (the oracle's match against the target set plus one zero row, index 1 =
        # n2) would replace d1 = FLT_MAX, and rows at d0 >= |a|^2 would take the padding as index0
        from oracle import sift3d as s3
        padded = np.vstack([p.ft.desc, np.zeros((1, p.ft.desc.shape[1]), np.float32)])
        pairs_padded, top2_padded, _ = s3.match(p.fr.desc, padded, p.ratio)
        assert n2 == 1 and n2 % 64 and (p.top2[:, 2] == np.finfo(np.float32).max).all()
        into_padding = int((top2_padded[:, 1] == n2).sum())
        assert into_padding > 0 and not np.array_equal(pairs_padded, p.pairs), (into_padding, pairs_padded, p.pairs)
        what = "%d pairs; with the padding scanned %d pairs, %d rows nearest to a padded column" % (len(p.pairs), len(pairs_padded),
                                                                                                    into_padding)
    elif name == "ties":
        d0, d1 = p.top2[:, 0], p.top2[:, 2]
        zero, pos = int(((d0 == 0) & (d1 == 0)).sum()), int(((d0 == d1) & (d0 > 0)).sum())
        assert zero > 0 and pos > 0 and len(p.pairs) > 0
        t = tie_spread(p, sm_count)
        assert t["tiles"] > 0 and t["segments"] > 0 and t["thread_groups"] > 0 and t["lane_order"] > 0, t
        assert split_branch(n1, n2, sm_count) == "partial last segment"
        what = "%d rows with d0 = d1 = 0, %d with d0 = d1 > 0; tied pairs %s" % (zero, pos, t)
    else:
        raise AssertionError("no branch check for " + name)
    return "%s: %s; %s" % (name, what, split_txt)


def _runs_at(name, ratio):
    from oracle import sift3d as s3
    p = products(name)
    return s3.match(p.fr.desc, p.ft.desc, ratio)[0]
