"""Synthetic speckle pairs / volumes with known displacement fields (SURVEY.md section 8(d)).

The reference ships no generator; bench.py and the tests use this one.  Gaussian-speckle model,
8-bit quantised then cast to float for 2D (the reference only ever sees 8-bit-valued floats in
2D, src/oc_image.cpp:39,56): I(x) = clip(B + (255 - B) * sum_k a_k exp(-|x - c_k|^2 / rho^2)), the
target is rendered analytically from displaced centres c_k' = c_k + u(c_k).

The background level B = 24 is a deliberate departure from SURVEY.md's formula (B = 0): the
reference treats ANY interpolated sample < 0 as "outside the image" (src/oc_icgn.cpp:251-255), and
bicubic/tricubic overshoot next to truly black pixels produces such samples, so a pattern with a
zero background makes the reference reject every POI with ZNCC = -3.
"""
import numpy as np

REF_SEED = 20260924
BACKGROUND = 24.0


def _render_torch(shape, centres, amps, rho, device):
    """Same as _render on a torch device (float64 accumulation); used for the large bench inputs."""
    import torch
    nd = len(shape)
    c = torch.as_tensor(centres, dtype=torch.float64, device=device)
    a = torch.as_tensor(amps, dtype=torch.float64, device=device)
    img = torch.zeros(int(np.prod(shape)), dtype=torch.float64, device=device)
    base = torch.floor(c).to(torch.int64)
    half = int(np.ceil(3.5 * rho))
    rng = torch.arange(-half, half + 1, device=device)
    offs = torch.stack([g.reshape(-1) for g in torch.meshgrid(*([rng] * nd), indexing="ij")], 1)
    lim = torch.tensor(shape, device=device)
    strides = torch.tensor([int(np.prod(shape[i + 1:])) for i in range(nd)], dtype=torch.int64, device=device)
    inv = 1.0 / (rho * rho)
    for o in offs:
        p = base + o
        ok = ((p >= 0) & (p < lim)).all(1)
        d2 = ((p[ok].to(torch.float64) - c[ok]) ** 2).sum(1)
        img.index_add_(0, (p[ok] * strides).sum(1), a[ok] * torch.exp(-d2 * inv))
    return img.reshape(shape).cpu().numpy()


def _render(shape, centres, amps, rho, device=None):
    """Sum of isotropic Gaussians, evaluated within +-3.5 rho of each centre (numpy, any dim)."""
    if device is not None:
        return _render_torch(shape, centres, amps, rho, device)
    nd = len(shape)
    img = np.zeros(int(np.prod(shape)), np.float64)
    base = np.floor(centres).astype(np.int64)
    half = int(np.ceil(3.5 * rho))
    rng = np.arange(-half, half + 1)
    grids = np.meshgrid(*([rng] * nd), indexing="ij")
    offs = np.stack([g.ravel() for g in grids], axis=1)  # [K, nd], order (z,)y,x
    inv = 1.0 / (rho * rho)
    strides = np.array([int(np.prod(shape[i + 1:])) for i in range(nd)], np.int64)
    for o in offs:
        p = base + o
        ok = np.all((p >= 0) & (p < np.array(shape)), axis=1)
        d2 = np.sum((p[ok] - centres[ok]) ** 2, axis=1)
        np.add.at(img, p[ok] @ strides, amps[ok] * np.exp(-d2 * inv))
    return img.reshape(shape)


def displacement_2d(x, y, width, height, second_order=False):
    """u, v at pixel positions (x, y); x~, y~ are relative to the image centre."""
    xt, yt = x - 0.5 * width, y - 0.5 * height
    u = 2.37 + 1.5e-3 * xt - 0.8e-3 * yt
    v = -1.62 + 0.6e-3 * xt + 2.1e-3 * yt
    if second_order:
        u = u + 2e-6 * xt * xt - 1e-6 * xt * yt + 1.5e-6 * yt * yt
        v = v + 1.5e-6 * xt * xt - 1e-6 * xt * yt + 2e-6 * yt * yt
    return u, v


def displacement_3d(x, y, z, dim_x, dim_y, dim_z):
    xt, yt, zt = x - 0.5 * dim_x, y - 0.5 * dim_y, z - 0.5 * dim_z
    return 1.3 + 1e-3 * xt, -0.7 + 1.2e-3 * yt, 2.4 - 1.5e-3 * zt


def speckle_pair_2d(width, height, second_order=False, rho=2.0, seed=REF_SEED, quantise=True, device=None, background=BACKGROUND):
    """(ref, tar) float32 [height, width].  background=0 is SURVEY.md's formula (truly black gaps between the speckles)."""
    rng = np.random.default_rng(seed)
    n = int(0.5 * width * height / (np.pi * rho * rho))
    cx = rng.uniform(-8, width + 8, n)
    cy = rng.uniform(-8, height + 8, n)
    amp = rng.uniform(0.4, 1.0, n)
    ref = _render((height, width), np.stack([cy, cx], 1), amp, rho, device)
    u, v = displacement_2d(cx, cy, width, height, second_order)
    tar = _render((height, width), np.stack([cy + v, cx + u], 1), amp, rho, device)
    out = []
    for im in (ref, tar):
        im = np.clip(background + (255.0 - background) * im, 0, 255)
        if quantise:
            im = np.round(im)
        out.append(im.astype(np.float32))
    return out[0], out[1]


def speckle_pair_3d(dim_x, dim_y, dim_z, rho=2.0, seed=REF_SEED, quantise=True, device=None, background=BACKGROUND):
    """(ref, tar) float32 [dim_z, dim_y, dim_x]."""
    rng = np.random.default_rng(seed)
    n = int(0.35 * dim_x * dim_y * dim_z / (4.0 / 3.0 * np.pi * rho ** 3))
    cx = rng.uniform(-8, dim_x + 8, n)
    cy = rng.uniform(-8, dim_y + 8, n)
    cz = rng.uniform(-8, dim_z + 8, n)
    amp = rng.uniform(0.4, 1.0, n)
    ref = _render((dim_z, dim_y, dim_x), np.stack([cz, cy, cx], 1), amp, rho, device)
    u, v, w = displacement_3d(cx, cy, cz, dim_x, dim_y, dim_z)
    tar = _render((dim_z, dim_y, dim_x), np.stack([cz + w, cy + v, cx + u], 1), amp, rho, device)
    out = []
    for im in (ref, tar):
        im = np.clip(background + (255.0 - background) * im, 0, 255)
        if quantise:
            im = np.round(im)
        out.append(im.astype(np.float32))
    return out[0], out[1]


def speckle_series_3d(dim_x, dim_y, dim_z, n_frames, rho=2.0, seed=REF_SEED, device=None, background=BACKGROUND):
    """(ref [dim_z, dim_y, dim_x], tars [n_frames, dim_z, dim_y, dim_x]) float32, 8-bit valued: the speckles of speckle_pair_3d
    moved by (f + 1) / n_frames of displacement_3d in frame f, so the last frame carries the whole field."""
    rng = np.random.default_rng(seed)
    n = int(0.35 * dim_x * dim_y * dim_z / (4.0 / 3.0 * np.pi * rho ** 3))
    cx = rng.uniform(-8, dim_x + 8, n)
    cy = rng.uniform(-8, dim_y + 8, n)
    cz = rng.uniform(-8, dim_z + 8, n)
    amp = rng.uniform(0.4, 1.0, n)
    u, v, w = displacement_3d(cx, cy, cz, dim_x, dim_y, dim_z)

    def volume(s):
        im = _render((dim_z, dim_y, dim_x), np.stack([cz + s * w, cy + s * v, cx + s * u], 1), amp, rho, device)
        return np.round(np.clip(background + (255.0 - background) * im, 0, 255)).astype(np.float32)

    return volume(0.0), np.stack([volume((f + 1) / n_frames) for f in range(n_frames)])


def _rotation(rv):
    """Rotation matrix of a rotation vector (angle-axis), float64."""
    rv = np.asarray(rv, np.float64)
    th = np.linalg.norm(rv)
    if th == 0:
        return np.eye(3)
    k = rv / th
    kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * kx + (1 - np.cos(th)) * kx @ kx


def _render_plane(shape, hom, to_px, centres, amps, rho, half, device=None):
    """Gaussian speckles on a plane seen through a homography: pixel (c, r) shows material point hom @ (c, r, 1) (dehomogenised),
    and I = sum_k a_k exp(-|m - c_k|^2 / rho^2) over the material centres c_k [K, 2] (x, y).  to_px maps material points to
    pixels (the inverse of hom); each speckle is evaluated on the pixels within +-half of its image."""
    if device is not None:
        import torch
        xp, f = torch, lambda a: torch.as_tensor(np.asarray(a, np.float64), device=device)
    else:
        xp, f = np, lambda a: np.asarray(a, np.float64)
    h, w = shape
    H, G, c, a = f(hom), f(to_px), f(centres), f(amps)
    q = c @ G[:, :2].T + G[:, 2]
    base = xp.floor(q[:, :2] / q[:, 2:3])
    img = xp.zeros(h * w, dtype=base.dtype) if device is None else torch.zeros(h * w, dtype=torch.float64, device=device)
    inv = 1.0 / (rho * rho)
    for dy in range(-half, half + 1):
        for dx in range(-half, half + 1):
            px, py = base[:, 0] + dx, base[:, 1] + dy
            ok = (px >= 0) & (px < w) & (py >= 0) & (py < h)
            px, py, ck, ak = px[ok], py[ok], c[ok], a[ok]
            m = px[:, None] * H[:, 0] + py[:, None] * H[:, 1] + H[:, 2]
            d2 = (m[:, 0] / m[:, 2] - ck[:, 0]) ** 2 + (m[:, 1] / m[:, 2] - ck[:, 1]) ** 2
            idx = py * w + px
            if device is None:
                np.add.at(img, idx.astype(np.int64), ak * np.exp(-d2 * inv))
            else:
                img.index_add_(0, idx.to(torch.int64), ak * torch.exp(-d2 * inv))
    img = img.reshape(h, w)
    return img.cpu().numpy() if device is not None else img


# Stereo rig of speckle_stereo_series: two pinhole cameras (no lens distortion) 600 mm from a planar specimen, the second one
# 120 mm to the side and turned towards the specimen's centre; 1 px is about 0.2 mm on the specimen.
STEREO_Z0, STEREO_BASELINE, STEREO_F = 600.0, 120.0, 3000.0
# displacement of the specimen point (X, Y, Z0) in the last frame, X and Y in mm from the specimen's centre:
# (ex X + tx, ey Y + ty, tz + gx X) -- a stretch in the plane, a rigid translation and an out-of-plane w with a tilt
STEREO_FIELD = dict(ex=4e-3, ey=-2.5e-3, tx=0.8, ty=-0.5, tz=3.0, gx=0.01)


def stereo_rig(width, height):
    """(intrinsics [2, 13], extrinsics [2, 6]) of the speckle_stereo_series cameras, in the order Calibration takes them:
    fx fy fs cx cy k1..k6 p1 p2 and tx ty tz rx ry rz (world -> camera: R X + t)."""
    phi = np.arctan2(STEREO_BASELINE, STEREO_Z0)
    r2 = _rotation([0.0, phi, 0.0])
    t2 = -r2 @ np.array([STEREO_BASELINE, 0.0, 0.0])
    intr = np.zeros((2, 13), np.float32)
    intr[:, 0:5] = [STEREO_F, STEREO_F, 0.0, 0.5 * width, 0.5 * height]
    extr = np.array([[0, 0, 0, 0, 0, 0], [t2[0], t2[1], t2[2], 0.0, phi, 0.0]], np.float32)
    return intr, extr


def speckle_stereo_series(width, height, n_frames, points=None, rho=2.0, seed=REF_SEED, device=None, background=BACKGROUND):
    """A stereo load series of a planar speckled specimen seen by the two cameras of stereo_rig.

    Frame f moves every specimen point by (f + 1) / n_frames of STEREO_FIELD, an affine 3D displacement, so the deformed specimen
    is still a plane.  Each pixel is rendered by intersecting its ray with that plane, mapping the hit back to material
    coordinates and evaluating the Gaussian speckle texture (speckle radius rho px at the specimen's centre) there; images are
    8-bit valued float32 like speckle_pair_2d's.

    Returns a dict: ref1, r2 (height, width), tars1, tars2 (n_frames, height, width), intrinsics, extrinsics (stereo_rig), and
    for points (n, 2) of the view-1 reference image: material (n, 3), the specimen point under each point; displaced
    (n_frames, n, 3), its position in every frame; r2_true (n, 2), its projection into the view-2 reference image; t1_true,
    t2_true (n_frames, n, 2), its projections into both views of every frame (float64)."""
    intr, extr = stereo_rig(width, height)
    K = np.array([[STEREO_F, 0, 0.5 * width], [0, STEREO_F, 0.5 * height], [0, 0, 1]])
    cams = [(np.eye(3), np.zeros(3)), (_rotation(extr[1, 3:6].astype(np.float64)), extr[1, 0:3].astype(np.float64))]
    fd = STEREO_FIELD

    def plane(s):  # the specimen in a frame with load s: P(X, Y) = o + X a + Y b
        return (np.array([s * fd["tx"], s * fd["ty"], STEREO_Z0 + s * fd["tz"]]), np.array([1 + s * fd["ex"], 0, s * fd["gx"]]),
                np.array([0, 1 + s * fd["ey"], 0]))

    def to_px(cam, s):  # material (X, Y, 1) -> homogeneous pixel
        R, t = cams[cam]
        o, a, b = plane(s)
        return K @ np.stack([R @ a, R @ b, R @ o + t], 1)

    pix = STEREO_Z0 / STEREO_F
    rng = np.random.default_rng(seed)
    hw, hh = 0.75 * width * pix + 8, 0.75 * height * pix + 8  # the specimen outgrows both views in every frame
    n = int(0.5 * (2 * hw) * (2 * hh) / (np.pi * (rho * pix) ** 2))
    centres = np.stack([rng.uniform(-hw, hw, n), rng.uniform(-hh, hh, n)], 1)
    amps = rng.uniform(0.4, 1.0, n)
    half = int(np.ceil(3.5 * rho * 1.15)) + 1

    def image(cam, s):
        G = to_px(cam, s)
        im = _render_plane((height, width), np.linalg.inv(G), G, centres, amps, rho * pix, half, device)
        return np.round(np.clip(background + (255.0 - background) * im, 0, 255)).astype(np.float32)

    loads = [(f + 1) / n_frames for f in range(n_frames)]
    out = dict(ref1=image(0, 0.0), r2=image(1, 0.0), tars1=np.stack([image(0, s) for s in loads]),
               tars2=np.stack([image(1, s) for s in loads]), intrinsics=intr, extrinsics=extr)
    if points is not None:
        p = np.asarray(points, np.float64).reshape(-1, 2)
        m = np.c_[p, np.ones(len(p))] @ np.linalg.inv(to_px(0, 0.0)).T
        m = m[:, :2] / m[:, 2:3]

        def proj(cam, s):
            q = np.c_[m, np.ones(len(m))] @ to_px(cam, s).T
            return q[:, :2] / q[:, 2:3]

        def pos(s):
            o, a, b = plane(s)
            return o + m[:, 0:1] * a + m[:, 1:2] * b

        out.update(material=pos(0.0), displaced=np.stack([pos(s) for s in loads]), r2_true=proj(1, 0.0),
                   t1_true=np.stack([proj(0, s) for s in loads]), t2_true=np.stack([proj(1, s) for s in loads]))
    return out


def grid_2d(x0, y0, nx, ny, sx, sy):
    """POI grid, row-major over y then x like the reference examples (test_2d_dic_fftcc_icgn1.cpp:57-66)."""
    ys, xs = np.meshgrid(y0 + sy * np.arange(ny), x0 + sx * np.arange(nx), indexing="ij")
    return np.stack([xs.ravel(), ys.ravel()], 1).astype(np.float32)


def grid_3d(x0, y0, z0, nx, ny, nz, sx, sy, sz):
    zs, ys, xs = np.meshgrid(z0 + sz * np.arange(nz), y0 + sy * np.arange(ny), x0 + sx * np.arange(nx), indexing="ij")
    return np.stack([xs.ravel(), ys.ravel(), zs.ravel()], 1).astype(np.float32)


# BASELINE.json configs (SURVEY.md section 8(d)): image size, POI grid, subset radius, path
CONFIGS = {
    "A": dict(kind="2d", size=(512, 512), grid=(48, 48, 20, 10, 20, 40), r=15, order=1, conv=1e-3, stop=10),
    "B": dict(kind="2d", size=(2048, 2048), grid=(64, 64, 250, 200, 7, 9), r=16, order=1, conv=1e-3, stop=10),
    "C": dict(kind="2d", size=(2048, 2048), grid=(64, 64, 250, 200, 7, 9), r=20, order=2, conv=1e-3, stop=10),
    "D": dict(kind="3d", size=(256, 256, 256), grid=(40, 40, 40, 40, 25, 20, 4, 7, 8), r=16, order=1, conv=1e-3, stop=20),
    "E": dict(kind="2d", size=(4096, 4096), grid=(128, 128, 1000, 500, 3, 7), r=16, order=1, conv=1e-3, stop=10),
    # not a BASELINE.json config: the geometry of the reference's own DVC example (examples/test_dvc_fftcc_icgn1.cpp:
    # 61^3 subvolumes, stop 20) on a synthetic volume (bench.py --config F)
    "F": dict(kind="3d", size=(288, 288, 288), grid=(40, 40, 40, 12, 12, 12, 19, 19, 19), r=30, order=1, conv=1e-3, stop=20),
}
