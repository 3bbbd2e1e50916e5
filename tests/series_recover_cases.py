"""The series recovery calls (ocb_icgn2d_series_recover, ocb_icgn3d_series_recover): the loop they equal, a model of the 2D call's
frame-inner schedule, and the GPU workloads.

series_loop is the contract of include/opencorr_b200.h: for every frame f, register_all(f, q) registers the queue q (frame f - 1's
final records; frame 0: the seeds) and recover(f, q) runs the recovery on it in place.  On the GPU (dev_loop) these are
set_images_*(ref, tars[f]), the prepare, the _dev pair call on all n POIs and icgn*_recover_dev; on the CPU they are stubs and
recover is region_recover_cases.witness_loop.  frame_inner restates the 2D call's schedule (one series pass, a scan for each POI's
first unreliable frame, the rounds in each frame that holds one, the accepted POIs carried through the later frames and the
frame's POIs scanned again), so the CPU tests can show it gives what the loop gives."""
from dataclasses import dataclass

import numpy as np

import region_recover_cases as rr
import subset_series_cases as sc

COLS = rr.COLS


@dataclass
class Params:
    conv: float = 0.001
    stop: float = 10
    radius: float = 20.0
    k_min: int = 9
    zncc_high: float = 0.9
    zncc_low: float = 0.5
    max_rounds: int = 20

    def recover_args(self):
        return (self.conv, self.stop, self.radius, self.k_min, self.zncc_high, self.zncc_low, self.max_rounds)


def series_loop(q, n_frames, register_all, recover, max_rounds):
    """q: a torch tensor [n, 25 | 31] (the seeds), updated frame by frame.  recover(f, q) -> (recovered: max_rounds ints,
    remaining).  Returns (out [F, n, C], recovered [F, max_rounds], remaining [F]) as numpy arrays."""
    import torch
    out, rec, left = [], [], []
    for f in range(n_frames):
        register_all(f, q)
        recovered, remaining = recover(f, q)
        out.append(q.clone())
        rec.append(list(recovered) + [0] * (max_rounds - len(recovered)))
        left.append(remaining)
    return torch.stack(out).cpu().numpy(), np.array(rec, np.int64).reshape(n_frames, max_rounds), np.array(left, np.int64)


def frame_inner(seeds, n_frames, register_all, recover, conv, zncc_low, max_rounds):
    """The 2D call's schedule on a numpy queue of seeds, with register_all(f, q) a per-POI function of the record and the frame.
    Returns what series_loop returns."""
    import torch
    zc, cc = COLS[seeds.shape[1]]

    def carry(q, f0):  # the series pass of the records q over frames f0 ... F - 1
        t = torch.from_numpy(q.copy())
        frames = []
        for f in range(f0, n_frames):
            register_all(f, t)
            frames.append(t.clone().numpy())
        return np.stack(frames) if frames else np.zeros((0,) + q.shape, np.float32)

    def first_unreliable(f0, pois):
        for i in pois:
            hit = [f for f in range(f0, n_frames) if out[f, i, zc] < zncc_low or out[f, i, cc] > conv]
            first[i] = hit[0] if hit else -1

    out = carry(seeds, 0)
    rec = np.zeros((n_frames, max_rounds), np.int64)
    left = np.zeros(n_frames, np.int64)
    first = np.full(len(seeds), -1)
    first_unreliable(0, range(len(seeds)))
    for f in range(n_frames):
        pois = np.flatnonzero(first == f)
        if not len(pois):
            continue
        q = torch.from_numpy(out[f].copy())
        recovered, left[f] = recover(f, q)
        rec[f, :len(recovered)] = recovered
        accepted = np.flatnonzero((q.numpy().view(np.uint32) != out[f].view(np.uint32)).any(1))
        out[f] = q.numpy()
        if len(accepted):
            out[f + 1:, accepted] = carry(out[f, accepted], f + 1)
        first_unreliable(f + 1, pois)
    return out, rec, left


# ---- GPU ---------------------------------------------------------------------------------------------------------------------
W, H, FRAMES = 387, 320, 4  # W % 4 != 0: frame pointers of the stack are not 16-byte aligned
BLOCK = (130, 130, 200, 200)  # reference-frame region whose subsets frame K covers
K = 2


def occlusion_box(region, k, n_frames, r, margin=4):
    """The box of frame k (of sc.render_series(W, H, n_frames)) covering the subsets (radius r) of the POIs in `region`."""
    from opencorr_b200 import synth
    x0, y0, x1, y1 = region
    u, v = synth.displacement_2d((x0 + x1) / 2.0, (y0 + y1) / 2.0, W, H)
    s = (k + 1) / n_frames
    return (int(x0 + s * u - r - margin), int(y0 + s * v - r - margin), int(x1 + s * u + r + margin + 1), int(y1 + s * v + r + margin + 1))


def in_region(xy, region):
    x0, y0, x1, y1 = region
    return (xy[:, 0] >= x0) & (xy[:, 0] < x1) & (xy[:, 1] >= y0) & (xy[:, 1] < y1)


def occluded_series(n_frames=FRAMES, k=K, second_order=False):
    """(ref, clean stack, stack whose frame k covers BLOCK's subsets)"""
    ref, clean = sc.render_series(W, H, n_frames, second_order=second_order)
    return ref, clean, sc.occlude(clean, k, occlusion_box(BLOCK, k, n_frames, 20))


def garbage(seeds, mask):
    """seeds with the POIs of mask given a translation far beyond their subsets"""
    q = seeds.copy()
    q[mask, 2] += 23.0
    q[mask, 8] -= 19.0
    return q


def dev_loop(eng, dim, order, ref, tars, seeds, r, p):
    """The loop of existing calls the series recovery calls equal: for f: set_images_*(ref, tars[f]); prepare; the _dev pair
    call on all n POIs; icgn*_recover_dev.  r: the subset radius (2D) or radii (3D)."""
    import torch
    q = torch.from_numpy(seeds.copy()).cuda()
    n = len(seeds)

    def register_all(f, q):
        if dim == 2:
            eng.set_images_2d(ref, tars[f])
            eng.icgn2d_prepare()
            torch.cuda.synchronize()
            (eng.icgn2d1_dev if order == 1 else eng.icgn2d2_dev)(q.data_ptr(), n, r, r, p.conv, p.stop)
        else:
            eng.set_images_3d(ref, tars[f])
            eng.icgn3d_prepare()
            torch.cuda.synchronize()
            eng.icgn3d1_dev(q.data_ptr(), n, *r, p.conv, p.stop)
        eng.sync()

    def recover(f, q):
        if dim == 2:
            return eng.icgn2d_recover_dev(order, q.data_ptr(), n, r, r, *p.recover_args())
        return eng.icgn3d_recover_dev(q.data_ptr(), n, *r, *p.recover_args())

    return series_loop(q, len(tars), register_all, recover, p.max_rounds)
