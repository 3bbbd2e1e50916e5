"""The recovery calls (ocb_icgn2d_recover, ocb_icgn3d_recover): the witness, the reference example's loop restated, and the
GPU cases.

witness_loop is the loop of include/opencorr_b200.h written with the bookkeeping in torch: classify once, then per round
fit(reliable, work), register(work), accept, append, compact.  On the GPU (witness) fit is ocb_region_fit*_dev and register the
_dev pair call on the working records, so the pair kernel plans for |U| POIs exactly as the one call does.  example_loop restates
examples/test_3d_reconstruction_sift_icgn2_regfit.cpp:219-270 of the reference line by line, including the erase inside its index
loop that skips the POI after each accepted one for that round."""
from dataclasses import dataclass

import numpy as np

# field columns (ZNCC, convergence) and record length of POI2D and POI3D
COLS = {25: (16, 18), 31: (18, 20)}


def witness_loop(q, fit, register, conv, zncc_high, zncc_low, max_rounds):
    """q: a torch tensor [n, 25 | 31], updated in place.  Returns (recovered: max_rounds ints, remaining, rounds run)."""
    import torch
    zc, cc = COLS[q.shape[1]]
    z, c = q[:, zc], q[:, cc]
    unreliable = (z < zncc_low) | (c > conv)
    u_idx = torch.nonzero(unreliable).flatten()
    reliable = q[~unreliable & (z >= zncc_high)].contiguous()
    work = q[u_idx].contiguous()
    recovered = [0] * max_rounds
    rounds = 0
    while rounds < max_rounds and len(u_idx):
        fit(reliable, work)
        register(work)
        acc = (work[:, zc] >= zncc_high) & (work[:, cc] <= conv)
        q[u_idx[acc]] = work[acc]
        reliable = torch.cat([reliable, work[acc]]).contiguous()
        work, u_idx = work[~acc].contiguous(), u_idx[~acc]
        recovered[rounds] = int(acc.sum())
        rounds += 1
        if recovered[rounds - 1] == 0:
            break
    return recovered, len(u_idx), rounds


def example_loop(q, fit, register, conv, zncc_high, zncc_low, trial_rounds):
    """The reference example's loop on a numpy queue q (updated in place), with fit / register taking stacked records as the
    witness's do.  Returns (success_counter per round (trial_rounds ints), POIs left unreliable)."""
    zc, cc = COLS[q.shape[1]]
    reliable, unreliable, unreliable_idx = [], [], []
    for i in range(len(q)):
        if q[i, zc] < zncc_low or q[i, cc] > conv:
            unreliable.append(q[i].copy())
            unreliable_idx.append(i)
        elif q[i, zc] >= zncc_high:
            reliable.append(q[i].copy())
    counts = [0] * trial_rounds
    for i in range(trial_rounds):
        success = 0
        work = np.array(unreliable, np.float32).reshape(-1, q.shape[1])
        fit(np.array(reliable, np.float32).reshape(-1, q.shape[1]), work)
        register(work)
        unreliable = [r.copy() for r in work]
        queue_size = len(unreliable)
        if queue_size == 0:
            break
        j = 0
        while j < queue_size:  # for (int j = 0; j < queue_size; j++), with the erase and queue_size update inside
            if unreliable[j][zc] >= zncc_high and unreliable[j][cc] <= conv:
                q[unreliable_idx[j]] = unreliable[j]
                reliable.append(unreliable[j])
                del unreliable[j]
                del unreliable_idx[j]
                success += 1
            queue_size = len(unreliable)
            j += 1
        counts[i] = success
        if success == 0:
            break
    return counts, len(unreliable)


# ---- GPU cases --------------------------------------------------------------------------------------------------------------
@dataclass
class Case:
    name: str
    dim: int
    ref: np.ndarray
    tar: np.ndarray
    q: np.ndarray           # the registered queue the recovery starts from
    r: tuple                # subset radii
    conv: float
    stop: float
    radius: float
    k_min: int
    zncc_high: float
    zncc_low: float
    max_rounds: int
    clean: np.ndarray = None  # the same queue registered without the garbage seeds (synthetic cases)
    block: np.ndarray = None  # the POIs seeded with garbage


def _register_2d(engine, ref, tar, xy, order, r, conv, stop, garbage=None):
    """FFTCC2D then ICGN2D<order> over the POIs xy; the POIs in `garbage` are re-seeded far off and registered again."""
    import opencorr_b200 as ob
    engine.set_images_2d(ref, tar)
    engine.icgn2d_prepare()
    q = ob.make_poi2d(xy)
    engine.fftcc2d(q, r, r)
    icgn = engine.icgn2d1 if order == 1 else engine.icgn2d2
    icgn(q, r, r, conv, stop)
    clean = q.copy()
    if garbage is not None and len(garbage):
        q[garbage, 2:14] = 0
        q[garbage, 2], q[garbage, 8] = 23.0, -19.0  # garbage seeds, far beyond the subset
        sub = np.ascontiguousarray(q[garbage])
        icgn(sub, r, r, conv, stop)
        q[garbage] = sub
    return q, clean


def speckle_block(engine, order):
    """The second-order speckle pair of test_recovery_loop with a 12 x 12 block of POIs seeded with garbage."""
    from opencorr_b200 import synth
    ref, tar = synth.speckle_pair_2d(512, 512, second_order=True)
    xy = synth.grid_2d(40, 40, 55, 55, 8, 8)
    gx, gy = (xy[:, 0] - 40) / 8, (xy[:, 1] - 40) / 8
    block = np.flatnonzero((gx >= 20) & (gx < 32) & (gy >= 18) & (gy < 30))
    q, clean = _register_2d(engine, ref, tar, xy, order, 16, 0.001, 10, block)
    return Case("speckle_block_o%d" % order, 2, ref, tar, q, (16, 16), 0.001, 10, 20.0, 9, 0.9, 0.5, 20, clean, block)


def speckle_dead_disc(engine, order):
    """speckle_block with a disc of zero pixels in the target: the POIs whose subsets sit in it can never recover, so the loop
    ends on a round that recovers none."""
    from opencorr_b200 import synth
    ref, tar = synth.speckle_pair_2d(512, 512, second_order=True)
    yy, xx = np.mgrid[0:512, 0:512]
    tar = tar.copy()
    tar[(xx - 330) ** 2 + (yy - 300) ** 2 < 45 ** 2] = 0
    xy = synth.grid_2d(40, 40, 55, 55, 8, 8)
    gx, gy = (xy[:, 0] - 40) / 8, (xy[:, 1] - 40) / 8
    block = np.flatnonzero((gx >= 20) & (gx < 40) & (gy >= 18) & (gy < 38))
    q, clean = _register_2d(engine, ref, tar, xy, order, 16, 0.001, 10, block)
    return Case("speckle_dead_disc_o%d" % order, 2, ref, tar, q, (16, 16), 0.001, 10, 20.0, 9, 0.9, 0.5, 20, clean, block)


def oht_cfrp(engine):
    """The reference's 2D example pair and grid (examples/test_2d_dic_fftcc_icgn1.cpp:44-66): FFTCC2D -> ICGN2D1, then the regfit
    example's recovery parameters (0.9 / 0.5, radius 12, 9 neighbours, 20 rounds) around the specimen's hole."""
    import util
    from opencorr_b200 import synth
    ref, tar = util.oht_cfrp_pair()
    ref, tar = ref.astype(np.float32), tar.astype(np.float32)
    xy = synth.grid_2d(30, 30, 100, 300, 2, 2)
    q, _ = _register_2d(engine, ref, tar, xy, 1, 16, 0.001, 10)
    return Case("oht_cfrp", 2, ref, tar, q, (16, 16), 0.001, 10, 12.0, 9, 0.9, 0.5, 20)


def config_b_discs(engine, order=1):
    """Config B's geometry (2048^2, 250 x 200 POIs at 7 x 9 px, r = 16) with 10 % of the POIs seeded with garbage in discs."""
    from opencorr_b200 import synth
    cfg = synth.CONFIGS["B"]
    ref, tar = synth.speckle_pair_2d(*cfg["size"])
    xy = synth.grid_2d(*cfg["grid"])
    bad = discs(xy, 0.10, (20.0, 60.0), np.random.default_rng(7))
    q, clean = _register_2d(engine, ref, tar, xy, order, cfg["r"], cfg["conv"], cfg["stop"], np.flatnonzero(bad))
    return Case("config_b_discs_o%d" % order, 2, ref, tar, q, (16, 16), cfg["conv"], cfg["stop"], 20.0, 9, 0.9, 0.5, 20, clean,
                np.flatnonzero(bad))


def discs(pos, frac, radii, rng):
    """A mask of the POIs inside random discs / balls, grown until it holds frac of them."""
    bad = np.zeros(len(pos), bool)
    lo, hi = pos.min(0), pos.max(0)
    while bad.mean() < frac:
        c = rng.uniform(lo, hi)
        bad |= ((pos - c) ** 2).sum(1) < rng.uniform(*radii) ** 2
    return bad


def ball_3d(engine, size=96, grid=(20, 20, 20, 8, 8, 8, 8, 8, 8), r=8):
    """A synthetic volume pair, FFTCC3D -> ICGN3D1, with a ball of POIs seeded with garbage."""
    import opencorr_b200 as ob
    from opencorr_b200 import synth
    ref, tar = synth.speckle_pair_3d(size, size, size)
    xyz = synth.grid_3d(*grid)
    engine.set_images_3d(ref, tar)
    engine.icgn3d_prepare()
    q = ob.make_poi3d(xyz)
    engine.fftcc3d(q, r, r, r)
    engine.icgn3d1(q, r, r, r, 0.001, 20)
    clean = q.copy()
    centre = xyz.mean(0)
    block = np.flatnonzero(((xyz - centre) ** 2).sum(1) < (0.3 * (xyz.max(0) - xyz.min(0)).min()) ** 2)
    q[block, 3:15] = 0
    q[block, 3], q[block, 7], q[block, 11] = 11.0, -9.0, 13.0
    sub = np.ascontiguousarray(q[block])
    engine.icgn3d1(sub, r, r, r, 0.001, 20)
    q[block] = sub
    return Case("ball_3d", 3, ref, tar, q, (r, r, r), 0.001, 20, 20.0, 12, 0.9, 0.5, 20, clean, block)


def set_pair(engine, c):
    if c.dim == 2:
        engine.set_images_2d(c.ref, c.tar)
        engine.icgn2d_prepare()
    else:
        engine.set_images_3d(c.ref, c.tar)
        engine.icgn3d_prepare()


def witness(engine, c, q=None, order=1, **over):
    """The witness loop on the GPU over a copy of c.q (or q), with the parameters of c overridden by `over`.  Returns (records,
    recovered, remaining, rounds run)."""
    import torch
    p = dict(radius=c.radius, k_min=c.k_min, zncc_high=c.zncc_high, zncc_low=c.zncc_low, max_rounds=c.max_rounds, conv=c.conv)
    p.update(over)
    d_q = torch.from_numpy((c.q if q is None else q).copy()).cuda()
    kind = "2d" if c.dim == 2 else "3d"

    def fit(rel, work):
        torch.cuda.synchronize()
        engine.region_fit_dev(kind, rel.data_ptr() if len(rel) else 0, len(rel), work.data_ptr(), len(work), p["radius"], p["k_min"])
        engine.sync()

    def register(work):
        torch.cuda.synchronize()
        if c.dim == 3:
            engine.icgn3d1_dev(work.data_ptr(), len(work), *c.r, p["conv"], c.stop)
        elif order == 1:
            engine.icgn2d1_dev(work.data_ptr(), len(work), *c.r, p["conv"], c.stop)
        else:
            engine.icgn2d2_dev(work.data_ptr(), len(work), *c.r, p["conv"], c.stop)
        engine.sync()

    recovered, remaining, rounds = witness_loop(d_q, fit, register, p["conv"], p["zncc_high"], p["zncc_low"], p["max_rounds"])
    torch.cuda.synchronize()
    return d_q.cpu().numpy(), np.array(recovered, np.int64), remaining, rounds
