"""GPU: the recovery calls (ocb_icgn2d_recover, ocb_icgn3d_recover and their _dev variants) against the witness of
tests/region_recover_cases.py, the same loop written with ocb_region_fit*_dev and the _dev pair calls and torch bookkeeping.
The records, `recovered` and `remaining` must be byte-identical.  Then the edge cases of the classification, the launch count,
the refusals, a group context, the state the call must not touch, and the recovered POIs against the clean run and the truth."""
import ctypes

import numpy as np
import pytest

import opencorr_b200 as ob
from opencorr_b200 import _capi, synth
import region_recover_cases as rr

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def reliable(c, q):
    zc, cc = rr.COLS[q.shape[1]]
    return (q[:, zc] >= c.zncc_high) & (q[:, cc] <= c.conv)


def call(engine, c, dev, q=None, order=1, **over):
    """The one call on a copy of c.q (or q), host or _dev.  Returns (records, recovered, remaining)."""
    p = dict(radius=c.radius, k_min=c.k_min, zncc_high=c.zncc_high, zncc_low=c.zncc_low, max_rounds=c.max_rounds, conv=c.conv)
    p.update(over)
    args = (p["conv"], c.stop, p["radius"], p["k_min"], p["zncc_high"], p["zncc_low"], p["max_rounds"])
    src = (c.q if q is None else q).copy()
    if not dev:
        if c.dim == 2:
            rec, left = engine.icgn2d_recover(order, src, *c.r, *args)
        else:
            rec, left = engine.icgn3d_recover(src, *c.r, *args)
        return src, rec, left
    d = torch.from_numpy(src).cuda()
    torch.cuda.synchronize()
    if c.dim == 2:
        rec, left = engine.icgn2d_recover_dev(order, d.data_ptr(), len(src), *c.r, *args)
    else:
        rec, left = engine.icgn3d_recover_dev(d.data_ptr(), len(src), *c.r, *args)
    return d.cpu().numpy(), rec, left


def check(engine, c, dev, q=None, order=1, **over):
    """The call against the witness, byte for byte; returns the witness's (records, recovered, remaining, rounds)."""
    rr.set_pair(engine, c)
    w = rr.witness(engine, c, q, order, **over)
    got, rec, left = call(engine, c, dev, q, order, **over)
    assert np.array_equal(rec, w[1]) and left == w[2], (c.name, rec, w[1], left, w[2])
    bad = np.flatnonzero((bits(got) != bits(w[0])).any(1))
    assert not len(bad), "%s: %d records differ from the witness, first %d" % (c.name, len(bad), bad[0])
    return w


@pytest.fixture(scope="module")
def cases(engine):
    out = {}
    for order in (1, 2):
        out["speckle_block_o%d" % order] = (rr.speckle_block(engine, order), order)
        out["speckle_dead_disc_o%d" % order] = (rr.speckle_dead_disc(engine, order), order)
    out["oht_cfrp"] = (rr.oht_cfrp(engine), 1)
    out["ball_3d"] = (rr.ball_3d(engine), 1)
    return out


NAMES = ["speckle_block_o1", "speckle_block_o2", "speckle_dead_disc_o1", "speckle_dead_disc_o2", "oht_cfrp", "ball_3d"]


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
@pytest.mark.parametrize("name", NAMES)
def test_against_the_witness(engine, cases, name, dev):
    c, order = cases[name]
    w = check(engine, c, dev, order=order)
    zc, cc = rr.COLS[c.q.shape[1]]
    unreliable = (c.q[:, zc] < c.zncc_low) | (c.q[:, cc] > c.conv)
    print("%s %s: %d unreliable of %d, recovered %s, %d remain after %d rounds" % (name, "dev" if dev else "host", unreliable.sum(), len(c.q),
                                                                                 w[1][:w[3]].tolist(), w[2], w[3]))
    assert w[3] >= 1 and unreliable.any()
    if name.startswith("speckle_dead_disc"):
        assert w[2] > 0 and w[1][w[3] - 1] == 0  # the disc never recovers: the loop ends on "0 recovered"
    if c.block is not None and not name.startswith("speckle_dead_disc"):
        assert reliable(c, w[0][c.block]).all(), "%d block POIs still unreliable" % (~reliable(c, w[0][c.block])).sum()


@pytest.mark.parametrize("max_rounds", [0, 1, 2, 1000])
def test_max_rounds(engine, cases, max_rounds):
    c, order = cases["speckle_dead_disc_o2"]
    for dev in (False, True):
        w = check(engine, c, dev, order=order, max_rounds=max_rounds)
        assert len(w[1]) == max_rounds and w[3] <= max_rounds
    if max_rounds == 0:
        got, rec, left = call(engine, c, False, order=order, max_rounds=0)
        assert np.array_equal(bits(got), bits(c.q)) and left > 0


def test_unchanged_bytes(engine, cases):
    """Reliable POIs, POIs in neither set and POIs never accepted keep every byte; the accepted ones are IC-GN records."""
    c, order = cases["speckle_dead_disc_o1"]
    rr.set_pair(engine, c)
    got, rec, left = call(engine, c, False, order=order)
    zc, cc = rr.COLS[25]
    u = (c.q[:, zc] < c.zncc_low) | (c.q[:, cc] > c.conv)
    accepted = (bits(got) != bits(c.q)).any(1)
    assert not accepted[~u].any()
    assert accepted.sum() == rec.sum() and (u & ~accepted).sum() == left
    assert (got[accepted, zc] >= c.zncc_high).all() and (got[accepted, cc] <= c.conv).all()


def test_edge_sets(engine, cases):
    """An empty U (nothing launched after the classification), an empty R, min_neighbors above |R|."""
    c, order = cases["speckle_block_o1"]
    rr.set_pair(engine, c)
    zc, cc = rr.COLS[25]
    q = c.q.copy()
    q[:, zc], q[:, cc] = 0.95, 0.0  # every POI reliable: U empty
    before = engine.launch_count()
    got, rec, left = call(engine, c, False, q, order)
    assert engine.launch_count() - before == 2 and left == 0 and not rec.any() and np.array_equal(bits(got), bits(q))
    q = c.q.copy()
    q[:, zc] = np.where(q[:, zc] >= c.zncc_high, 0.7, q[:, zc])  # no reliable POI: every fit finds no neighbour
    assert not reliable(c, q).any()
    for dev in (False, True):
        check(engine, c, dev, q, order)
    for dev in (False, True):
        check(engine, c, dev, order=order, k_min=len(c.q))  # more neighbours needed than there are reliable POIs


def test_nan_positions_and_fields(engine, cases):
    c, order = cases["speckle_block_o2"]
    zc, cc = rr.COLS[25]
    rng = np.random.default_rng(5)
    q = c.q.copy()
    pick = rng.choice(len(q), 200, replace=False)
    q[pick[:40], 0] = np.nan             # NaN positions, in every set
    q[c.block[:10], 1] = np.nan          # unreliable POIs with a NaN position
    q[pick[40:80], zc] = np.nan          # NaN ZNCC: neither set unless the convergence is above conv
    q[pick[60:80], cc] = 1.0
    q[pick[80:120], cc] = np.nan         # NaN convergence: reliable with a high ZNCC
    q[pick[120:160], 2] = np.nan         # NaN displacement
    for dev in (False, True):
        check(engine, c, dev, q, order)


def test_config_b_queue(engine):
    """Config B's 50 000 POIs, 10 % seeded with garbage in discs: far more POIs than one launch's resident warps."""
    for order in (1, 2):
        c = rr.config_b_discs(engine, order)
        for dev in (False, True):
            w = check(engine, c, dev, order=order)
        print("config B order %d: %d garbage-seeded, recovered %s, %d remain" % (order, len(c.block), w[1][:w[3]].tolist(), w[2]))


def test_recovered_blocks_match_the_clean_run(engine, cases):
    """The recovered block POIs are within IC-GN's tolerance of the clean run and of the synthetic truth."""
    for name in ("speckle_block_o1", "speckle_block_o2", "ball_3d"):
        c, order = cases[name]
        rr.set_pair(engine, c)
        got, rec, left = call(engine, c, False, order=order)
        b = c.block
        if c.dim == 2:
            W, H = c.ref.shape[1], c.ref.shape[0]
            u, v = synth.displacement_2d(got[b, 0].astype(np.float64), got[b, 1].astype(np.float64), W, H, True)
            err = np.hypot(got[b, 2] - u, got[b, 8] - v).max()
            clean_err = np.hypot(c.clean[b, 2] - u, c.clean[b, 8] - v).max()
            diff = np.abs(got[b][:, [2, 8]] - c.clean[b][:, [2, 8]]).max()
        else:
            dz, dy, dx = c.ref.shape
            u, v, ww = synth.displacement_3d(got[b, 0], got[b, 1], got[b, 2], dx, dy, dz)
            err = np.sqrt((got[b, 3] - u) ** 2 + (got[b, 7] - v) ** 2 + (got[b, 11] - ww) ** 2).max()
            clean_err = np.sqrt((c.clean[b, 3] - u) ** 2 + (c.clean[b, 7] - v) ** 2 + (c.clean[b, 11] - ww) ** 2).max()
            diff = np.abs(got[b][:, [3, 7, 11]] - c.clean[b][:, [3, 7, 11]]).max()
        print("%s: %d block POIs, max |d| vs truth %.2e (clean %.2e), vs clean %.2e" % (name, len(b), err, clean_err, diff))
        assert reliable(c, got[b]).all() and err < max(2 * clean_err, 0.01) and diff < 5e-3, (name, err, clean_err, diff)


def test_launches_per_round_do_not_depend_on_n(engine, cases):
    """Two for the classification, one move, and nine per round: RegionFit's five, IC-GN, two selections and one move."""
    for name in ("speckle_dead_disc_o1", "oht_cfrp"):
        c, order = cases[name]
        rr.set_pair(engine, c)
        w = rr.witness(engine, c, order=order)
        before = engine.launch_count()
        call(engine, c, True, order=order)
        assert engine.launch_count() - before == 3 + 9 * w[3], (name, engine.launch_count() - before, w[3])


def _raw(engine, c, dev, q, n, order=1, rx=16, conv=0.001, zh=0.9, zl=0.5, rounds=5, rec=None, left=None):
    if c.dim == 2:
        fn = engine._lib.ocb_icgn2d_recover_dev if dev else engine._lib.ocb_icgn2d_recover
        head = (order, q, n, rx, c.r[1])
    else:
        fn = engine._lib.ocb_icgn3d_recover_dev if dev else engine._lib.ocb_icgn3d_recover
        head = (q, n, rx, c.r[1], c.r[2])
    return fn(engine._ctx, *head, ctypes.c_float(conv), ctypes.c_float(c.stop), ctypes.c_float(c.radius), c.k_min, ctypes.c_float(zh),
              ctypes.c_float(zl), rounds, rec, left)


def test_refusals_write_nothing(engine, cases):
    nan = float("nan")
    for name in ("speckle_block_o1", "ball_3d"):
        c, _ = cases[name]
        rr.set_pair(engine, c)
        for dev in (False, True):
            q = c.q.copy()
            d = torch.from_numpy(q.copy()).cuda() if dev else None
            qp = ctypes.c_void_p(d.data_ptr() if dev else q.ctypes.data)
            rec = np.full(5, 77, np.uint64)
            left = ctypes.c_size_t(99)
            out = (ctypes.c_void_p(rec.ctypes.data), ctypes.byref(left))
            refusals = [dict(rounds=-1), dict(conv=nan), dict(zh=nan), dict(zl=nan), dict(rx=0), dict(rx=4000)]
            if c.dim == 2:
                refusals += [dict(order=0), dict(order=3)]
            for kw in refusals:
                rc = _raw(engine, c, dev, qp, len(q), **kw, rec=out[0], left=out[1])
                assert rc in (_capi.OCB_ERR_ARG, _capi.OCB_ERR_UNSUPPORTED), (name, dev, kw, rc)
            assert _raw(engine, c, dev, None, len(q), rec=out[0], left=out[1]) == _capi.OCB_ERR_ARG
            assert _raw(engine, c, dev, qp, 1 << 31, rec=out[0], left=out[1]) == _capi.OCB_ERR_ARG
            assert (rec == 77).all() and left.value == 99
            got = d.cpu().numpy() if dev else q
            assert np.array_equal(bits(got), bits(c.q)), (name, dev)
            # n = 0: nothing to do, the counts are zero
            assert _raw(engine, c, dev, None, 0, rec=out[0], left=out[1]) == _capi.OCB_OK and not rec.any() and left.value == 0
    fresh = ob.Engine(0)
    try:
        c, _ = cases["speckle_block_o1"]
        q = c.q.copy()
        assert _raw(fresh, c, False, ctypes.c_void_p(q.ctypes.data), len(q)) == _capi.OCB_ERR_STATE  # no images set
        assert np.array_equal(bits(q), bits(c.q))
    finally:
        fresh.close()
    with pytest.raises(ValueError):
        engine.icgn2d_recover(1, c.q[:, :24].copy(), 16, 16, 0.001, 10, 20.0, 9, 0.9, 0.5, 3)


def test_group_context(engine, cases):
    n_dev = _capi.load().ocb_device_count()
    grp = ob.Engine(list(range(n_dev)))
    try:
        for name in ("speckle_dead_disc_o2", "ball_3d"):
            c, order = cases[name]
            rr.set_pair(engine, c)
            rr.set_pair(grp, c)
            a = call(engine, c, False, order=order)
            b = call(grp, c, False, order=order)
            assert np.array_equal(bits(a[0]), bits(b[0])) and np.array_equal(a[1], b[1]) and a[2] == b[2], name
        c, _ = cases["speckle_block_o1"]
        d = torch.from_numpy(c.q.copy()).cuda()
        assert _raw(grp, c, True, ctypes.c_void_p(d.data_ptr()), len(c.q)) == _capi.OCB_ERR_ARG
        assert np.array_equal(bits(d.cpu().numpy()), bits(c.q))
    finally:
        grp.close()


def test_pair_prepare_and_series_state_untouched(engine, cases):
    """After a recovery call the pair gives the same IC-GN records, needs no new prepare, and a series set before gives the same
    records as before."""
    c, order = cases["speckle_block_o2"]
    ref, tar = c.ref, c.tar
    engine.set_series_2d(ref, np.stack([tar, tar]))
    rr.set_pair(engine, c)
    probe = c.clean[:300].copy()
    probe[:, 16:19] = 0
    first = probe.copy()
    engine.icgn2d2(first, 16, 16, 0.001, 10)
    series = engine.icgn2d_series(2, probe, 16, 16, 0.001, 10)
    call(engine, c, False, order=order)
    call(engine, c, True, order=order)
    again = probe.copy()
    engine.icgn2d2(again, 16, 16, 0.001, 10)
    assert np.array_equal(bits(again), bits(first))
    assert np.array_equal(bits(engine.icgn2d_series(2, probe, 16, 16, 0.001, 10)), bits(series))
