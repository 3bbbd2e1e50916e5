"""CPU: the loop the series recovery calls equal (tests/series_recover_cases.py series_loop, built on
region_recover_cases.witness_loop) and the 2D call's frame-inner schedule (frame_inner), with stub registration and fit
functions.

The stubs make a POI's history a schedule.  The series registration (track) carries a record whose ZNCC is negative unchanged
(the guard) and otherwise adds 1 to u and sets zncc 0.95; in the frame its subset is occluded (column OCC) it ends with the
sentinel -1, and a dead POI (column DEAD) always ends with zncc 0.3.  The fit writes the mean u of the reliable set with zncc 0;
the recovery's registration counts its trials (column TRIALS) and passes a POI (zncc 0.95, convergence 0) unless it is dead or
occluded in that frame."""
import numpy as np
import pytest

import region_recover_cases as rr
import series_recover_cases as src

torch = pytest.importorskip("torch")
ZC, CC, OCC, DEAD, TRIALS = 16, 18, 20, 21, 22
CONV, HIGH, LOW = 0.001, 0.9, 0.5


def track(f, q):
    ok = q[:, ZC] >= 0
    occluded = q[:, OCC] == f
    dead = q[:, DEAD] > 0
    q[ok, 2] += 1.0
    q[ok, CC] = 0.0
    q[ok, ZC] = 0.95
    q[ok & dead, ZC] = 0.3
    q[ok & occluded, ZC] = -1.0


def fit(f, rel, work):
    work[:, 2] = float(rel[:, 2].mean()) if len(rel) else 0.0
    work[:, ZC] = 0.0


def register(f, work):
    work[:, TRIALS] += 1
    fail = (work[:, DEAD] > 0) | (work[:, OCC] == f)
    work[:, CC] = 0.0
    work[:, ZC] = 0.95
    work[fail, ZC] = -1.0


def seeds(n, occluded=(), dead=(), failed=()):
    """n POIs: occluded = [(POI, frame)], dead and failed (seeded with the sentinel) POI indices"""
    q = np.zeros((n, 25), np.float32)
    q[:, 0] = np.arange(n)
    q[:, ZC] = 0.95
    q[:, OCC] = -1
    for i, f in occluded:
        q[i, OCC] = f
    q[list(dead), DEAD] = 1
    q[list(failed), ZC] = -1.0
    return q


def loop(q, n_frames, rounds):
    def recover(f, t):
        rec, left, _ = rr.witness_loop(t, lambda rel, work: fit(f, rel, work), lambda work: register(f, work), CONV, HIGH, LOW, rounds)
        return rec, left
    return src.series_loop(torch.from_numpy(q.copy()), n_frames, track, recover, rounds)


def inner(q, n_frames, rounds):
    def recover(f, t):
        rec, left, _ = rr.witness_loop(t, lambda rel, work: fit(f, rel, work), lambda work: register(f, work), CONV, HIGH, LOW, rounds)
        return rec, left
    return src.frame_inner(q, n_frames, track, recover, CONV, LOW, rounds)


def plain(q, n_frames):
    t = torch.from_numpy(q.copy())
    out = []
    for f in range(n_frames):
        track(f, t)
        out.append(t.clone().numpy())
    return np.stack(out)


def same(a, b):
    return np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32))


def test_accepted_poi_carries_its_recovered_record():
    q = seeds(12, occluded=[(4, 1), (5, 1)])
    out, rec, left = loop(q, 4, 5)
    base = plain(q, 4)
    assert (base[1:, 4:6, ZC] == -1).all(), "control: the plain series loses the occluded POIs for good"
    assert left[1] == 2 and rec[1, 0] == 0, "occluded in frame 1: the rounds of frame 1 cannot recover them"
    assert rec[2, 0] == 2 and left[2] == 0, "frame 2 recovers them"
    fitted = out[2, 4, 2]
    assert fitted == np.float32(base[2, 0, 2]), "frame 2's record of POI 4 is the fit of its reliable neighbours"
    for f in (3,):  # frame 3 is registered from the recovered record
        assert out[f, 4, 2] == out[f - 1, 4, 2] + 1 and out[f, 4, ZC] == np.float32(0.95)


def test_never_accepted_poi_keeps_its_bytes():
    q = seeds(10, dead=[3], occluded=[(6, 0)])
    out, rec, left = loop(q, 3, 4)
    base = plain(q, 3)
    assert same(out[:, 3], base[:, 3]), "a dead POI keeps the series' records in every frame"
    assert list(rec[:, 0]) == [0, 1, 0] and (rec[:, 1:] == 0).all(), "POI 6, occluded in frame 0, comes back in frame 1"
    assert list(left) == [2, 1, 1], "the dead POI takes one round per frame and is never recovered"
    assert (out[:, 3, TRIALS] == 0).all(), "a POI never accepted keeps its bytes: its trials stay in the working records"


def test_counts_layout():
    q = seeds(16, occluded=[(1, 0), (2, 2)], dead=[9], failed=[12])
    rounds = 3
    out, rec, left = loop(q, 4, rounds)
    assert rec.shape == (4, rounds) and left.shape == (4,)
    # frame 0: POI 12 (failed seed) recovered in round 0, POI 1 occluded, POI 9 dead: a round that accepts none ends the frame
    assert list(rec[0]) == [1, 0, 0] and left[0] == 2
    assert list(rec[1]) == [1, 0, 0] and left[1] == 1  # POI 1 back in frame 1
    assert list(rec[2]) == [0, 0, 0] and left[2] == 2  # POI 2 occluded in frame 2
    assert list(rec[3]) == [1, 0, 0] and left[3] == 1


def test_max_rounds_0_is_the_plain_series():
    q = seeds(20, occluded=[(1, 0), (2, 2), (7, 1)], dead=[9], failed=[12, 13])
    out, rec, left = loop(q, 5, 0)
    assert same(out, plain(q, 5))
    assert rec.shape == (5, 0)
    zc, cc = ZC, CC
    assert list(left) == [int(((out[f, :, zc] < LOW) | (out[f, :, cc] > CONV)).sum()) for f in range(5)]


@pytest.mark.parametrize("rounds", [0, 1, 2, 20])
def test_frame_inner_schedule_equals_the_loop(rounds):
    rng = np.random.default_rng(rounds)
    for trial in range(40):
        n, n_frames = int(rng.integers(1, 30)), int(rng.integers(1, 7))
        occ = [(int(i), int(rng.integers(0, n_frames))) for i in rng.choice(n, int(rng.integers(0, n)), replace=False)]
        dead = rng.choice(n, int(rng.integers(0, max(1, n // 4))), replace=False)
        failed = rng.choice(n, int(rng.integers(0, max(1, n // 4))), replace=False)
        q = seeds(n, occ, dead, failed)
        a = loop(q, n_frames, rounds)
        b = inner(q, n_frames, rounds)
        assert same(a[0], b[0]), trial
        assert np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2]), (trial, a[1:], b[1:])
