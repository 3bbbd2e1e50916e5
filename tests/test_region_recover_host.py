"""CPU: the bookkeeping of the recovery witness (tests/region_recover_cases.py witness_loop) against a plain restatement of the
reference example's loop (example_loop), with stub fit and registration functions.

The stubs make a POI's fate a schedule: the fit writes the reliable set's size into u (so the fit sees the set the round
reads), and the registration counts the POI's trials in eyy and passes it (zncc 0.95, convergence 0) once it has had `need`
trials (exx), else fails it (zncc 0.3).  Where no two POIs adjacent in the unreliable list pass in the same round, the two loops
agree byte for byte.  Where two do, the example skips the second for that round and registers it once more: the one documented
difference."""
import numpy as np
import pytest

import region_recover_cases as rr

torch = pytest.importorskip("torch")
ZC, CC, NEED, TRIALS = 16, 18, 20, 21
CONV, HIGH, LOW = 0.001, 0.9, 0.5


def fit(rel, work):
    work[:, 2] = float(len(rel))
    work[:, ZC] = 0.0


def register(work):
    work[:, TRIALS] += 1
    ok = work[:, TRIALS] >= work[:, NEED]
    work[:, ZC] = 0.3
    work[:, CC] = 0.0
    work[ok, ZC] = 0.95


def queue(kinds, need):
    """kinds: 'r' reliable, 'u' unreliable (low ZNCC), 'c' unreliable (convergence above conv), 'n' neither; need: trials to
    pass, per POI."""
    q = np.zeros((len(kinds), 25), np.float32)
    zncc = {"r": 0.95, "u": 0.2, "c": 0.95, "n": 0.7}
    for i, k in enumerate(kinds):
        q[i, ZC] = zncc[k]
        q[i, CC] = 0.5 if k == "c" else 0.0
        q[i, NEED] = need[i]
        q[i, 0] = i
    return q


def both(q, rounds):
    a = q.copy()
    ex, ex_left = rr.example_loop(a, fit, register, CONV, HIGH, LOW, rounds)
    b = torch.from_numpy(q.copy())
    wi, wi_left, _ = rr.witness_loop(b, fit, register, CONV, HIGH, LOW, rounds)
    return a, ex, ex_left, b.numpy(), wi, wi_left


def adjacent_accepts(q, rounds):
    """Does the example ever accept a POI and then find the POI it skipped passing too?"""
    u = [i for i in range(len(q)) if q[i, ZC] < LOW or q[i, CC] > CONV]
    trials = {i: 0 for i in u}
    for _ in range(rounds):
        for i in u:
            trials[i] += 1
        passing = [i for i in u if trials[i] >= q[i, NEED]]
        if not passing:
            return False
        if any(u[j] in passing and u[j + 1] in passing for j in range(len(u) - 1)):
            return True
        u = [i for i in u if i not in passing]
        if not u:
            return False
    return False


def test_agrees_with_the_example_without_adjacent_accepts():
    rng = np.random.default_rng(0)
    checked = 0
    for trial in range(300):
        n = int(rng.integers(1, 40))
        kinds = rng.choice(list("rucn"), n, p=[0.4, 0.3, 0.15, 0.15])
        need = rng.integers(1, 8, n).astype(np.float32)
        rounds = int(rng.integers(0, 10))
        q = queue(kinds, need)
        if adjacent_accepts(q, rounds):
            continue
        a, ex, ex_left, b, wi, wi_left = both(q, rounds)
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), trial
        assert ex == wi and ex_left == wi_left, (trial, ex, wi)
        checked += 1
    assert checked > 100


def test_distinct_schedules_agree():
    """Every unreliable POI passes in a round of its own: never two accepts in one round."""
    kinds = list("rurcnuurcu")
    u = [i for i, k in enumerate(kinds) if k in "uc"]
    need = np.zeros(len(kinds), np.float32)
    passing = [i for i in u if i != u[2]]
    need[passing] = np.arange(1, len(passing) + 1)[::-1]
    need[u[2]] = 99  # never passes: the loop ends on a round that recovers none
    q = queue(kinds, need)
    a, ex, ex_left, b, wi, wi_left = both(q, 12)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    assert ex == wi and ex_left == wi_left == 1
    assert wi[:len(u)].count(1) == len(u) - 1
    # the POI never accepted keeps the bytes it came in with; reliable and neither POIs are never written
    keep = [u[2]] + [i for i, k in enumerate(kinds) if k in "rn"]
    assert np.array_equal(b[keep].view(np.uint32), q[keep].view(np.uint32))


def test_adjacent_accepts_are_the_documented_difference():
    """Two adjacent unreliable POIs that both pass in round 1: the example accepts the first, skips the second, registers it
    again in round 2 and accepts it there with a second trial; the call accepts both in round 1."""
    q = queue(list("ruur"), [0, 1, 1, 0])
    a, ex, ex_left, b, wi, wi_left = both(q, 5)
    assert wi == [2, 0, 0, 0, 0] and wi_left == 0
    assert ex == [1, 1, 0, 0, 0] and ex_left == 0
    assert b[1, TRIALS] == b[2, TRIALS] == 1
    assert a[1, TRIALS] == 1 and a[2, TRIALS] == 2
    assert a[2, 2] == 3 and b[2, 2] == 2  # the example's second fit saw the reliable set grown by the first accept


def test_classification_literal_comparisons():
    """NaN fails every comparison: a NaN ZNCC is unreliable only through its convergence, a NaN convergence leaves a POI
    reliable when its ZNCC is high (no convergence test for R), and neither set is ever written."""
    q = queue(list("rrrr"), [1, 1, 1, 1])
    q[0, ZC] = np.nan                 # neither
    q[1, ZC], q[1, CC] = np.nan, 1.0  # unreliable through its convergence
    q[2, CC] = np.nan                 # reliable
    q[3, ZC] = 0.5                    # not < 0.5 and below 0.9: neither
    b = torch.from_numpy(q.copy())
    wi, left, rounds = rr.witness_loop(b, fit, register, CONV, HIGH, LOW, 3)
    assert wi == [1, 0, 0] and left == 0 and rounds == 1
    assert b[1, 2] == 1  # the fit saw one reliable POI: POI 2
    keep = [0, 2, 3]
    assert np.array_equal(b.numpy()[keep].view(np.uint32), q[keep].view(np.uint32))
