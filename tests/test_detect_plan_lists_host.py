"""The per-slot rule of a detect receivers plan's lists (libcimbar_b200/csrc/receivers_core.cuh: plan_slot, run on the device by
k_detect_plan_lists), compiled for the CPU and compared with the direct call's host builder (detect_lists, also compiled for the CPU)
on random candidate masks and receiver maps of up to 3 000 slots, with empty slots of both kinds (no candidate bit below n_modes,
a receiver outside [0, receivers)), high candidate bits and out-of-range receivers:
  - a slot is empty exactly when its receiver is out of range or its candidates have no bit below n_modes; an empty slot has no
    mode, is present in no geometry and has position -1 everywhere;
  - for every geometry g, its present slots are the direct call's sub-batch U_g over the non-empty slots alone;
  - compacted over those slots, each mode's raw receivers are the first half of detect_lists' map, and make_order of them is its
    second half (the plan's k_receivers_order builds that order; tests/test_receivers_order_host.py checks it against make_order);
  - each position at[k][i] is i or -1, and its rank among geometry g's present slots is detect_lists' position."""
import os
import subprocess

import numpy as np
import pytest
from cpu_support import run

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INT_MIN, INT_MAX = -2 ** 31, 2 ** 31 - 1


@pytest.fixture(scope="module")
def exes(tmp_path_factory):
    d = tmp_path_factory.mktemp("detect_plan_lists")
    out = {}
    for name in ("detect_plan_lists_host", "detect_lists_host"):
        out[name] = str(d / name)
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-o", out[name], os.path.join(ROOT, "tests", "cpp", name + ".cpp")])
    return out


def plan_lists(exe, cand, of, receivers, group):
    n, k, ng = len(cand), len(group), max(group) + 1
    data = np.concatenate([np.array([n, receivers, k, ng], np.int32), np.asarray(group, np.int32), np.asarray(cand, np.uint32).view(np.int32),
                           np.asarray(of, np.int32)]).tobytes()
    out = subprocess.run([exe], input=data, stdout=subprocess.PIPE, check=True).stdout
    words = np.frombuffer(out[:8 * k * n], np.int32)
    present = np.frombuffer(out[8 * k * n:], np.uint8)
    assert len(present) == ng * n
    return words[:k * n].reshape(k, n), words[k * n:].reshape(k, n), present.reshape(ng, n)


def direct_lists(exe, cand, of, receivers, group):
    """detect_lists over these (non-empty) pictures: (U_g per geometry, counts, maps, positions)"""
    return run(exe, cand, of, receivers, group)


def make_order(of):
    return np.argsort(np.asarray(of, np.int64), kind="stable").astype(np.int32)


def check(exes, cand, of, receivers, group):
    cand = np.asarray(cand, np.int64).astype(np.uint32)
    of = np.asarray(of, np.int64).astype(np.int32)
    n, K, ng = len(cand), len(group), max(group) + 1
    raw, at, present = plan_lists(exes["detect_plan_lists_host"], cand, of, receivers, group)
    low = cand & np.uint32((1 << K) - 1)
    full = np.flatnonzero((of >= 0) & (of < receivers) & (low != 0))           # the non-empty slots
    empty = np.setdiff1d(np.arange(n), full)
    assert (raw[:, empty] == -1).all() and (at[:, empty] == -1).all() and not present[:, empty].any()
    assert set(np.unique(present)) <= {0, 1}
    if not len(full):
        return
    slots, counts, maps, pos = direct_lists(exes["detect_lists_host"], low[full], of[full], receivers, group)
    for g in range(ng):
        assert np.array_equal(np.flatnonzero(present[g]), full[slots[g]]), g       # U_g, over the non-empty slots
    for k in range(K):
        g = group[k]
        u = np.flatnonzero(present[g])
        mine = raw[k, u]
        assert counts[k] == int((mine >= 0).sum()), k
        if counts[k]:
            m = len(u)
            assert np.array_equal(mine, maps[k][:m]), k
            assert np.array_equal(make_order(np.where(mine < 0, receivers, mine)), maps[k][m:]), k
        else:
            assert len(maps[k]) == 0 and (mine == -1).all(), k
        inside = at[k] >= 0
        assert np.array_equal(at[k][inside], np.flatnonzero(inside)), k            # identity positions
        rank = np.full(n, -1, np.int32)
        rank[u] = np.arange(len(u))
        want = np.full(n, -1, np.int32)
        want[full] = pos[k]
        assert np.array_equal(np.where(inside, rank, -1), want), k


GROUPS = {"one": [0], "one-geometry": [0, 0, 0], "recv": [0, 1, 2, 1], "five": [0, 1, 1, 2, 0]}


@pytest.mark.parametrize("grouping", list(GROUPS))
@pytest.mark.parametrize("n,receivers", [(1, 1), (7, 3), (64, 16), (257, 64), (3000, 40)])
def test_random_patterns(exes, grouping, n, receivers):
    group = GROUPS[grouping]
    K = len(group)
    rng = np.random.default_rng(n * 11 + receivers + K)
    # any candidate pattern, high bits and zero included, and receivers partly out of range
    cand = rng.integers(0, 1 << min(K + 3, 31), n)
    of = rng.integers(-3, receivers + 3, n)
    check(exes, cand, of, receivers, group)
    # sessions: locked receivers pass one bit, auto ones every bit; a few empty slots of each kind
    locked = rng.integers(0, K, receivers)
    auto = rng.random(receivers) < 0.2
    of = rng.integers(0, receivers, n)
    cand = np.where(auto[of], (1 << K) - 1, 1 << locked[of])
    cand[rng.random(n) < 0.1] = 0
    cand[rng.random(n) < 0.05] |= 1 << 31
    hole = rng.random(n) < 0.1
    of[hole] = rng.choice([-1, receivers, INT_MIN, INT_MAX], int(hole.sum()))
    check(exes, cand, of, receivers, group)
    check(exes, np.full(n, (1 << K) - 1), of, receivers, group)                # every mode (candidates = NULL)


def test_all_empty_and_only_high_bits(exes):
    n, group = 100, [0, 1, 2, 1]
    rng = np.random.default_rng(1)
    of = rng.integers(0, 5, n)
    check(exes, np.full(n, 1 << 4), of, 5, group)                             # bits at or above n_modes only: every slot empty
    check(exes, np.full(n, 0xFFFFFFF0), of, 5, group)
    check(exes, np.full(n, 0b1111), np.full(n, -1), 5, group)                  # every receiver out of range
    check(exes, np.full(n, 0b1111), np.full(n, INT_MAX), 5, group)


def test_a_geometry_or_mode_without_slots(exes):
    n, receivers, group = 500, 20, [0, 1, 2, 1]
    rng = np.random.default_rng(3)
    of = rng.integers(0, receivers, n)
    check(exes, np.full(n, 1 << 1), of, receivers, group)                      # one mode: geometries 0 and 2 absent everywhere
    check(exes, np.full(n, 0b1010), of, receivers, group)
    check(exes, rng.choice([0b0001, 0b0100, 0, 0b10000], n), of, receivers, group)
