"""The host builder of a detect receivers call's lists (libcimbar_b200/csrc/receivers_core.cuh: detect_lists), compiled for the CPU
and compared with a plain model on random candidate patterns, geometry groupings and receiver maps of up to 20 000 pictures:
  - U_g, the sub-batch of geometry g, is the batch-ordered union of P_k over its modes (P_k: the pictures with candidate bit k);
  - picture i's position under mode k is its index in U_g when i is in P_k, else -1;
  - mode k's map gives each position of U_g its receiver, -1 (an empty slot) where the picture is not in P_k;
  - its order lists the non-empty positions first, and those are make_order over P_k (the direct receivers call's order); the empty
    positions follow, in batch order."""
import os
import subprocess

import numpy as np
import pytest
from cpu_support import run

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("detect_lists") / "detect_lists_host")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-o", path, os.path.join(ROOT, "tests", "cpp", "detect_lists_host.cpp")])
    return path


def model_order(of, receivers):
    """make_order: a stable counting sort by receiver"""
    return np.argsort(np.asarray(of, np.int64), kind="stable").astype(np.int32)


def check(exe, cand, of, receivers, group):
    cand = np.asarray(cand, np.uint32)
    of = np.asarray(of, np.int32)
    n, K = len(cand), len(group)
    slots, counts, maps, pos = run(exe, cand, of, receivers, group)
    for g in range(K):
        modes = [k for k in range(K) if group[k] == g]
        bits = np.uint32(sum(1 << k for k in modes))
        assert np.array_equal(slots[g], np.flatnonzero(cand & bits)), g           # U_g in batch order
    for k in range(K):
        P = np.flatnonzero(cand >> np.uint32(k) & np.uint32(1))
        u = slots[group[k]]
        assert counts[k] == len(P), k
        want_pos = np.full(n, -1, np.int32)
        want_pos[u] = np.arange(len(u))
        want_pos[np.setdiff1d(np.arange(n), P)] = -1
        assert np.array_equal(pos[k], want_pos), k
        if not len(P):
            assert len(maps[k]) == 0, k                    # a mode without pictures builds nothing
            continue
        m = len(u)
        rec, order = maps[k][:m], maps[k][m:]
        inside = np.isin(u, P)
        assert np.array_equal(rec, np.where(inside, of[u], -1)), k
        assert np.array_equal(u[order[:len(P)]], P[model_order(of[P], receivers)]), k     # make_order over P_k
        assert np.array_equal(order[len(P):], np.flatnonzero(~inside)), k                 # empties last, in batch order
        assert np.array_equal(np.sort(order), np.arange(m)), k


GROUPS = {"one": [0], "one-geometry": [0, 0, 0], "recv": [0, 1, 2, 1], "five": [0, 1, 1, 2, 0]}


@pytest.mark.parametrize("grouping", list(GROUPS))
@pytest.mark.parametrize("n,receivers", [(1, 1), (7, 3), (64, 16), (257, 64), (2000, 5), (20000, 1000)])
def test_random_patterns(exe, grouping, n, receivers):
    group = GROUPS[grouping]
    K = len(group)
    rng = np.random.default_rng(n * 7 + receivers + K)
    check(exe, rng.integers(1, 1 << K, n), rng.integers(0, receivers, n), receivers, group)
    # sessions: locked receivers pass one bit, auto ones every bit
    locked = rng.integers(0, K, receivers)
    auto = rng.random(receivers) < 0.1
    of = rng.integers(0, receivers, n)
    cand = np.where(auto[of], (1 << K) - 1, 1 << locked[of])
    check(exe, cand, of, receivers, group)


def test_a_mode_or_a_geometry_without_pictures(exe):
    rng = np.random.default_rng(3)
    n, receivers = 500, 20
    of = rng.integers(0, receivers, n)
    check(exe, np.full(n, 1 << 1), of, receivers, [0, 1, 2, 1])           # one mode: geometries 0 and 2 empty, mode 3 too
    check(exe, np.full(n, 0b1010), of, receivers, [0, 1, 2, 1])          # two modes of one geometry: no empty slots
    check(exe, rng.choice([0b0001, 0b0100], n), of, receivers, [0, 1, 2, 1])
    check(exe, np.full(n, 0b1111), of, receivers, [0, 1, 2, 1])          # every mode decodes every picture


def test_one_picture_per_receiver_and_huge_receiver_indices(exe):
    rng = np.random.default_rng(4)
    n = 3000
    check(exe, rng.integers(1, 16, n), rng.permutation(n), n, [0, 1, 2, 1])
    receivers = 10 ** 6
    check(exe, rng.integers(1, 8, n), rng.choice([0, 5, 2 ** 19, receivers - 1], n), receivers, [0, 0, 1])
