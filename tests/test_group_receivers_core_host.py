"""The receivers form of the grouping rule (cb200_scan_extract_decode_chunks_grouped_receivers_dev; libcimbar_b200/csrc/combine_core.cuh:
pair_tiles, segment_starts, assign_segment and the numbering that k_pair_match and k_assign_groups run) compiled for the host
(tests/cpp/group_receivers_core_host.cpp) and checked against a numpy restatement: group_fixtures.assign applied to each receiver's
pictures alone, with the leaders numbered in batch order across the receivers.  The match rows are given by position of the
receiver-major order, with random bits wherever two receivers meet: the assignment must never read them."""
import ctypes as C

import numpy as np
import pytest

from group_fixtures import assign
from host_harness import build_harness

TILE = 64


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    L = build_harness(tmp_path_factory, "group_receivers_core_host")
    L.grc_order.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    L.grc_tiles.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int]
    L.grc_assign.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                             C.c_void_p]
    return L


def receiver_map(rng, n, kind):
    if kind == "one":
        return np.zeros(n, np.int32), 1
    if kind == "every":
        return rng.permutation(n).astype(np.int32), max(n, 1)
    k = int(rng.integers(2, 8))
    return rng.integers(0, k, n).astype(np.int32), k + int(rng.integers(0, 3))       # some receivers without a picture


def order_of(lib, of, receivers):
    order = np.zeros(max(len(of), 1), np.int32)
    lib.grc_order(of.ctypes.data, len(of), receivers, order.ctypes.data)
    return order[:len(of)]


def position_rows(match, of, order, rng):
    """row p, bit q = match(order[p], order[q]) where both have one receiver, random bits elsewhere (and from q = p on)"""
    n = len(of)
    words = max(1, (n + 31) // 32)
    m = match[np.ix_(order, order)]
    same = of[order][:, None] == of[order][None, :]
    lower = np.tril(np.ones((n, n), bool), -1)
    bits = np.where(same & lower, m, rng.random((n, n)) < 0.5)
    padded = np.zeros((n, 32 * words), bool)
    padded[:, :n] = bits
    return np.ascontiguousarray(np.packbits(padded, axis=1, bitorder="little").view(np.uint32)), words


def expected(match, status, of):
    """group_fixtures.assign on each receiver's pictures, leaders numbered in batch order: (group_of, count, receiver of each group)"""
    n = len(of)
    elig = np.isin(status, (1, 2))
    local = np.full(n, -1)
    leaders = []                                           # (leader's batch index, receiver, local group)
    for r in np.unique(of):
        idx = np.flatnonzero(of == r)
        sub, _ = assign(match[np.ix_(idx, idx)], elig[idx])
        for k, g in enumerate(sub):
            if g >= 0:
                local[idx[k]] = g
        for g in range(max(sub, default=-1) + 1):
            leaders.append((int(idx[sub.index(g)]), int(r), g))
    leaders.sort()
    number = {(r, g): k for k, (_, r, g) in enumerate(leaders)}
    group_of = [number[(int(of[i]), int(local[i]))] if local[i] >= 0 else -1 for i in range(n)]
    return group_of, len(leaders), [r for _, r, _ in leaders]


def run(lib, rows, words, status, of, receivers):
    n = len(of)
    slots = n // 2
    group_of = np.full(max(n, 1), -7, np.int32)
    offsets = np.full(slots + 1, -7, np.int32)
    members = np.full(max(n, 1), -7, np.int32)
    grec = np.full(max(slots, 1), -7, np.int32)
    status = np.ascontiguousarray(status, np.int32)
    count = lib.grc_assign(rows.ctypes.data, words, status.ctypes.data, of.ctypes.data, n, receivers, slots, group_of.ctypes.data,
                           offsets.ctypes.data, members.ctypes.data, grec.ctypes.data)
    return group_of[:n].tolist(), count, offsets, members[:offsets[slots]], grec[:slots].tolist()


@pytest.mark.parametrize("kind", ["one", "few", "every"])
@pytest.mark.parametrize("seed", range(3))
def test_assignment_equals_the_rule_per_receiver(lib, seed, kind):
    rng = np.random.default_rng([seed, len(kind)])
    sizes = [0, 1, 2, 33, 97, int(rng.integers(100, 700))] + ([1024, 4096] if kind != "one" else [1024])
    for n in sizes:
        of, receivers = receiver_map(rng, n, kind)
        density = float(rng.choice([0.0, 0.05, 0.3, 1.0]))
        m = rng.random((n, n)) < density
        m = m | m.T
        status = rng.choice([-4, -1, 0, 1, 2, 3], n, p=[0.03, 0.05, 0.1, 0.4, 0.4, 0.02]).astype(np.int32)
        elig = np.isin(status, (1, 2))
        m &= elig[:, None] & elig[None, :]
        order = order_of(lib, of, receivers)
        assert order.tolist() == np.argsort(of, kind="stable").tolist()
        rows, words = position_rows(m, of, order, rng)
        want_of, want_count, want_receivers = expected(m, status, of)
        group_of, count, offsets, members, grec = run(lib, rows, words, status, of, receivers)
        assert (group_of, count) == (want_of, want_count), (seed, kind, n, density)
        want_members = [i for g in range(count) for i in range(n) if group_of[i] == g]
        assert members.tolist() == want_members
        sizes_g = [group_of.count(g) for g in range(count)]
        assert offsets.tolist() == [0] + np.cumsum(sizes_g).tolist() + [len(want_members)] * (n // 2 - count)
        assert grec == want_receivers + [-1] * (n // 2 - count)
        assert all(len({int(of[i]) for i in range(n) if group_of[i] == g}) == 1 for g in range(count))


def test_one_frame_in_two_receivers_forms_two_groups(lib):
    n = 8
    of = np.array([0, 1, 0, 1, 0, 1, 0, 1], np.int32)      # every picture shows one frame, alternately held by two receivers
    m = np.ones((n, n), bool)
    order = order_of(lib, of, 2)
    rows, words = position_rows(m, of, order, np.random.default_rng(1))
    group_of, count, offsets, members, grec = run(lib, rows, words, [1] * n, of, 2)
    assert (group_of, count) == ([0, 1] * 4, 2)
    assert members.tolist() == [0, 2, 4, 6, 1, 3, 5, 7] and grec == [0, 1, -1, -1]


def test_the_cap_applies_per_receiver(lib):
    of = np.array([1] * 20 + [0] * 18, np.int32)
    n = len(of)
    order = order_of(lib, of, 2)
    rows, words = position_rows(np.ones((n, n), bool), of, order, np.random.default_rng(2))
    group_of, count, _, _, grec = run(lib, rows, words, [2] * n, of, 2)
    assert count == 4 and group_of == [0] * 16 + [1] * 4 + [2] * 16 + [3] * 2
    assert grec[:4] == [1, 1, 0, 0]


def pair_tiles_by_brute_force(of, order):
    n = len(of)
    want = set()
    pos_of = of[order]
    s = 0
    while s < n:
        e = s + 1
        while e < n and pos_of[e] == pos_of[s]:
            e += 1
        if e - s >= 2:
            p, q = np.tril_indices(e - s, -1)
            t = np.unique(((p + s) // TILE) * 65536 + (q + s) // TILE)
            want.update((int(k) // 65536, int(k) % 65536) for k in t)
        s = e
    return want


@pytest.mark.parametrize("kind", ["one", "few", "every"])
@pytest.mark.parametrize("seed", range(3))
def test_tile_pairs_cover_every_same_receiver_pair_once(lib, seed, kind):
    rng = np.random.default_rng([seed, 7, len(kind)])
    for n in (0, 1, 2, 63, 64, 65, 130, int(rng.integers(200, 1500)), 4096):
        of, receivers = receiver_map(rng, n, kind)
        if kind == "few" and n > 100 and seed == 2:
            of = np.repeat(np.arange(n // 40, dtype=np.int32), 40)[:n]                  # runs that start inside tiles
            of = np.concatenate([of, np.full(n - len(of), n // 40, np.int32)])
            receivers = n // 40 + 1
            rng.shuffle(of)
        order = order_of(lib, of, receivers)
        cap = 1 + ((n + TILE - 1) // TILE) ** 2
        ij = np.zeros((cap, 2), np.int32)
        k = lib.grc_tiles(of.ctypes.data, n, receivers, TILE, ij.ctypes.data, cap)
        got = [tuple(map(int, t)) for t in ij[:k]]
        assert got == sorted(set(got)), "each tile pair once, in (I, J) order"
        assert all(J <= I for I, J in got)
        assert set(got) == pair_tiles_by_brute_force(of, order), (seed, kind, n)
        if kind == "every":
            assert k == 0


def test_tile_pairs_follow_the_sum_of_squares(lib):
    """64 receivers of 16 pictures each, interleaved in batch order: the 16 diagonal tiles, not the 136 tile pairs of one receiver's
    1024 pictures"""
    of = np.tile(np.arange(64, dtype=np.int32), 16)
    ij = np.zeros((200, 2), np.int32)
    assert lib.grc_tiles(of.ctypes.data, len(of), 64, TILE, ij.ctypes.data, 200) == 16
    assert [tuple(t) for t in ij[:16].tolist()] == [(k, k) for k in range(16)]
    one = np.zeros(1024, np.int32)
    assert lib.grc_tiles(one.ctypes.data, 1024, 1, TILE, ij.ctypes.data, 200) == 136
