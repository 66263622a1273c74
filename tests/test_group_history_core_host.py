"""The history rule of the grouped history call (libcimbar_b200/csrc/combine_core.cuh: position statuses, the assignment over the
positions, the "at least one batch member" numbering, the done-group and keep rule and the last-H compaction) compiled for the host
(tests/cpp/group_history_core_host.cpp) and checked against the numpy restatement tests/history_fixtures.history_rule on random match
matrices, masks and capacities."""
import ctypes as C

import numpy as np
import pytest

from history_fixtures import history_rule
from host_harness import build_harness


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    L = build_harness(tmp_path_factory, "group_history_core_host")
    L.gh_rule.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                          C.c_void_p, C.c_void_p]
    L.gh_complete.argtypes = [C.c_uint32, C.c_int]
    L.gh_destination.argtypes = [C.c_int, C.c_int, C.c_int]
    return L


def device_rows(match, H, h, rng):
    """the match rows over the device's positions: history picture q at slot q, empty slots h .. H, batch picture i at H + i; the
    bits of pairs with an empty slot and from j = i on are random (the rule never reads them)"""
    n = len(match) - h
    N = H + n
    where = list(range(h)) + [H + i for i in range(n)]
    words = max(1, (N + 31) // 32)
    bits = rng.random((N, N)) < 0.5
    for a, pa in enumerate(where):
        for b, pb in enumerate(where):
            if pb < pa:
                bits[pa, pb] = match[a][b]
    rows = np.zeros((N, words), np.uint32)
    for i in range(N):
        for j in np.flatnonzero(bits[i]):
            rows[i, j // 32] |= np.uint32(1 << (j % 32))
    return rows, words, where


def check(lib, rng, H, h, n, density, cpf, frames=None):
    N = h + n
    if frames is None:
        m = rng.random((N, N)) < density
    else:                                            # pictures of a few frames: every picture matches its frame's others
        f = rng.integers(0, frames, N)
        m = (f[:, None] == f[None, :]) & (rng.random((N, N)) < 1 - density)
    m = m | m.T
    status = rng.choice([-1, 0, 1, 2, 3], n, p=[0.05, 0.15, 0.4, 0.35, 0.05]).astype(np.int32)
    full = (1 << cpf) - 1 if cpf < 32 else 0xFFFFFFFF
    pick = lambda k: np.where(rng.random(k) < 0.3, full, rng.integers(0, full, k, dtype=np.uint64) & full).astype(np.uint32)
    own, gmask = pick(max(n, 1)), pick(max(n, 1))
    want_of, want_count, groups, kept = history_rule(m, h, np.isin(status, (1, 2)), own[:n] == full,
                                                     lambda g, members: gmask[g] == full, H)
    rows, words, where = device_rows(m, H, h, rng)
    of = np.full(max(n, 1), -7, np.int32)
    pos_group = np.full(H + n, -7, np.int32)
    src = np.full(H, -7, np.int32)
    r = lib.gh_rule(rows.ctypes.data, words, H, h, status.ctypes.data, n, own.ctypes.data, gmask.ctypes.data, cpf, of.ctypes.data,
                    pos_group.ctypes.data, src.ctypes.data)
    count, new_h = r >> 16, r & 0xFFFF
    assert (of[:n].tolist(), count) == (want_of, want_count), (H, h, n)
    for g, members in enumerate(groups):
        assert [p for p in range(H + n) if pos_group[p] == g] == [where[q] for q in members]
    assert src[:new_h].tolist() == [where[q] for q in kept], (H, h, n)
    return count, len(kept), max((len(g) for g in groups), default=0)


@pytest.mark.parametrize("seed", range(8))
def test_rule_equals_the_restatement(lib, seed):
    rng = np.random.default_rng(seed)
    seen_cut = False
    for _ in range(40):
        H = int(rng.choice([1, 2, 3, 8, 31, 32, 33, 64, 256]))
        h = int(rng.integers(0, H + 1))
        n = int(rng.choice([0, 1, 2, 5, 17, int(rng.integers(30, 90))]))
        cpf = int(rng.choice([1, 7, 10, 31, 32]))
        _, kept, _ = check(lib, rng, H, h, n, float(rng.choice([0.0, 0.05, 0.3, 0.9])), cpf,
                           frames=int(rng.integers(1, 6)) if rng.random() < 0.5 else None)
        seen_cut |= kept > 0 and kept == H
    assert seen_cut                                  # premise: more survivors than the capacity in some case


def test_groups_capped_at_sixteen_and_h_below_the_survivors(lib):
    rng = np.random.default_rng(99)
    """one frame: every eligible picture matches every other, so groups fill to 16; the survivors outnumber H"""
    for H, h, n in ((2, 2, 30), (8, 8, 40), (20, 10, 25), (256, 200, 60)):
        _, kept, biggest = check(lib, rng, H, h, n, 0.0, 10, frames=1)
        assert biggest == 16


def test_complete_and_destination(lib):
    assert [lib.gh_complete(m, 7) for m in (0x7F, 0x3F, 0xFF)] == [1, 0, 0]
    assert lib.gh_complete(0xFFFFFFFF, 32) == 1 and lib.gh_complete(0x7FFFFFFF, 32) == 0
    assert [lib.gh_destination(r, 5, 2) for r in range(5)] == [-3, -2, -1, 0, 1]
    assert [lib.gh_destination(r, 2, 4) for r in range(2)] == [0, 1]
