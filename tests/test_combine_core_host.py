"""The combined call's per-cell vote and group table (libcimbar_b200/csrc/combine_core.cuh, run on the device by k_combine) compiled
for the host (tests/cpp/combine_core_host.cpp) and checked against a literal numpy restatement of the rule in include/cb200.h:
(1) the value most participating pictures hold, (2) among values tied on count the one with the smallest walk distance among its
pictures, (3) the value of the earliest picture.  The group table is a stable counting sort of group_of into CSR offsets."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("combine_core") / "combine_core_host.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-shared", "-fPIC", "-o", so, os.path.join(ROOT, "tests", "cpp", "combine_core_host.cpp")])
    L = C.CDLL(so)
    L.cc_vote.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    L.cc_takes_part.argtypes = [C.c_int32]
    L.cc_group_error.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_int)]
    L.cc_group_table.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    return L


def vote_rule(values, dists):
    """the rule, literally: one picture's value bits and distance per entry, in batch order"""
    values = [int(v) & 0x7F for v in values]
    cands = []
    for v in dict.fromkeys(values):                                # distinct values in order of first appearance
        mine = [i for i, x in enumerate(values) if x == v]
        cands.append((-len(mine), min(int(dists[i]) for i in mine), mine[0], v))
    return min(cands)[3]


def device_vote(lib, v, d):
    k, cells = v.shape
    v = np.ascontiguousarray(v, np.uint8)
    d = np.ascontiguousarray(d, np.uint8)
    out = np.zeros(cells, np.uint8)
    lib.cc_vote(v.ctypes.data, d.ctypes.data, k, cells, out.ctypes.data)
    return out


@pytest.mark.parametrize("seed", range(6))
def test_vote_matches_the_rule_on_random_groups(lib, seed):
    rng = np.random.default_rng(seed)
    assert lib.cc_max_group() == 16
    for k in range(1, 17):
        cells = 400
        # few distinct values and distances: many ties on count, on distance, and on both
        nv = int(rng.integers(1, 5))
        palette = rng.integers(0, 256, nv, dtype=np.uint8)
        v = palette[rng.integers(0, nv, (k, cells))]
        d = rng.integers(0, int(rng.integers(1, 4)), (k, cells), dtype=np.uint8)
        if seed % 2:                                               # bit 7 (K1's dirty marker) is not part of the value
            v = v | (rng.integers(0, 2, (k, cells), dtype=np.uint8) << 7)
        got = device_vote(lib, v, d)
        want = np.array([vote_rule(v[:, c], d[:, c]) for c in range(cells)], np.uint8)
        assert np.array_equal(got, want), (seed, k)


def test_vote_cases():
    assert vote_rule([5], [9]) == 5
    assert vote_rule([5, 6], [3, 2]) == 6                          # two pictures: the lower distance
    assert vote_rule([5, 6], [2, 2]) == 5                          # tied: the earlier picture
    assert vote_rule([5, 6, 6], [0, 9, 9]) == 6                    # a majority beats a better distance
    assert vote_rule([5, 6, 7, 6, 5], [4, 3, 0, 5, 4]) == 6        # 5 and 6 tied on count, 6 has the smaller distance


def test_vote_cases_on_the_device_rule(lib):
    for v, d, want in [([5], [9], 5), ([5, 6], [3, 2], 6), ([5, 6], [2, 2], 5), ([5, 6, 6], [0, 9, 9], 6),
                       ([5, 6, 7, 6, 5], [4, 3, 0, 5, 4], 6), ([0x85, 5], [1, 0], 5), ([0x80 | 3, 3, 4], [7, 7, 0], 3)]:
        got = device_vote(lib, np.array(v, np.uint8).reshape(-1, 1), np.array(d, np.uint8).reshape(-1, 1))
        assert int(got[0]) == want & 0x7F, (v, d)


def test_participating_statuses(lib):
    assert [lib.cc_takes_part(s) for s in (-4, -3, -2, -1, 0, 1, 2, 3)] == [0, 0, 0, 0, 0, 1, 1, 0]


def table(lib, of, m):
    of = np.ascontiguousarray(of, np.int32)
    offsets = np.full(m + 1, -7, np.int32)
    members = np.full(len(of) + 1, -7, np.int32)
    lib.cc_group_table(of.ctypes.data, len(of), m, offsets.ctypes.data, members.ctypes.data)
    return offsets, members[:offsets[m]], members[offsets[m]:]


def error(lib, of, m):
    of = np.ascontiguousarray(of, np.int32)
    at = C.c_int(-9)
    return lib.cc_group_error(of.ctypes.data, len(of), m, C.byref(at)), at.value


@pytest.mark.parametrize("seed", range(8))
def test_group_table_is_a_stable_sort(lib, seed):
    rng = np.random.default_rng(100 + seed)
    n = int(rng.integers(0, 200))
    m = int(rng.integers(1, 40))
    of = rng.integers(-1, m, n).astype(np.int32)
    if seed == 0:
        of[:] = -1                                                 # every picture outside the groups
    counts = np.bincount(of[of >= 0], minlength=m)
    assert error(lib, of, m)[0] == (2 if counts.max(initial=0) > 16 else 0)
    offsets, members, rest = table(lib, of, m)
    want = np.argsort(np.where(of < 0, m, of), kind="stable")[:int((of >= 0).sum())]
    assert np.array_equal(members, want)
    assert np.array_equal(offsets, np.concatenate([[0], np.cumsum(counts)]))
    assert (rest == -7).all()                                      # nothing written past the members
    for g in range(m):                                             # empty groups have empty ranges
        assert np.array_equal(members[offsets[g]:offsets[g + 1]], np.flatnonzero(of == g))


def test_group_table_without_groups(lib):
    offsets, members, _ = table(lib, [-1, -1, -1], 0)
    assert offsets.tolist() == [0] and len(members) == 0
    offsets, members, _ = table(lib, [], 3)
    assert offsets.tolist() == [0, 0, 0, 0] and len(members) == 0


def test_group_errors(lib):
    assert error(lib, [0, 1, -1], 2) == (0, -9)
    assert error(lib, [0, 2, -1], 2) == (1, 1)
    assert error(lib, [0, 1, -2], 2) == (1, 2)
    assert error(lib, [0], 0) == (1, 0)
    assert error(lib, [-1] * 5, 0) == (0, -9)
    assert error(lib, [3] * 16, 4) == (0, -9)                      # the cap itself
    assert error(lib, [3] * 17, 4) == (2, 16)                      # the 17th picture is named
    of = [0, 1] * 16 + [1, 0]
    assert error(lib, of, 2) == (2, 32)
    assert error(lib, [2 ** 31 - 1], 5) == (1, 0)
    assert error(lib, [-2 ** 31], 5) == (1, 0)
