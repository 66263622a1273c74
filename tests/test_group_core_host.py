"""The grouping rule of the grouped camera call (libcimbar_b200/csrc/combine_core.cuh: agree, match, the packed-symbol count of
k_pair_match and the assignment k_assign_groups runs) compiled for the host (tests/cpp/group_core_host.cpp) and checked against the
numpy restatement of include/cb200.h in tests/group_fixtures.py; then the rule on the oracle's cells of the sample photographs and
of synthetic captures of distinct frames, which must group by frame."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from group_fixtures import assign

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("group_core") / "group_core_host.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-shared", "-fPIC", "-o", so, os.path.join(ROOT, "tests", "cpp", "group_core_host.cpp")])
    L = C.CDLL(so)
    L.gc_agree.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    L.gc_agree_packed.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    L.gc_match.argtypes = [C.c_int, C.c_int]
    L.gc_assign.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    return L


@pytest.mark.parametrize("seed", range(6))
def test_agree_counts_equal_symbol_bits_only(lib, seed):
    rng = np.random.default_rng(seed)
    for cells in (8, 5376, 8592, 12400):
        a = rng.integers(0, 256, cells, dtype=np.uint8)
        b = a.copy()
        flip = rng.random(cells) < rng.uniform(0, 1)
        b[flip] = rng.integers(0, 16, int(flip.sum()), dtype=np.uint8)            # other symbols on some cells
        b ^= (rng.integers(0, 16, cells, dtype=np.uint8) << 4)                      # colour bits and bit 7 differ everywhere
        for bits in (4, 3, 2):
            want = int((((a ^ b) & ((1 << bits) - 1)) == 0).sum())
            assert lib.gc_agree(a.ctypes.data, b.ctypes.data, cells, bits) == want, (cells, bits)
            assert lib.gc_agree_packed(a.ctypes.data, b.ctypes.data, cells, bits) == want, (cells, bits)


def test_match_is_half_the_cells_or_more(lib):
    assert [lib.gc_match(a, 12400) for a in (0, 6199, 6200, 12400)] == [0, 0, 1, 1]
    assert [lib.gc_match(a, 5) for a in (2, 3)] == [0, 1]


def rows_of(match):
    """the match rows as the device stores them: row i, bit j of word j / 32; the bits from j = i on are set at random, unread"""
    n = len(match)
    words = max(1, (n + 31) // 32)
    rng = np.random.default_rng(n)
    rows = np.zeros((n, words), np.uint32)
    for i in range(n):
        for j in range(n):
            if (match[i][j] if j < i else rng.random() < 0.5):
                rows[i, j // 32] |= np.uint32(1 << (j % 32))
    return rows, words


def run(lib, match, status):
    n = len(status)
    rows, words = rows_of(match)
    status = np.ascontiguousarray(status, np.int32)
    slots = n // 2
    of = np.full(max(n, 1), -7, np.int32)
    offsets = np.full(slots + 1, -7, np.int32)
    members = np.full(max(n, 1), -7, np.int32)
    count = lib.gc_assign(rows.ctypes.data, words, status.ctypes.data, n, slots, of.ctypes.data, offsets.ctypes.data, members.ctypes.data)
    return of[:n].tolist(), count, offsets, members[:offsets[slots]]


@pytest.mark.parametrize("density", [0.0, 0.02, 0.2, 0.6, 1.0])
@pytest.mark.parametrize("seed", range(3))
def test_assignment_equals_the_rule(lib, seed, density):
    rng = np.random.default_rng([seed, int(density * 100)])
    for n in (0, 1, 2, 31, 32, 33, 97, int(rng.integers(100, 320))):
        m = rng.random((n, n)) < density
        m = m | m.T
        status = rng.choice([-1, 0, 1, 2, 3], n, p=[0.05, 0.1, 0.4, 0.4, 0.05]).astype(np.int32)
        elig = np.isin(status, (1, 2))
        m &= elig[:, None] & elig[None, :]
        want_of, want_count = assign(m, elig)
        of, count, offsets, members = run(lib, m, status)
        assert (of, count) == (want_of, want_count), (seed, density, n)
        want_members = [i for g in range(count) for i in range(n) if of[i] == g]
        assert members.tolist() == want_members
        sizes = [of.count(g) for g in range(count)]
        assert offsets.tolist() == [0] + np.cumsum(sizes).tolist() + [len(want_members)] * (n // 2 - count)
        assert all(2 <= s <= 16 for s in sizes)


def test_ineligible_pictures_and_singletons(lib):
    n = 6
    m = np.ones((n, n), bool)
    status = [1, 0, -2, 2, 3, 1]                      # 1, 2 and 3 do not take part, whatever their match bits say
    of, count, _, _ = run(lib, m, status)
    assert (of, count) == ([0, -1, -1, 0, -1, 0], 1)
    of, count, _, _ = run(lib, np.zeros((n, n), bool), [1] * n)
    assert (of, count) == ([-1] * n, 0)              # every picture alone: no group
    m = np.zeros((4, 4), bool)
    m[3, 1] = m[1, 3] = True
    assert run(lib, m, [2, 2, 2, 2])[:2] == ([-1, 0, -1, 0], 1)


def test_the_cap_of_sixteen(lib):
    of, count, offsets, members = run(lib, np.ones((40, 40), bool), [1] * 40)
    assert count == 3 and [of.count(g) for g in range(3)] == [16, 16, 8]
    assert of == [0] * 16 + [1] * 16 + [2] * 8
    assert offsets.tolist() == [0, 16, 32, 40] + [40] * 17
    of, count, offsets, members = run(lib, np.ones((18, 18), bool), [2] * 18)
    assert count == 2 and of == [0] * 16 + [1] * 2
    assert members.tolist() == list(range(18)) and offsets.tolist() == [0, 16, 18] + [18] * 7


def test_a_full_group_leaves_later_pictures_to_the_next_leader(lib):
    """picture 17 matches leader 0 (full) and leader 16: it joins 16, which leads because it matched no open leader"""
    n = 18
    m = np.zeros((n, n), bool)
    m[:16, :16] = True
    m[16, :16] = m[:16, 16] = True
    m[17, 0] = m[0, 17] = m[17, 16] = m[16, 17] = True
    of, count, _, _ = run(lib, m, [1] * n)
    assert of == [0] * 16 + [1, 1] and count == 2


# ---- the rule on the oracle's cells

def per_picture(mode_val, pics):
    from combine_fixtures import picture_cells
    return [picture_cells(mode_val, p) for p in pics]


def golden(name):
    import cv2
    return cv2.cvtColor(cv2.imread(os.path.join(ROOT, "tests", "golden", name.replace("/", "__"))), cv2.COLOR_BGR2RGB)


def test_the_sample_photographs_group_by_frame():
    from group_fixtures import rule_groups
    names = ["6bit/4_30_f0_627.jpg", "6bit/4_30_f0_177_ccm.jpg", "6bit/4_30_f1_360.jpg", "6bit/4_30_f2_246.jpg", "6bit/4_30_f2_734.jpg",
             "6bit/4_30_802.jpg"]
    of, count = rule_groups(4, per_picture(4, [golden(nm) for nm in names]))
    assert (of, count) == ([0, 0, -1, 1, 1, -1], 2)


def test_the_mode_b_photographs_form_one_group():
    from group_fixtures import rule_groups
    of, count = rule_groups(68, per_picture(68, [golden("b/ex2434.jpg"), golden("b/ex380.jpg")]))
    assert (of, count) == ([0, 0], 1)


@pytest.mark.parametrize("mode_val", [68, 4])
def test_captures_of_seeded_frames_group_by_frame(mode_val):
    from group_fixtures import frame_captures, rule_groups
    pics, frame_of = frame_captures(mode_val, [3, 2, 2, 3], seed=3)
    order = np.random.default_rng(mode_val).permutation(len(pics))
    per = per_picture(mode_val, [pics[i] for i in order])
    assert all(p[0] in (1, 2) for p in per)
    of, count = rule_groups(mode_val, per)
    frames = [frame_of[i] for i in order]
    assert count == 4
    for a in range(len(of)):
        for b in range(len(of)):
            assert (of[a] == of[b]) == (frames[a] == frames[b]), (a, b)
