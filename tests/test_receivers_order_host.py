"""The receiver map of a receivers camera plan (libcimbar_b200/csrc/receivers_core.cuh, built on the device at each launch by
k_receivers_order) compiled for the host and run as the kernel runs it (each slot's rank summed over 8 interleaved lanes).  On the
slots whose receiver lies in [0, receivers) the order must be make_order's stable receiver-major order (make_order itself, run on
the same receivers renumbered densely); the empty slots (receiver outside the range) follow in batch order, with map entry -1.
The rule allocates nothing: its work and memory depend on the number of slots, not on the number of receivers."""
import os
import subprocess

import numpy as np
import pytest

from host_harness import build_harness

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INT_MIN, INT_MAX = -2 ** 31, 2 ** 31 - 1


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("receivers_order") / "receivers_order_host")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-o", path, os.path.join(ROOT, "tests", "cpp", "receivers_order_host.cpp")])
    return path


@pytest.fixture(scope="module")
def make_order(tmp_path_factory):
    """make_order through the existing host harness of the carry (tests/cpp/receivers_core_host.cpp)"""
    import ctypes as C
    lib = build_harness(tmp_path_factory, "receivers_core_host")
    lib.rc_order.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]

    def run(of, receivers):
        of = np.ascontiguousarray(of, np.int32)
        order = np.zeros(len(of), np.int32)
        lib.rc_order(of.ctypes.data, len(of), receivers, order.ctypes.data)
        return order
    return run


def rule(exe, of, receivers, parts=8):
    of = np.ascontiguousarray(of, np.int64).astype(np.int32)
    n = len(of)
    data = np.concatenate([np.array([n, receivers, parts], np.int32), of]).tobytes()
    out = np.frombuffer(subprocess.run([exe], input=data, stdout=subprocess.PIPE, check=True).stdout, np.int32)
    assert len(out) == 2 * n + 1
    return out[:n], out[n:2 * n], int(out[2 * n])


def check(exe, make_order, of, receivers, parts=8):
    of = np.asarray(of, np.int64)
    got_map, got_order, allocations = rule(exe, of, receivers, parts)
    assert allocations == 0
    inside = (of >= 0) & (of < receivers)
    assert np.array_equal(got_map, np.where(inside, of, -1))
    full = np.flatnonzero(inside)
    dense = np.unique(of[full], return_inverse=True)[1].astype(np.int32)   # the same receivers renumbered 0 .. k-1
    want = full[make_order(dense, int(dense.max()) + 1 if len(dense) else 1)] if len(full) else full
    assert np.array_equal(got_order[:len(full)], want)
    assert np.array_equal(got_order[len(full):], np.flatnonzero(~inside))
    assert np.array_equal(np.sort(got_order), np.arange(len(of)))


def with_empties(rng, of, receivers, p):
    """about a fraction p of the slots made empty, with every kind of out-of-range index"""
    of = np.array(of, np.int64)
    pick = rng.random(len(of)) < p
    of[pick] = rng.choice([-1, receivers, INT_MIN, INT_MAX, -7, receivers + 5], int(pick.sum()))
    return of


@pytest.mark.parametrize("n,receivers", [(1, 1), (2, 1), (31, 3), (32, 32), (33, 5), (1023, 100), (1024, 7), (1025, 1000), (5000, 64)])
def test_random_maps(exe, make_order, n, receivers):
    rng = np.random.default_rng(n * 31 + receivers)
    check(exe, make_order, rng.integers(0, receivers, n), receivers)
    check(exe, make_order, with_empties(rng, rng.integers(0, receivers, n), receivers, 0.3), receivers)


def test_twenty_thousand_slots_and_huge_receiver_indices(exe, make_order):
    rng = np.random.default_rng(20000)
    receivers = INT_MAX                                          # every index but INT_MAX itself is in range
    of = rng.choice(np.array([0, 1, 5, 2 ** 20, 2 ** 30 + 3, INT_MAX - 1], np.int64), 20000)
    of[rng.random(20000) < 0.1] = INT_MAX                        # empty: the bound itself
    of[rng.random(20000) < 0.05] = -1
    check(exe, make_order, of, receivers)
    check(exe, make_order, rng.integers(0, 10 ** 6, 20000), 10 ** 6)


def test_empty_slots_in_every_position(exe, make_order):
    n, receivers = 40, 4
    rng = np.random.default_rng(5)
    base = rng.integers(0, receivers, n)
    for i in range(n):
        of = base.copy()
        of[i] = -1
        check(exe, make_order, of, receivers)
    check(exe, make_order, np.full(n, -1), receivers)             # every slot empty
    of = base.copy()
    of[:n // 2] = INT_MIN                                        # a leading run, then a trailing one
    check(exe, make_order, of, receivers)
    of = base.copy()
    of[n // 2:] = receivers
    check(exe, make_order, of, receivers)


@pytest.mark.parametrize("parts", [1, 3, 8])
def test_the_lanes_do_not_change_the_order(exe, make_order, parts):
    rng = np.random.default_rng(parts)
    check(exe, make_order, with_empties(rng, rng.integers(0, 50, 3001), 50, 0.2), 50, parts)
