"""The segmented CCM carry of a batch of several receivers (libcimbar_b200/csrc/receivers_core.cuh) compiled for the host and run
as k_ccm_carry_receivers runs it (1024 threads, each over a contiguous range of the receiver-major order, combined by a block max
scan), against a sequential carry per receiver: a picture takes the fit of its receiver's last picture with a fit at or before it,
else its receiver's entry state, and each receiver's last picture writes the exit state.  The GPU test (tests/test_gpu_receivers.py)
compares whole calls."""
import ctypes as C

import numpy as np
import pytest

from host_harness import build_harness


@pytest.fixture(scope="module")
def core(tmp_path_factory):
    lib = build_harness(tmp_path_factory, "receivers_core_host")
    lib.rc_carry.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    lib.rc_order.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    return lib


def sequential(of, valid, receivers):
    """one decoder per receiver, taking its pictures in batch order"""
    src = np.full(len(of), -1, np.int32)
    last = np.full(receivers, -1, np.int32)
    fit = {}
    for f, r in enumerate(of):
        if valid[f]:
            fit[r] = f
        src[f] = fit.get(r, -1)
        last[r] = f
    return src, last


def run(core, of, valid, receivers, threads=1024):
    of = np.ascontiguousarray(of, np.int32)
    valid = np.ascontiguousarray(valid, np.uint8)
    src = np.full(len(of), -7, np.int32)
    last = np.full(receivers, -7, np.int32)
    core.rc_carry(of.ctypes.data, valid.ctypes.data, len(of), receivers, threads, src.ctypes.data, last.ctypes.data)
    return src, last


def check(core, of, valid, receivers, threads=1024):
    got = run(core, of, valid, receivers, threads)
    want = sequential(of, valid, receivers)
    assert np.array_equal(got[0], want[0])
    assert np.array_equal(got[1], want[1])


def test_order_is_stable_and_receiver_major(core):
    rng = np.random.default_rng(3)
    of = rng.integers(0, 37, 5000).astype(np.int32)
    order = np.zeros(len(of), np.int32)
    core.rc_order(of.ctypes.data, len(of), 37, order.ctypes.data)
    assert np.array_equal(order, np.argsort(of, kind="stable"))


@pytest.mark.parametrize("n", [1, 2, 7, 1023, 1024, 1025, 3000, 7777])
def test_one_receiver_is_the_plain_carry(core, n):
    rng = np.random.default_rng(n)
    check(core, np.zeros(n, np.int32), rng.random(n) < 0.3, 1)


@pytest.mark.parametrize("n,receivers,p_fit", [(5, 3, 0.5), (64, 8, 0.2), (1000, 100, 0.1), (3000, 17, 0.05), (4096, 700, 0.3),
                                               (6000, 3, 0.001), (6000, 2500, 0.5), (5000, 5000, 0.5)])
def test_random_patterns(core, n, receivers, p_fit):
    rng = np.random.default_rng(n * 7 + receivers)
    for _ in range(3):
        check(core, rng.integers(0, receivers, n), rng.random(n) < p_fit, receivers)


def test_no_fits_and_all_fits(core):
    rng = np.random.default_rng(11)
    of = rng.integers(0, 50, 4000)
    check(core, of, np.zeros(4000, bool), 50)
    check(core, of, np.ones(4000, bool), 50)


def test_absent_receivers_are_not_written(core):
    rng = np.random.default_rng(12)
    of = rng.choice([3, 9, 10, 40], 2500)
    src, last = run(core, of, rng.random(2500) < 0.2, 64)
    assert set(np.flatnonzero(last >= 0)) == {3, 9, 10, 40}
    check(core, of, rng.random(2500) < 0.2, 64)


def test_segments_cross_thread_ranges(core):
    """each of the 1024 threads owns several positions, and receivers' segments start and end inside and across those ranges: one
    fit early in a long segment must reach its last picture three threads on, and must not leak into the next receiver"""
    n = 5 * 1024 + 3
    of = np.repeat(np.arange(n // 17 + 1), 17)[:n]
    valid = np.zeros(n, bool)
    valid[::41] = True
    check(core, of, valid, int(of.max()) + 1)
    rng = np.random.default_rng(13)
    of = np.sort(rng.integers(0, 9, n))
    valid = np.zeros(n, bool)
    valid[[0, 5, 2000]] = True
    check(core, rng.permutation(of), valid, 9)
    check(core, of, valid, 9)
    check(core, of, valid, 9, threads=7)
