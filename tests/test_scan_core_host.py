"""The device anchor-scan code (libcimbar_b200/csrc/scan_core.cuh: what the kernels of scan.cu are made of) compiled for the
host and run as a one-thread CTA against the oracle -- the logic check that is possible without a GPU.  The GPU parity test
(tests/test_gpu_scan.py) runs the same comparisons through the C ABI."""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as ol
from scan_oracle_lib import ScanOracle, join
from host_harness import build_harness
from cpu_support import pictures

SO = ScanOracle()


@pytest.fixture(scope="module")
def core(tmp_path_factory):
    lib = build_harness(tmp_path_factory, "scan_core_host", "-ffp-contract=off")
    lib.sc_scan.argtypes = [C.POINTER(C.c_uint8), C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_uint), C.POINTER(C.c_int)]
    lib.sc_sort_check.argtypes = [C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    return lib


@pytest.mark.parametrize("name,rgb", pictures(), ids=[p[0] for p in pictures()])
def test_device_scan_code_matches_oracle_on_the_host(core, name, rgb):
    t, bin_, blurred = SO.preprocess(rgb)
    want, want_cutoff = SO.scan(rgb)
    h, w = rgb.shape[:2]
    anchors = (C.c_int * 16)(); cutoff = C.c_uint(0); status = C.c_int(0)
    n = core.sc_scan(ol._ptr(np.ascontiguousarray(blurred)), w, h, t, anchors, C.byref(cutoff), C.byref(status))
    got = [tuple(anchors[4 * i + k] for k in range(4)) for i in range(n)]
    assert status.value == 0
    assert got == want, (join(got), join(want))
    assert cutoff.value == want_cutoff


def test_restated_std_sort_is_this_toolchains_std_sort(core):
    rng = np.random.default_rng(17)
    for trial in range(400):
        n = int(rng.choice([1, 2, 3, 5, 15, 16, 17, 18, 31, 33, 64, 100, 257]))
        sizes = rng.integers(1, 6 if trial % 2 else 60, n)             # few distinct sizes: many ties
        a = np.zeros((n, 4), np.int32)
        a[:, 0] = np.arange(n)                                          # x identifies the element, xmax - x is its size
        a[:, 1] = a[:, 0] + sizes
        mine = np.zeros((n, 4), np.int32); std = np.zeros((n, 4), np.int32)
        same = core.sc_sort_check(a.ctypes.data_as(C.POINTER(C.c_int)), n, mine.ctypes.data_as(C.POINTER(C.c_int)),
                                  std.ctypes.data_as(C.POINTER(C.c_int)))
        assert same == 1, (trial, n)
