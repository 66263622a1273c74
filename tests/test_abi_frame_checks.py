"""One check sequence on every frame entry point, without a GPU: the flags come first, then the selection, then the context.  With
a NULL context, CC_SIMPLE together with CC_FIT is refused as exclusive on every call that honours CC_FIT, at n = 1 and at n = 0
alike.  The raw and cell calls ignore CC_FIT, so the pair reaches their context check."""
import numpy as np
import pytest

import libcimbar_b200 as cb
from libcimbar_b200 import build as cbbuild


@pytest.fixture(scope="module", autouse=True)
def built():
    cbbuild.build()


def lib():
    return cb.load_library()


BUF = np.zeros(256, np.uint8)
P = BUF.ctypes.data                                     # stand-in addresses: never dereferenced before the checks
SEL = np.ones(1, np.uint8).ctypes.data
BOTH = cb.FLAG_CC_SIMPLE | cb.FLAG_CC_FIT


def fit_calls(n, flags):
    """the frame entry points that honour CC_FIT (NULL context): (name, thunk)"""
    L = lib()
    yield "decode", lambda: L.cb200_decode(None, P, n, flags, P, None, None)
    yield "decode_chunks_dev", lambda: L.cb200_decode_chunks_dev(None, P, n, flags, P, P, None)
    yield "decode_chunks_sharpen_dev", lambda: L.cb200_decode_chunks_sharpen_dev(None, P, n, flags, SEL, P, P, None)
    yield "decode_fountain", lambda: L.cb200_decode_fountain(None, P, n, flags, P, P, None, None)
    yield "decode_fountain_sharpen", lambda: L.cb200_decode_fountain_sharpen(None, P, n, flags, SEL, P, P, None, None)
    yield "decode_fountain_from_dev", lambda: L.cb200_decode_fountain_from_dev(None, P, n, flags, P, P, None, None)


def raw_and_cell_calls(n, flags):
    """the frame entry points that ignore CC_FIT (NULL context)"""
    L = lib()
    yield "decode_raw", lambda: L.cb200_decode_raw(None, P, n, flags, P, None)
    yield "decode_raw_dev", lambda: L.cb200_decode_raw_dev(None, P, n, flags, P, None)
    yield "decode_cells", lambda: L.cb200_decode_cells(None, P, n, flags, P, P)
    yield "decode_cells_means", lambda: L.cb200_decode_cells_means(None, P, n, flags, P, P, P)


def refused(thunk):
    rc = thunk()
    return rc, lib().cb200_last_error().decode()


@pytest.mark.parametrize("n", [1, 0])
def test_good_arguments_reach_the_context_check(n):
    for name, thunk in [*fit_calls(n, 0), *raw_and_cell_calls(n, 0)]:
        rc, msg = refused(thunk)
        assert rc == -1 and "null context" in msg, (name, msg)


@pytest.mark.parametrize("n", [1, 0])
def test_cc_simple_with_cc_fit_is_refused_before_the_context(n):
    for name, thunk in fit_calls(n, BOTH):
        rc, msg = refused(thunk)
        assert rc == -1 and "CC_SIMPLE and CC_FIT are exclusive" in msg, (name, msg)


@pytest.mark.parametrize("n", [1, 0])
def test_the_raw_and_cell_calls_ignore_cc_fit(n):
    for name, thunk in raw_and_cell_calls(n, BOTH):
        rc, msg = refused(thunk)
        assert rc == -1 and "null context" in msg, (name, msg)
