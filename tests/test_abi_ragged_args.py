"""CPU-side checks of the ragged-batch entry points (cb200_scan_ragged[_dev], cb200_scan_blurred_ragged,
cb200_extract_decode_fountain_ragged_dev, cb200_scan_extract_decode_fountain_ragged): every argument error comes before any CUDA
call, and a bad picture is named by its index.  The context is NULL here, so a call whose arguments are all good fails on the
context instead; n > max_frames needs a context and is checked on the GPU (tests/test_gpu_scan_ragged.py)."""
import ctypes as C

import numpy as np
import pytest

import libcimbar_b200 as cb
from libcimbar_b200 import build as cbbuild


@pytest.fixture(scope="module", autouse=True)
def built():
    cbbuild.build()


LIB = None


def lib():
    global LIB
    if LIB is None:
        LIB = cb.load_library()
    return LIB


def err(rc, text):
    msg = lib().cb200_last_error()
    assert rc == -1 and text in msg, msg


def batch(shapes):
    """host pictures of the given (h, w), their pointer array and wh"""
    pics = [np.zeros((h, w, 3), np.uint8) for h, w in shapes]
    ptrs = (C.c_void_p * len(pics))(*[p.ctypes.data for p in pics])
    wh = np.array([(w, h) for h, w in shapes], np.int32).reshape(-1, 2)
    return pics, ptrs, wh


GOOD = [(960, 1280), (1280, 960), (637, 955)]


def calls(ptrs, wh, n, flags=0):
    """each ragged entry point with these pictures (NULL context); yields (name, rc)"""
    L = lib()
    whp = None if wh is None else wh.ctypes.data
    cnt, st = (C.c_uint32 * 8)(), (C.c_int32 * 8)()
    out = np.zeros(64, np.uint8)
    corners = np.zeros(64, np.float32)
    dev = None if ptrs is None else out.ctypes.data          # a stand-in device address: never dereferenced before the checks
    yield "scan_ragged", L.cb200_scan_ragged(None, ptrs, whp, n, None, cnt, None)
    yield "scan_ragged_dev", L.cb200_scan_ragged_dev(None, dev, whp, n, None, cnt, None)
    yield "extract_decode_ragged_dev", L.cb200_extract_decode_fountain_ragged_dev(None, dev, whp, n, corners.ctypes.data, flags,
                                                                                  out.ctypes.data, cnt, None, None)
    yield "scan_extract_decode_ragged", L.cb200_scan_extract_decode_fountain_ragged(None, ptrs, whp, n, flags, out.ctypes.data, cnt,
                                                                                    None, None, st)


def test_good_arguments_reach_the_context_check():
    _, ptrs, wh = batch(GOOD)
    for name, rc in calls(ptrs, wh, len(GOOD)):
        err(rc, b"null context")


def test_negative_n_null_wh_and_null_pictures():
    _, ptrs, wh = batch(GOOD)
    for name, rc in calls(ptrs, wh, -1):
        err(rc, b"n < 0")
    for name, rc in calls(ptrs, None, len(GOOD)):
        err(rc, b"null wh")
    for name, rc in calls(None, wh, len(GOOD)):
        err(rc, b"null pictures")
    err(lib().cb200_scan_blurred_ragged(None, None, None, wh.ctypes.data, -1), b"n < 0")
    err(lib().cb200_scan_blurred_ragged(None, None, None, None, 1), b"null wh")
    err(lib().cb200_scan_blurred_ragged(None, None, None, wh.ctypes.data, 1), b"no scan")


@pytest.mark.parametrize("bad,index", [((59, 1280), 1), ((1280, 59), 2), ((4500, 4600), 0), ((4600, 4500), 3), ((30, 30), 1)])
def test_out_of_range_picture_is_named(bad, index):
    shapes = GOOD + [(960, 1280)]
    shapes[index] = bad
    _, ptrs, wh = batch(shapes)
    for name, rc in calls(ptrs, wh, len(shapes)):
        err(rc, b"picture %d is %d x %d" % (index, bad[1], bad[0]))


def test_the_largest_accepted_sizes_pass():
    # short side 60 (row step 1) and 4499 (9-tap Gaussian): the checks let them through to the context
    wh = np.array([(60, 100), (4499, 4600), (5000, 60)], np.int32)
    ptrs = (C.c_void_p * 3)(*[1, 2, 3])
    for name, rc in calls(ptrs, wh, 3):
        err(rc, b"null context")


def test_null_host_picture_is_named():
    _, ptrs, wh = batch(GOOD)
    ptrs[2] = None
    L = lib()
    cnt, st = (C.c_uint32 * 8)(), (C.c_int32 * 8)()
    out = np.zeros(64, np.uint8)
    err(L.cb200_scan_ragged(None, ptrs, wh.ctypes.data, 3, None, cnt, None), b"picture 2 is a null pointer")
    err(L.cb200_scan_extract_decode_fountain_ragged(None, ptrs, wh.ctypes.data, 3, 0, out.ctypes.data, cnt, None, None, st),
        b"picture 2 is a null pointer")


def test_both_sharpen_flags_are_refused():
    _, ptrs, wh = batch(GOOD)
    both = cb.FLAG_SHARPEN | cb.FLAG_SHARPEN_IF_NEEDED
    for name, rc in list(calls(ptrs, wh, len(GOOD), flags=both))[2:]:
        err(rc, b"exclusive")


def test_ragged_samples_are_the_recorded_pictures():
    # the two photographs kept for the ragged tests decode to the RGB recorded with them, and the stand-in for the sample directory's
    # largest photograph is, like it, portrait and past the 9-tap threshold (short side >= 2560)
    from ragged_samples import BIG, GLOB, sample
    shapes = [sample(s).shape for s in GLOB]
    assert len(shapes) == 8 and all(a != b for a, b in zip(shapes, shapes[1:]))
    h, w, _ = sample(BIG).shape
    assert (h, w) == (3584, 2688) and min(h, w) >= 2560


def test_python_lists_are_checked():
    with pytest.raises(cb.Cb200Error):
        cb._ragged([np.zeros((100, 100), np.uint8)])
    pics, ptrs, wh = cb._ragged([np.zeros((70, 90, 3), np.uint8), np.zeros((100, 80, 3), np.uint8)])
    assert wh.tolist() == [[90, 70], [80, 100]] and ptrs[0] == pics[0].ctypes.data
