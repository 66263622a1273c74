"""One check sequence on every camera and corner entry point, without a GPU: the flags come first, then the pictures, then the
context.  With a NULL context (a list of NULL contexts for detect), CC_SIMPLE together with CC_FIT is refused as exclusive, and a
packed picture spanning 4 GB or more (k_deskew's offsets inside a picture are 32-bit) is refused by name, both before the context
check.  The scan-only entry points do not deskew, so such a picture reaches their context check."""
import ctypes as C

import numpy as np
import pytest

import libcimbar_b200 as cb
from libcimbar_b200 import build as cbbuild
from cpu_support import PHOTO
from png_corpus import BASE as PNG


@pytest.fixture(scope="module", autouse=True)
def built():
    cbbuild.build()


def lib():
    return cb.load_library()


BUF = np.zeros(256, np.uint8)
DEV = BUF.ctypes.data                                   # stand-in addresses: never dereferenced before the checks
OUT = np.zeros(64, np.uint32)
CORNERS = np.zeros(64, np.float32)
GOOD = (1280, 960)
HUGE = (400000, 4000)                                   # short side in range, 3 w h >= 4 GB


def sizes(w, h, n=2):
    return np.array([(w, h)] * n, np.int32)


def host_ptrs(n=2):
    return (C.c_void_p * n)(*([DEV] * n))


def files(data, n=2):
    return (C.c_char_p * n)(*([data] * n)), (C.c_uint64 * n)(*([len(data)] * n))


def camera_calls(w, h, flags):
    """every camera and corner entry point on pictures of w x h (NULL context): (name, thunk)"""
    L, o = lib(), OUT.ctypes.data
    wh = sizes(w, h)
    picture = [cb.Picture(DEV, w, h, 3 * w, 0, cb.LAYOUT_RGB)] * 2
    pics = (cb.Picture * 2)(*picture)
    yield "host_uniform", lambda: L.cb200_scan_extract_decode_fountain(None, DEV, w, h, 2, flags, DEV, o, None, None, o)
    yield "host_ragged", lambda: L.cb200_scan_extract_decode_fountain_ragged(None, host_ptrs(), wh.ctypes.data, 2, flags, DEV, o, None, None, o)
    yield "dev_uniform", lambda: L.cb200_scan_extract_decode_chunks_dev(None, DEV, w, h, 2, flags, DEV, o, None, o)
    yield "dev_ragged", lambda: L.cb200_scan_extract_decode_chunks_ragged_dev(None, DEV, wh.ctypes.data, 2, flags, DEV, o, None, o)
    yield "descriptors", lambda: L.cb200_scan_extract_decode_chunks_pictures_dev(None, C.cast(pics, C.c_void_p), 2, flags, DEV, o, None, o)
    yield "plan", lambda: L.cb200_camera_plan_create(None, wh.ctypes.data, 2, flags, DEV, DEV, o, None, o, C.byref(C.c_void_p()))
    yield "detect", lambda: L.cb200_detect_scan_extract_decode_chunks_dev((C.c_void_p * 2)(None, None), 2, DEV, wh.ctypes.data, 2, flags,
                                                                          DEV, o, o, o, None)
    c = CORNERS.ctypes.data
    yield "corner_host", lambda: L.cb200_extract_decode_fountain(None, DEV, w, h, 2, c, flags, DEV, o, None, None)
    yield "corner_dev", lambda: L.cb200_extract_decode_fountain_dev(None, DEV, w, h, 2, c, flags, DEV, o, None, None)
    yield "corner_ragged_dev", lambda: L.cb200_extract_decode_fountain_ragged_dev(None, DEV, wh.ctypes.data, 2, c, flags, DEV, o, None, None)


def file_calls(flags):
    L, o = lib(), OUT.ctypes.data
    for name, data, fn in (("jpeg", PHOTO, L.cb200_jpeg_scan_extract_decode_chunks_dev), ("png", PNG, L.cb200_png_scan_extract_decode_chunks_dev)):
        f, s = files(data)
        yield name, lambda fn=fn, f=f, s=s: fn(None, f, s, 2, flags, DEV, o, None, o)


def scan_calls(w, h):
    """the scan-only entry points (NULL context)"""
    L, o = lib(), OUT.ctypes.data
    wh = sizes(w, h)
    yield "scan", lambda: L.cb200_scan(None, DEV, w, h, 2, None, o, None)
    yield "scan_dev", lambda: L.cb200_scan_dev(None, DEV, w, h, 2, None, o, None)
    yield "scan_ragged", lambda: L.cb200_scan_ragged(None, host_ptrs(), wh.ctypes.data, 2, None, o, None)
    yield "scan_ragged_dev", lambda: L.cb200_scan_ragged_dev(None, DEV, wh.ctypes.data, 2, None, o, None)


def deskew_calls(w, h):
    L, m9 = lib(), np.eye(3).ctypes.data
    yield "deskew", lambda: L.cb200_deskew(None, DEV, w, h, 2, m9, DEV)
    yield "deskew_dev", lambda: L.cb200_deskew_dev(None, DEV, w, h, 2, m9, DEV)


def refused(thunk):
    rc = thunk()
    return rc, lib().cb200_last_error().decode()


def test_good_arguments_reach_the_context_check():
    for name, thunk in [*camera_calls(*GOOD, 0), *file_calls(0), *scan_calls(*GOOD), *deskew_calls(*GOOD)]:
        rc, msg = refused(thunk)
        assert rc == -1 and ("null context" in msg or "context 0 is null" in msg), (name, msg)


def test_cc_simple_with_cc_fit_is_refused_before_the_context():
    for name, thunk in [*camera_calls(*GOOD, cb.FLAG_CC_SIMPLE | cb.FLAG_CC_FIT), *file_calls(cb.FLAG_CC_SIMPLE | cb.FLAG_CC_FIT)]:
        rc, msg = refused(thunk)
        assert rc == -1 and "CC_SIMPLE and CC_FIT are exclusive" in msg, (name, msg)


def test_a_picture_spanning_4_gb_is_refused_before_the_context():
    for name, thunk in [*camera_calls(*HUGE, 0), *deskew_calls(*HUGE)]:
        rc, msg = refused(thunk)
        assert rc == -1 and "picture 0 spans 4 GB or more" in msg, (name, msg)


def test_the_scan_only_calls_take_a_picture_spanning_4_gb():
    for name, thunk in scan_calls(*HUGE):
        rc, msg = refused(thunk)
        assert rc == -1 and "null context" in msg, (name, msg)
