"""CPU-side checks of the group history (cb200_group_history_*) and cb200_scan_extract_decode_chunks_grouped_history_dev: every
argument error comes before any CUDA call.  The call refuses what the grouped call refuses, in its order, then a null history; the
context is NULL here, so a call whose other arguments are all good fails on the context.  A history of another context and
n > max_frames need a context and are checked on the GPU (tests/test_gpu_grouped_history.py)."""
import ctypes as C

import numpy as np
import pytest

import libcimbar_b200 as cb
from libcimbar_b200 import build as cbbuild
from cpu_support import good, with_

GROUP_OUTPUTS = ("group_of", "count", "chunks", "mask", "used")


@pytest.fixture(scope="module", autouse=True)
def built():
    cbbuild.build()


def lib():
    return cb.load_library()


def last():
    return lib().cb200_last_error()


def err(rc, text):
    msg = last()
    assert rc == -1 and text in msg, msg


def call(pics, n=None, flags=0, null_array=False, outputs=True, missing=(), history=None):
    arr = (cb.Picture * max(1, len(pics)))(*pics)
    out = np.zeros(64, np.uint8)                         # stand-in device addresses: never dereferenced before the checks
    st = np.zeros(8, np.int32)
    o = out.ctypes.data if outputs else None
    g = [None if k in missing else out.ctypes.data for k in GROUP_OUTPUTS]
    return lib().cb200_scan_extract_decode_chunks_grouped_history_dev(
        None, history, None if null_array else C.cast(arr, C.c_void_p), len(pics) if n is None else n, flags, o, o, None,
        st.ctypes.data if outputs else None, *g)


def grouped_call(pics, n=None, flags=0, null_array=False, outputs=True, missing=()):
    arr = (cb.Picture * max(1, len(pics)))(*pics)
    out = np.zeros(64, np.uint8)
    st = np.zeros(8, np.int32)
    o = out.ctypes.data if outputs else None
    g = [None if k in missing else out.ctypes.data for k in GROUP_OUTPUTS]
    return lib().cb200_scan_extract_decode_chunks_grouped_dev(
        None, None if null_array else C.cast(arr, C.c_void_p), len(pics) if n is None else n, flags, o, o, None,
        st.ctypes.data if outputs else None, *g)


def test_good_arguments_reach_the_context_check():
    err(call(good()), b"null context")
    err(call(good(), flags=cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT | cb.FLAG_NO_INTERLEAVE), b"null context")
    for n in (0, 1):
        err(call(good()[:n]), b"null context")


@pytest.mark.parametrize("n", [0, 1, 4])
def test_no_fallback_is_refused(n):
    err(call(good()[:n], flags=cb.FLAG_NO_FALLBACK), b"CB200_FLAG_NO_FALLBACK: the vote needs every picture's walk")


@pytest.mark.parametrize("which", GROUP_OUTPUTS)
@pytest.mark.parametrize("n", [0, 1, 4])
def test_each_null_group_output_is_refused(which, n):
    err(call(good()[:n], missing=(which,)), b"null group output")


CASES = [
    ("good", lambda: (good(), {})),
    ("negative n", lambda: (good(), {"n": -1})),
    ("null array", lambda: (good(), {"null_array": True})),
    ("null data", lambda: (with_(0, data=None), {})),
    ("layout", lambda: (with_(1, layout=5), {})),
    ("pitch", lambda: (with_(3, row_pitch=-4), {})),
    ("size", lambda: (with_(1, h=59, w=1280, row_pitch=4 * 1280), {})),
    ("row pitch", lambda: (with_(0, row_pitch=3 * 1280 - 1), {})),
    ("planes", lambda: (with_(2, plane_pitch=1280 * 1024 - 1), {})),
    ("4 GB", lambda: (with_(3, row_pitch=1 << 32), {})),
    ("sharpen flags", lambda: (good(), {"flags": cb.FLAG_SHARPEN | cb.FLAG_SHARPEN_IF_NEEDED})),
    ("cc flags", lambda: (good(), {"flags": cb.FLAG_CC_SIMPLE | cb.FLAG_CC_FIT})),
    ("no fallback", lambda: (good(), {"flags": cb.FLAG_NO_FALLBACK})),
    ("group outputs", lambda: (good(), {"missing": ("mask",)})),
    ("outputs", lambda: (good(), {"outputs": False})),
    ("flags before no fallback", lambda: (good(), {"flags": cb.FLAG_CC_SIMPLE | cb.FLAG_CC_FIT | cb.FLAG_NO_FALLBACK})),
    ("pictures before group outputs", lambda: (with_(2, data=None), {"missing": GROUP_OUTPUTS, "flags": cb.FLAG_NO_FALLBACK})),
    ("group outputs before outputs", lambda: (good(), {"missing": ("used",), "outputs": False})),
]


@pytest.mark.parametrize("name,case", CASES, ids=[c[0] for c in CASES])
def test_it_refuses_what_the_grouped_call_refuses_in_its_order(name, case):
    pics, kw = case()
    rc_g = grouped_call(pics, **kw)
    want = last()
    rc = call(pics, **kw)
    assert (rc, last()) == (rc_g, want), name


def test_create_read_reset_destroy_checks():
    L = lib()
    out = C.c_void_p(1)
    err(L.cb200_group_history_create(None, 8, None), b"null output")
    err(L.cb200_group_history_create(None, 8, C.byref(out)), b"null context")
    assert out.value is None                                         # *out is cleared before the other checks
    fake = C.c_void_p(1)                                             # never dereferenced: the capacity check comes first
    for capacity in (0, -1, 257, 1 << 30):
        err(L.cb200_group_history_create(fake, capacity, C.byref(out)), b"capacity = %d outside [1, 256]" % capacity)
    count = C.c_int32()
    tags = np.zeros(4, np.int64)
    err(L.cb200_group_history_read(None, tags.ctypes.data, 4, C.byref(count)), b"null history")
    err(L.cb200_group_history_read(fake, tags.ctypes.data, 4, None), b"null count")
    err(L.cb200_group_history_read(fake, tags.ctypes.data, -1, C.byref(count)), b"max = -1 < 0")
    err(L.cb200_group_history_read(fake, None, 1, C.byref(count)), b"null tags with max > 0")
    err(L.cb200_group_history_reset(None), b"null history")
    err(L.cb200_group_history_destroy(None), b"null history")


def test_python_wrapper_checks_the_orders():
    ctx = cb.Context.__new__(cb.Context)
    with pytest.raises(cb.Cb200Error, match="1 orders for 2 pictures"):
        cb.Context.scan_extract_decode_chunks_grouped_history_dev(ctx, [None, None], None, 0, 0, 0, 0, 0, 0, 0, 0, order=["bgr"])
