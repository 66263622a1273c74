"""CPU-side checks of cb200_scan_extract_decode_chunks_grouped_dev (the groups of a batch found on the device): every argument error
comes before any CUDA call, in check_camera_call's order.  The context is NULL here, so a call whose arguments are all good fails on
the context instead; the pictures' null outputs and n > max_frames need a context and are checked on the GPU
(tests/test_gpu_grouped.py).  Apart from CB200_FLAG_NO_FALLBACK, the call refuses exactly what the pictures call refuses."""
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


def call(pics, n=None, flags=0, null_array=False, outputs=True, missing=()):
    arr = (cb.Picture * max(1, len(pics)))(*pics)
    out = np.zeros(64, np.uint8)                         # stand-in device addresses: never dereferenced before the checks
    st = np.zeros(8, np.int32)
    o = out.ctypes.data if outputs else None
    g = [None if k in missing else out.ctypes.data for k in GROUP_OUTPUTS]
    return lib().cb200_scan_extract_decode_chunks_grouped_dev(
        None, None if null_array else C.cast(arr, C.c_void_p), len(pics) if n is None else n, flags, o, o, None,
        st.ctypes.data if outputs else None, *g)


def pictures_call(pics, n=None, flags=0, null_array=False):
    arr = (cb.Picture * max(1, len(pics)))(*pics)
    out = np.zeros(64, np.uint8)
    st = np.zeros(8, np.int32)
    return lib().cb200_scan_extract_decode_chunks_pictures_dev(None, None if null_array else C.cast(arr, C.c_void_p),
                                                               len(pics) if n is None else n, flags, out.ctypes.data,
                                                               out.ctypes.data, None, st.ctypes.data)


def test_good_arguments_reach_the_context_check():
    err(call(good()), b"null context")
    err(call(good(), flags=cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT | cb.FLAG_NO_INTERLEAVE), b"null context")
    err(call(good() * 10), b"null context")
    for n in (0, 1):
        err(call(good()[:n]), b"null context")


@pytest.mark.parametrize("n", [0, 1, 4])
def test_no_fallback_is_refused(n):
    err(call(good()[:n], flags=cb.FLAG_NO_FALLBACK), b"CB200_FLAG_NO_FALLBACK: the vote needs every picture's walk")


@pytest.mark.parametrize("which", GROUP_OUTPUTS)
@pytest.mark.parametrize("n", [0, 1, 4])
def test_each_null_group_output_is_refused(which, n):
    err(call(good()[:n], missing=(which,)), b"null group output")


def test_the_order_of_the_checks():
    # the pictures call's flag and batch checks first, then NO_FALLBACK, the group outputs, the context and the pictures' outputs
    err(call(good(), flags=cb.FLAG_CC_SIMPLE | cb.FLAG_CC_FIT | cb.FLAG_NO_FALLBACK, missing=GROUP_OUTPUTS), b"exclusive")
    err(call(with_(2, data=None), flags=cb.FLAG_NO_FALLBACK, missing=GROUP_OUTPUTS), b"picture 2 has a null data pointer")
    err(call(with_(3, row_pitch=1 << 32), flags=cb.FLAG_NO_FALLBACK), b"picture 3 spans 4 GB or more")
    err(call(good(), n=-1, flags=cb.FLAG_NO_FALLBACK), b"n")
    err(call(good(), flags=cb.FLAG_NO_FALLBACK, missing=GROUP_OUTPUTS, outputs=False), b"CB200_FLAG_NO_FALLBACK")
    err(call(good(), missing=("used",), outputs=False), b"null group output")
    err(call(good(), outputs=False), b"null context")


PICTURE_CASES = [
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
]


@pytest.mark.parametrize("name,case", PICTURE_CASES, ids=[c[0] for c in PICTURE_CASES])
def test_it_refuses_what_the_pictures_call_refuses(name, case):
    pics, kw = case()
    rc_p = pictures_call(pics, **kw)
    want = last()
    rc = call(pics, **kw)
    assert (rc, last()) == (rc_p, want), name


def test_python_wrapper_checks_the_orders():
    ctx = cb.Context.__new__(cb.Context)
    with pytest.raises(cb.Cb200Error, match="1 orders for 2 pictures"):
        cb.Context.scan_extract_decode_chunks_grouped_dev(ctx, [None, None], 0, 0, 0, 0, 0, 0, 0, 0, order=["bgr"])
