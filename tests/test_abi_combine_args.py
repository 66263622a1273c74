"""CPU-side checks of cb200_scan_extract_decode_chunks_combined_dev (several pictures of one frame decoded as a group): every argument
error comes before any CUDA call, in check_camera_call's order, and names the offending picture.  The context is NULL here, so a call
whose arguments are all good fails on the context instead; m > max_frames and the pictures' null outputs need a context and are
checked on the GPU (tests/test_gpu_combine.py).  With m = 0 and every group_of -1 the call refuses exactly what the pictures call
refuses."""
import ctypes as C

import numpy as np
import pytest

import libcimbar_b200 as cb
from libcimbar_b200 import build as cbbuild
from test_abi_layout_args import good, with_


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


def call(pics, group_of, m, n=None, flags=0, null_array=False, outputs=True, group_outputs=True, ctx=None):
    arr = (cb.Picture * max(1, len(pics)))(*pics)
    out = np.zeros(64, np.uint8)                         # stand-in device addresses: never dereferenced before the checks
    st = np.zeros(8, np.int32)
    of = None if group_of is None else np.ascontiguousarray(group_of, np.int32)
    g = out.ctypes.data if group_outputs else None
    o = out.ctypes.data if outputs else None
    return lib().cb200_scan_extract_decode_chunks_combined_dev(
        ctx, None if null_array else C.cast(arr, C.c_void_p), len(pics) if n is None else n, None if of is None else of.ctypes.data, m,
        flags, o, o, None, st.ctypes.data if outputs else None, g, g, g)


def pictures_call(pics, n=None, flags=0, null_array=False):
    arr = (cb.Picture * max(1, len(pics)))(*pics)
    out = np.zeros(64, np.uint8)
    st = np.zeros(8, np.int32)
    return lib().cb200_scan_extract_decode_chunks_pictures_dev(None, None if null_array else C.cast(arr, C.c_void_p),
                                                               len(pics) if n is None else n, flags, out.ctypes.data,
                                                               out.ctypes.data, None, st.ctypes.data)


def test_good_arguments_reach_the_context_check():
    err(call(good(), [0, 0, 1, -1], 2), b"null context")
    err(call(good(), [-1, -1, -1, -1], 5), b"null context")          # groups without pictures are allowed
    err(call(good(), None, 0), b"null context")
    err(call(good(), [0] * 4, 1, flags=cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT | cb.FLAG_NO_INTERLEAVE), b"null context")
    pics = good() * 4                                                # 16 pictures in one group: the cap itself
    err(call(pics, [0] * 16, 1), b"null context")


def test_no_fallback_is_refused_with_groups():
    err(call(good(), [0, 0, 1, -1], 2, flags=cb.FLAG_NO_FALLBACK), b"CB200_FLAG_NO_FALLBACK with m > 0")
    err(call(good(), [-1] * 4, 0, flags=cb.FLAG_NO_FALLBACK), b"null context")


def test_negative_m_is_refused():
    err(call(good(), [-1] * 4, -1), b"m = -1 < 0")
    err(call(good(), None, -3), b"m = -3 < 0")


def test_null_group_of_is_refused_with_groups():
    err(call(good(), None, 1), b"null group_of with m > 0")


@pytest.mark.parametrize("at,value,m", [(0, 2, 2), (3, -2, 2), (1, 1, 1), (2, 0, 0), (1, 7, 3), (3, -2 ** 31, 4)])
def test_entry_outside_the_groups_is_named(at, value, m):
    of = [-1, 0 if m else -1, -1, -1]
    of[at] = value
    err(call(good(), of, m), b"picture %d: group %d outside [-1, %d)" % (at, value, m))


def test_seventeenth_picture_of_a_group_is_named():
    pics = good() * 5
    of = [1] * 20
    of[3] = 0
    err(call(pics, of, 2), b"picture 17: group 1 has more than 16 pictures")
    of[17] = 0
    err(call(pics, of, 2), b"picture 18: group 1 has more than 16 pictures")
    of = [0, 1] * 10                                                 # 10 per group
    err(call(pics, of, 2), b"null context")


def test_null_group_outputs_are_refused_with_groups():
    err(call(good(), [0, 0, 1, -1], 2, group_outputs=False), b"null group output")
    err(call(good(), [-1] * 4, 0, group_outputs=False), b"null context")


def test_the_order_of_the_checks():
    # the pictures call's flag and batch checks come first, then the groups', then the context
    err(call(good(), None, -1, flags=cb.FLAG_CC_SIMPLE | cb.FLAG_CC_FIT), b"exclusive")
    err(call(with_(2, data=None), None, -1), b"picture 2 has a null data pointer")
    err(call(with_(3, row_pitch=1 << 32), [9] * 4, 1), b"picture 3 spans 4 GB or more")
    err(call(good(), [9] * 4, 1, flags=cb.FLAG_NO_FALLBACK), b"CB200_FLAG_NO_FALLBACK")
    err(call(good(), None, -1), b"m = -1 < 0")
    err(call(good(), [9] * 4, 1, group_outputs=False), b"picture 0: group 9")
    err(call(good(), [0] * 4, 1, group_outputs=False, outputs=False), b"null group output")
    err(call(good(), [0] * 4, 1, outputs=False), b"null context")


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
    ("no fallback", lambda: (good(), {"flags": cb.FLAG_NO_FALLBACK})),
]


@pytest.mark.parametrize("name,case", PICTURE_CASES, ids=[c[0] for c in PICTURE_CASES])
def test_without_groups_it_refuses_what_the_pictures_call_refuses(name, case):
    pics, kw = case()
    rc_p = pictures_call(pics, **kw)
    want = last()
    for of in (None, [-1] * len(pics)):
        rc = call(pics, of, 0, **kw)
        assert (rc, last()) == (rc_p, want), name


def test_python_wrapper_checks_the_group_list():
    ctx = cb.Context.__new__(cb.Context)
    with pytest.raises(cb.Cb200Error, match="3 group_of entries for 2 pictures"):
        cb.Context.scan_extract_decode_chunks_combined_dev(ctx, [None, None], [0, 0, 0], 1, 0, 0, 0, 0, 0, 0)


def test_a_huge_m_is_answered_at_once():
    """m is checked against max_frames only after the context, so the group checks before it must not size anything by m"""
    import time
    for of, want in (([-1] * 4, b"null context"), ([0, 1, 2 ** 31 - 2, -1], b"null context"), ([0] * 4, b"null context"),
                     ([0, -2, 0, 0], b"picture 1: group -2 outside [-1, 2147483647)")):
        t0 = time.perf_counter()
        err(call(good(), of, 2 ** 31 - 1), want)
        assert time.perf_counter() - t0 < 0.5
    pics = good() * 5
    t0 = time.perf_counter()
    err(call(pics, [2 ** 31 - 2] * 20, 2 ** 31 - 1), b"picture 16: group 2147483646 has more than 16 pictures")
    assert time.perf_counter() - t0 < 0.5
