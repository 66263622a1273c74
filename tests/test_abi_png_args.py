"""CPU-side checks of the PNG entry points (cb200_png_info, cb200_png_decode_dev, cb200_png_scan_extract_decode_chunks_dev): a file
outside the supported set, a bad size or a null pointer is refused with CB200_ERR_ARG before any CUDA call, and the message names the
picture and the reason.  The context is NULL here, so a call whose files are all good fails on the context instead.

The crafted corruptions are checked against cv2 as well: where cv2 returns None, the file is refused here or fails on the device
(the host build of the device functions, tests/cpp/png_core_host.cpp, reports -2); where cv2 decodes it, it is decoded to cv2's
bytes or refused."""
import ctypes as C

import numpy as np
import pytest

import libcimbar_b200 as cb
from libcimbar_b200 import build as cbbuild
from png_matrix import cv2_rgb
from host_harness import build_harness
from png_corpus import ACCEPTED, BASE, CORRUPT, FRAME, REFUSED, tail_after_rows


@pytest.fixture(scope="module", autouse=True)
def built():
    cbbuild.build()


def lib():
    return cb.load_library()


@pytest.fixture(scope="module")
def core(tmp_path_factory):
    L = build_harness(tmp_path_factory, "png_core_host")
    L.pc_decode.argtypes = [C.c_char_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_char_p, C.c_int]
    return L


def host_decode(core, data):
    out = np.zeros(3 * 200 * 8200, np.uint8)
    wh = np.zeros(2, np.int32)
    why = C.create_string_buffer(256)
    rc = core.pc_decode(data, len(data), out.ctypes.data, out.size, wh.ctypes.data, why, 256)
    return rc, (out[:3 * wh[0] * wh[1]].reshape(wh[1], wh[0], 3) if rc == 0 else None)


def calls(files, sizes=None, n=None, flags=0):
    """each PNG entry point with these files (NULL context); yields (name, rc)"""
    L = lib()
    n = len(files) if n is None else n
    ptrs = None if files is None else (C.c_char_p * max(len(files), 1))(*files)
    if sizes is None and files is not None:
        sizes = (C.c_uint64 * max(len(files), 1))(*[len(f) if f is not None else 0 for f in files])
    buf = np.zeros(64, np.uint8)
    yield "decode_dev", L.cb200_png_decode_dev(None, ptrs, sizes, n, buf.ctypes.data, buf.ctypes.data)
    yield "camera_dev", L.cb200_png_scan_extract_decode_chunks_dev(None, ptrs, sizes, n, flags, buf.ctypes.data, buf.ctypes.data,
                                                                   None, buf.ctypes.data)


def last_error():
    return lib().cb200_last_error().decode()


@pytest.mark.parametrize("what,data,reason", REFUSED, ids=[r[0] for r in REFUSED])
def test_refused_files_name_the_picture(what, data, reason):
    for name, rc in calls([FRAME, data, FRAME]):
        assert rc == -1, name
        msg = last_error()
        assert "picture 1" in msg and reason in msg, (name, msg)
    w, h = C.c_int32(), C.c_int32()
    assert lib().cb200_png_info(data, len(data), C.byref(w), C.byref(h)) == -1
    assert reason in last_error()
    with pytest.raises(cb.Cb200Error, match=reason):
        cb.png_info(data)


@pytest.mark.parametrize("what,data", CORRUPT, ids=[c[0] for c in CORRUPT])
def test_corrupt_files_fail_where_cv2_fails(core, what, data):
    assert cv2_rgb(data) is None                                     # premise: cv2 rejects the file
    rc, _ = host_decode(core, data)
    assert rc == -2, rc


@pytest.mark.parametrize("what,data", ACCEPTED, ids=[a[0] for a in ACCEPTED])
def test_files_cv2_accepts_decode_to_its_bytes(core, what, data):
    want = cv2_rgb(data)
    assert want is not None                                          # premise: cv2 decodes the file
    rc, got = host_decode(core, data)
    assert rc == 0 and np.array_equal(got, want), rc


def test_corrupt_data_after_the_rows_in_a_later_read_is_minus_2():
    """the documented deviation: libpng only warns about corrupt data it reads after the last row in a later zlib call (cv2
    decodes the file), and the device reports it -2; in the same read as the last row both fail the file (CORRUPT above)"""
    data = tail_after_rows(False)
    assert cv2_rgb(data) is not None


def test_corrupt_data_after_the_rows_in_a_later_read_decodes_to_minus_2(core):
    rc, _ = host_decode(core, tail_after_rows(False))
    assert rc == -2


def test_refused_files_are_not_decoded_by_cv2_or_listed():
    """every refusal above is either a file cv2 rejects too or one of the deliberate ones (APNG, repeated eXIf, sizes)"""
    deliberate = {"APNG", "two eXIf", "too small", "too large"}
    for what, data, _ in REFUSED:
        if what not in deliberate:
            assert cv2_rgb(data) is None, what


def test_good_files_fail_only_on_the_context():
    for name, rc in calls([FRAME, BASE]):
        assert rc == -1 and "null context" in last_error(), name


def test_null_pointers():
    for name, rc in calls(None, n=1):
        assert rc == -1 and "null files" in last_error(), name
    files = (C.c_char_p * 1)(FRAME)
    L = lib()
    buf = np.zeros(64, np.uint8)
    assert L.cb200_png_decode_dev(None, files, None, 1, buf.ctypes.data, None) == -1 and "null sizes" in last_error()
    for name, rc in calls([FRAME, None]):
        assert rc == -1 and "picture 1 is a null pointer" in last_error(), name
    for name, rc in calls([FRAME], n=-1):
        assert rc == -1 and "n < 0" in last_error(), name
    w = C.c_int32()
    assert L.cb200_png_info(None, 10, C.byref(w), C.byref(w)) == -1
    assert L.cb200_png_info(FRAME, len(FRAME), None, C.byref(w)) == -1


def test_camera_flags_checked_before_cuda():
    for name, rc in calls([FRAME], flags=cb.FLAG_CC_FIT | cb.FLAG_CC_SIMPLE):
        if name == "camera_dev":
            assert rc == -1 and "exclusive" in last_error()
