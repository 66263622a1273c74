"""CPU-side checks of the per-frame sharpen surface: the argument errors of the new entry points and flag come before any CUDA
call, and the C++ test of the Decoder mirror's per-frame overload compiles (it runs on the GPU in tests/test_gpu_sharpen_select.py)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import libcimbar_b200 as cb
from libcimbar_b200 import build as cbbuild

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module", autouse=True)
def built():
    cbbuild.build()


def test_sharpen_selection_arguments_are_checked_without_touching_a_gpu():
    # the two sharpen flags together, CB200_FLAG_SHARPEN_IF_NEEDED on an entry point that takes frames, CB200_FLAG_SHARPEN with a
    # selection and a missing selection are CB200_ERR_ARG before any CUDA call; the message names the offending argument (the
    # context is NULL here, so without the offending argument the call fails on the context instead)
    lib = cb.load_library()
    buf = np.zeros(64 * 64 * 3, np.uint8)
    cnt, st = (C.c_uint32 * 1)(), (C.c_int32 * 1)()
    sel = np.ones(1, np.uint8)
    corners = np.zeros(8, np.float32)
    both = cb.FLAG_SHARPEN | cb.FLAG_SHARPEN_IF_NEEDED

    def err(rc, text):
        assert rc == -1 and text in lib.cb200_last_error(), lib.cb200_last_error()

    err(lib.cb200_scan_extract_decode_fountain(None, buf.ctypes.data, 64, 64, 1, both, buf.ctypes.data, cnt, None, None, st), b"exclusive")
    err(lib.cb200_extract_decode_fountain(None, buf.ctypes.data, 64, 64, 1, corners.ctypes.data, both, buf.ctypes.data, cnt, None, None), b"exclusive")
    err(lib.cb200_extract_decode_fountain_dev(None, buf.ctypes.data, 64, 64, 1, corners.ctypes.data, both, buf.ctypes.data, cnt, None, None), b"exclusive")
    ifn = cb.FLAG_SHARPEN_IF_NEEDED
    err(lib.cb200_decode_fountain(None, buf.ctypes.data, 1, ifn, buf.ctypes.data, cnt, None, None), b"not to frames")
    err(lib.cb200_decode_fountain_from_dev(None, buf.ctypes.data, 1, ifn, buf.ctypes.data, cnt, None, None), b"not to frames")
    err(lib.cb200_decode_chunks_dev(None, buf.ctypes.data, 1, ifn, buf.ctypes.data, cnt, None), b"not to frames")
    err(lib.cb200_decode_raw_dev(None, buf.ctypes.data, 1, ifn, buf.ctypes.data, None), b"not to frames")
    err(lib.cb200_decode_raw(None, buf.ctypes.data, 1, ifn, buf.ctypes.data, None), b"not to frames")
    err(lib.cb200_decode(None, buf.ctypes.data, 1, ifn, buf.ctypes.data, None, None), b"not to frames")
    err(lib.cb200_decode_cells(None, buf.ctypes.data, 1, ifn, buf.ctypes.data, buf.ctypes.data), b"not to frames")
    err(lib.cb200_decode_chunks_sharpen_dev(None, buf.ctypes.data, 1, ifn, sel.ctypes.data, buf.ctypes.data, cnt, None), b"not to frames")
    err(lib.cb200_decode_fountain_sharpen(None, buf.ctypes.data, 1, ifn, sel.ctypes.data, buf.ctypes.data, cnt, None, None), b"not to frames")
    err(lib.cb200_decode_chunks_sharpen_dev(None, buf.ctypes.data, 1, cb.FLAG_SHARPEN, sel.ctypes.data, buf.ctypes.data, cnt, None), b"per-frame")
    err(lib.cb200_decode_fountain_sharpen(None, buf.ctypes.data, 1, cb.FLAG_SHARPEN, sel.ctypes.data, buf.ctypes.data, cnt, None, None), b"per-frame")
    err(lib.cb200_decode_chunks_sharpen_dev(None, buf.ctypes.data, 1, 0, None, buf.ctypes.data, cnt, None), b"null sharpen")
    err(lib.cb200_decode_fountain_sharpen(None, buf.ctypes.data, 1, 0, None, buf.ctypes.data, cnt, None, None), b"null sharpen")
    err(lib.cb200_decode_fountain_sharpen(None, buf.ctypes.data, 1, 0, sel.ctypes.data, buf.ctypes.data, cnt, None, None), b"null context")


def test_python_selection_must_have_one_entry_per_frame():
    with pytest.raises(cb.Cb200Error):
        cb._selection([True, False], 3)
    assert cb._selection([True, 0, 2], 3).tolist() == [1, 0, 1]


def test_decoder_per_frame_overload_test_compiles():
    subprocess.check_call(["g++", "-std=c++17", "-fsyntax-only", os.path.join(ROOT, "tests", "cpp", "decoder_sharpen_test.cpp")])
