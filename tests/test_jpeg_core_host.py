"""The device JPEG decoder's functions (libcimbar_b200/csrc/jpeg_core.cuh: parse, segment decoder, ISLOW IDCT, fancy upsampling,
YCbCr -> RGB, EXIF orientation -- what jpeg.cu's kernels run) compiled for the host and pinned against cv2: every golden JPEG and
every file of the generated matrix decodes to exactly cv2.imread + cvtColor(BGR2RGB), and cb200_jpeg_info gives cv2's size."""
import ctypes as C
import os
import subprocess

import cv2
import numpy as np
import pytest

import libcimbar_b200 as cb
from libcimbar_b200 import build as cbbuild
from jpeg_matrix import cv2_rgb, golden_files, matrix

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FILES = golden_files() + matrix()


@pytest.fixture(scope="module")
def core(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("jpeg_core") / "jpeg_core_host.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-shared", "-fPIC", "-o", so, os.path.join(ROOT, "tests", "cpp", "jpeg_core_host.cpp")])
    lib = C.CDLL(so)
    lib.jc_decode.argtypes = [C.c_char_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_char_p, C.c_int]
    lib.jc_info.argtypes = [C.c_char_p, C.c_uint64, C.c_void_p, C.c_char_p, C.c_int]
    return lib


def decode(core, data, like=None):
    want = cv2_rgb(data if like is None else like)
    out = np.zeros(want.size + 16, np.uint8)
    wh = np.zeros(2, np.int32)
    why = C.create_string_buffer(256)
    rc = core.jc_decode(data, len(data), out.ctypes.data, out.size, wh.ctypes.data, why, 256)
    return rc, why.value.decode(), wh, out, want


def test_premise_the_matrix_covers_the_layouts():
    names = [n for n, _ in FILES]
    assert len(names) == 9 + 64 + 2 + 1 + 8
    assert any(n.startswith("prog_420") for n in names) and any(n.startswith("base_440") for n in names)


@pytest.mark.parametrize("name,data", FILES, ids=[n for n, _ in FILES])
def test_decodes_like_cv2(core, name, data):
    rc, why, wh, out, want = decode(core, data)
    assert rc == 0, why
    h, w = want.shape[:2]
    assert (wh[0], wh[1]) == (w, h)
    got = out[:want.size].reshape(want.shape)
    assert np.array_equal(got, want), (name, int(np.count_nonzero(got != want)))


@pytest.mark.parametrize("name,data", FILES, ids=[n for n, _ in FILES])
def test_info_agrees_with_cv2(name, data):
    cbbuild.build()
    h, w = cv2_rgb(data).shape[:2]
    assert cb.jpeg_info(data) == (w, h)


def test_exif_orientations_differ():
    """premise: the eight PIL files do exercise eight different orientations in cv2"""
    pics = [cv2_rgb(d) for n, d in FILES if n.startswith("exif_")]
    assert len({(p.shape, p.tobytes()) for p in pics}) == 8


def test_corrupt_data_is_reported(core):
    data = dict(FILES)["base_420_q95_opt0_rst0"]
    rc, _, _, _, _ = decode(core, data[:len(data) // 2], data)
    assert rc == -2
    # a run of 32 one bits (FF 00 stuffed four times) in the data cannot be decoded: no Huffman code is all ones
    sos = data.index(b"\xff\xda")
    mid = sos + (len(data) - sos) // 2
    bad = data[:mid] + b"\xff\x00" * 4 + data[mid + 8:]
    rc, _, _, _, _ = decode(core, bad, data)
    assert rc == -2
