"""The device JPEG decoder's functions (libcimbar_b200/csrc/jpeg_core.cuh: parse, segment decoder, ISLOW IDCT, fancy upsampling,
YCbCr -> RGB, EXIF orientation -- what jpeg.cu's kernels run) compiled for the host and pinned against cv2: every golden JPEG and
every file of the generated matrix decodes to exactly cv2.imread + cvtColor(BGR2RGB), and cb200_jpeg_info gives cv2's size."""
import cv2
import numpy as np
import pytest

import libcimbar_b200 as cb
from libcimbar_b200 import build as cbbuild
from jpeg_matrix import cv2_rgb, golden_files, matrix
from cpu_support import core, decode  # noqa: F401

FILES = golden_files() + matrix()


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
