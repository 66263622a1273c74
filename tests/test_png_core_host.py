"""The device PNG decoder's functions (libcimbar_b200/csrc/png_core.cuh: chunk walk, IDAT CRC pieces, inflate, unfilter, expand --
what png.cu's kernels run) compiled for the host and pinned against cv2: every golden PNG and every file of the generated matrix
decodes to exactly cv2.imread + cvtColor(BGR2RGB), and cb200_png_info gives cv2's size for each file the camera path takes."""
import ctypes as C

import numpy as np
import pytest

import libcimbar_b200 as cb
from libcimbar_b200 import build as cbbuild
from png_matrix import cv2_rgb, golden_files, matrix, premise
from host_harness import build_harness

FILES = golden_files() + matrix()


@pytest.fixture(scope="module")
def core(tmp_path_factory):
    lib = build_harness(tmp_path_factory, "png_core_host")
    lib.pc_decode.argtypes = [C.c_char_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_char_p, C.c_int]
    lib.pc_info.argtypes = [C.c_char_p, C.c_uint64, C.c_void_p, C.c_char_p, C.c_int]
    return lib


def decode(core, data, size_of=None):
    """(rc, why, (w, h), rgb or None) of the host build"""
    want = cv2_rgb(size_of if size_of is not None else data)
    n = want.size if want is not None else 3 * 4500 * 4500
    out = np.zeros(n + 16, np.uint8)
    wh = np.zeros(2, np.int32)
    why = C.create_string_buffer(256)
    rc = core.pc_decode(data, len(data), out.ctypes.data, out.size, wh.ctypes.data, why, 256)
    rgb = out[:3 * wh[0] * wh[1]].reshape(wh[1], wh[0], 3) if rc == 0 else None
    return rc, why.value.decode(), (int(wh[0]), int(wh[1])), rgb


def test_premise_the_matrix_covers_every_block_filter_colour_and_depth():
    p = premise(FILES)
    assert p["blocks"] == {0, 1, 2}
    assert p["filters"] == {0, 1, 2, 3, 4}
    assert p["colour"] == {(0, 1), (0, 2), (0, 4), (0, 8), (0, 16), (2, 8), (2, 16), (3, 1), (3, 2), (3, 4), (3, 8), (4, 8), (4, 16),
                           (6, 8), (6, 16)}
    names = [n for n, _ in FILES]
    assert len([n for n in names if n.startswith("cv2_frame_c")]) == 50 and len([n for n in names if n.startswith("cv2_photo_c")]) == 50
    # the eXIf files do exercise different orientations in cv2
    pics = [cv2_rgb(d) for n, d in FILES if n.startswith("exif_")]
    assert len({(p.shape, p.tobytes()) for p in pics}) == 4


@pytest.mark.parametrize("name,data", FILES, ids=[n for n, _ in FILES])
def test_decodes_like_cv2(core, name, data):
    want = cv2_rgb(data)
    assert want is not None, name
    rc, why, wh, got = decode(core, data)
    assert rc == 0, why
    assert wh == (want.shape[1], want.shape[0])
    assert np.array_equal(got, want), (name, int(np.count_nonzero(got != want)))


@pytest.mark.parametrize("name,data", FILES, ids=[n for n, _ in FILES])
def test_info_agrees_with_cv2(name, data):
    cbbuild.build()
    h, w = cv2_rgb(data).shape[:2]
    if min(w, h) < 60:
        with pytest.raises(cb.Cb200Error, match="smaller than 60"):
            cb.png_info(data)
    else:
        assert cb.png_info(data) == (w, h)
