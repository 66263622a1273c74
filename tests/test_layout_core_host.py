"""The per-layout pixel fetch of the camera kernels (libcimbar_b200/csrc/layout_core.cuh) compiled for the host and compared with
numpy and cv2: the gray k_scan_blur4 takes (byte fetch and word path) is cvtColor(RGB2GRAY) of the packed RGB copy, and the tap
pairs k_deskew reads are that copy's pixels, in every layout, at odd widths, unaligned bases and padded pitches.  The GPU test
(tests/test_gpu_camera_layouts.py) compares the whole camera call."""
import ctypes as C

import cv2
import numpy as np
import pytest

import libcimbar_b200 as cb
from host_harness import build_harness

LAYOUTS = {"rgb": cb.LAYOUT_RGB, "bgr": cb.LAYOUT_BGR, "rgba": cb.LAYOUT_RGBA, "bgra": cb.LAYOUT_BGRA, "planar": cb.LAYOUT_RGB_PLANAR}


@pytest.fixture(scope="module")
def core(tmp_path_factory):
    lib = build_harness(tmp_path_factory, "layout_core_host")
    lib.lc_gray.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int64, C.c_int64, C.c_int, C.c_int, C.c_void_p]
    lib.lc_taps.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int64, C.c_int64, C.c_int, C.c_void_p, C.c_int, C.c_void_p]
    lib.lc_picture_abi.argtypes = [C.c_void_p]
    return lib


def place(rgb, name, base_off, pad):
    """rgb (h, w, 3) in layout `name` inside a buffer of 0xFF bytes: the picture starts base_off bytes in, its rows `pad` bytes
    longer than they need to be (planes: one padded row more).  Returns (buffer, offset, row pitch, plane pitch)"""
    h, w, _ = rgb.shape
    if name == "planar":
        pitch = w + pad
        plane = (h + 1) * pitch
        buf = np.full(base_off + 3 * plane + 16, 0xFF, np.uint8)
        for k in range(3):
            v = buf[base_off + k * plane: base_off + k * plane + h * pitch].reshape(h, pitch)
            v[:, :w] = rgb[:, :, k]
        return buf, base_off, pitch, plane
    conv = {"rgb": rgb, "bgr": cv2.cvtColor(rgb, cv2.COLOR_RGB2BGR), "rgba": cv2.cvtColor(rgb, cv2.COLOR_RGB2RGBA),
            "bgra": cv2.cvtColor(rgb, cv2.COLOR_RGB2BGRA)}[name]
    ch = conv.shape[2]
    if ch == 4:
        conv = conv.copy()
        conv[:, :, 3] = np.random.default_rng(5).integers(0, 256, (h, w), dtype=np.uint8)     # the alpha must not matter
    pitch = w * ch + pad
    buf = np.full(base_off + h * pitch + 16, 0xFF, np.uint8)
    buf[base_off: base_off + h * pitch].reshape(h, pitch)[:, :w * ch] = conv.reshape(h, w * ch)
    return buf, base_off, pitch, 0


CASES = [(37, 61, 0, 0), (40, 64, 1, 3), (33, 127, 2, 5), (24, 96, 3, 8), (17, 250, 0, 4), (29, 66, 1, 1)]


@pytest.mark.parametrize("name", list(LAYOUTS))
@pytest.mark.parametrize("h,w,base_off,pad", CASES)
def test_gray_is_cvtcolor_of_the_rgb_copy(core, name, h, w, base_off, pad):
    rng = np.random.default_rng(h * 1000 + w)
    rgb = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    want = cv2.cvtColor(rgb, cv2.COLOR_RGB2GRAY)
    buf, off, pitch, plane = place(rgb, name, base_off, pad)
    for words in (0, 1):
        got = np.zeros((h, w), np.uint8)
        core.lc_gray(buf.ctypes.data + off, w, h, pitch, plane, LAYOUTS[name], words, got.ctypes.data)
        assert np.array_equal(got, want), (name, words)


@pytest.mark.parametrize("name", list(LAYOUTS))
@pytest.mark.parametrize("h,w,base_off,pad", CASES)
def test_tap_pairs_are_the_rgb_copys_pixels(core, name, h, w, base_off, pad):
    rng = np.random.default_rng(h * 7 + w)
    rgb = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    buf, off, pitch, plane = place(rgb, name, base_off, pad)
    cy = [(c, y) for y in (0, h // 2, h - 1) for c in (0, 1, 2, 3, w // 2, w - 3, w - 2)]      # the last pair of the last row too
    cy += [(int(rng.integers(0, w - 1)), int(rng.integers(0, h))) for _ in range(200)]
    cy = np.array(cy, np.int32)
    got = np.zeros((len(cy), 6), np.uint8)
    core.lc_taps(buf.ctypes.data + off, w, h, pitch, plane, LAYOUTS[name], cy.ctypes.data, len(cy), got.ctypes.data)
    want = np.concatenate([rgb[cy[:, 1], cy[:, 0]], rgb[cy[:, 1], cy[:, 0] + 1]], axis=1)
    assert np.array_equal(got, want), name


def test_picture_struct_matches_the_c_header(core):
    out = (C.c_int64 * 7)()
    core.lc_picture_abi(out)
    P = cb.Picture
    assert list(out) == [C.sizeof(P), P.data.offset, P.w.offset, P.h.offset, P.row_pitch.offset, P.plane_pitch.offset, P.layout.offset]
