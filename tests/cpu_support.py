"""Helpers shared by the CPU test files (and the GPU tests that reuse their inputs).  Test infrastructure only.  A fixture defined
here reaches a test file by import (`from cpu_support import core  # noqa: F401`)."""
import ctypes as C
import subprocess

import cv2
import numpy as np
import pytest

import libcimbar_b200 as cb
import oracle_lib as ol
from host_harness import build_harness
from jpeg_matrix import cv2_rgb, golden_files


# ------------------------------------------------------------------------------------------------ the ragged and layout ABI checks
LIB = None


def lib():
    global LIB
    if LIB is None:
        LIB = cb.load_library()
    return LIB


def err(rc, text):
    msg = lib().cb200_last_error()
    assert rc == -1 and text in msg, msg


def batch(shapes):
    """host pictures of the given (h, w), their pointer array and wh"""
    pics = [np.zeros((h, w, 3), np.uint8) for h, w in shapes]
    ptrs = (C.c_void_p * len(pics))(*[p.ctypes.data for p in pics])
    wh = np.array([(w, h) for h, w in shapes], np.int32).reshape(-1, 2)
    return pics, ptrs, wh


GOOD = [(960, 1280), (1280, 960), (637, 955)]


def good():
    """descriptors of four well-formed pictures (stand-in addresses: never dereferenced before the checks)"""
    return [cb.Picture(0x10000, 1280, 960, 3 * 1280, 0, cb.LAYOUT_BGR), cb.Picture(0x20001, 955, 637, 4 * 955 + 9, 0, cb.LAYOUT_RGBA),
            cb.Picture(0x30003, 960, 1280, 1024, 1024 * 1300, cb.LAYOUT_RGB_PLANAR), cb.Picture(0x40000, 640, 480, 4 * 640, 0, cb.LAYOUT_BGRA)]


def with_(i, **kw):
    pics = good()
    for k, v in kw.items():
        setattr(pics[i], k, v)
    return pics


# ------------------------------------------------------------------------------------------------ JPEG files
PHOTO = dict(golden_files())["6bit__4_30_f0_627.jpg"]


@pytest.fixture(scope="module")
def core(tmp_path_factory):
    lib = build_harness(tmp_path_factory, "jpeg_core_host")
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


def decode_wide(core, data):
    """(rc, wide, rgb or None) of the host build's jc_decode_wide"""
    core.jc_decode_wide.argtypes = [C.c_char_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_char_p, C.c_int, C.c_void_p]
    wh = np.zeros(2, np.int32)
    why = C.create_string_buffer(256)
    assert core.jc_info(data, len(data), wh.ctypes.data, why, 256) == 0, why.value
    out = np.zeros(3 * int(wh[0]) * int(wh[1]), np.uint8)
    wide = np.zeros(1, np.int32)
    rc = core.jc_decode_wide(data, len(data), out.ctypes.data, out.size, wh.ctypes.data, why, 256, wide.ctypes.data)
    return rc, int(wide[0]), out.reshape(wh[1], wh[0], 3) if rc == 0 else None


# ------------------------------------------------------------------------------------------------ pictures, models and harness runs
def pictures():
    """camera pictures, clean frames, rotations, shrunken and enlarged copies, and pictures without a code"""
    out = []
    for s in ("6bit/4_30_f0_627.jpg", "6bit/4_30_f2_734.jpg", "6bit/4_30_f2_246.jpg", "6bit/4_30_f1_360.jpg",
              "6bit/4color_ecc30_fountain_0.png", "b/ex2434.jpg", "b/tr_0.png"):
        out.append((s, ol.load_sample(s)))
    cam = out[0][1]
    out.append(("627 rot90", np.ascontiguousarray(np.rot90(cam))))
    out.append(("627 rot180", np.ascontiguousarray(np.rot90(cam, 2))))
    out.append(("627 x0.6", cv2.resize(cam, None, fx=0.6, fy=0.6, interpolation=cv2.INTER_AREA)))
    out.append(("627 x1.7 (blur 5)", cv2.resize(cam, None, fx=1.7, fy=1.7)))
    out.append(("627 cropped (anchor cut off)", np.ascontiguousarray(cam[:, 260:])))
    out.append(("627 odd width (1277 x 957: no 4-byte aligned rows)", np.ascontiguousarray(cam[2:959, 1:1278])))
    rng = np.random.default_rng(3)
    out.append(("noise", rng.integers(0, 256, (480, 640, 3), dtype=np.uint8)))
    out.append(("black", np.zeros((300, 400, 3), np.uint8)))
    pad = np.full((1400, 1500, 3), 40, np.uint8)
    pad[150:1174, 300:1324] = ol.load_sample("b/tr_1.png")
    out.append(("clean frame on a dark table", pad))
    return out


def camera_view(frame, quad, size):
    """a synthetic camera image: the 1024x1024 frame seen in perspective inside a larger picture (made with cv2)"""
    import cv2
    h, w = frame.shape[:2]
    src = np.float32([[0, 0], [w, 0], [0, h], [w, h]])
    M = cv2.getPerspectiveTransform(src, np.float32(quad))
    return cv2.warpPerspective(frame, M, size, flags=cv2.INTER_LINEAR)


U = np.uint32
NT = 128


def prmt(a, b, sel):
    """__byte_perm(a, b, sel) on arrays of uint32."""
    a = a.astype(np.uint64); b = b.astype(np.uint64)
    src = a | (b << np.uint64(32))
    out = np.zeros_like(a)
    for i in range(4):
        n = (sel >> (4 * i)) & 0x7
        out |= ((src >> np.uint64(8 * n)) & np.uint64(0xFF)) << np.uint64(8 * i)
    return out.astype(U)


def vmaxu2(a, b):
    lo = np.maximum(a & U(0xFFFF), b & U(0xFFFF)); hi = np.maximum(a >> U(16), b >> U(16))
    return (lo | (hi << U(16))).astype(U)


def vminu2(a, b):
    lo = np.minimum(a & U(0xFFFF), b & U(0xFFFF)); hi = np.minimum(a >> U(16), b >> U(16))
    return (lo | (hi << U(16))).astype(U)


def run(exe, cand, of, receivers, group):
    n, k = len(cand), len(group)
    data = np.concatenate([np.array([n, receivers, k], np.int32), np.asarray(group, np.int32), np.asarray(cand, np.uint32).view(np.int32),
                           np.asarray(of, np.int32)]).tobytes()
    out = np.frombuffer(subprocess.run([exe], input=data, stdout=subprocess.PIPE, check=True).stdout, np.int32)
    at = 0
    slots, counts, maps = [], [], []
    for _ in range(k):
        m = int(out[at]); slots.append(out[at + 1:at + 1 + m]); at += 1 + m
    for _ in range(k):
        counts.append(int(out[at])); m = int(out[at + 1]); maps.append(out[at + 2:at + 2 + m]); at += 2 + m
    pos = out[at:].reshape(k, n)
    assert at + k * n == len(out)
    return slots, counts, maps, pos
