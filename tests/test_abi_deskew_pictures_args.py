"""CPU-side checks of cb200_deskew_pictures_dev (the deskew of pictures in the caller's layout): the pictures are checked as the
pictures camera call checks them, with its messages, before the context and any CUDA call.  The context is NULL here, so a call
whose pictures are all good fails on the context instead; a singular transform needs a context and is checked on the GPU
(tests/test_gpu_deskew_corpus.py)."""
import ctypes as C

import numpy as np
import pytest

import libcimbar_b200 as cb
from libcimbar_b200 import build as cbbuild
from cpu_support import err, good, with_

M9 = np.tile(np.eye(3).reshape(9), 8)
OUT = np.zeros(64, np.uint8)


@pytest.fixture(scope="module", autouse=True)
def built():
    cbbuild.build()


def call(pics, n=None, null_array=False, m9=M9.ctypes.data, dst=OUT.ctypes.data):
    arr = (cb.Picture * max(1, len(pics)))(*pics)
    return cb.load_library().cb200_deskew_pictures_dev(None, None if null_array else C.cast(arr, C.c_void_p),
                                                       len(pics) if n is None else n, m9, dst)


def test_good_arguments_reach_the_context_check():
    err(call(good()), b"null context")
    err(call(good(), m9=None), b"null context")
    err(call(good(), dst=None), b"null context")
    err(call([], n=0), b"null context")
    for lay, ch in ((cb.LAYOUT_RGB, 3), (cb.LAYOUT_BGR, 3), (cb.LAYOUT_RGBA, 4), (cb.LAYOUT_BGRA, 4), (cb.LAYOUT_RGB_PLANAR, 1)):
        err(call([cb.Picture(0x1001, 61, 60, 61 * ch, 60 * 61 * ch, lay)]), b"null context")


def test_n_and_the_array():
    err(call(good(), n=-1), b"n < 0")
    err(call(good(), null_array=True), b"null pictures")
    err(call([], n=0, null_array=True), b"null pictures")


@pytest.mark.parametrize("i", [0, 3])
def test_null_data_pointer_is_named(i):
    err(call(with_(i, data=None)), b"picture %d has a null data pointer" % i)


@pytest.mark.parametrize("lay", [-1, 5])
def test_unknown_layout_is_named(lay):
    err(call(with_(2, layout=lay)), b"picture 2 has an unknown layout %d" % lay)


@pytest.mark.parametrize("i,field", [(1, "row_pitch"), (2, "plane_pitch")])
def test_negative_pitch_is_named(i, field):
    err(call(with_(i, **{field: -4})), b"picture %d has a negative %s pitch" % (i, field.split("_")[0].encode()))


@pytest.mark.parametrize("bad,index", [((59, 1280), 1), ((1280, 59), 2), ((4500, 4600), 0), ((2, 2), 3), ((5, 7), 1)])
def test_the_scan_size_rule_holds_here_too(bad, index):
    """tiny and huge pictures are refused by name (the uniform cb200_deskew / cb200_deskew_dev take 2 x 2 and up)"""
    pics = with_(index, h=bad[0], w=bad[1], row_pitch=4 * bad[1], plane_pitch=4 * bad[1] * bad[0])
    err(call(pics), b"picture %d is %d x %d" % (index, bad[1], bad[0]))


def test_the_largest_accepted_sizes_pass():
    pics = [cb.Picture(0x1000, 4600, 4499, 3 * 4600, 0, cb.LAYOUT_BGR), cb.Picture(0x2000, 60, 100, 240, 0, cb.LAYOUT_RGBA)]
    err(call(pics), b"null context")


@pytest.mark.parametrize("i", [0, 1, 2, 3])
def test_row_pitch_below_a_row_is_named(i):
    p = good()[i]
    row = p.w * {cb.LAYOUT_BGR: 3, cb.LAYOUT_RGBA: 4, cb.LAYOUT_RGB_PLANAR: 1, cb.LAYOUT_BGRA: 4}[p.layout]
    err(call(with_(i, row_pitch=row - 1)), b"picture %d has a row pitch of %d bytes, below w x channels = %d" % (i, row - 1, row))
    err(call(with_(i, row_pitch=row)), b"null context")


def test_overlapping_planes_are_named():
    p = good()[2]
    err(call(with_(2, plane_pitch=p.h * p.row_pitch - 1)), b"picture 2 has overlapping planes")
    err(call(with_(2, plane_pitch=p.h * p.row_pitch)), b"null context")


def test_pictures_of_4_gb_or_more_are_refused():
    """k_deskew's byte offsets inside a picture are 32-bit"""
    err(call(with_(3, row_pitch=1 << 32)), b"picture 3 spans 4 GB or more")
    err(call(with_(0, row_pitch=(1 << 32) // 959)), b"picture 0 spans 4 GB or more")
    err(call(with_(2, plane_pitch=(1 << 31))), b"picture 2 spans 4 GB or more")
