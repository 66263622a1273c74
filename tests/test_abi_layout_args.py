"""CPU-side checks of cb200_scan_extract_decode_chunks_pictures_dev (camera pictures in the caller's layout): every argument error
comes before any CUDA call and names the picture.  The context is NULL here, so a call whose arguments are all good fails on the
context instead; n > max_frames and null outputs need a context and are checked on the GPU (tests/test_gpu_camera_layouts.py).
Also the Python side: which tensors make a picture and which are refused rather than copied."""
import ctypes as C

import numpy as np
import pytest

import libcimbar_b200 as cb
from libcimbar_b200 import build as cbbuild
from cpu_support import err, good, with_


@pytest.fixture(scope="module", autouse=True)
def built():
    cbbuild.build()


def lib():
    return cb.load_library()


CH = {cb.LAYOUT_RGB: 3, cb.LAYOUT_BGR: 3, cb.LAYOUT_RGBA: 4, cb.LAYOUT_BGRA: 4, cb.LAYOUT_RGB_PLANAR: 1}


def call(pics, n=None, flags=0, null_array=False):
    arr = (cb.Picture * max(1, len(pics)))(*pics)
    out = np.zeros(64, np.uint8)
    st = np.zeros(8, np.int32)
    return lib().cb200_scan_extract_decode_chunks_pictures_dev(None, None if null_array else C.cast(arr, C.c_void_p),
                                                               len(pics) if n is None else n, flags, out.ctypes.data,
                                                               out.ctypes.data, None, st.ctypes.data)


def test_good_arguments_reach_the_context_check():
    err(call(good()), b"null context")
    for lay in CH:                                  # every layout at its tightest pitch
        err(call([cb.Picture(0x1001, 61, 60, 61 * CH[lay], 60 * 61 * CH[lay], lay)]), b"null context")


def test_n_and_the_array():
    err(call(good(), n=-1), b"n < 0")
    err(call(good(), null_array=True), b"null pictures")
    err(call([], n=0, null_array=True), b"null pictures")


@pytest.mark.parametrize("i", [0, 2, 3])
def test_null_data_pointer_is_named(i):
    err(call(with_(i, data=None)), b"picture %d has a null data pointer" % i)


@pytest.mark.parametrize("lay", [-1, 5, 12, 420])
def test_unknown_layout_is_named(lay):
    err(call(with_(1, layout=lay)), b"picture 1 has an unknown layout %d" % lay)


@pytest.mark.parametrize("i,field", [(0, "row_pitch"), (3, "row_pitch"), (2, "plane_pitch"), (1, "plane_pitch")])
def test_negative_pitch_is_named(i, field):
    err(call(with_(i, **{field: -4})), b"picture %d has a negative %s pitch" % (i, field.split("_")[0].encode()))


@pytest.mark.parametrize("bad,index", [((59, 1280), 1), ((1280, 59), 2), ((4500, 4600), 0), ((4600, 4500), 3), ((30, 30), 1)])
def test_size_rule_names_the_picture(bad, index):
    pics = with_(index, h=bad[0], w=bad[1], row_pitch=4 * bad[1], plane_pitch=4 * bad[1] * bad[0])
    err(call(pics), b"picture %d is %d x %d" % (index, bad[1], bad[0]))


def test_the_largest_accepted_sizes_pass():
    pics = [cb.Picture(0x1000, 4600, 4499, 3 * 4600, 0, cb.LAYOUT_BGR), cb.Picture(0x2000, 60, 100, 240, 0, cb.LAYOUT_RGBA)]
    err(call(pics), b"null context")


@pytest.mark.parametrize("i", [0, 1, 2, 3])
def test_row_pitch_below_a_row_is_named(i):
    p = good()[i]
    row = p.w * CH[p.layout]
    err(call(with_(i, row_pitch=row - 1)), b"picture %d has a row pitch of %d bytes, below w x channels = %d" % (i, row - 1, row))
    err(call(with_(i, row_pitch=row)), b"null context")


def test_overlapping_planes_are_named():
    p = good()[2]
    err(call(with_(2, plane_pitch=p.h * p.row_pitch - 1)), b"picture 2 has overlapping planes")
    err(call(with_(2, plane_pitch=p.h * p.row_pitch)), b"null context")
    err(call(with_(0, plane_pitch=5)), b"null context")           # ignored outside the planar layout


def test_pictures_of_4_gb_or_more_are_refused():
    err(call(with_(3, row_pitch=1 << 32)), b"picture 3 spans 4 GB or more")
    err(call(with_(0, row_pitch=(1 << 32) // 959)), b"picture 0 spans 4 GB or more")
    err(call(with_(2, plane_pitch=(1 << 31))), b"picture 2 spans 4 GB or more")


def test_flags_the_ragged_call_refuses():
    err(call(good(), flags=cb.FLAG_SHARPEN | cb.FLAG_SHARPEN_IF_NEEDED), b"exclusive")
    err(call(good(), flags=cb.FLAG_CC_SIMPLE | cb.FLAG_CC_FIT), b"exclusive")


def test_layout_values_are_the_headers():
    import os
    import re
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "cb200.h")).read()
    vals = dict(re.findall(r"#define CB200_(LAYOUT_\w+)\s+(\d+)", hdr))
    assert {k: int(v) for k, v in vals.items()} == {k: getattr(cb, k) for k in vals} and len(vals) == 5


# ---- the Python side: tensors -> descriptors (CPU tensors are refused last, so the stride rules can be checked without a GPU)
def test_tensor_strides_that_do_not_fit_are_refused():
    import torch
    hwc = torch.zeros(100, 120, 3, dtype=torch.uint8)
    with pytest.raises(cb.Cb200Error, match="stride"):
        cb.picture(hwc[:, ::2])                                     # stride(1) == 6
    with pytest.raises(cb.Cb200Error, match="stride"):
        cb.picture(torch.zeros(100, 3, 120, dtype=torch.uint8).permute(0, 2, 1))      # channels not innermost
    with pytest.raises(cb.Cb200Error, match="stride"):
        cb.picture(torch.zeros(3, 120, 100, dtype=torch.uint8).transpose(1, 2))       # planar rows not contiguous
    with pytest.raises(cb.Cb200Error, match="uint8"):
        cb.picture(torch.zeros(100, 120, 3, dtype=torch.float32))
    with pytest.raises(cb.Cb200Error, match="order"):
        cb.picture(torch.zeros(3, 100, 120, dtype=torch.uint8), "bgr")
    with pytest.raises(cb.Cb200Error, match="order"):
        cb.picture(hwc, "yuv")
    with pytest.raises(cb.Cb200Error, match=r"\(h, w, 3 \| 4\)"):
        cb.picture(torch.zeros(100, 120, 2, dtype=torch.uint8))
    # fitting strides (a crop, padded rows) get as far as the device check: nothing is copied
    with pytest.raises(cb.Cb200Error, match="device memory"):
        cb.picture(torch.zeros(100, 130, 4, dtype=torch.uint8)[5:, 3:125])
    with pytest.raises(cb.Cb200Error, match="device memory"):
        cb.picture(torch.zeros(3, 100, 128, dtype=torch.uint8)[:, :, :120])
