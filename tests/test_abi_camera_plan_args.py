"""CPU-side checks of cb200_camera_plan_create: every argument error comes before any CUDA call, with the checks and messages of
cb200_scan_extract_decode_chunks_ragged_dev and a picture named by its index, plus the plan's own refusals (no pictures, no place for
the plan).  The context is NULL here, so a call whose arguments are all good fails on the context instead; a context attached to a
CCM chain, n > max_frames and buffers frozen by a live plan need a context and are checked on the GPU
(tests/test_gpu_camera_plan.py)."""
import ctypes as C

import numpy as np
import pytest

import libcimbar_b200 as cb
from libcimbar_b200 import build as cbbuild
from test_abi_ragged_args import GOOD, batch, err, lib


@pytest.fixture(scope="module", autouse=True)
def built():
    cbbuild.build()


def create(wh, n, flags=0, ctx=None, pictures=True, chunks=True, mask=True, status=True, out=True):
    buf = np.zeros(64, np.uint8)
    dev = buf.ctypes.data                                # stand-in device addresses: never dereferenced before the checks
    h = C.c_void_p()
    whp = None if wh is None else wh.ctypes.data
    return lib().cb200_camera_plan_create(ctx, whp, n, flags, dev if pictures else None, dev if chunks else None, dev if mask else None,
                                          None, dev if status else None, C.byref(h) if out else None)


def test_good_arguments_reach_the_context_check():
    _, _, wh = batch(GOOD)
    err(create(wh, len(GOOD)), b"null context")


def test_negative_n_null_wh_and_null_pictures():
    _, _, wh = batch(GOOD)
    err(create(wh, -1), b"n < 0")
    err(create(None, len(GOOD)), b"null wh")
    err(create(wh, len(GOOD), pictures=False), b"null pictures")


def test_no_pictures_is_refused():
    _, _, wh = batch(GOOD)
    err(create(wh, 0), b"n = 0")


def test_null_plan_is_refused():
    _, _, wh = batch(GOOD)
    err(create(wh, len(GOOD), out=False), b"null plan")


@pytest.mark.parametrize("bad,index", [((59, 1280), 1), ((1280, 59), 2), ((4500, 4600), 0), ((30, 30), 1)])
def test_out_of_range_picture_is_named(bad, index):
    shapes = GOOD + [(960, 1280)]
    shapes[index] = bad
    _, _, wh = batch(shapes)
    err(create(wh, len(shapes)), b"picture %d is %d x %d" % (index, bad[1], bad[0]))


def test_null_outputs_are_refused():
    _, _, wh = batch(GOOD)
    fake = C.c_void_p(1)                                 # a non-null context that is never dereferenced before these checks
    for kw in ({"chunks": False}, {"mask": False}, {"status": False}):
        err(create(wh, len(GOOD), **kw), b"null context")
        err(create(wh, len(GOOD), ctx=fake, **kw), b"null output")


@pytest.mark.parametrize("flags", ["SHARPEN|SHARPEN_IF_NEEDED", "CC_SIMPLE|CC_FIT"])
def test_exclusive_flags_are_refused(flags):
    _, _, wh = batch(GOOD)
    f = 0
    for name in flags.split("|"):
        f |= getattr(cb, "FLAG_" + name)
    err(create(wh, len(GOOD), flags=f), b"exclusive")


def test_plan_calls_refuse_a_null_plan():
    g = C.c_void_p()
    err(lib().cb200_camera_plan_launch(None), b"null plan")
    err(lib().cb200_camera_plan_graph(None, C.byref(g)), b"bad arguments")
    assert lib().cb200_camera_plan_destroy(None) == 0
