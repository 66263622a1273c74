"""CPU-side checks of the enqueue-only camera entry points (cb200_scan_extract_decode_chunks[_ragged]_dev, cb200_camera_transforms):
every argument error comes before any CUDA call, with the messages of the ragged entry points.  The context is NULL here, so a call
whose arguments are all good fails on the context instead; n > max_frames needs a context and is checked on the GPU
(tests/test_gpu_camera_dev.py)."""
import numpy as np
import pytest

import libcimbar_b200 as cb
from libcimbar_b200 import build as cbbuild
from cpu_support import GOOD, batch, err, lib


@pytest.fixture(scope="module", autouse=True)
def built():
    cbbuild.build()


def call(wh, n, flags=0, pictures=True, chunks=True, mask=True, status=True, ragged=True):
    out = np.zeros(64, np.uint8)
    dev = out.ctypes.data                                # stand-in device addresses: never dereferenced before the checks
    whp = None if wh is None else wh.ctypes.data
    args = (dev if chunks else None, dev if mask else None, None, dev if status else None)
    if ragged:
        return lib().cb200_scan_extract_decode_chunks_ragged_dev(None, dev if pictures else None, whp, n, flags, *args)
    return lib().cb200_scan_extract_decode_chunks_dev(None, dev if pictures else None, int(wh[0, 0]), int(wh[0, 1]), n, flags, *args)


def test_good_arguments_reach_the_context_check():
    _, _, wh = batch(GOOD)
    err(call(wh, len(GOOD)), b"null context")
    err(call(wh[:1], 3, ragged=False), b"null context")


def test_negative_n_null_wh_and_null_pictures():
    _, _, wh = batch(GOOD)
    err(call(wh, -1), b"n < 0")
    err(call(wh[:1], -1, ragged=False), b"n < 0")
    err(call(None, len(GOOD)), b"null wh")
    err(call(wh, len(GOOD), pictures=False), b"null pictures")
    err(call(wh[:1], 2, pictures=False, ragged=False), b"null pictures")


@pytest.mark.parametrize("bad,index", [((59, 1280), 1), ((1280, 59), 2), ((4500, 4600), 0), ((30, 30), 1)])
def test_out_of_range_picture_is_named(bad, index):
    shapes = GOOD + [(960, 1280)]
    shapes[index] = bad
    _, _, wh = batch(shapes)
    err(call(wh, len(shapes)), b"picture %d is %d x %d" % (index, bad[1], bad[0]))
    err(call(wh[index:index + 1], 2, ragged=False), b"picture 0 is %d x %d" % (bad[1], bad[0]))


def test_null_outputs_are_refused():
    _, _, wh = batch(GOOD)
    for kw in ({"chunks": False}, {"mask": False}, {"status": False}):
        err(call(wh, len(GOOD), **kw), b"null context")          # the context comes first, as on the ragged entry points
    import ctypes as C
    h = C.c_void_p(1)                                             # a non-null context that is never dereferenced before the checks
    out = np.zeros(64, np.uint8)
    for args in ((None, out.ctypes.data, out.ctypes.data), (out.ctypes.data, None, out.ctypes.data), (out.ctypes.data, out.ctypes.data, None)):
        rc = lib().cb200_scan_extract_decode_chunks_ragged_dev(h, out.ctypes.data, wh.ctypes.data, len(GOOD), 0, args[0], args[1], None, args[2])
        err(rc, b"null output")


def test_exclusive_flags_are_refused():
    _, _, wh = batch(GOOD)
    err(call(wh, len(GOOD), flags=cb.FLAG_SHARPEN | cb.FLAG_SHARPEN_IF_NEEDED), b"exclusive")
    err(call(wh, len(GOOD), flags=cb.FLAG_CC_SIMPLE | cb.FLAG_CC_FIT), b"exclusive")


def test_camera_transforms_arguments():
    out = np.zeros(9, np.float64)
    err(lib().cb200_camera_transforms(None, out.ctypes.data, 1), b"bad arguments")
    err(lib().cb200_camera_transforms(None, None, 1), b"bad arguments")
