"""Argument checks of the auto-mode call (cb200_detect_scan_extract_decode_chunks_dev): every refusal is CB200_ERR_ARG with a
message naming it, before any CUDA call.  The checks that need no context come first, so they run here with a list of NULL contexts;
the ones that read a context (distinct modes, one device and stream, no CCM chain, no camera plans, n against max_frames) need real
contexts and run on the GPU, where the refused call must launch nothing."""
import ctypes as C

import numpy as np
import pytest

import libcimbar_b200 as cb
from libcimbar_b200 import build as cbbuild
from cpu_support import GOOD, batch, err, lib


@pytest.fixture(scope="module", autouse=True)
def built():
    cbbuild.build()


OUT = np.zeros(64, np.uint8)
DEV = OUT.ctypes.data                                   # stand-in device addresses: never dereferenced before the checks


def call(ctxs, n_modes, wh, n, flags=0, pictures=True, chunks=True, mask=True, status=True, mode=True, list_ok=True):
    hs = (C.c_void_p * max(len(ctxs), 1))(*ctxs)
    whp = None if wh is None else wh.ctypes.data
    return lib().cb200_detect_scan_extract_decode_chunks_dev(hs if list_ok else None, n_modes, DEV if pictures else None, whp, n, flags,
                                                             DEV if chunks else None, DEV if mask else None, DEV if status else None,
                                                             DEV if mode else None, None)


NULLS = [None] * 4


def test_good_arguments_reach_the_context_checks():
    _, _, wh = batch(GOOD)
    err(call(NULLS, 4, wh, len(GOOD)), b"context 0 is null")
    err(call(NULLS, 4, wh, len(GOOD), list_ok=False), b"null context list")


@pytest.mark.parametrize("n_modes", [0, -1, 6])
def test_n_modes_out_of_range(n_modes):
    _, _, wh = batch(GOOD)
    err(call([None] * 6, n_modes, wh, len(GOOD)), b"n_modes = %d: between 1 and 5" % n_modes)


def test_flags_are_checked_first():
    _, _, wh = batch(GOOD)
    err(call(NULLS, 4, wh, len(GOOD), flags=cb.FLAG_SHARPEN | cb.FLAG_SHARPEN_IF_NEEDED), b"exclusive")
    err(call(NULLS, 4, wh, len(GOOD), flags=cb.FLAG_CC_SIMPLE | cb.FLAG_CC_FIT), b"CC_SIMPLE and CC_FIT are exclusive")


def test_negative_n_null_wh_and_null_pictures():
    _, _, wh = batch(GOOD)
    err(call(NULLS, 4, wh, -1), b"n < 0")
    err(call(NULLS, 4, None, len(GOOD)), b"null wh")
    err(call(NULLS, 4, wh, len(GOOD), pictures=False), b"null pictures")


@pytest.mark.parametrize("bad,index", [((59, 1280), 1), ((1280, 59), 2), ((4500, 4600), 0), ((30, 30), 1)])
def test_out_of_range_picture_is_named(bad, index):
    shapes = GOOD + [(960, 1280)]
    shapes[index] = bad
    _, _, wh = batch(shapes)
    err(call(NULLS, 4, wh, len(shapes)), b"picture %d is %d x %d" % (index, bad[1], bad[0]))


@pytest.mark.parametrize("missing", ["chunks", "mask", "status", "mode"])
def test_null_outputs_are_refused(missing):
    _, _, wh = batch(GOOD)
    err(call(NULLS, 4, wh, len(GOOD), **{missing: False}), b"null output")


def test_a_null_context_is_named():
    _, _, wh = batch(GOOD)
    fake = C.c_void_p(1).value                          # never dereferenced: the null entry is found first
    err(call([fake, fake, None, fake], 4, wh, len(GOOD)), b"context 2 is null")


# ---- the checks that read the contexts
def _dev_call(ctxs, n, flags=0):
    import torch
    wh = np.array([(1280, 960)] * n, np.int32).reshape(-1, 2)
    pics = torch.zeros(max(n, 1) * 1280 * 960 * 3, dtype=torch.uint8, device="cuda")
    chunks = torch.zeros(max(n, 1) * 8750, dtype=torch.uint8, device="cuda")
    words = torch.zeros(max(n, 1) * 8, dtype=torch.int32, device="cuda")
    hs = (C.c_void_p * len(ctxs))(*[c._h.value for c in ctxs])
    before = cb.launch_count()
    rc = lib().cb200_detect_scan_extract_decode_chunks_dev(hs, len(ctxs), pics.data_ptr(), wh.ctypes.data, n, flags, chunks.data_ptr(),
                                                           words.data_ptr(), words.data_ptr(), words.data_ptr(), None)
    assert cb.launch_count() == before                  # refused before any launch
    return rc


@pytest.mark.gpu
def test_context_refusals():
    import torch
    st, side = torch.cuda.Stream(), torch.cuda.Stream()
    ctx = {m: cb.Context(m, max_frames=4) for m in (68, 4, 67)}
    for c in ctx.values():
        c.set_stream(st.cuda_stream)
    try:
        twin = cb.Context(68, max_frames=4)
        twin.set_stream(st.cuda_stream)
        err(_dev_call([ctx[68], ctx[4], twin], 2), b"contexts 0 and 2 are both mode 68")
        twin.close()
        err(_dev_call([ctx[68], cb.Context(4, max_frames=4)], 2), b"context 1 is on another stream than context 0")   # its own stream
        ctx[4].set_stream(side.cuda_stream)
        err(_dev_call([ctx[68], ctx[4]], 2), b"context 1 is on another stream than context 0")
        ctx[4].set_stream(st.cuda_stream)
        err(_dev_call([ctx[68], ctx[4], ctx[67]], 5), b"n = 5 > max_frames = 4 of context 0")
        big = cb.Context(66, max_frames=8)
        big.set_stream(st.cuda_stream)
        err(_dev_call([big, ctx[68]], 6), b"n = 6 > max_frames = 4 of context 1")
        big.close()
        # a context with a live camera plan
        wh = np.array([(1280, 960)], np.int32)
        pics = torch.zeros(1280 * 960 * 3, dtype=torch.uint8, device="cuda")
        chunks = torch.zeros(7500, dtype=torch.uint8, device="cuda")
        words = torch.zeros(4, dtype=torch.int32, device="cuda")
        plan = ctx[4].camera_plan(wh, 0, pics.data_ptr(), chunks.data_ptr(), words.data_ptr(), None, words.data_ptr())
        err(_dev_call([ctx[68], ctx[4]], 1), b"context 1 has live camera plans")
        plan.close()
        assert _dev_call([ctx[68], ctx[4]], 0) == 0     # nothing to do, but every check passed
        torch.cuda.synchronize()
    finally:
        for c in ctx.values():
            c.close()


@pytest.mark.gpu
def test_chained_context_is_refused():
    import torch
    st = torch.cuda.Stream()
    a, b = cb.Context(68, max_frames=2), cb.Context(4, max_frames=2)
    a.set_stream(st.cuda_stream)
    b.set_stream(st.cuda_stream)
    try:
        b.ccm_chain_root_create(1)
        b.ccm_chain_attach(0, 1)
        err(_dev_call([a, b], 1), b"context 1 is linked to a CCM chain")
    finally:
        a.close(); b.close()
