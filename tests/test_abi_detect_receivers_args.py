"""Argument checks of the auto mode for receivers (cb200_detect_scan_extract_decode_chunks_receivers_dev): every refusal is
CB200_ERR_ARG with a message naming the violation -- and its picture or mode -- before any CUDA call.  The checks that need no
context come first, so they run here with a list of NULL contexts: a call whose other arguments are all good fails on "context 0 is
null".  The ones that read the contexts (distinct modes, one stream, no CCM chain, no live plans, max_frames) run on the GPU, where
the refused call must launch nothing."""
import ctypes as C

import numpy as np
import pytest

import libcimbar_b200 as cb
from libcimbar_b200 import build as cbbuild


@pytest.fixture(scope="module", autouse=True)
def built():
    cbbuild.build()


def lib():
    return cb.load_library()


BUF = np.zeros(1 << 16, np.uint8)
P = BUF.ctypes.data                                     # stand-in addresses: never dereferenced before the checks
ENTRY = 40                                              # bytes of one cb200_receiver_state
GOOD_OF = np.array([0, 2, 1, 2], np.int32)
GOOD_CAND = np.array([0b1111, 0b0010, 0b1001, 0b0100], np.uint32)


def pictures(n, w=1280, h=960):
    return (cb.Picture * max(1, n))(*[cb.Picture(P, w, h, 3 * w, 0, cb.LAYOUT_RGB) for _ in range(n)])


def tables(n_modes, count=3, gap=None):
    """n_modes state tables of `count` entries, `gap` bytes apart (default: just not overlapping)"""
    step = ENTRY * count if gap is None else gap
    return [P + 64 + k * step for k in range(n_modes)]


def call(n_modes=4, n=4, cand=GOOD_CAND, of=GOOD_OF, count=3, states="good", flags=0, pics=None, ctxs=None, outputs=(P, P, P, P),
         list_ok=True):
    ctxs = [None] * max(n_modes, 1) if ctxs is None else ctxs
    hs = (C.c_void_p * len(ctxs))(*ctxs)
    candp = None if cand is None else np.ascontiguousarray(cand, np.uint32).ctypes.data
    ofp = None if of is None else np.ascontiguousarray(of, np.int32).ctypes.data
    if states == "good":
        states = tables(max(n_modes, 1), count)
    sp = None if states is None else (C.c_void_p * len(states))(*states)
    descs = pictures(max(n, 0)) if pics is None else pics
    return lib().cb200_detect_scan_extract_decode_chunks_receivers_dev(hs if list_ok else None, n_modes, C.cast(descs, C.c_void_p), n, flags,
                                                                       candp, ofp, count, sp, *outputs, None)


def refused(rc):
    return rc, lib().cb200_last_error().decode()


def test_good_arguments_reach_the_context_checks():
    assert refused(call()) == (-1, "context 0 is null")
    assert refused(call(cand=None)) == (-1, "context 0 is null")                  # NULL candidates: every picture under every mode
    assert refused(call(list_ok=False)) == (-1, "null context list")
    assert refused(call(n=0, of=np.zeros(1, np.int32)))[1] == "context 0 is null"
    fake = C.c_void_p(1).value                                                    # never dereferenced: the null entry is found first
    assert refused(call(ctxs=[fake, None, fake, fake]))[1] == "context 1 is null"


@pytest.mark.parametrize("n_modes", [0, -1, 6])
def test_n_modes_out_of_range(n_modes):
    assert refused(call(n_modes=n_modes, cand=None))[1] == "n_modes = %d: between 1 and 5 candidate modes" % n_modes


def test_what_the_detect_call_refuses():
    assert refused(call(flags=cb.FLAG_SHARPEN | cb.FLAG_SHARPEN_IF_NEEDED))[1] == "CB200_FLAG_SHARPEN and CB200_FLAG_SHARPEN_IF_NEEDED are exclusive"
    assert refused(call(flags=cb.FLAG_CC_SIMPLE | cb.FLAG_CC_FIT))[1] == "CC_SIMPLE and CC_FIT are exclusive"
    for missing in range(4):
        outs = [P] * 4
        outs[missing] = None
        assert refused(call(outputs=tuple(outs))) == (-1, "null output"), missing


def test_what_the_receivers_camera_call_refuses():
    assert refused(call(n=-1))[1] == "n < 0"
    bad = pictures(4)
    bad[2].layout = 9
    msg = refused(call(pics=bad))[1]
    assert "picture 2" in msg, msg
    small = pictures(4, w=50, h=40)
    msg = refused(call(pics=small))[1]
    assert "picture 0" in msg, msg
    assert refused(call(of=None)) == (-1, "null receiver_of")
    assert refused(call(count=0, states=tables(4, 1))) == (-1, "n_receivers < 1")
    assert refused(call(count=-3, states=tables(4, 1))) == (-1, "n_receivers < 1")
    assert refused(call(of=[0, 1, 3, 2])) == (-1, "picture 2: receiver 3 outside [0, 3)")
    assert refused(call(of=[0, -1, 1, 2])) == (-1, "picture 1: receiver -1 outside [0, 3)")


def test_candidates_are_checked_per_picture():
    assert refused(call(cand=[0b1111, 0, 1, 1])) == (-1, "picture 1 has no candidate mode (candidates = 0)")
    assert refused(call(cand=[1, 1, 0b10000, 1])) == (-1, "picture 2: candidates = 16 has a bit at or above n_modes = 4")
    assert refused(call(n_modes=2, cand=[1, 2, 3, 4], states=tables(2)))[1] == "picture 3: candidates = 4 has a bit at or above n_modes = 2"
    assert refused(call(n_modes=1, cand=[1, 1, 1, 1 << 31], states=tables(1)))[1] == \
        "picture 3: candidates = 2147483648 has a bit at or above n_modes = 1"
    assert refused(call(n_modes=5, cand=[31, 16, 1, 2], states=tables(5)))[1] == "context 0 is null"


def test_state_tables_are_named():
    assert refused(call(states=None)) == (-1, "null d_states")
    t = tables(4)
    t[2] = None
    assert refused(call(states=t)) == (-1, "d_states[2] (the state table of context 2) is null")
    t = tables(4)
    t[3] += 2
    assert refused(call(states=t)) == (-1, "d_states[3] (the state table of context 3) is not 4-byte aligned")


def test_overlapping_state_tables_are_refused():
    # tables of 3 entries, 120 bytes: one entry apart overlap, exactly one table apart do not
    assert refused(call(states=tables(4, 3, gap=ENTRY)))[1] == "d_states[0] and d_states[1] overlap: each candidate mode needs its own 3-entry table"
    t = tables(4)
    t[3] = t[1] + ENTRY * 2                                        # the last entry of table 1
    assert refused(call(states=t))[1] == "d_states[1] and d_states[3] overlap: each candidate mode needs its own 3-entry table"
    t = tables(4)
    t[2] = t[0]
    assert refused(call(states=t))[1] == "d_states[0] and d_states[2] overlap: each candidate mode needs its own 3-entry table"
    assert refused(call(states=tables(4, 3, gap=3 * ENTRY)))[1] == "context 0 is null"


def test_the_checks_come_in_order():
    both = cb.FLAG_CC_SIMPLE | cb.FLAG_CC_FIT
    assert refused(call(n_modes=0, flags=both, of=None))[1].startswith("n_modes = 0")
    assert refused(call(flags=both, of=None, cand=[0, 0, 0, 0]))[1] == "CC_SIMPLE and CC_FIT are exclusive"
    assert refused(call(outputs=(P, None, P, P), of=None))[1] == "null output"
    assert refused(call(cand=[0, 0, 0, 0], of=None))[1] == "picture 0 has no candidate mode (candidates = 0)"
    assert refused(call(of=None, states=None))[1] == "null receiver_of"


def test_python_wrapper_refuses_mismatched_lists():
    torch = pytest.importorskip("torch")
    with pytest.raises(cb.Cb200Error, match="2 state tables for 3 contexts"):
        cb.detect_scan_extract_decode_chunks_receivers_dev([None] * 3, [], [], [torch.zeros(10, dtype=torch.int32)] * 2, 0, 0, 0, 0)


# ---- the checks that read the contexts
def _dev_call(ctxs, n, cand=None, count=2):
    import torch
    pics = [torch.zeros((960, 1280, 3), dtype=torch.uint8, device="cuda") for _ in range(max(n, 1))]
    descs = (cb.Picture * max(n, 1))(*[cb.picture(t, "rgb") for t in pics[:max(n, 1)]])
    chunks = torch.zeros(max(n, 1) * 8750, dtype=torch.uint8, device="cuda")
    words = torch.zeros(max(n, 1) * 8, dtype=torch.int32, device="cuda")
    states = [torch.zeros(count * 10, dtype=torch.int32, device="cuda") for _ in ctxs]
    of = np.zeros(max(n, 1), np.int32)
    hs = (C.c_void_p * len(ctxs))(*[c._h.value for c in ctxs])
    sp = (C.c_void_p * len(ctxs))(*[s.data_ptr() for s in states])
    candp = None if cand is None else np.ascontiguousarray(cand, np.uint32).ctypes.data
    before = cb.launch_count()
    rc = lib().cb200_detect_scan_extract_decode_chunks_receivers_dev(hs, len(ctxs), C.cast(descs, C.c_void_p), n, 0, candp, of.ctypes.data, count,
                                                                     sp, chunks.data_ptr(), words.data_ptr(), words.data_ptr(), words.data_ptr(),
                                                                     None)
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
        err = refused(_dev_call([ctx[68], ctx[4], twin], 2))[1]
        assert err.startswith("contexts 0 and 2 are both mode 68"), err
        twin.close()
        ctx[4].set_stream(side.cuda_stream)
        assert refused(_dev_call([ctx[68], ctx[4]], 2))[1].startswith("context 1 is on another stream than context 0")
        ctx[4].set_stream(st.cuda_stream)
        assert refused(_dev_call([ctx[68], ctx[4], ctx[67]], 5))[1] == "n = 5 > max_frames = 4 of context 0"
        wh = np.array([(1280, 960)], np.int32)
        pics = torch.zeros(1280 * 960 * 3, dtype=torch.uint8, device="cuda")
        chunks = torch.zeros(7500, dtype=torch.uint8, device="cuda")
        words = torch.zeros(4, dtype=torch.int32, device="cuda")
        plan = ctx[4].camera_plan(wh, 0, pics.data_ptr(), chunks.data_ptr(), words.data_ptr(), None, words.data_ptr())
        # a mode none of whose pictures it decodes is still a candidate: its plans refuse the call
        assert refused(_dev_call([ctx[68], ctx[4]], 1, cand=[1]))[1].startswith("context 1 has live camera plans")
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
        assert refused(_dev_call([a, b], 1))[1].startswith("context 1 is linked to a CCM chain")
    finally:
        a.close(); b.close()
