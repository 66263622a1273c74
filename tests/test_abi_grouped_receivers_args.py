"""CPU-side checks of cb200_scan_extract_decode_chunks_grouped_receivers_dev and its _flags_ form (the groups of a receivers batch
found within each receiver): every argument error comes before any CUDA call, in this order -- the flags form's table and flags, the
receiver arguments, then what the grouped call refuses in its order (the flags, the pictures, CB200_FLAG_NO_FALLBACK, a null group
output, the context).  The context is NULL here, so a call whose arguments are all good fails on the context instead; the pictures'
null outputs, n > max_frames and a chain-linked context need a context and are checked on the GPU
(tests/test_gpu_grouped_receivers.py)."""
import ctypes as C

import numpy as np
import pytest

import libcimbar_b200 as cb
from libcimbar_b200 import build as cbbuild
from cpu_support import good, with_

GROUP_OUTPUTS = ("group_of", "count", "chunks", "mask", "used", "receiver")
BUF = np.zeros(4096, np.uint8)
P = (BUF.ctypes.data + 63) & ~63                        # stand-in addresses: never dereferenced before the checks
STATES = P + 64
WORDS = P + 192
GOOD_OF = np.array([0, 2, 1, 2], np.int32)
PER_RECEIVER = [cb.FLAG_SHARPEN, cb.FLAG_SHARPEN_IF_NEEDED, cb.FLAG_CC_SIMPLE, cb.FLAG_CC_FIT]


@pytest.fixture(scope="module", autouse=True)
def built():
    cbbuild.build()


def lib():
    return cb.load_library()


def refused(rc):
    return rc, lib().cb200_last_error().decode()


def call(form, pics=None, n=None, flags=0, of=GOOD_OF, count=3, states=STATES, words=WORDS, outputs=True, missing=()):
    pics = good() if pics is None else pics
    arr = (cb.Picture * max(1, len(pics)))(*pics)
    ofp = None if of is None else np.ascontiguousarray(of, np.int32).ctypes.data
    o = P if outputs else None
    g = [None if k in missing else P for k in GROUP_OUTPUTS]
    n = len(pics) if n is None else n
    if form == "plain":
        return lib().cb200_scan_extract_decode_chunks_grouped_receivers_dev(None, C.cast(arr, C.c_void_p), n, flags, ofp, count, states, o, o,
                                                                            None, o, *g)
    return lib().cb200_scan_extract_decode_chunks_grouped_receivers_flags_dev(None, C.cast(arr, C.c_void_p), n, flags, ofp, count, states,
                                                                              words, o, o, None, o, *g)


def receivers_call(form, pics=None, n=None, flags=0, of=GOOD_OF, count=3, states=STATES, words=WORDS):
    """the mirrored receivers call on the same arguments"""
    pics = good() if pics is None else pics
    arr = (cb.Picture * max(1, len(pics)))(*pics)
    ofp = None if of is None else np.ascontiguousarray(of, np.int32).ctypes.data
    n = len(pics) if n is None else n
    if form == "plain":
        return lib().cb200_scan_extract_decode_chunks_receivers_dev(None, C.cast(arr, C.c_void_p), n, flags, ofp, count, states, P, P, None, P)
    return lib().cb200_scan_extract_decode_chunks_receivers_flags_dev(None, C.cast(arr, C.c_void_p), n, flags, ofp, count, states, words, P, P,
                                                                      None, P)


FORMS = ["plain", "flags"]


@pytest.mark.parametrize("form", FORMS)
def test_good_arguments_reach_the_context_check(form):
    assert refused(call(form)) == (-1, "null context")
    assert refused(call(form, flags=cb.FLAG_NO_INTERLEAVE)) == (-1, "null context")
    if form == "plain":
        assert refused(call(form, flags=cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT)) == (-1, "null context")
    for n in (0, 1):
        assert refused(call(form, pics=good()[:n], of=GOOD_OF[:n])) == (-1, "null context")


def test_the_flags_table_comes_first():
    assert refused(call("flags", words=None, of=None, states=None, flags=cb.FLAG_NO_FALLBACK, missing=GROUP_OUTPUTS)) == \
        (-1, "null d_receiver_flags")
    for off in (1, 2, 3):
        assert refused(call("flags", words=WORDS + off, of=None)) == (-1, "d_receiver_flags is not 4-byte aligned")
    why = "flags hold a per-receiver bit (SHARPEN, SHARPEN_IF_NEEDED, CC_SIMPLE, CC_FIT): those come from d_receiver_flags"
    for bit in PER_RECEIVER:
        assert refused(call("flags", flags=bit, of=None, missing=GROUP_OUTPUTS)) == (-1, why), bit


RECEIVER_CASES = [
    ("null map", {"of": None}, "null receiver_of"),
    ("null states", {"states": None}, "null d_states"),
    ("misaligned states", {"states": STATES + 2}, "d_states is not 4-byte aligned"),
    ("no receivers", {"count": 0}, "n_receivers < 1"),
    ("receiver out of range", {"of": np.array([0, 3, 1, 2], np.int32)}, "picture 1: receiver 3 outside [0, 3)"),
    ("negative receiver", {"of": np.array([0, 1, -1, 2], np.int32)}, "picture 2: receiver -1 outside [0, 3)"),
]


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("name,kw,msg", RECEIVER_CASES, ids=[c[0] for c in RECEIVER_CASES])
def test_the_receiver_arguments_before_the_grouped_checks(form, name, kw, msg):
    assert refused(call(form, **kw)) == (-1, msg)
    assert refused(receivers_call(form, **kw)) == (-1, msg)
    # before the batch, NO_FALLBACK, the group outputs and the pictures' outputs
    assert refused(call(form, pics=with_(2, data=None), flags=cb.FLAG_NO_FALLBACK, missing=GROUP_OUTPUTS, outputs=False, **kw)) == (-1, msg)


PICTURE_CASES = [
    ("negative n", lambda: (good(), {"n": -1})),
    ("null data", lambda: (with_(0, data=None), {})),
    ("layout", lambda: (with_(1, layout=5), {})),
    ("pitch", lambda: (with_(3, row_pitch=-4), {})),
    ("size", lambda: (with_(1, h=59, w=1280, row_pitch=4 * 1280), {})),
    ("row pitch", lambda: (with_(0, row_pitch=3 * 1280 - 1), {})),
    ("planes", lambda: (with_(2, plane_pitch=1280 * 1024 - 1), {})),
    ("4 GB", lambda: (with_(3, row_pitch=1 << 32), {})),
    ("sharpen flags", lambda: (good(), {"flags": cb.FLAG_SHARPEN | cb.FLAG_SHARPEN_IF_NEEDED})),
    ("cc flags", lambda: (good(), {"flags": cb.FLAG_CC_SIMPLE | cb.FLAG_CC_FIT})),
]


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("name,case", PICTURE_CASES, ids=[c[0] for c in PICTURE_CASES])
def test_it_refuses_what_the_receivers_call_refuses(form, name, case):
    pics, kw = case()
    rc_r = receivers_call(form, pics=pics, **kw)
    want = refused(rc_r)
    assert want[0] == -1 and want[1] != "null context", name
    assert refused(call(form, pics=pics, **kw)) == want, name
    # and before NO_FALLBACK and the group outputs
    kw = dict(kw, flags=kw.get("flags", 0) | cb.FLAG_NO_FALLBACK)
    assert refused(call(form, pics=pics, missing=GROUP_OUTPUTS, **kw))[1] == refused(receivers_call(form, pics=pics, **kw))[1], name


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("n", [0, 1, 4])
def test_no_fallback_is_refused(form, n):
    msg = "CB200_FLAG_NO_FALLBACK: the vote needs every picture's walk"
    assert refused(call(form, pics=good()[:n], of=GOOD_OF[:n], flags=cb.FLAG_NO_FALLBACK)) == (-1, msg)
    # before the group outputs and the pictures' outputs
    assert refused(call(form, pics=good()[:n], of=GOOD_OF[:n], flags=cb.FLAG_NO_FALLBACK, missing=GROUP_OUTPUTS, outputs=False)) == (-1, msg)


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("which", GROUP_OUTPUTS)
@pytest.mark.parametrize("n", [0, 1, 4])
def test_each_null_group_output_is_refused(form, which, n):
    assert refused(call(form, pics=good()[:n], of=GOOD_OF[:n], missing=(which,))) == (-1, "null group output")
    # before the context and the pictures' outputs
    assert refused(call(form, pics=good()[:n], of=GOOD_OF[:n], missing=(which,), outputs=False)) == (-1, "null group output")


def test_python_wrapper_refuses_what_its_siblings_refuse():
    import torch
    ctx = cb.Context.__new__(cb.Context)
    f = cb.Context.scan_extract_decode_chunks_grouped_receivers_dev
    with pytest.raises(cb.Cb200Error, match="1 orders for 2 pictures"):
        f(ctx, [None, None], [0, 0], None, 0, 0, 0, 0, 0, 0, 0, 0, 0, order=["bgr"])
    with pytest.raises(cb.Cb200Error, match="3 receiver indices for 2 pictures"):
        f(ctx, [None, None], [0, 0, 1], None, 0, 0, 0, 0, 0, 0, 0, 0, 0)
    with pytest.raises(cb.Cb200Error, match="receiver states are a contiguous CUDA tensor"):
        f(ctx, [None, None], [0, 0], torch.zeros(20, dtype=torch.float32), 0, 0, 0, 0, 0, 0, 0, 0, 0)
    # the siblings say the same
    with pytest.raises(cb.Cb200Error, match="1 orders for 2 pictures"):
        cb.Context.scan_extract_decode_chunks_receivers_dev(ctx, [None, None], [0, 0], None, 0, 0, 0, order=["bgr"])
    with pytest.raises(cb.Cb200Error, match="3 receiver indices for 2 pictures"):
        cb.Context.scan_extract_decode_chunks_receivers_dev(ctx, [None, None], [0, 0, 1], None, 0, 0, 0)
