"""CPU-side checks of the receiver flags calls (cb200_scan_extract_decode_chunks_receivers_flags_dev,
cb200_camera_plan_create_receivers_pictures_flags_dev): the flags table's pointer and the call's flags are refused first, before any
CUDA call, with messages that name the cause, and then the mirrored function's checks apply in their order.  The context is NULL, so
a call whose arguments are all good fails on the context instead."""
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


BUF = np.zeros(4096, np.uint8)
P = (BUF.ctypes.data + 63) & ~63                        # stand-in addresses: never dereferenced before the checks
PICS = P + 256                                          # 8-byte aligned stand-in for d_pics
OF = P + 128                                            # 4-byte aligned stand-ins for d_receiver_of, d_states, d_receiver_flags
STATES = P + 64
WORDS = P + 192
GOOD_OF = np.array([0, 2, 1, 2], np.int32)
BOUNDS = (60, 1080, 1920)
PER_RECEIVER = [cb.FLAG_SHARPEN, cb.FLAG_SHARPEN_IF_NEEDED, cb.FLAG_CC_SIMPLE, cb.FLAG_CC_FIT]


def pictures(n, w=1280, h=960):
    return (cb.Picture * max(1, n))(*[cb.Picture(P, w, h, 3 * w, 0, cb.LAYOUT_RGB) for _ in range(n)])


def direct(n=4, of=GOOD_OF, count=3, states=STATES, words=WORDS, flags=0, pics=None, status=P):
    ofp = None if of is None else np.ascontiguousarray(of, np.int32).ctypes.data
    descs = pictures(max(n, 0)) if pics is None else pics
    return lib().cb200_scan_extract_decode_chunks_receivers_flags_dev(None, C.cast(descs, C.c_void_p), n, flags, ofp, count, states, words,
                                                                      P, P, None, status)


def plan(n=4, of=OF, count=3, states=STATES, words=WORDS, flags=0, pics=PICS, bounds=BOUNDS, status=P):
    bd = None if bounds is None else C.cast((C.c_int32 * 3)(*bounds), C.c_void_p)
    h = C.c_void_p()
    return lib().cb200_camera_plan_create_receivers_pictures_flags_dev(None, pics, n, bd, flags, of, count, states, words, P, P, None, status,
                                                                       C.byref(h))


CALLS = {"direct": direct, "plan": plan}


def refused(rc):
    return rc, lib().cb200_last_error().decode()


@pytest.mark.parametrize("kind", list(CALLS))
def test_good_arguments_reach_the_context_check(kind):
    assert refused(CALLS[kind]()) == (-1, "null context")
    # the call's own flags keep the bits that are not per receiver
    assert refused(CALLS[kind](flags=cb.FLAG_NO_INTERLEAVE | cb.FLAG_NO_FALLBACK)) == (-1, "null context")


@pytest.mark.parametrize("kind", list(CALLS))
def test_table_pointer_first(kind):
    call = CALLS[kind]
    # a null table comes before every other refusal, a bad map and bad flags included
    assert refused(call(words=None, of=None, flags=cb.FLAG_CC_FIT, states=None)) == (-1, "null d_receiver_flags")
    for off in (1, 2, 3):
        assert refused(call(words=WORDS + off, of=None)) == (-1, "d_receiver_flags is not 4-byte aligned"), off


@pytest.mark.parametrize("kind", list(CALLS))
def test_per_receiver_bits_in_the_call_flags(kind):
    call = CALLS[kind]
    why = ("flags hold a per-receiver bit (SHARPEN, SHARPEN_IF_NEEDED, CC_SIMPLE, CC_FIT): those come from d_receiver_flags")
    for bit in PER_RECEIVER:
        assert refused(call(flags=bit, of=None)) == (-1, why), bit
        assert refused(call(flags=bit | cb.FLAG_NO_INTERLEAVE)) == (-1, why), bit
    # before the mirrored function's pair rule
    assert refused(call(flags=cb.FLAG_CC_SIMPLE | cb.FLAG_CC_FIT)) == (-1, why)


def test_direct_then_the_mirrored_checks_in_order():
    assert refused(direct(of=None)) == (-1, "null receiver_of")
    assert refused(direct(states=None)) == (-1, "null d_states")
    assert refused(direct(states=STATES + 2)) == (-1, "d_states is not 4-byte aligned")
    assert refused(direct(count=0)) == (-1, "n_receivers < 1")
    assert refused(direct(of=np.array([0, 3, 1, 2], np.int32))) == (-1, "picture 1: receiver 3 outside [0, 3)")
    # the receiver arguments come before the outputs, as in cb200_scan_extract_decode_chunks_receivers_dev
    assert refused(direct(of=None, status=None)) == (-1, "null receiver_of")
    # then the batch: a picture the mirrored call refuses
    bad = pictures(4)
    bad[2].data = None
    assert refused(direct(pics=bad))[1].startswith("picture 2")


def test_plan_then_the_mirrored_checks_in_order():
    assert refused(plan(of=None, pics=None, bounds=None)) == (-1, "null d_receiver_of")
    assert refused(plan(of=OF + 2)) == (-1, "d_receiver_of is not 4-byte aligned")
    assert refused(plan(states=None, pics=None)) == (-1, "null d_states")
    assert refused(plan(count=0, bounds=(1, 0, 0))) == (-1, "n_receivers < 1")
    assert refused(plan(pics=None, bounds=None)) == (-1, "null d_pics")
    assert refused(plan(pics=PICS + 4)) == (-1, "d_pics is not 8-byte aligned")
    assert refused(plan(bounds=None)) == (-1, "null bounds")
    assert refused(plan(bounds=(59, 1080, 1920)))[1].startswith("min_short < 60")


CTXS = (C.c_void_p * 2)(None, None)
TABLES = (C.c_void_p * 2)(STATES, STATES + 400)


def detect(n=4, n_modes=2, of=GOOD_OF, count=3, words=WORDS, flags=0, pics=None, mode=P):
    ofp = None if of is None else np.ascontiguousarray(of, np.int32).ctypes.data
    descs = pictures(max(n, 0)) if pics is None else pics
    return lib().cb200_detect_scan_extract_decode_chunks_receivers_flags_dev(CTXS, n_modes, C.cast(descs, C.c_void_p), n, flags, None, ofp,
                                                                             count, TABLES, words, P, P, P, mode, None)


def detect_plan(n=4, n_modes=2, of=OF, count=3, words=WORDS, flags=0, pics=PICS, bounds=BOUNDS, mode=P):
    bd = None if bounds is None else C.cast((C.c_int32 * 3)(*bounds), C.c_void_p)
    h = C.c_void_p()
    return lib().cb200_camera_plan_create_detect_receivers_pictures_flags_dev(CTXS, n_modes, pics, n, bd, flags, None, of, count, TABLES,
                                                                              words, P, P, P, mode, None, C.byref(h))


DETECT = {"detect": detect, "detect_plan": detect_plan}


@pytest.mark.parametrize("kind", list(DETECT))
def test_detect_forms_table_and_flags_first(kind):
    call = DETECT[kind]
    assert refused(call()) == (-1, "context 0 is null")
    assert refused(call(words=None, n_modes=0, of=None, flags=cb.FLAG_CC_FIT)) == (-1, "null d_receiver_flags")
    assert refused(call(words=WORDS + 2, n_modes=0)) == (-1, "d_receiver_flags is not 4-byte aligned")
    why = ("flags hold a per-receiver bit (SHARPEN, SHARPEN_IF_NEEDED, CC_SIMPLE, CC_FIT): those come from d_receiver_flags")
    for bit in PER_RECEIVER:
        assert refused(call(flags=bit, n_modes=0)) == (-1, why), bit
    # then the mirrored function's checks in their order: n_modes first, the output, the receivers
    assert refused(call(n_modes=0)) == (-1, "n_modes = 0: between 1 and 5 candidate modes")
    assert refused(call(mode=None)) == (-1, "null output")
    assert refused(call(of=None)) == (-1, "null d_receiver_of" if kind == "detect_plan" else "null receiver_of")


def test_detect_plan_then_the_descriptor_checks():
    assert refused(detect_plan(pics=None, bounds=None)) == (-1, "null d_pics")
    assert refused(detect_plan(bounds=None)) == (-1, "null bounds")
