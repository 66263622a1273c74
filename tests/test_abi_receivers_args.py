"""CPU-side checks of the receivers calls (cb200_decode_chunks_receivers_dev, cb200_scan_extract_decode_chunks_receivers_dev): the
receiver arguments are refused before any CUDA call, with messages that name the violation, and then the mirrored call's checks
apply unchanged.  The context is NULL here, so a call whose arguments are all good fails on the context instead; the CCM chain
refusal needs a context and is checked on the GPU (tests/test_gpu_receivers.py).  Also the layout of cb200_receiver_state as C
compiles it from include/cb200.h and as the Python module declares it."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import libcimbar_b200 as cb
from libcimbar_b200 import build as cbbuild

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module", autouse=True)
def built():
    cbbuild.build()


def lib():
    return cb.load_library()


BUF = np.zeros(4096, np.uint8)
P = BUF.ctypes.data                                     # stand-in addresses: never dereferenced before the checks
STATES = P + 64                                         # 4-byte aligned
GOOD_OF = np.array([0, 2, 1, 2], np.int32)


def pictures(n, w=1280, h=960):
    return (cb.Picture * max(1, n))(*[cb.Picture(P, w, h, 3 * w, 0, cb.LAYOUT_RGB) for _ in range(n)])


def frame_call(n=4, of=GOOD_OF, count=3, states=STATES, flags=0, rgb=P, chunks=P):
    ofp = None if of is None else np.ascontiguousarray(of, np.int32).ctypes.data
    return lib().cb200_decode_chunks_receivers_dev(None, rgb, n, flags, ofp, count, states, chunks, P, None)


def camera_call(n=4, of=GOOD_OF, count=3, states=STATES, flags=0, pics=None, status=P):
    ofp = None if of is None else np.ascontiguousarray(of, np.int32).ctypes.data
    descs = pictures(max(n, 0)) if pics is None else pics
    return lib().cb200_scan_extract_decode_chunks_receivers_dev(None, C.cast(descs, C.c_void_p), n, flags, ofp, count, states, P, P, None,
                                                                status)


CALLS = {"frames": frame_call, "camera": camera_call}


def refused(rc):
    return rc, lib().cb200_last_error().decode()


@pytest.mark.parametrize("kind", list(CALLS))
def test_good_arguments_reach_the_context_check(kind):
    assert refused(CALLS[kind]()) == (-1, "null context")
    assert refused(CALLS[kind](n=0, of=np.zeros(1, np.int32)))[1] == "null context"


@pytest.mark.parametrize("kind", list(CALLS))
def test_receiver_arguments(kind):
    call = CALLS[kind]
    assert refused(call(of=None)) == (-1, "null receiver_of")
    assert refused(call(states=None)) == (-1, "null d_states")
    assert refused(call(states=STATES + 2)) == (-1, "d_states is not 4-byte aligned")
    assert refused(call(count=0)) == (-1, "n_receivers < 1")
    assert refused(call(count=-3)) == (-1, "n_receivers < 1")
    assert refused(call(of=[0, 1, 3, 2])) == (-1, "picture 2: receiver 3 outside [0, 3)")
    assert refused(call(of=[0, -1, 1, 2])) == (-1, "picture 1: receiver -1 outside [0, 3)")
    assert refused(call(of=[0, 1, 2, 3], count=4))[1] == "null context"


@pytest.mark.parametrize("kind", list(CALLS))
def test_the_receivers_are_checked_before_the_mirrored_call(kind):
    call = CALLS[kind]
    both = cb.FLAG_CC_SIMPLE | cb.FLAG_CC_FIT
    assert refused(call(of=None, flags=both)) == (-1, "null receiver_of")
    assert refused(call(flags=both)) == (-1, "CC_SIMPLE and CC_FIT are exclusive")


def test_the_frame_call_refuses_what_decode_chunks_dev_refuses():
    assert refused(frame_call(flags=cb.FLAG_SHARPEN_IF_NEEDED))[1] == "CB200_FLAG_SHARPEN_IF_NEEDED applies to camera pictures, not to frames"
    assert refused(frame_call(flags=cb.FLAG_CC_SIMPLE | cb.FLAG_CC_FIT))[1] == "CC_SIMPLE and CC_FIT are exclusive"


def test_the_camera_call_refuses_what_the_pictures_call_refuses():
    both = cb.FLAG_SHARPEN | cb.FLAG_SHARPEN_IF_NEEDED
    assert refused(camera_call(flags=both))[1] == "CB200_FLAG_SHARPEN and CB200_FLAG_SHARPEN_IF_NEEDED are exclusive"
    assert refused(camera_call(n=-1))[1] == "n < 0"
    bad = pictures(4)
    bad[2].layout = 9
    msg = refused(camera_call(pics=bad))[1]
    assert "picture 2" in msg, msg
    small = pictures(4, w=50, h=40)
    msg = refused(camera_call(pics=small))[1]
    assert "picture 0" in msg, msg


def test_receiver_state_layout(tmp_path):
    assert C.sizeof(cb.ReceiverState) == 40
    assert cb.ReceiverState.ccm.offset == 0 and cb.ReceiverState.active.offset == 36
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "cb200.h"\n'
                   'int main(void) { printf("%zu %zu %zu %zu", sizeof(cb200_receiver_state), offsetof(cb200_receiver_state, ccm),'
                   ' offsetof(cb200_receiver_state, active), sizeof(((cb200_receiver_state*)0)->active)); return 0; }\n')
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    assert subprocess.check_output([str(exe)]).decode().split() == ["40", "0", "36", "4"]


def test_state_tensor_helpers_round_trip():
    torch = pytest.importorskip("torch")
    m = np.arange(9, dtype=np.float32).reshape(3, 3) / 7
    a = np.zeros((3, 10), np.float32)
    words = a.view(np.uint32)
    a[0, :9] = m.reshape(9)
    words[0, 9] = 1
    host = torch.from_numpy(a.view(np.int32))
    back = cb.read_receiver_states(host)
    assert back[1] is None and back[2] is None and np.array_equal(back[0], m)
