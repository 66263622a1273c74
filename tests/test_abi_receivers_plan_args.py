"""CPU-side checks of cb200_camera_plan_create_receivers: every refusal comes before any CUDA call, with a message that names its
cause -- the receiver arguments first (the map is a device pointer here, so its indices are not checked), then what the receivers
camera call and cb200_camera_plan_create refuse.  The context is NULL, so a call whose arguments are all good fails on the context
instead; the CCM chain refusal needs a context and is checked on the GPU (tests/test_gpu_receivers_plan.py)."""
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
P = BUF.ctypes.data                                     # stand-in addresses: never dereferenced before the checks
OF = P + 128                                            # 4-byte aligned stand-ins for d_receiver_of and d_states
STATES = P + 64


def pictures(n, w=1280, h=960):
    return (cb.Picture * max(1, n))(*[cb.Picture(P, w, h, 3 * w, 0, cb.LAYOUT_RGB) for _ in range(n)])


def create(n=4, of=OF, count=3, states=STATES, flags=0, pics=None, chunks=P, mask=P, status=P, out=True, ctx=None):
    descs = pictures(max(n, 0)) if pics is None else pics
    h = C.c_void_p()
    return lib().cb200_camera_plan_create_receivers(ctx, C.cast(descs, C.c_void_p), n, flags, of, count, states, chunks, mask, None, status,
                                                    C.byref(h) if out else None)


def refused(rc):
    return rc, lib().cb200_last_error().decode()


def test_good_arguments_reach_the_context_check():
    assert refused(create()) == (-1, "null context")


def test_receiver_arguments():
    assert refused(create(of=None)) == (-1, "null d_receiver_of")
    assert refused(create(of=OF + 2)) == (-1, "d_receiver_of is not 4-byte aligned")
    assert refused(create(of=OF + 1)) == (-1, "d_receiver_of is not 4-byte aligned")
    assert refused(create(states=None)) == (-1, "null d_states")
    assert refused(create(states=STATES + 2)) == (-1, "d_states is not 4-byte aligned")
    assert refused(create(count=0)) == (-1, "n_receivers < 1")
    assert refused(create(count=-3)) == (-1, "n_receivers < 1")
    assert refused(create(count=2 ** 31 - 1))[1] == "null context"


def test_the_receivers_are_checked_first():
    both = cb.FLAG_CC_SIMPLE | cb.FLAG_CC_FIT
    assert refused(create(of=None, flags=both)) == (-1, "null d_receiver_of")
    assert refused(create(count=0, n=0)) == (-1, "n_receivers < 1")


def test_what_the_receivers_camera_call_refuses():
    assert refused(create(flags=cb.FLAG_CC_SIMPLE | cb.FLAG_CC_FIT)) == (-1, "CC_SIMPLE and CC_FIT are exclusive")
    both = cb.FLAG_SHARPEN | cb.FLAG_SHARPEN_IF_NEEDED
    assert refused(create(flags=both))[1] == "CB200_FLAG_SHARPEN and CB200_FLAG_SHARPEN_IF_NEEDED are exclusive"
    assert refused(create(n=-1))[1] == "n < 0"
    bad = pictures(4)
    bad[2].layout = 9
    msg = refused(create(pics=bad))[1]
    assert "picture 2" in msg, msg
    small = pictures(4, w=50, h=40)
    msg = refused(create(pics=small))[1]
    assert "picture 0" in msg, msg
    pitch = pictures(4)
    pitch[3].row_pitch = 100
    msg = refused(create(pics=pitch))[1]
    assert "picture 3" in msg, msg
    nulls = pictures(4)
    nulls[1].data = None
    msg = refused(create(pics=nulls))[1]
    assert "picture 1" in msg, msg


def test_what_camera_plan_create_refuses():
    assert refused(create(n=0)) == (-1, "n = 0: a camera plan needs at least one picture")
    assert refused(create(out=False)) == (-1, "null plan")
    fake = C.c_void_p(1)                                 # a non-null context that is never dereferenced before these checks
    for kw in ({"chunks": None}, {"mask": None}, {"status": None}):
        assert refused(create(**kw)) == (-1, "null context"), kw
        assert refused(create(ctx=fake, **kw)) == (-1, "null output"), kw


def test_python_refuses_a_host_map():
    torch = pytest.importorskip("torch")
    ctx = object.__new__(cb.Context)                      # no device: the wrapper's own checks come first
    with pytest.raises(cb.Cb200Error, match="int32 CUDA tensor"):
        cb.Context.receivers_camera_plan(ctx, [], torch.zeros(0, dtype=torch.int32), None, 0, 0, 0)
