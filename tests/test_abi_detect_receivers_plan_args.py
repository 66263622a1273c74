"""CPU-side checks of cb200_camera_plan_create_detect_receivers: every refusal is CB200_ERR_ARG with a message naming its cause,
before any CUDA call, in this order -- n_modes, the flags, the pictures and the plan's own rules (n == 0, a null plan), the null
outputs, the device pointers of the candidates and the map (their entries are only read by a launch), n_receivers and the state
tables, then the contexts.  The contexts are NULL here, so a call whose other arguments are all good fails on "context 0 is null";
the checks that read the contexts (one stream, a CCM chain) run on the GPU (tests/test_gpu_detect_receivers_plan.py)."""
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
CAND = P + 256                                          # 4-byte aligned stand-ins for d_candidates and d_receiver_of
OF = P + 512


def pictures(n, w=1280, h=960):
    return (cb.Picture * max(1, n))(*[cb.Picture(P, w, h, 3 * w, 0, cb.LAYOUT_RGB) for _ in range(n)])


def tables(n_modes, count=3, gap=None):
    step = ENTRY * count if gap is None else gap
    return [P + 1024 + k * step for k in range(n_modes)]


def create(n_modes=4, n=4, cand=CAND, of=OF, count=3, states="good", flags=0, pics=None, ctxs=None, outputs=(P, P, P, P), out=True,
           list_ok=True):
    ctxs = [None] * max(n_modes, 1) if ctxs is None else ctxs
    hs = (C.c_void_p * len(ctxs))(*ctxs)
    if states == "good":
        states = tables(max(n_modes, 1), count)
    sp = None if states is None else (C.c_void_p * len(states))(*states)
    descs = pictures(max(n, 0)) if pics is None else pics
    h = C.c_void_p()
    return lib().cb200_camera_plan_create_detect_receivers(hs if list_ok else None, n_modes, C.cast(descs, C.c_void_p), n, flags, cand, of, count,
                                                           sp, *outputs, None, C.byref(h) if out else None)


def refused(rc):
    return rc, lib().cb200_last_error().decode()


def test_good_arguments_reach_the_context_checks():
    assert refused(create()) == (-1, "context 0 is null")
    assert refused(create(cand=None)) == (-1, "context 0 is null")               # NULL candidates: every mode
    assert refused(create(list_ok=False)) == (-1, "null context list")
    fake = C.c_void_p(1).value                                                    # never dereferenced: the null entry is found first
    assert refused(create(ctxs=[fake, None, fake, fake]))[1] == "context 1 is null"


@pytest.mark.parametrize("n_modes", [0, -1, 6])
def test_n_modes_out_of_range(n_modes):
    assert refused(create(n_modes=n_modes, cand=None))[1] == "n_modes = %d: between 1 and 5 candidate modes" % n_modes


def test_what_the_detect_call_refuses():
    assert refused(create(flags=cb.FLAG_SHARPEN | cb.FLAG_SHARPEN_IF_NEEDED))[1] == "CB200_FLAG_SHARPEN and CB200_FLAG_SHARPEN_IF_NEEDED are exclusive"
    assert refused(create(flags=cb.FLAG_CC_SIMPLE | cb.FLAG_CC_FIT))[1] == "CC_SIMPLE and CC_FIT are exclusive"
    for missing in range(4):
        outs = [P] * 4
        outs[missing] = None
        assert refused(create(outputs=tuple(outs))) == (-1, "null output"), missing


def test_what_the_pictures_refuse():
    assert refused(create(n=-1))[1] == "n < 0"
    bad = pictures(4)
    bad[2].layout = 9
    assert "picture 2" in refused(create(pics=bad))[1]
    small = pictures(4, w=50, h=40)
    assert "picture 0" in refused(create(pics=small))[1]
    pitch = pictures(4)
    pitch[3].row_pitch = 100
    assert "picture 3" in refused(create(pics=pitch))[1]
    nulls = pictures(4)
    nulls[1].data = None
    assert "picture 1" in refused(create(pics=nulls))[1]


def test_the_plan_rules():
    assert refused(create(n=0)) == (-1, "n = 0: a camera plan needs at least one picture")
    assert refused(create(out=False)) == (-1, "null plan")
    assert refused(create(n=0, outputs=(None, P, P, P)))[1] == "n = 0: a camera plan needs at least one picture"   # before the outputs


def test_the_device_arrays():
    assert refused(create(of=None)) == (-1, "null d_receiver_of")
    assert refused(create(of=OF + 2)) == (-1, "d_receiver_of is not 4-byte aligned")
    assert refused(create(of=OF + 1)) == (-1, "d_receiver_of is not 4-byte aligned")
    assert refused(create(cand=CAND + 2)) == (-1, "d_candidates is not 4-byte aligned")
    assert refused(create(cand=CAND + 3, of=None)) == (-1, "d_candidates is not 4-byte aligned")          # the candidates first
    assert refused(create(of=None, count=0)) == (-1, "null d_receiver_of")                             # then the map
    # their entries are not read at create: a stand-in full of garbage is fine
    BUF[256:1024] = 0xFF
    assert refused(create()) == (-1, "context 0 is null")


def test_receivers_and_tables():
    assert refused(create(count=0)) == (-1, "n_receivers < 1")
    assert refused(create(count=-3)) == (-1, "n_receivers < 1")
    assert refused(create(states=None)) == (-1, "null d_states")
    assert refused(create(states=[tables(4)[0], None, *tables(4)[2:]])) == (-1, "d_states[1] (the state table of context 1) is null")
    assert refused(create(states=[tables(4)[0] + 2, *tables(4)[1:]])) == (-1, "d_states[0] (the state table of context 0) is not 4-byte aligned")
    msg = refused(create(states=tables(4, 3, gap=ENTRY * 2)))[1]
    assert msg == "d_states[0] and d_states[1] overlap: each candidate mode needs its own 3-entry table", msg
    assert refused(create(count=2 ** 31 - 1, states=tables(4, 1, gap=ENTRY)))[1].endswith("needs its own 2147483647-entry table")


def test_order_of_the_groups():
    both = cb.FLAG_CC_SIMPLE | cb.FLAG_CC_FIT
    assert refused(create(n_modes=0, flags=both))[1].startswith("n_modes = 0")
    assert refused(create(flags=both, n=0))[1] == "CC_SIMPLE and CC_FIT are exclusive"
    assert refused(create(outputs=(P, None, P, P), of=None)) == (-1, "null output")
    assert refused(create(of=None, states=None)) == (-1, "null d_receiver_of")
    assert refused(create(count=0, list_ok=False)) == (-1, "n_receivers < 1")


def test_python_refuses_host_arrays():
    torch = pytest.importorskip("torch")
    with pytest.raises(cb.Cb200Error, match="receiver_of is a contiguous int32 CUDA tensor"):
        cb.detect_receivers_camera_plan([], [], None, torch.zeros(0, dtype=torch.int32), [], 0, 0, 0, 0)
    with pytest.raises(cb.Cb200Error, match="state tables for"):
        cb.detect_receivers_camera_plan([None], [], None, None, [], 0, 0, 0, 0)
