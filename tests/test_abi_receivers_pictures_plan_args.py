"""CPU-side checks of cb200_camera_plan_create_receivers_pictures_dev: every refusal comes before any CUDA call, in order, with a
message that names its cause -- the receiver arguments, the flags, the descriptors' pointer and bounds (their contents are read only
by the launches), then what cb200_camera_plan_create_receivers refuses.  The context is NULL (or a stand-in that is never
dereferenced), so a call whose arguments are all good fails on the context instead."""
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
OF = P + 128                                            # 4-byte aligned stand-ins for d_receiver_of and d_states
STATES = P + 64
GOOD = (60, 1080, 1920)


def create(n=4, pics=PICS, bounds=GOOD, of=OF, count=3, states=STATES, flags=0, chunks=P, mask=P, status=P, out=True, ctx=None):
    bd = None if bounds is None else C.cast((C.c_int32 * 3)(*bounds), C.c_void_p)
    h = C.c_void_p()
    return lib().cb200_camera_plan_create_receivers_pictures_dev(ctx, pics, n, bd, flags, of, count, states, chunks, mask, None, status,
                                                                 C.byref(h) if out else None)


def refused(rc):
    return rc, lib().cb200_last_error().decode()


def test_good_arguments_reach_the_context_check():
    assert refused(create()) == (-1, "null context")
    assert refused(create(bounds=(60, 4499, 4499)))[1] == "null context"
    assert refused(create(bounds=(4499, 4499, 2 ** 20), n=1))[1] == "null context"


def test_receiver_arguments_come_first():
    assert refused(create(of=None, pics=None, bounds=None)) == (-1, "null d_receiver_of")
    assert refused(create(of=OF + 2)) == (-1, "d_receiver_of is not 4-byte aligned")
    assert refused(create(states=None, pics=None)) == (-1, "null d_states")
    assert refused(create(states=STATES + 2)) == (-1, "d_states is not 4-byte aligned")
    assert refused(create(count=0, bounds=(1, 0, 0))) == (-1, "n_receivers < 1")


def test_flags_before_the_descriptors():
    both = cb.FLAG_CC_SIMPLE | cb.FLAG_CC_FIT
    assert refused(create(flags=both, pics=None)) == (-1, "CC_SIMPLE and CC_FIT are exclusive")
    sharpen = cb.FLAG_SHARPEN | cb.FLAG_SHARPEN_IF_NEEDED
    assert refused(create(flags=sharpen, bounds=None))[1] == "CB200_FLAG_SHARPEN and CB200_FLAG_SHARPEN_IF_NEEDED are exclusive"


def test_descriptor_pointer_and_bounds_in_order():
    assert refused(create(n=-1, pics=None)) == (-1, "n < 0")
    assert refused(create(pics=None, bounds=None)) == (-1, "null d_pics")
    for off in (1, 2, 4):
        assert refused(create(pics=PICS + off, bounds=None)) == (-1, "d_pics is not 8-byte aligned"), off
    assert refused(create(bounds=None)) == (-1, "null bounds")
    cases = [
        ((59, 1080, 1920), "min_short < 60"),
        ((-5, 1080, 1920), "min_short < 60"),
        ((60, 4500, 4500), "max_short > 4499"),
        ((59, 4500, 4500), "min_short < 60"),
        ((61, 60, 1920), "min_short > max_short"),
        ((60, 1080, 1079), "max_long < max_short"),
        ((61, 60, 59), "min_short > max_short"),
    ]
    for bounds, why in cases:
        rc, msg = refused(create(bounds=bounds))
        assert rc == -1 and msg.startswith(why), (bounds, msg)
        assert f"(bounds {bounds[0]}, {bounds[1]}, {bounds[2]})" in msg, msg


def test_bounds_that_would_overflow():
    # 4499 x 2^31 - 1: 141 x 67 108 864 tiles even for one slot
    rc, msg = refused(create(n=1, bounds=(4499, 4499, 2 ** 31 - 1)))
    assert rc == -1 and "blur tiles" in msg, msg
    # one slot of 60 x 2^31 - 1 has 2^26 tiles, but 2^32 scan rows
    rc, msg = refused(create(n=1, bounds=(60, 60, 2 ** 31 - 1)))
    assert rc == -1 and "scan rows" in msg, msg
    # the tile limit scales with n: 4096 x 4096 has 32 x 128 tiles, so 2^31 / 4096 slots fit and one more does not
    assert refused(create(n=2 ** 31 // 4096 - 1, bounds=(4096, 4096, 4096)))[1] == "null context"
    rc, msg = refused(create(n=2 ** 31 // 4096, bounds=(4096, 4096, 4096)))
    assert rc == -1 and "blur tiles" in msg, msg


def test_what_camera_plan_create_refuses():
    assert refused(create(n=0)) == (-1, "n = 0: a camera plan needs at least one picture")
    assert refused(create(out=False)) == (-1, "null plan")
    fake = C.c_void_p(1)                                 # a non-null context that is never dereferenced before these checks
    for kw in ({"chunks": None}, {"mask": None}, {"status": None}):
        assert refused(create(**kw)) == (-1, "null context"), kw
        assert refused(create(ctx=fake, **kw)) == (-1, "null output"), kw


def test_python_checks_its_tensors():
    torch = pytest.importorskip("torch")
    ctx = object.__new__(cb.Context)                      # no device: the wrapper's own checks come first
    with pytest.raises(cb.Cb200Error, match="uint8 CUDA tensor"):
        cb.Context.receivers_camera_plan_pictures_dev(ctx, torch.zeros((2, 40), dtype=torch.uint8), GOOD, None, None, 0, 0, 0)
    with pytest.raises(cb.Cb200Error, match="uint8 CUDA tensor"):
        cb.Context.receivers_camera_plan_pictures_dev(ctx, np.zeros((2, 40), np.uint8), GOOD, None, None, 0, 0, 0)


def test_descriptor_bytes_are_the_c_struct():
    assert C.sizeof(cb.Picture) == 40
    d = cb.Picture(0x1234560, 640, 480, 2048, 0, cb.LAYOUT_BGR)
    raw = np.frombuffer(bytes(d), np.uint8)
    assert raw[:8].view(np.uint64)[0] == 0x1234560 and tuple(raw[8:16].view(np.int32)) == (640, 480)
    assert raw[16:24].view(np.int64)[0] == 2048 and raw[32:36].view(np.int32)[0] == cb.LAYOUT_BGR


# ---- cb200_camera_plan_create_detect_receivers_pictures_dev: n_modes, the flags, d_pics and the bounds, the plan's own rules, the
# outputs, the candidates' and map's pointers, the state tables, then the contexts (NULL here: "context 0 is null")
ENTRY = 40
CAND = P + 512


def create_detect(n_modes=3, n=4, pics=PICS, bounds=GOOD, cand=CAND, of=OF, count=3, states="good", flags=0, outputs=(P, P, P, P), out=True):
    hs = (C.c_void_p * max(n_modes, 1))(*([None] * max(n_modes, 1)))
    if states == "good":
        states = [P + 1024 + k * ENTRY * count for k in range(max(n_modes, 1))]
    sp = None if states is None else (C.c_void_p * len(states))(*states)
    bd = None if bounds is None else C.cast((C.c_int32 * 3)(*bounds), C.c_void_p)
    h = C.c_void_p()
    return lib().cb200_camera_plan_create_detect_receivers_pictures_dev(hs, n_modes, pics, n, bd, flags, cand, of, count, sp, *outputs, None,
                                                                        C.byref(h) if out else None)


def test_detect_good_arguments_reach_the_context_checks():
    assert refused(create_detect()) == (-1, "context 0 is null")
    assert refused(create_detect(cand=None)) == (-1, "context 0 is null")        # NULL candidates: every mode


def test_detect_refusals_in_order():
    assert refused(create_detect(n_modes=0, pics=None))[1] == "n_modes = 0: between 1 and 5 candidate modes"
    assert refused(create_detect(n_modes=6, bounds=None))[1] == "n_modes = 6: between 1 and 5 candidate modes"
    assert refused(create_detect(flags=cb.FLAG_CC_SIMPLE | cb.FLAG_CC_FIT, pics=None))[1] == "CC_SIMPLE and CC_FIT are exclusive"
    assert refused(create_detect(n=-1, pics=None))[1] == "n < 0"
    assert refused(create_detect(pics=None, bounds=None, outputs=(None,) * 4)) == (-1, "null d_pics")
    assert refused(create_detect(pics=PICS + 4, bounds=None)) == (-1, "d_pics is not 8-byte aligned")
    assert refused(create_detect(bounds=None, outputs=(None,) * 4)) == (-1, "null bounds")
    for bounds, why in (((59, 1080, 1920), "min_short < 60"), ((60, 4500, 4500), "max_short > 4499"), ((61, 60, 1920), "min_short > max_short"),
                        ((60, 1080, 1079), "max_long < max_short")):
        rc, msg = refused(create_detect(bounds=bounds, outputs=(None,) * 4))
        assert rc == -1 and msg.startswith(why), (bounds, msg)
    rc, msg = refused(create_detect(n=1, bounds=(4499, 4499, 2 ** 31 - 1)))
    assert rc == -1 and "blur tiles" in msg, msg
    assert refused(create_detect(n=0, outputs=(None,) * 4)) == (-1, "n = 0: a camera plan needs at least one picture")
    assert refused(create_detect(out=False, outputs=(None,) * 4)) == (-1, "null plan")
    for missing in range(4):
        outs = [P] * 4
        outs[missing] = None
        assert refused(create_detect(outputs=tuple(outs), of=None)) == (-1, "null output"), missing
    assert refused(create_detect(cand=CAND + 2, of=None)) == (-1, "d_candidates is not 4-byte aligned")
    assert refused(create_detect(of=None)) == (-1, "null d_receiver_of")
    assert refused(create_detect(of=OF + 1)) == (-1, "d_receiver_of is not 4-byte aligned")
    assert refused(create_detect(count=0)) == (-1, "n_receivers < 1")
    assert refused(create_detect(states=None)) == (-1, "null d_states")


def test_detect_python_checks_its_tensors():
    torch = pytest.importorskip("torch")
    with pytest.raises(cb.Cb200Error, match="uint8 CUDA tensor"):
        cb.detect_receivers_camera_plan_pictures_dev([], torch.zeros((2, 40), dtype=torch.uint8), GOOD, None, None, [], 0, 0, 0, 0)
