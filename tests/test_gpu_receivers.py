"""Batches of several receivers (cb200_decode_chunks_receivers_dev, cb200_scan_extract_decode_chunks_receivers_dev): each receiver is
one decoder with its own colour-correction state.  The expected result is always the per-receiver sequence of direct calls: for
every receiver, a context set to its entry state decodes its pictures alone, in batch order; its records, masks, frame flags,
statuses and transforms are those pictures' in the receivers call, and its cb200_get_ccm afterwards is the receiver's new state.
Each test also asserts its premise: one plain call on the same batch gives a different result, so the receivers really matter."""
import os
import sys
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import chain_batches as CB  # noqa: E402
from gpu_support import cb, entries, frames  # noqa: F401  (fixtures)
from gpu_support import camera_call, layouts, same_ccm


# ------------------------------------------------------------------------------------------------------------------- frames
def frame_call(cb, ctx, frames, flags, receiver_of=None, states=None):
    """one frame call (plain, or receivers when receiver_of is given): (chunks, masks, frame flags, launches)"""
    import torch
    n = len(frames)
    d = torch.from_numpy(np.ascontiguousarray(frames)).cuda()
    chunks = torch.full((n, ctx.info.data_bytes), 0xA5, dtype=torch.uint8, device="cuda")
    mask = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    ff = torch.full((n,), 0xEE, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    l0 = cb.launch_count()
    if receiver_of is None:
        ctx.decode_chunks_dev(d.data_ptr(), n, chunks.data_ptr(), mask.data_ptr(), ff.data_ptr(), flags=flags)
    else:
        ctx.decode_chunks_receivers_dev(d.data_ptr(), n, receiver_of, states, chunks.data_ptr(), mask.data_ptr(), ff.data_ptr(), flags=flags)
    launches = cb.launch_count() - l0
    ctx.sync()
    return chunks.cpu().numpy(), mask.cpu().numpy(), ff.cpu().numpy(), launches


def frames_expected(cb, frames, of, entries, flags, mode=68):
    """the per-receiver sequence of direct calls: (chunks, masks, frame flags, exit states, per-picture CCMs of CC_FIT calls)"""
    n = len(frames)
    ctx = cb.Context(mode, max_frames=n)
    chunks = np.zeros((n, ctx.info.data_bytes), np.uint8)
    masks = np.zeros(n, np.int32)
    ff = np.zeros(n, np.uint8)
    used = np.full((n, 3, 3), np.nan, np.float32)
    exits = list(entries)
    for r in range(len(entries)):
        idx = np.flatnonzero(of == r)
        if not len(idx):
            continue
        ctx.set_ccm(entries[r])
        c, m, f, _ = frame_call(cb, ctx, frames[idx], flags)
        chunks[idx], masks[idx], ff[idx] = c, m, f
        exits[r] = ctx.get_ccm()
        if flags & cb.FLAG_CC_FIT:
            used[idx] = ctx.frame_ccms(len(idx))
    ctx.close()
    return chunks, masks, ff, exits, used


def check_frames(cb, frames, of, entries, flags, mode=68, plain_launches=None):
    import torch
    of = np.asarray(of, np.int32)
    want = frames_expected(cb, frames, of, entries, flags, mode)
    ctx = cb.Context(mode, max_frames=len(frames))
    states = cb.receiver_states(entries)
    c, m, f, launches = frame_call(cb, ctx, frames, flags, of, states)
    torch.cuda.synchronize()
    assert np.array_equal(c, want[0]) and np.array_equal(m, want[1]) and np.array_equal(f, want[2])
    got = cb.read_receiver_states(states)
    for r in range(len(entries)):
        assert same_ccm(got[r], want[3][r]), r
    if flags & cb.FLAG_CC_FIT:
        assert np.array_equal(ctx.frame_ccms(len(frames)), want[4], equal_nan=True)
    assert ctx.get_ccm() is None                          # the context's own CCM is untouched
    if plain_launches is not None:
        assert launches == plain_launches
    # premise: one plain call over the batch from receiver 0's state gives other records or leaves another state
    ctx.set_ccm(entries[0])
    pc, pm, _, _ = frame_call(cb, ctx, frames, flags)
    last = ctx.get_ccm()
    ctx.close()
    assert not np.array_equal(pc, want[0]) or not np.array_equal(pm, want[1]) or \
        any(not same_ccm(last, want[3][r]) for r in set(of.tolist()))
    return launches


FLAGS = {"none": 0, "cc_simple": 4, "cc_fit": 8}
IDX = [0, 2, 6, 2, 7, 3, 2, 9, 2, 7, 5, 2]


@pytest.mark.parametrize("flag", list(FLAGS))
def test_interleaved_receivers(cb, frames, entries, flag):
    of = [0, 1, 2, 3, 1, 0, 2, 3, 3, 1, 2, 0]
    check_frames(cb, frames[IDX], of, entries, FLAGS[flag])


@pytest.mark.parametrize("flag", list(FLAGS))
def test_each_picture_its_own_receiver(cb, frames, entries, flag):
    n = len(IDX)
    check_frames(cb, frames[IDX], np.arange(n), [entries[i % 4] for i in range(n)], FLAGS[flag])


@pytest.mark.parametrize("flag", list(FLAGS))
def test_a_receiver_of_headerless_pictures(cb, frames, entries, flag):
    idx = [2, 0, 7, 2, 4, 2, 7, 1]
    of = [0, 1, 0, 0, 1, 2, 0, 2]                          # receiver 0 has only headerless frames
    for e in ([entries[1], None, entries[2]], [None, entries[3], entries[1]], [entries[2], entries[1], None]):
        check_frames(cb, frames[idx], of, e, FLAGS[flag])


@pytest.mark.parametrize("flag", list(FLAGS))
@pytest.mark.parametrize("entry", [0, 1, 2, 3])
def test_one_receiver_is_the_plain_call(cb, frames, entries, flag, entry):
    """one receiver for every picture is the plain call from that state; CC_FIT launches exactly the plain call's kernels (the
    segmented carry replaces the carry), the other routes one small kernel more (the gather, or CC_SIMPLE's write-back)"""
    flags = FLAGS[flag]
    ctx = cb.Context(68, max_frames=len(IDX))
    ctx.set_ccm(entries[entry])
    _, _, _, plain = frame_call(cb, ctx, frames[IDX], flags)
    ctx.close()
    ours = frame_call_one_receiver(cb, frames[IDX], entries[entry], flags)
    assert ours == plain + (0 if flags & cb.FLAG_CC_FIT else 1), (ours, plain)


def frame_call_one_receiver(cb, frames, entry, flags):
    want = frames_expected(cb, frames, np.zeros(len(frames), np.int32), [entry], flags)
    ctx = cb.Context(68, max_frames=len(frames))
    states = cb.receiver_states([entry])
    c, m, f, launches = frame_call(cb, ctx, frames, flags, np.zeros(len(frames), np.int32), states)
    assert np.array_equal(c, want[0]) and np.array_equal(m, want[1]) and np.array_equal(f, want[2])
    assert same_ccm(cb.read_receiver_states(states)[0], want[3][0])
    ctx.close()
    return launches


def test_scale_more_frames_than_four_waves(cb, frames, entries):
    """4 x SMs + 1 frames of about 100 receivers under CC_FIT: every thread of the carry owns a range that crosses receivers"""
    import torch
    n = 4 * torch.cuda.get_device_properties(0).multi_processor_count + 1
    rng = np.random.default_rng(71)
    idx = rng.choice([0, 1, 2, 2, 2, 3, 4, 7, 7, 8], n)
    of = rng.integers(0, 100, n)
    ents = [entries[i % 4] for i in range(100)]
    check_frames(cb, frames[idx], of, ents, cb.FLAG_CC_FIT)


# ------------------------------------------------------------------------------------------------------------------- camera
def check_camera(cb, mode, pics, of, entries, flags):
    of = np.asarray(of, np.int32)
    ts, orders = layouts(pics)
    n = len(ts)
    ref = cb.Context(mode, max_frames=n)
    want = [None] * 5
    exits = list(entries)
    for r in range(len(entries)):
        idx = np.flatnonzero(of == r)
        if not len(idx):
            continue
        ref.set_ccm(entries[r])
        got = camera_call(cb, ref, [ts[i] for i in idx], [orders[i] for i in idx], flags)
        for k, a in enumerate(got):
            if want[k] is None:
                want[k] = np.zeros((n,) + a.shape[1:], a.dtype)
            want[k][idx] = a
        exits[r] = ref.get_ccm()
    ctx = cb.Context(mode, max_frames=n)
    states = cb.receiver_states(entries)
    got = camera_call(cb, ctx, ts, orders, flags, of, states)
    for k in range(5):
        assert np.array_equal(got[k], want[k]), k
    st = cb.read_receiver_states(states)
    for r in range(len(entries)):
        assert same_ccm(st[r], exits[r]), r
    assert ctx.get_ccm() is None
    ref.set_ccm(entries[0])
    plain = camera_call(cb, ref, ts, orders, flags)
    assert any(not np.array_equal(plain[k], want[k]) for k in range(4)), "premise: the plain call gives the same records"
    ref.close()
    ctx.close()


def test_camera_mode_b(cb, entries):
    import torch
    pics = CB.camera_pictures()
    ctx = cb.Context(68, max_frames=1)                    # a matrix fitted under the camera cast
    ts, orders = layouts(pics[1:2])
    camera_call(cb, ctx, ts, orders, cb.FLAG_CC_FIT)
    cam = ctx.get_ccm()
    assert cam is not None
    ctx.close()
    torch.cuda.synchronize()
    of = [0, 1, 2, 3, 1, 0, 3, 2, 1, 4, 0, 2]
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    check_camera(cb, 68, pics, of, [None, cam, entries[2], cam, entries[1]], flags)
    check_camera(cb, 68, pics, of, [cam, None, cam, entries[1], None], flags)


@pytest.mark.parametrize("cc", [0, 8])
def test_camera_legacy_4c(cb, cc):
    """mode 4C never fits: CC_FIT leaves every state as it was, and each picture decodes with its receiver's matrix"""
    pics = CB.legacy_pictures()
    cast = np.diag([0.55, 1.0, 1.25]).astype(np.float32)
    of = [i % 3 for i in range(len(pics))]
    check_camera(cb, 4, pics, of, [None, cast, np.eye(3, dtype=np.float32)], cb.FLAG_SHARPEN_IF_NEEDED | cc)


# ------------------------------------------------------------------------------------------------------------------- across calls
def test_two_calls_carry_and_absent_receivers_stay(cb, frames, entries):
    import torch
    ents = [entries[1], None, entries[2], entries[3], None]
    a_idx, a_of = [0, 2, 2, 4, 2, 1], [0, 1, 0, 1, 2, 2]
    b_idx, b_of = [2, 2, 3, 2, 2], [1, 0, 1, 2, 0]
    allf = frames[a_idx + b_idx]
    all_of = np.array(a_of + b_of, np.int32)
    want = frames_expected(cb, allf, all_of, ents, cb.FLAG_CC_FIT)
    ctx = cb.Context(68, max_frames=8)
    before = frames[[0]]
    ctx.set_ccm(None)
    frame_call(cb, ctx, before, cb.FLAG_CC_FIT)           # the context holds its own fitted matrix
    own = ctx.get_ccm()
    assert own is not None
    states = cb.receiver_states(ents)
    raw = states.view(torch.int32).reshape(-1, 10)
    raw[4] = torch.tensor([0x7FC00001] * 9 + [0xDEAD], dtype=torch.int32, device="cuda")    # a poisoned absent receiver
    raw[3, 9] = 5                                          # a nonzero activity other than 1
    poisoned = raw[3:].clone()
    ca, ma, _, _ = frame_call(cb, ctx, frames[a_idx], cb.FLAG_CC_FIT, np.array(a_of, np.int32), states)
    cb_, mb, _, _ = frame_call(cb, ctx, frames[b_idx], cb.FLAG_CC_FIT, np.array(b_of, np.int32), states)
    torch.cuda.synchronize()
    assert np.array_equal(np.concatenate([ca, cb_]), want[0]) and np.array_equal(np.concatenate([ma, mb]), want[1])
    got = cb.read_receiver_states(states)
    for r in range(3):
        assert same_ccm(got[r], want[3][r]), r
    assert torch.equal(raw[3:], poisoned)                  # receivers 3 and 4 had no picture: byte for byte as they were
    assert same_ccm(ctx.get_ccm(), own)
    # a direct CC_FIT call afterwards is the one a context that never ran the receivers calls makes
    fresh = cb.Context(68, max_frames=8)
    fresh.set_ccm(None)
    frame_call(cb, fresh, before, cb.FLAG_CC_FIT)
    after = frames[[2, 2, 1, 2]]
    x = frame_call(cb, ctx, after, cb.FLAG_CC_FIT)
    y = frame_call(cb, fresh, after, cb.FLAG_CC_FIT)
    assert all(np.array_equal(p, q) for p, q in zip(x[:3], y[:3]))
    assert same_ccm(ctx.get_ccm(), fresh.get_ccm())
    ctx.close()
    fresh.close()


def test_calls_only_enqueue(cb, frames, entries):
    """receivers calls queued behind a sleeping stream return at once and give what they give one at a time"""
    import torch
    pics = CB.camera_pictures()[:6]
    ts, orders = layouts(pics)
    of = np.array([0, 1, 0, 2, 1, 2], np.int32)
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    ents = [None, entries[1], entries[2]]
    ctx = cb.Context(68, max_frames=len(IDX))
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    d = torch.from_numpy(np.ascontiguousarray(frames[IDX])).cuda()
    n = len(IDX)
    fof = np.array([i % 3 for i in range(n)], np.int32)
    bufs = [torch.zeros((n, ctx.info.data_bytes), dtype=torch.uint8, device="cuda") for _ in range(4)]
    masks = [torch.zeros(n, dtype=torch.int32, device="cuda") for _ in range(4)]
    status = torch.zeros(n, dtype=torch.int32, device="cuda")

    def calls(states):
        ctx.scan_extract_decode_chunks_receivers_dev(ts, of, states, bufs[0].data_ptr(), masks[0].data_ptr(), status.data_ptr(), flags=flags,
                                                     order=orders)
        ctx.decode_chunks_receivers_dev(d.data_ptr(), n, fof, states, bufs[1].data_ptr(), masks[1].data_ptr(), flags=cb.FLAG_CC_FIT)
        ctx.scan_extract_decode_chunks_receivers_dev(ts, of, states, bufs[2].data_ptr(), masks[2].data_ptr(), status.data_ptr(), flags=flags,
                                                     order=orders)

    s1 = cb.receiver_states(ents)
    torch.cuda.synchronize()
    calls(s1)                                              # warm-up: every buffer at its size
    ctx.sync()
    want = [b.cpu().clone() for b in bufs[:3]] + [m.cpu().clone() for m in masks[:3]]
    s2 = cb.receiver_states(ents)
    torch.cuda.synchronize()
    with torch.cuda.stream(stream):
        torch.cuda._sleep(int(1.5e9))
    t0 = time.perf_counter()
    calls(s2)
    spent = time.perf_counter() - t0
    busy = not stream.query()
    ctx.sync()
    assert busy, "the stream finished before the third call returned"
    assert spent < 0.25, spent
    got = [b.cpu() for b in bufs[:3]] + [m.cpu() for m in masks[:3]]
    assert all(torch.equal(a, b) for a, b in zip(got, want))
    assert torch.equal(s1, s2)
    ctx.close()


def test_a_chained_context_is_refused(cb):
    ctx = cb.Context(68, max_frames=2)
    handle = ctx.ccm_chain_root_create(1)
    ctx.ccm_chain_attach(0, 1)
    states = cb.receiver_states([None])
    lib = cb.load_library()
    of = np.zeros(1, np.int32)
    before = cb.launch_count()
    rc = lib.cb200_decode_chunks_receivers_dev(ctx._h, 16, 1, 0, of.ctypes.data, 1, states.data_ptr(), 16, 16, None)
    assert rc == -1 and b"CCM chain" in lib.cb200_last_error()
    assert cb.launch_count() == before
    del handle
    ctx.close()
