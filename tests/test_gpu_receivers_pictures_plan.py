"""Receivers camera plans over device descriptors (cb200_camera_plan_create_receivers_pictures_dev): the descriptors are read from
device memory at every launch, so every launch may put pictures of other sizes, layouts and buffers in every slot.  The expected
result of a launch is a direct receivers call (cb200_scan_extract_decode_chunks_receivers_dev) on a second context with its own state
table, on the launch's accepted non-empty slots alone, in slot order: records, masks, frame flags, statuses, transforms, frame CCMs
and states, bit for bit.  Empty slots (receiver out of range) give EXTRACT_EMPTY, refused slots (a descriptor a direct call would
refuse, or outside the bounds) EXTRACT_REFUSED; both give mask 0 and touch no state.  Every descriptor here points at real device
memory, refused ones included: a refused picture that were decoded would change the records or the states."""
import os
import sys
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from gpu_support import cb, entries, frames  # noqa: E402,F401  (fixtures)
from gpu_support import KINDS, as_tensor, bounds_of, direct, fresh, graph_kernel_nodes, pool, resized  # noqa: E402

FLAGS = {"0": 0, "cc_simple": 4, "cc_fit": 8, "sharpen_if_needed|cc_fit": 0x20 | 8}


def radius(w, h):
    s = min(w, h)
    return 1 if s < 1500 else (2 if s < 2500 else 4)


class Plan:
    """n slots: the device descriptors and map, the outputs, and the tensors behind every descriptor ever written (kept alive, so
    that a stale descriptor still points at device memory)"""

    def __init__(self, cb, ctx, n, bounds, states, flags):
        import torch
        self.cb, self.ctx, self.n = cb, ctx, n
        self.d_pics = torch.zeros((n, 40), dtype=torch.uint8, device="cuda")
        self.of = torch.full((n,), -1, dtype=torch.int32, device="cuda")
        self.chunks = torch.full((n, ctx.info.data_bytes), 0xA5, dtype=torch.uint8, device="cuda")
        self.mask = torch.full((n,), -1, dtype=torch.int32, device="cuda")
        self.status = torch.full((n,), 7, dtype=torch.int32, device="cuda")
        self.flags = torch.full((n,), 0xEE, dtype=torch.uint8, device="cuda")
        self.keep = []
        torch.cuda.synchronize()
        self.plan = ctx.receivers_camera_plan_pictures_dev(self.d_pics, bounds, self.of, states, self.chunks.data_ptr(), self.mask.data_ptr(),
                                                           self.status.data_ptr(), self.flags.data_ptr(), flags=flags)

    def descriptors(self, ts, orders, tamper=None):
        """the host bytes of these tensors' descriptors, with tamper(i, Picture) applied to slot i"""
        d = self.cb.picture_descriptors(ts, orders)
        if tamper:
            for i in range(len(ts)):
                p = self.cb.Picture.from_buffer_copy(d[i].tobytes())
                if tamper(i, p):
                    d[i] = np.frombuffer(bytes(p), np.uint8)
        return d

    def write(self, desc, of):
        import torch
        self.d_pics.copy_(torch.from_numpy(np.ascontiguousarray(desc)))
        self.of.copy_(torch.from_numpy(np.asarray(of, np.int64).astype(np.int32)))

    def records(self):
        return [t.cpu().numpy() for t in (self.chunks, self.mask, self.status, self.flags)]


def launch_and_check(cb, slots, ts, orders, of, n_receivers, refused, states, ref, ref_states, flags, launch=None):
    """one launch (of the descriptors and map already written) against the direct call on its accepted non-empty slots.  launch:
    a replay of an outer graph instead, which leaves the context's host state -- the transforms' picture count -- alone"""
    import torch
    torch.cuda.synchronize()
    (launch or slots.plan.launch)()
    slots.ctx.sync()
    torch.cuda.synchronize()
    got = slots.records()
    of = np.asarray(of, np.int64)
    inside = (of >= 0) & (of < n_receivers)
    refused = np.asarray(refused, bool) & inside
    take = np.flatnonzero(inside & ~refused)
    want = direct(cb, ref, [ts[i] for i in take], [orders[i] for i in take], of[take], ref_states, flags)
    if want is not None:
        for k in range(4):
            assert np.array_equal(got[k][take], want[0][k]), k
        if launch is None:
            assert np.array_equal(slots.ctx.camera_transforms(slots.n)[take], want[1])
            assert np.array_equal(slots.ctx.frame_ccms(slots.n)[take], want[2], equal_nan=True)
    assert (got[1][~inside] == 0).all() and (got[2][~inside] == cb.EXTRACT_EMPTY).all()
    assert (got[1][refused] == 0).all() and (got[2][refused] == cb.EXTRACT_REFUSED).all()
    assert torch.equal(states, ref_states)
    return got


@pytest.mark.parametrize("flag", list(FLAGS))
@pytest.mark.parametrize("mode", [68, 4])
def test_mixed_sizes_every_launch_equal_the_direct_call(cb, entries, mode, flag):
    import torch
    flags = FLAGS[flag]
    p = pool(mode)
    assert {radius(x.shape[1], x.shape[0]) for x in p} == {1, 2, 4}          # premise: 3, 5 and 9 taps
    n, receivers = 8, 6
    bounds = bounds_of(p)
    ents = [entries[i % 4] for i in range(receivers)]
    ctx, ref = cb.Context(mode, max_frames=n), cb.Context(mode, max_frames=n)
    states, ref_states = cb.receiver_states(ents), cb.receiver_states(ents)
    slots = Plan(cb, ctx, n, bounds, states, flags)
    rng = np.random.default_rng(mode * 100 + flags)
    for k in range(5):
        pick = rng.permutation(len(p))[:n]                                    # a new assignment of pictures to slots
        ts, orders = fresh([p[i] for i in pick], rng)
        slots.keep.append(ts)
        of = rng.integers(0, receivers, n)
        if k >= 3:
            of[rng.choice(n, 2, replace=False)] = -1
        slots.write(slots.descriptors(ts, orders), of)
        launch_and_check(cb, slots, ts, orders, of, receivers, np.zeros(n, bool), states, ref, ref_states, flags)
    assert ctx.get_ccm() is None
    slots.plan.close()
    ctx.close()
    ref.close()


def test_refused_and_empty_slots_touch_nothing(cb, entries):
    import torch
    p = pool(68)
    n, receivers = 10, 4
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    lo, hi, lng = bounds_of(p)
    bounds = (lo, hi, lng)
    small = resized(p[0], lo - 100)                                         # outside the bounds: a short side below min_short
    ents = [entries[1], None, entries[2], entries[3]]
    ctx, ref = cb.Context(68, max_frames=n), cb.Context(68, max_frames=n)
    table = cb.receiver_states([entries[0]] + ents + [entries[0]])           # guard rows around the bound table
    raw = table.view(torch.int32).reshape(-1, 10)
    raw[0] = torch.tensor([0x7FC00001] * 9 + [0xDEAD], dtype=torch.int32, device="cuda")
    raw[-1] = torch.tensor([0x7FC00002] * 9 + [0xBEEF], dtype=torch.int32, device="cuda")
    guards = (raw[0].clone(), raw[-1].clone())
    states = table[1:receivers + 1]
    ref_states = cb.receiver_states(ents)
    slots = Plan(cb, ctx, n, bounds, states, flags)
    rng = np.random.default_rng(3)

    def pitch_small(i, d):
        d.row_pitch = d.w * (1 if d.layout == cb.LAYOUT_RGB_PLANAR else (4 if d.layout in (cb.LAYOUT_RGBA, cb.LAYOUT_BGRA) else 3)) - 1
        return True

    def overlap(i, d):
        d.plane_pitch = d.h * d.row_pitch - 1
        return True

    def unknown(i, d):
        d.layout = 7
        return True

    stale = None
    for k in range(4):
        pick = rng.permutation(len(p))[:n]
        pics = [p[i] for i in pick]
        kinds = [KINDS[int(rng.integers(len(KINDS)))] for _ in range(n)]
        bad = {1: (pitch_small, "rgb"), 4: (overlap, "planar"), 6: (unknown, "bgr"), 8: (None, "small")}
        for i, (_, kind) in bad.items():
            kinds[i] = "rgb" if kind == "small" else kind
            if kind == "small":
                pics[i] = small
        made = [as_tensor(x, kd) for x, kd in zip(pics, kinds)]
        ts, orders = [t for t, _ in made], [o for _, o in made]
        slots.keep.append(ts)
        desc = slots.descriptors(ts, orders, lambda i, d: bad[i][0](i, d) if i in bad and bad[i][0] else False)
        of = rng.integers(0, receivers, n)
        empty = [3, 9] if k % 2 else [0]
        of[empty] = [-1, receivers][:len(empty)] if len(empty) == 2 else [-1]
        if stale is not None:                                               # an empty slot keeps last launch's descriptor
            desc[empty[0]] = stale[empty[0]]
        refused = np.zeros(n, bool)
        refused[list(bad)] = True
        slots.write(desc, of)
        launch_and_check(cb, slots, ts, orders, of, receivers, refused, states, ref, ref_states, flags)
        assert torch.equal(raw[0], guards[0]) and torch.equal(raw[-1], guards[1])
        stale = desc
    before = table.clone()
    # every slot refused, then every slot empty
    desc = slots.descriptors(ts, orders, unknown)
    of = rng.integers(0, receivers, n)
    slots.write(desc, of)
    got = launch_and_check(cb, slots, ts, orders, of, receivers, np.ones(n, bool), states, ref, ref_states, flags)
    assert (got[2] == cb.EXTRACT_REFUSED).all()
    slots.write(desc, np.full(n, -1))
    got = launch_and_check(cb, slots, ts, orders, np.full(n, -1), receivers, np.zeros(n, bool), states, ref, ref_states, flags)
    assert (got[2] == cb.EXTRACT_EMPTY).all()
    assert torch.equal(table, before)
    slots.plan.close()
    ctx.close()
    ref.close()


def test_launch_count_is_the_same_for_every_descriptor_set(cb, entries):
    p = pool(68)
    n = 6
    ctx = cb.Context(68, max_frames=n)
    states = cb.receiver_states([entries[i % 4] for i in range(3)])
    slots = Plan(cb, ctx, n, bounds_of(p), states, cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT)
    rng = np.random.default_rng(8)
    counts = []
    for k in range(3):
        ts, orders = fresh([p[i] for i in rng.permutation(len(p))[:n]], rng)
        slots.keep.append(ts)
        of = rng.integers(-1, 3, n)
        slots.write(slots.descriptors(ts, orders), of)
        import torch
        torch.cuda.synchronize()
        before = cb.launch_count()
        slots.plan.launch()
        counts.append(cb.launch_count() - before)
        ctx.sync()
    assert counts[0] == counts[1] == counts[2] == graph_kernel_nodes(slots.plan.graph), counts
    slots.plan.close()
    ctx.close()


def test_inside_an_outer_graph_with_captured_descriptor_copies(cb, entries):
    import torch
    p = pool(68)
    n, receivers = 6, 5
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    ents = [entries[i % 4] for i in range(receivers)]
    ctx, ref = cb.Context(68, max_frames=n), cb.Context(68, max_frames=n)
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    states, ref_states = cb.receiver_states(ents), cb.receiver_states(ents)
    slots = Plan(cb, ctx, n, bounds_of(p), states, flags)
    staged_pics = torch.zeros((n, 40), dtype=torch.uint8, device="cuda")
    staged_of = torch.zeros(n, dtype=torch.int32, device="cuda")
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=stream):
        slots.d_pics.copy_(staged_pics)
        slots.of.copy_(staged_of)
        slots.plan.launch()
    rng = np.random.default_rng(77)
    for k in range(3):
        ts, orders = fresh([p[i] for i in rng.permutation(len(p))[:n]], rng)
        slots.keep.append(ts)
        of = rng.integers(-1, receivers, n)
        staged_pics.copy_(torch.from_numpy(slots.descriptors(ts, orders)))
        staged_of.copy_(torch.from_numpy(of.astype(np.int32)))
        launch_and_check(cb, slots, ts, orders, of, receivers, np.zeros(n, bool), states, ref, ref_states, flags, launch=g.replay)
    del g
    slots.plan.close()
    ctx.close()
    ref.close()


def test_two_plans_double_buffered_freezing_and_a_chained_context(cb, entries):
    import torch
    p = pool(68)
    n, receivers = 6, 4
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    ents = [entries[1], None, entries[2], entries[3]]
    ctx, ref = cb.Context(68, max_frames=2 * n), cb.Context(68, max_frames=n)
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    states, ref_states = cb.receiver_states(ents), cb.receiver_states(ents)
    bounds = bounds_of(p)
    buf = [Plan(cb, ctx, n, bounds, states, flags), Plan(cb, ctx, n, bounds, states, flags)]
    rng = np.random.default_rng(5)
    batches = []
    for k in range(4):
        ts, orders = fresh([p[i] for i in rng.permutation(len(p))[:n]], rng)
        batches.append((ts, orders, rng.integers(-1, receivers, n)))
    for k in range(2):
        buf[k].write(buf[k].descriptors(*batches[k][:2]), batches[k][2])
    torch.cuda.synchronize()
    with torch.cuda.stream(stream):
        torch.cuda._sleep(int(1.5e9))
    t0 = time.perf_counter()
    buf[0].plan.launch()
    buf[1].plan.launch()
    spent = time.perf_counter() - t0
    busy = not stream.query()
    ctx.sync()
    assert busy and spent < 0.25, (busy, spent)
    got = [buf[0].records(), buf[1].records()]
    for k in range(2, 4):
        with torch.cuda.stream(stream):
            buf[k % 2].write(buf[k % 2].descriptors(*batches[k][:2]), batches[k][2])
        buf[k % 2].plan.launch()
        ctx.sync()
        got.append(buf[k % 2].records())
    for k, (ts, orders, of) in enumerate(batches):
        idx = np.flatnonzero(of >= 0)
        want = direct(cb, ref, [ts[i] for i in idx], [orders[i] for i in idx], of[idx], ref_states, flags)
        for j in range(4):
            assert np.array_equal(got[k][j][idx], want[0][j]), (k, j)
    torch.cuda.synchronize()
    assert torch.equal(states, ref_states)
    # frozen: a plan with larger bounds, or more slots, would grow the scan's buffers
    with pytest.raises(cb.Cb200Error, match="would grow"):
        Plan(cb, ctx, n, (bounds[0], bounds[1], bounds[2] + 500), states, flags)
    with pytest.raises(cb.Cb200Error, match="would grow"):
        Plan(cb, ctx, 2 * n, bounds, states, flags)
    for b in buf:
        b.plan.close()
    Plan(cb, ctx, 2 * n, bounds, states, flags).plan.close()
    ctx.close()
    ref.close()
    chained = cb.Context(68, max_frames=2)
    handle = chained.ccm_chain_root_create(1)
    chained.ccm_chain_attach(0, 1)
    before = cb.launch_count()
    with pytest.raises(cb.Cb200Error, match="CCM chain"):
        Plan(cb, chained, 1, bounds, states, 0)
    assert cb.launch_count() == before
    del handle
    chained.close()
