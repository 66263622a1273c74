"""Receivers camera plans (cb200_camera_plan_create_receivers): the receivers camera call captured once, its receiver map read from
device memory and grouped on the device at every launch.  The expected result of a launch is always a direct receivers call
(cb200_scan_extract_decode_chunks_receivers_dev) on a second context with its own state table, on the launch's non-empty slots
alone, in batch order: records, masks, frame flags, statuses, transforms, frame CCMs and states, bit for bit.  Empty slots (a
receiver outside [0, n_receivers)) give mask 0 and status EXTRACT_EMPTY and touch no state."""
import os
import sys
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import chain_batches as CB  # noqa: E402
from gpu_support import cb, entries, frames  # noqa: E402,F401  (fixtures)
from gpu_support import direct, graph_kernel_nodes, layouts, same_ccm  # noqa: E402

INT_MIN, INT_MAX = -2 ** 31, 2 ** 31 - 1
EXTRA_KERNELS = 1                      # k_receivers_order: every other kernel of the graph is the direct receivers call's


def variant(pics, k):
    """the pixels of launch k: the same sizes, other content"""
    f = [lambda p: p, lambda p: (p.astype(np.uint16) * 3 // 4).astype(np.uint8), lambda p: p[::-1, ::-1], lambda p: p][k % 4]
    return [np.ascontiguousarray(f(p)) for p in pics]


class Slots:
    """n bound pictures in mixed layouts, the bound map and outputs of one plan (or of the direct calls)"""

    def __init__(self, ctx, pics):
        import torch
        self.pics = pics
        self.ts, self.orders = layouts(pics)
        n = self.n = len(pics)
        self.of = torch.full((n,), -1, dtype=torch.int32, device="cuda")
        self.chunks = torch.full((n, ctx.info.data_bytes), 0xA5, dtype=torch.uint8, device="cuda")
        self.mask = torch.full((n,), -1, dtype=torch.int32, device="cuda")
        self.status = torch.full((n,), 7, dtype=torch.int32, device="cuda")
        self.flags = torch.full((n,), 0xEE, dtype=torch.uint8, device="cuda")

    def write(self, k):
        """launch k's pixels into the bound pictures (on the current stream)"""
        for t, s in zip(self.ts, layouts(variant(self.pics, k))[0]):
            t.copy_(s)

    def plan(self, ctx, states, flags):
        return ctx.receivers_camera_plan(self.ts, self.of, states, self.chunks.data_ptr(), self.mask.data_ptr(), self.status.data_ptr(),
                                         self.flags.data_ptr(), flags=flags, order=self.orders)

    def records(self):
        return [t.cpu().numpy() for t in (self.chunks, self.mask, self.status, self.flags)]


def launch_and_check(cb, ctx, plan, slots, of, n_receivers, states, ref, ref_states, flags):
    """one launch with map `of` against the direct call on its non-empty slots; the plan's and the direct call's states after it"""
    import torch
    of = np.asarray(of, np.int64)
    slots.of.copy_(torch.from_numpy(of.astype(np.int32)))
    torch.cuda.synchronize()                                             # the pixels and the map, before the context's stream
    plan.launch()
    ctx.sync()
    got = slots.records()
    inside = (of >= 0) & (of < n_receivers)
    idx = np.flatnonzero(inside)
    want = direct(cb, ref, [slots.ts[i] for i in idx], [slots.orders[i] for i in idx], of[idx], ref_states, flags)
    if want is not None:
        for k in range(4):
            assert np.array_equal(got[k][idx], want[0][k]), k
        assert np.array_equal(ctx.camera_transforms(slots.n)[idx], want[1])
        assert np.array_equal(ctx.frame_ccms(slots.n)[idx], want[2], equal_nan=True)
    empty = np.flatnonzero(~inside)
    assert (got[1][empty] == 0).all() and (got[2][empty] == cb.EXTRACT_EMPTY).all()
    assert torch.equal(states, ref_states)
    return got


FLAGS = {"0": 0, "cc_simple": 4, "cc_fit": 8, "sharpen_if_needed|cc_fit": 0x20 | 8}


def maps(n, receivers, rng):
    """six launches: interleaved receivers, one receiver for all, one per slot, a permutation, receivers absent, and a mix"""
    return [np.arange(n) % 4, np.full(n, 2), np.arange(n), rng.permutation(n), rng.choice([1, 3], n),
            rng.integers(0, receivers, n)]


def pictures(mode):
    return CB.camera_pictures() if mode == 68 else CB.legacy_pictures()


@pytest.mark.parametrize("flag", list(FLAGS))
@pytest.mark.parametrize("mode", [68, 4])
def test_replay_equals_the_direct_sequence(cb, entries, mode, flag):
    import torch
    flags = FLAGS[flag]
    pics = pictures(mode)
    n = len(pics)
    receivers = n + 2
    ents = [entries[i % 4] for i in range(receivers)]
    ctx, ref = cb.Context(mode, max_frames=n), cb.Context(mode, max_frames=n)
    slots = Slots(ctx, pics)
    states, ref_states = cb.receiver_states(ents), cb.receiver_states(ents)
    torch.cuda.synchronize()
    plan = slots.plan(ctx, states, flags)
    rng = np.random.default_rng(mode * 10 + flags)
    for k, of in enumerate(maps(n, receivers, rng)):
        slots.write(k)
        launch_and_check(cb, ctx, plan, slots, of, receivers, states, ref, ref_states, flags)
    assert ctx.get_ccm() is None
    plan.close()
    ctx.close()
    ref.close()


def test_empty_slots_and_guarded_states(cb, entries):
    import torch
    pics = CB.camera_pictures()
    n, receivers = len(pics), 4
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    ents = [entries[1], None, entries[2], entries[3]]
    ctx, ref = cb.Context(68, max_frames=n), cb.Context(68, max_frames=n)
    slots = Slots(ctx, pics)
    table = cb.receiver_states([entries[0]] + ents + [entries[0]])       # guard rows before and after the bound table
    raw = table.view(torch.int32).reshape(-1, 10)
    raw[0] = torch.tensor([0x7FC00001] * 9 + [0xDEAD], dtype=torch.int32, device="cuda")
    raw[-1] = torch.tensor([0x7FC00002] * 9 + [0xBEEF], dtype=torch.int32, device="cuda")
    guards = (raw[0].clone(), raw[-1].clone())
    states = table[1:receivers + 1]
    ref_states = cb.receiver_states(ents)
    torch.cuda.synchronize()
    plan = slots.plan(ctx, states, flags)
    bad = [-1, receivers, INT_MIN, INT_MAX]
    rng = np.random.default_rng(9)
    for k in range(4):
        of = rng.integers(0, receivers, n).astype(np.int64)
        pick = rng.choice(n, 4 + k, replace=False)
        of[pick] = [bad[(j + k) % 4] for j in range(len(pick))]
        slots.write(k)
        launch_and_check(cb, ctx, plan, slots, of, receivers, states, ref, ref_states, flags)
        assert torch.equal(raw[0], guards[0]) and torch.equal(raw[-1], guards[1])
    before = table.clone()
    launch_and_check(cb, ctx, plan, slots, np.full(n, -1), receivers, states, ref, ref_states, flags)    # every slot empty
    assert torch.equal(table, before)
    plan.close()
    ctx.close()
    ref.close()


def test_more_than_1024_slots(cb, entries):
    """one launch of 1 100 slots over about 100 receivers (the same few pictures, each bound to many slots) under CC_FIT, with a
    few empty slots"""
    import torch
    base = CB.camera_pictures()
    n, receivers = 1100, 100
    rng = np.random.default_rng(1100)
    ctx, ref = cb.Context(68, max_frames=n), cb.Context(68, max_frames=n)
    small = Slots(ctx, base)
    pick = rng.integers(0, len(base), n)

    class Many(Slots):
        def __init__(self):
            self.pics, self.n = [base[i] for i in pick], n
            self.ts, self.orders = [small.ts[i] for i in pick], [small.orders[i] for i in pick]
            self.of = torch.full((n,), -1, dtype=torch.int32, device="cuda")
            self.chunks = torch.full((n, ctx.info.data_bytes), 0xA5, dtype=torch.uint8, device="cuda")
            self.mask = torch.full((n,), -1, dtype=torch.int32, device="cuda")
            self.status = torch.full((n,), 7, dtype=torch.int32, device="cuda")
            self.flags = torch.full((n,), 0xEE, dtype=torch.uint8, device="cuda")
    slots = Many()
    ents = [entries[i % 4] for i in range(receivers)]
    states, ref_states = cb.receiver_states(ents), cb.receiver_states(ents)
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    torch.cuda.synchronize()
    plan = slots.plan(ctx, states, flags)
    of = rng.integers(0, receivers, n)
    of[rng.choice(n, 7, replace=False)] = -1
    got = launch_and_check(cb, ctx, plan, slots, of, receivers, states, ref, ref_states, flags)
    assert (got[1] != 0).sum() > n // 4                                   # premise: many pictures decode
    plan.close()
    ctx.close()
    ref.close()


@pytest.mark.parametrize("flag", list(FLAGS))
def test_launch_count(cb, entries, flag):
    """a launch counts its graph's kernel nodes: the direct receivers call's kernels on the same batch, and k_receivers_order"""
    import torch
    flags = FLAGS[flag]
    pics = CB.camera_pictures()
    n = len(pics)
    ctx, ref = cb.Context(68, max_frames=n), cb.Context(68, max_frames=n)
    slots = Slots(ctx, pics)
    ents = [entries[i % 4] for i in range(4)]
    states, ref_states = cb.receiver_states(ents), cb.receiver_states(ents)
    of = np.arange(n) % 4
    slots.of.copy_(torch.from_numpy(of.astype(np.int32)))
    torch.cuda.synchronize()
    plan = slots.plan(ctx, states, flags)
    before = cb.launch_count()
    plan.launch()
    per_launch = cb.launch_count() - before
    ctx.sync()
    before = cb.launch_count()
    direct(cb, ref, slots.ts, slots.orders, of, ref_states, flags)
    direct_launches = cb.launch_count() - before
    assert per_launch == graph_kernel_nodes(plan.graph) == direct_launches + EXTRA_KERNELS, (per_launch, direct_launches)
    plan.close()
    ctx.close()
    ref.close()


def test_context_state_and_plain_calls_around_it(cb, entries):
    """launches leave the context's CCM alone, and plain plans and direct calls on the same context give what they give on a context
    without the receivers plan"""
    import torch
    pics = CB.camera_pictures()
    n = len(pics)
    fit = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    m9 = np.array([[1.05, 0.02, 0], [0, 0.95, 0.01], [0.01, 0, 1.0]], np.float32)
    wh = np.array([(p.shape[1], p.shape[0]) for p in pics], np.int32)
    packed = torch.cat([torch.from_numpy(np.ascontiguousarray(p).reshape(-1)) for p in pics]).cuda()
    runs = []
    for with_receivers in (True, False):
        ctx = cb.Context(68, max_frames=n)
        ctx.set_ccm(m9)
        slots = Slots(ctx, pics)
        states = cb.receiver_states([entries[1], None, entries[3]])
        chunks = torch.zeros((n, ctx.info.data_bytes), dtype=torch.uint8, device="cuda")
        mask = torch.zeros(n, dtype=torch.int32, device="cuda")
        status = torch.zeros(n, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        rplan = slots.plan(ctx, states, fit) if with_receivers else None
        plain = ctx.camera_plan(wh, fit, packed.data_ptr(), chunks.data_ptr(), mask.data_ptr(), None, status.data_ptr())
        slots.of.copy_(torch.from_numpy((np.arange(n) % 3).astype(np.int32)))
        torch.cuda.synchronize()
        rec = []
        for step in range(4):
            if rplan is not None:
                rplan.launch()
                ctx.sync()
                assert same_ccm(ctx.get_ccm(), m9 if step == 0 else rec[-1][-1])
            if step % 2 == 0:
                plain.launch()
            else:
                ctx.scan_extract_decode_chunks_dev(packed.data_ptr(), wh, chunks.data_ptr(), mask.data_ptr(), status.data_ptr(), flags=fit)
            ctx.sync()
            rec.append((chunks.cpu().numpy(), mask.cpu().numpy(), status.cpu().numpy(), ctx.get_ccm()))
        runs.append(rec)
        plain.close()
        if rplan is not None:
            rplan.close()
        ctx.close()
    for a, b in zip(*runs):
        assert all(np.array_equal(x, y) for x, y in zip(a[:3], b[:3])) and same_ccm(a[3], b[3])


def test_inside_an_outer_graph_with_a_captured_map(cb, entries):
    import torch
    pics = CB.camera_pictures()
    n, receivers = len(pics), 5
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    ents = [entries[i % 4] for i in range(receivers)]
    ctx, ref = cb.Context(68, max_frames=n), cb.Context(68, max_frames=n)
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    slots = Slots(ctx, pics)
    staged = torch.zeros(n, dtype=torch.int32, device="cuda")
    states, ref_states = cb.receiver_states(ents), cb.receiver_states(ents)
    torch.cuda.synchronize()
    plan = slots.plan(ctx, states, flags)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=stream):
        slots.of.copy_(staged)
        plan.launch()
    rng = np.random.default_rng(77)
    for k in range(3):
        of = rng.integers(-1, receivers, n)
        slots.write(k)
        staged.copy_(torch.from_numpy(of.astype(np.int32)))
        torch.cuda.synchronize()
        g.replay()
        torch.cuda.synchronize()
        got = slots.records()
        idx = np.flatnonzero(of >= 0)
        want = direct(cb, ref, [slots.ts[i] for i in idx], [slots.orders[i] for i in idx], of[idx], ref_states, flags)
        for j in range(4):
            assert np.array_equal(got[j][idx], want[0][j]), (k, j)
        assert (got[2][of < 0] == cb.EXTRACT_EMPTY).all()
        assert torch.equal(states, ref_states)
    del g
    plan.close()
    ctx.close()
    ref.close()


def test_two_plans_double_buffered_and_launch_only_enqueues(cb, entries):
    """two receivers plans over one state table, each with its own pictures, map and outputs, launched alternately behind a sleeping
    stream: the launches return at once, and the results are the direct sequence's"""
    import torch
    pics = CB.camera_pictures()
    n, receivers = len(pics), 4
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    ents = [entries[1], None, entries[2], entries[3]]
    ctx, ref = cb.Context(68, max_frames=n), cb.Context(68, max_frames=n)
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    buf = [Slots(ctx, pics), Slots(ctx, pics)]
    states, ref_states = cb.receiver_states(ents), cb.receiver_states(ents)
    rng = np.random.default_rng(5)
    ofs = [rng.integers(-1, receivers, n) for _ in range(4)]
    for k in range(2):
        buf[k].write(k)
        buf[k].of.copy_(torch.from_numpy(ofs[k].astype(np.int32)))
    torch.cuda.synchronize()
    plans = [buf[i].plan(ctx, states, flags) for i in range(2)]
    with torch.cuda.stream(stream):
        torch.cuda._sleep(int(1.5e9))
    t0 = time.perf_counter()
    plans[0].launch()
    plans[1].launch()
    spent = time.perf_counter() - t0
    busy = not stream.query()
    ctx.sync()
    assert busy, "the stream finished before the launches returned"
    assert spent < 0.25, spent
    got = [buf[0].records(), buf[1].records()]
    for k in range(2, 4):                                                # two more, fed in stream order
        with torch.cuda.stream(stream):
            buf[k % 2].write(k)
            buf[k % 2].of.copy_(torch.from_numpy(ofs[k].astype(np.int32)))
        plans[k % 2].launch()
        ctx.sync()
        got.append(buf[k % 2].records())
    for k in range(4):
        of = ofs[k]
        idx = np.flatnonzero(of >= 0)
        ts, orders = layouts(variant(pics, k))
        want = direct(cb, ref, [ts[i] for i in idx], [orders[i] for i in idx], of[idx], ref_states, flags)
        for j in range(4):
            assert np.array_equal(got[k][j][idx], want[0][j]), (k, j)
    torch.cuda.synchronize()
    assert torch.equal(states, ref_states)
    for p in plans:
        p.close()
    ctx.close()
    ref.close()


def test_live_plan_freezes_buffers_and_a_chained_context_is_refused(cb, entries):
    import torch
    pics = CB.camera_pictures()
    small, large = pics[:3], pics
    ctx = cb.Context(68, max_frames=len(large))
    slots = Slots(ctx, small)
    states = cb.receiver_states([None])
    big = Slots(ctx, large)
    torch.cuda.synchronize()
    plan = slots.plan(ctx, states, 0)
    plan.launch()
    ctx.sync()
    with pytest.raises(cb.Cb200Error, match="camera plan"):
        ctx.scan_extract_decode_chunks_receivers_dev(big.ts, np.zeros(len(large), np.int32), states, big.chunks.data_ptr(), big.mask.data_ptr(),
                                                     big.status.data_ptr(), order=big.orders)
    with pytest.raises(cb.Cb200Error, match="would grow"):
        big.plan(ctx, states, 0)
    plan.close()
    ctx.scan_extract_decode_chunks_receivers_dev(big.ts, np.zeros(len(large), np.int32), states, big.chunks.data_ptr(), big.mask.data_ptr(),
                                                 big.status.data_ptr(), order=big.orders)
    ctx.sync()
    ctx.close()
    chained = cb.Context(68, max_frames=2)
    handle = chained.ccm_chain_root_create(1)
    chained.ccm_chain_attach(0, 1)
    one = Slots(chained, pics[:1])
    before = cb.launch_count()
    with pytest.raises(cb.Cb200Error, match="CCM chain"):
        one.plan(chained, states, 0)
    assert cb.launch_count() == before
    del handle
    chained.close()
