"""Detect receivers camera plans (cb200_camera_plan_create_detect_receivers): the auto mode for receivers captured once, its candidate
masks and receiver map read from device memory at every launch.  The expected result of a launch is always the direct call
(cb200_detect_scan_extract_decode_chunks_receivers_dev) on a second set of contexts with cloned state tables, on the launch's
non-empty slots alone, in slot order, scattered back: records, masks, statuses, modes, every mode's mask and every table, bit for
bit.  A slot is empty when its receiver lies outside [0, n_receivers) or its candidates have no bit below n_modes: mode -1, mask 0,
a zeroed record, a zero row of mode masks, status EXTRACT_EMPTY, and no state read or written.
  - exactness under the detect tests' flag sets, for one mode, two modes of one geometry and all three geometries, over five
    launches with new pixels, candidates and maps (all-auto, locked, mixed, empty slots of both kinds, random), states carried;
  - receivers without a picture keep their entries byte for byte, poisoned ones included;
  - a batch locked to 68 walks one geometry: one long k_flood_walk, the two absent geometries' walks short; all-auto walks three;
  - the launch count is the graph's kernels whatever the map; the plan inside an outer torch graph with captured copies; two plans
    on the same contexts double-buffer and launch() only enqueues; a live plan freezes every context's buffers, the detect call's
    included, and keeps refusing direct detect calls; closing one context destroys the plan; a chained context is refused."""
import os
import sys
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from gpu_support import cb  # noqa: E402,F401  (fixtures)
from gpu_support import (  # noqa: E402
    FLAGS, RECV, close, entry_states, exact_pictures, graph_kernel_nodes, launches, layouts, nonempty, run, stream_contexts)


@pytest.fixture(scope="module")
def pics(cb):
    """the detect receivers tests' pool: mode-B / 4C photographs, rendered 66 and 67 frames, a noise picture"""
    return exact_pictures(cb)


def variant(pics, k):
    """the pixels of launch k: the same sizes, other content"""
    f = [lambda p: p, lambda p: (p.astype(np.uint16) * 3 // 4).astype(np.uint8), lambda p: p[::-1, ::-1], lambda p: p][k % 4]
    return [np.ascontiguousarray(f(p)) for p in pics]


class Slots:
    """n bound pictures in mixed layouts, the bound candidates, map and outputs of one plan"""

    def __init__(self, ctxs, pics):
        import torch
        self.pics, self.k = pics, len(ctxs)
        self.ts, self.orders = layouts(pics)
        n = self.n = len(pics)
        self.slot = max(c.info.data_bytes for c in ctxs)
        self.cand = torch.zeros(n, dtype=torch.int32, device="cuda")
        self.of = torch.full((n,), -1, dtype=torch.int32, device="cuda")
        self.chunks = torch.full((n, self.slot), 0xA5, dtype=torch.uint8, device="cuda")
        self.mask = torch.full((n,), -7, dtype=torch.int32, device="cuda")
        self.status = torch.full((n,), 7, dtype=torch.int32, device="cuda")
        self.mode = torch.full((n,), 9, dtype=torch.int32, device="cuda")
        self.mode_masks = torch.full((n, self.k), -7, dtype=torch.int32, device="cuda")

    def write(self, k):
        """launch k's pixels into the bound pictures (on the current stream)"""
        for t, s in zip(self.ts, layouts(variant(self.pics, k))[0]):
            t.copy_(s)

    def set(self, cand, of):
        import torch
        self.cand.copy_(torch.from_numpy(np.asarray(cand, np.uint32).view(np.int32)))
        self.of.copy_(torch.from_numpy(np.asarray(of, np.int32)))

    def plan(self, cb, ctxs, states, flags, null_candidates=False):
        return cb.detect_receivers_camera_plan(ctxs, self.ts, None if null_candidates else self.cand, self.of, states, self.chunks.data_ptr(),
                                               self.mask.data_ptr(), self.status.data_ptr(), self.mode.data_ptr(), self.mode_masks.data_ptr(),
                                               flags=flags, order=self.orders)

    def records(self):
        return (self.chunks.cpu().numpy(), self.mask.cpu().numpy().view(np.uint32), self.status.cpu().numpy(), self.mode.cpu().numpy(),
                self.mode_masks.cpu().numpy().view(np.uint32))


def check_launch(cb, got, refs, slots, ts, orders, cand, of, R, ref_states, flags):
    """got (a launch's records) against the direct call on refs over the non-empty slots alone; ref_states advance in place"""
    K = len(refs)
    idx = nonempty(cand, of, K, R)
    chunks, mask, status, mode, mode_masks = got
    if len(idx):
        want = run(cb, refs, [ts[i] for i in idx], [orders[i] for i in idx], np.asarray(of, np.int32)[idx], ref_states,
                   np.asarray(cand, np.uint32)[idx] & np.uint32((1 << K) - 1), flags)
        for j, (a, b) in enumerate(zip((chunks, mask, status, mode, mode_masks), want)):
            assert np.array_equal(a[idx], b), ("records", "mask", "status", "mode", "mode masks")[j]
    empty = np.setdiff1d(np.arange(len(of)), idx)
    assert (mode[empty] == -1).all() and (mask[empty] == 0).all() and not chunks[empty].any() and not mode_masks[empty].any()
    assert (status[empty] == cb.EXTRACT_EMPTY).all()
    return idx


# ------------------------------------------------------------------------------------------------ exactness
SETS = {"one-mode": [68], "one-geometry": [68, 4], "three-geometries": RECV}


@pytest.mark.parametrize("modes", list(SETS))
@pytest.mark.parametrize("sflag,ccflag", FLAGS)
def test_each_launch_equals_the_direct_call_on_its_nonempty_slots(cb, pics, modes, sflag, ccflag):
    import torch
    modes = SETS[modes]
    flags = (getattr(cb, "FLAG_" + sflag) if sflag else 0) | (getattr(cb, "FLAG_" + ccflag) if ccflag else 0)
    n, K, R = len(pics), len(modes), 6
    rng = np.random.default_rng(len(modes) * 100 + flags)
    ctxs, stream = stream_contexts(cb, modes, n)
    refs, _ = stream_contexts(cb, modes, n)
    try:
        entries = entry_states(R, flags + K)
        states = [cb.receiver_states(entries) for _ in modes]
        ref_states = [s.clone() for s in states]
        slots = Slots(ctxs, pics)
        torch.cuda.synchronize()
        plan = slots.plan(cb, ctxs, states, flags)
        decoded = 0
        for k, (cand, of) in enumerate(launches(n, K, R, rng, modes)):
            slots.write(k)
            slots.set(cand, of)
            torch.cuda.synchronize()
            plan.launch()
            ctxs[0].sync()
            got = slots.records()
            idx = check_launch(cb, got, refs, slots, slots.ts, slots.orders, cand, of, R, ref_states, flags)
            assert all(torch.equal(a, b) for a, b in zip(states, ref_states)), k
            decoded += int((got[3][idx] >= 0).sum())
        assert decoded > 0                                      # premise: pictures decode
        for s in states:                                        # the receiver without pictures, byte for byte
            assert np.array_equal(s.cpu().numpy().reshape(R, 10)[R - 1], cb.receiver_states(entries).cpu().numpy().reshape(R, 10)[R - 1])
        for c in ctxs:
            assert c.get_ccm() is None                          # no context's own CCM is read or changed
        plan.close()
    finally:
        close(ctxs, refs)


def test_null_candidates_and_untouched_receivers(cb, pics):
    """candidates = NULL decodes every non-empty slot under every mode; receivers without a picture keep their entries byte for
    byte, poisoned entries included"""
    import torch
    n, K, R = len(pics), len(RECV), 6
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    ctxs, _ = stream_contexts(cb, RECV, n)
    refs, _ = stream_contexts(cb, RECV, n)
    try:
        states = [cb.receiver_states(entry_states(R, 40 + k)) for k in range(K)]
        for s in states:
            s.view(torch.int32).reshape(-1, 10)[4] = torch.tensor([0x7FC00001] * 9 + [0xDEAD], dtype=torch.int32, device="cuda")
        before = [s.clone() for s in states]
        ref_states = [s.clone() for s in states]
        slots = Slots(ctxs, pics)
        torch.cuda.synchronize()
        plan = slots.plan(cb, ctxs, states, flags, null_candidates=True)
        for k, of in enumerate([np.arange(n) % 3, np.where(np.arange(n) % 4 == 0, -1, np.arange(n) % 2)]):   # 3 .. 5 never have one
            slots.write(k)
            slots.set(np.zeros(n), of)                            # ignored: no candidates are bound
            torch.cuda.synchronize()
            plan.launch()
            ctxs[0].sync()
            check_launch(cb, slots.records(), refs, slots, slots.ts, slots.orders, np.full(n, (1 << K) - 1), of, R, ref_states, flags)
            assert all(torch.equal(a, b) for a, b in zip(states, ref_states)), k
        for s, b in zip(states, before):
            assert torch.equal(s.reshape(R, 10)[3:], b.reshape(R, 10)[3:])
        plan.close()
    finally:
        close(ctxs, refs)


# ------------------------------------------------------------------------------------------------ premises
def walks(fn):
    """durations in ms of every k_flood_walk fn() runs (torch.profiler)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sorted(e.time_range.elapsed_us() / 1e3 for e in prof.events()
                  if e.device_type == torch.autograd.DeviceType.CUDA and "k_flood_walk" in e.name)


def test_a_locked_batch_walks_one_geometry(cb, pics):
    """on [66, 68, 67, 4], a launch locked to 68 runs one long walk (the 1024 x 1024 geometry's) and two short ones (66's and 67's
    geometries, whose slots are all absent); an all-auto launch runs three long walks"""
    import torch
    n, K, R = len(pics), len(RECV), 4
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    ctxs, _ = stream_contexts(cb, RECV, n)
    try:
        states = [cb.receiver_states(entry_states(R, 50)) for _ in RECV]
        slots = Slots(ctxs, pics)
        of = np.arange(n) % R
        torch.cuda.synchronize()
        plan = slots.plan(cb, ctxs, states, flags)
        slots.set(np.full(n, (1 << K) - 1), of)
        plan.launch()                                           # warm-up
        ctxs[0].sync()

        def launch():
            plan.launch()
            ctxs[0].sync()
        auto = walks(launch)
        slots.set(np.full(n, 1 << RECV.index(68)), of)
        locked = walks(launch)
        assert len(locked) == 3 and len(auto) == 3, (locked, auto)
        assert locked[2] > 10 and locked[1] < 1, locked
        assert auto[0] > 10, auto
        plan.close()
    finally:
        close(ctxs)


@pytest.mark.parametrize("flags", [0, 0x20 | 8])
def test_launch_count_is_the_graphs_kernels_for_every_map(cb, pics, flags):
    import torch
    n, K, R = len(pics), len(RECV), 5
    rng = np.random.default_rng(9)
    ctxs, _ = stream_contexts(cb, RECV, n)
    try:
        states = [cb.receiver_states(entry_states(R, 60)) for _ in RECV]
        slots = Slots(ctxs, pics)
        torch.cuda.synchronize()
        plan = slots.plan(cb, ctxs, states, flags)
        counts = []
        for cand, of in launches(n, K, R, rng, RECV):
            slots.set(cand, of)
            torch.cuda.synchronize()
            before = cb.launch_count()
            plan.launch()
            counts.append(cb.launch_count() - before)
            ctxs[0].sync()
        assert counts == [graph_kernel_nodes(plan.graph)] * len(counts), counts
        plan.close()
    finally:
        close(ctxs)


def test_inside_an_outer_graph_with_captured_copies(cb, pics):
    """the plan as a child node of a torch graph whose captured copies write the candidates and the map"""
    import torch
    n, K, R = len(pics), len(RECV), 5
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    rng = np.random.default_rng(77)
    ctxs, stream = stream_contexts(cb, RECV, n)
    refs, _ = stream_contexts(cb, RECV, n)
    try:
        states = [cb.receiver_states(entry_states(R, 70)) for _ in RECV]
        ref_states = [s.clone() for s in states]
        slots = Slots(ctxs, pics)
        staged_cand = torch.zeros(n, dtype=torch.int32, device="cuda")
        staged_of = torch.zeros(n, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        plan = slots.plan(cb, ctxs, states, flags)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=stream):
            slots.cand.copy_(staged_cand)
            slots.of.copy_(staged_of)
            plan.launch()
        for k, (cand, of) in enumerate(launches(n, K, R, rng, RECV)[2:]):
            slots.write(k)
            staged_cand.copy_(torch.from_numpy(np.asarray(cand, np.uint32).view(np.int32)))
            staged_of.copy_(torch.from_numpy(np.asarray(of, np.int32)))
            torch.cuda.synchronize()
            g.replay()
            torch.cuda.synchronize()
            check_launch(cb, slots.records(), refs, slots, slots.ts, slots.orders, cand, of, R, ref_states, flags)
            assert all(torch.equal(a, b) for a, b in zip(states, ref_states)), k
        del g
        plan.close()
    finally:
        close(ctxs, refs)


def test_two_plans_double_buffered_and_launch_only_enqueues(cb, pics):
    """two plans on the same contexts and state tables, each with its own pictures, candidates, map and outputs, launched alternately
    behind a sleeping stream: the launches return at once, and the results are the direct sequence's"""
    import torch
    n, K, R = len(pics), len(RECV), 5
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    rng = np.random.default_rng(5)
    ctxs, stream = stream_contexts(cb, RECV, n)
    refs, _ = stream_contexts(cb, RECV, n)
    try:
        states = [cb.receiver_states(entry_states(R, 80)) for _ in RECV]
        ref_states = [s.clone() for s in states]
        buf = [Slots(ctxs, pics), Slots(ctxs, pics)]
        batches = launches(n, K, R, rng, RECV)[:4]
        for k in range(2):
            buf[k].write(k)
            buf[k].set(*batches[k])
        torch.cuda.synchronize()
        plans = [buf[i].plan(cb, ctxs, states, flags) for i in range(2)]
        with torch.cuda.stream(stream):
            torch.cuda._sleep(int(1.5e9))
        t0 = time.perf_counter()
        plans[0].launch()
        plans[1].launch()
        spent = time.perf_counter() - t0
        busy = not stream.query()
        ctxs[0].sync()
        assert busy, "the stream finished before the launches returned"
        assert spent < 0.25, spent
        got = [buf[0].records(), buf[1].records()]
        for k in range(2, 4):                                   # two more, fed in stream order
            with torch.cuda.stream(stream):
                buf[k % 2].write(k)
                buf[k % 2].set(*batches[k])
            plans[k % 2].launch()
            ctxs[0].sync()
            got.append(buf[k % 2].records())
        for k in range(4):
            ts, orders = layouts(variant(pics, k))
            check_launch(cb, got[k], refs, buf[k % 2], ts, orders, batches[k][0], batches[k][1], R, ref_states, flags)
        torch.cuda.synchronize()
        assert all(torch.equal(a, b) for a, b in zip(states, ref_states))
        for p in plans:
            p.close()
    finally:
        close(ctxs, refs)


# ------------------------------------------------------------------------------------------------ lifecycle
def test_live_plan_freezes_every_context_and_closing_one_destroys_it(cb, pics):
    import torch
    n, R = len(pics), 3
    small = pics[:4]
    ctxs, _ = stream_contexts(cb, RECV, n)
    try:
        states = [cb.receiver_states(entry_states(R, 90)) for _ in RECV]
        # every context's own camera buffers at n pictures: only the detect call's buffers are still small
        for c in ctxs:
            out = Slots([c], pics)
            c.scan_extract_decode_chunks_pictures_dev(out.ts, out.chunks.data_ptr(), out.mask.data_ptr(), out.status.data_ptr(), order=out.orders)
            c.sync()
        few, many = Slots(ctxs, small), Slots(ctxs, pics)
        torch.cuda.synchronize()
        plan = few.plan(cb, ctxs, states, 0)
        few.set(np.full(len(small), 0b1111), np.arange(len(small)) % R)
        plan.launch()
        ctxs[0].sync()
        with pytest.raises(cb.Cb200Error, match="detect statuses"):
            many.plan(cb, ctxs, states, 0)
        with pytest.raises(cb.Cb200Error, match="live camera plans"):
            cb.detect_scan_extract_decode_chunks_receivers_dev(ctxs, few.ts, np.zeros(len(small), np.int32), states, few.chunks.data_ptr(),
                                                               few.mask.data_ptr(), few.status.data_ptr(), few.mode.data_ptr(), order=few.orders)
        largest = max(pics, key=lambda p: p.shape[0] * p.shape[1])
        for c in ctxs[1:]:                                      # the plan freezes every context, not only the first
            big = Slots([c], [largest] * n)                     # more pixels than any call so far: the scan's buffers would grow
            with pytest.raises(cb.Cb200Error, match="would grow"):
                c.scan_extract_decode_chunks_pictures_dev(big.ts, big.chunks.data_ptr(), big.mask.data_ptr(), big.status.data_ptr(),
                                                          order=big.orders)
            del big
        second = Slots(ctxs, small)                             # a second plan of the same size grows nothing: accepted
        plan2 = second.plan(cb, ctxs, states, 0)
        plan2.close()
        ctxs[2].close()                                         # destroys the plan on every context
        plan.close()                                            # safe: the plan went with the context
        rest = [ctxs[0], ctxs[1], ctxs[3]]
        out = Slots(rest, small)
        torch.cuda.synchronize()
        cb.detect_scan_extract_decode_chunks_receivers_dev(rest, out.ts, np.zeros(len(small), np.int32), [states[0], states[1], states[3]],
                                                           out.chunks.data_ptr(), out.mask.data_ptr(), out.status.data_ptr(), out.mode.data_ptr(),
                                                           order=out.orders)
        rest[0].sync()
    finally:
        close(ctxs)


def test_a_chained_context_is_refused(cb, pics):
    import torch
    chained = cb.Context(68, max_frames=2)
    other = cb.Context(4, max_frames=2)
    stream = torch.cuda.Stream()
    try:
        for c in (other, chained):
            c.set_stream(stream.cuda_stream)
        handle = chained.ccm_chain_root_create(1)
        chained.ccm_chain_attach(0, 1)
        one = Slots([other, chained], pics[:1])
        states = [cb.receiver_states([None]) for _ in range(2)]
        torch.cuda.synchronize()
        before = cb.launch_count()
        with pytest.raises(cb.Cb200Error, match="context 1 is linked to a CCM chain"):
            one.plan(cb, [other, chained], states, 0)
        assert cb.launch_count() == before
        del handle
    finally:
        close([other, chained])
