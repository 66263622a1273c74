"""Detect receivers camera plans over device descriptors (cb200_camera_plan_create_detect_receivers_pictures_dev): candidates, map and
picture descriptors are all read from device memory at every launch, so every launch may put pictures of other sizes, layouts and
buffers in every slot.  The expected result of a launch is the direct call (cb200_detect_scan_extract_decode_chunks_receivers_dev) on
a second set of contexts with cloned state tables, on the launch's accepted non-empty slots alone, in slot order: records, masks,
statuses, modes, every mode's mask and every table, bit for bit.  An empty slot (no candidate below n_modes, or a receiver out of
range) and a refused slot (a descriptor a direct call refuses, or outside the bounds) both get mode -1, mask 0, a zeroed record and
mode-mask row and touch no table; the status tells them apart (EXTRACT_EMPTY / EXTRACT_REFUSED).  Every descriptor points at real
device memory, refused ones included, and all-auto, locked and mixed candidate sets are covered."""
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from gpu_support import cb  # noqa: E402,F401  (fixtures)
from gpu_support import (  # noqa: E402
    FLAGS, KINDS, RECV, as_tensor, bounds_of, close, entry_states, exact_pictures, graph_kernel_nodes, launches, nonempty, resized,
    run, stream_contexts)


@pytest.fixture(scope="module")
def pool(cb):
    """the detect tests' pictures, a transposed photograph and a 5-tap upscale"""
    p = exact_pictures(cb)
    return p + [np.ascontiguousarray(np.transpose(p[0], (1, 0, 2))), resized(p[0], 1700)]


class Slots:
    def __init__(self, cb, ctxs, n, bounds, states, flags, null_candidates=False):
        import torch
        self.cb, self.n, self.k = cb, n, len(ctxs)
        self.slot = max(c.info.data_bytes for c in ctxs)
        self.d_pics = torch.zeros((n, 40), dtype=torch.uint8, device="cuda")
        self.cand = torch.zeros(n, dtype=torch.int32, device="cuda")
        self.of = torch.full((n,), -1, dtype=torch.int32, device="cuda")
        self.chunks = torch.full((n, self.slot), 0xA5, dtype=torch.uint8, device="cuda")
        self.mask = torch.full((n,), -7, dtype=torch.int32, device="cuda")
        self.status = torch.full((n,), 7, dtype=torch.int32, device="cuda")
        self.mode = torch.full((n,), 9, dtype=torch.int32, device="cuda")
        self.mode_masks = torch.full((n, self.k), -7, dtype=torch.int32, device="cuda")
        self.keep = []
        torch.cuda.synchronize()
        self.plan = cb.detect_receivers_camera_plan_pictures_dev(ctxs, self.d_pics, bounds, None if null_candidates else self.cand, self.of, states,
                                                                 self.chunks.data_ptr(), self.mask.data_ptr(), self.status.data_ptr(),
                                                                 self.mode.data_ptr(), self.mode_masks.data_ptr(), flags=flags)

    def write(self, ts, orders, cand, of, tamper=None):
        import torch
        d = self.cb.picture_descriptors(ts, orders)
        for i in range(len(ts)):
            if tamper and tamper(i):
                p = self.cb.Picture.from_buffer_copy(d[i].tobytes())
                p.layout = 7                                                   # unknown
                d[i] = np.frombuffer(bytes(p), np.uint8)
        self.keep.append(ts)
        self.d_pics.copy_(torch.from_numpy(d))
        self.cand.copy_(torch.from_numpy(np.asarray(cand, np.uint32).view(np.int32)))
        self.of.copy_(torch.from_numpy(np.asarray(of, np.int64).astype(np.int32)))

    def records(self):
        return (self.chunks.cpu().numpy(), self.mask.cpu().numpy().view(np.uint32), self.status.cpu().numpy(), self.mode.cpu().numpy(),
                self.mode_masks.cpu().numpy().view(np.uint32))


def check(cb, got, refs, ts, orders, cand, of, R, refused, ref_states, flags):
    K = len(refs)
    idx = nonempty(cand, of, K, R)
    take = idx[~refused[idx]]
    chunks, mask, status, mode, mode_masks = got
    if len(take):
        want = run(cb, refs, [ts[i] for i in take], [orders[i] for i in take], np.asarray(of, np.int32)[take], ref_states,
                   np.asarray(cand, np.uint32)[take] & np.uint32((1 << K) - 1), flags)
        for j, (a, b) in enumerate(zip((chunks, mask, status, mode, mode_masks), want)):
            assert np.array_equal(a[take], b), ("records", "mask", "status", "mode", "mode masks")[j]
    rest = np.setdiff1d(np.arange(len(of)), take)
    assert (mode[rest] == -1).all() and (mask[rest] == 0).all() and not chunks[rest].any() and not mode_masks[rest].any()
    ref_slots = np.intersect1d(idx, np.flatnonzero(refused))
    assert (status[ref_slots] == cb.EXTRACT_REFUSED).all()
    assert (status[np.setdiff1d(rest, ref_slots)] == cb.EXTRACT_EMPTY).all()
    return take


SETS = {"one-geometry": [68, 4], "three-geometries": RECV}


@pytest.mark.parametrize("modes", list(SETS))
@pytest.mark.parametrize("sflag,ccflag", [FLAGS[0], FLAGS[4]])
def test_mixed_sizes_and_candidates_every_launch_equal_the_direct_call(cb, pool, modes, sflag, ccflag):
    """five launches (all-auto, locked, mixed sessions, empty slots of both kinds, random), each with a new assignment of pictures to
    slots in new allocations and layouts; refused slots (unknown layout, a picture below min_short) in launches 2 .. 4"""
    import torch
    modes = SETS[modes]
    flags = (getattr(cb, "FLAG_" + sflag) if sflag else 0) | (getattr(cb, "FLAG_" + ccflag) if ccflag else 0)
    n, K, R = 10, len(modes), 6
    lo, hi, lng = bounds_of(pool)
    assert lo >= 160                                                       # premise: room for a picture below the bounds
    small = resized(pool[0], lo - 60)
    rng = np.random.default_rng(len(modes) * 100 + flags)
    ctxs, stream = stream_contexts(cb, modes, n)
    refs, _ = stream_contexts(cb, modes, n)
    try:
        entries = entry_states(R, flags + K)
        states = [cb.receiver_states(entries) for _ in modes]
        ref_states = [s.clone() for s in states]
        slots = Slots(cb, ctxs, n, (lo, hi, lng), states, flags)
        counts, decoded = [], 0
        for k, (cand, of) in enumerate(launches(n, K, R, rng, modes)):
            pics = [pool[i] for i in rng.permutation(len(pool))[:n]]
            refused = np.zeros(n, bool)
            if k >= 2:
                pics[n - 1] = small
                refused[[n - 1, n - 3]] = True
            made = [as_tensor(p, KINDS[int(rng.integers(len(KINDS)))]) for p in pics]
            ts, orders = [t for t, _ in made], [o for _, o in made]
            with torch.cuda.stream(stream):
                slots.write(ts, orders, cand, of, (lambda i: i == n - 3) if k >= 2 else None)
            torch.cuda.synchronize()
            before = cb.launch_count()
            slots.plan.launch()
            counts.append(cb.launch_count() - before)
            ctxs[0].sync()
            got = slots.records()
            take = check(cb, got, refs, ts, orders, cand, of, R, refused, ref_states, flags)
            assert all(torch.equal(a, b) for a, b in zip(states, ref_states)), k
            decoded += int((got[3][take] >= 0).sum())
        assert decoded > 0
        assert len(set(counts)) == 1 and counts[0] == graph_kernel_nodes(slots.plan.graph), counts
        slots.plan.close()
    finally:
        close(ctxs, refs)


def test_all_refused_then_all_empty_with_stale_descriptors(cb, pool):
    import torch
    modes = RECV
    n, K, R = 6, len(modes), 4
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    ctxs, stream = stream_contexts(cb, modes, n)
    try:
        entries = entry_states(R, 5)
        states = [cb.receiver_states(entries) for _ in modes]
        before = [s.clone() for s in states]
        slots = Slots(cb, ctxs, n, bounds_of(pool), states, flags)
        rng = np.random.default_rng(4)
        made = [as_tensor(p, KINDS[i % len(KINDS)]) for i, p in enumerate(pool[:n])]
        ts, orders = [t for t, _ in made], [o for _, o in made]
        of = rng.integers(0, R, n)
        with torch.cuda.stream(stream):
            slots.write(ts, orders, np.full(n, (1 << K) - 1), of, lambda i: True)
        slots.plan.launch()
        ctxs[0].sync()
        got = slots.records()
        assert (got[2] == cb.EXTRACT_REFUSED).all() and (got[3] == -1).all() and not got[0].any() and not got[4].any()
        # every slot empty (no candidates, or no receiver), the descriptors left from the launch before
        with torch.cuda.stream(stream):
            slots.cand.copy_(torch.from_numpy(np.where(np.arange(n) % 2, 0, (1 << K) - 1).astype(np.int32)))
            slots.of.copy_(torch.from_numpy(np.where(np.arange(n) % 2, 0, -1).astype(np.int32)))
        slots.plan.launch()
        ctxs[0].sync()
        got = slots.records()
        assert (got[2] == cb.EXTRACT_EMPTY).all() and (got[3] == -1).all() and not got[0].any() and not got[4].any()
        assert all(torch.equal(a, b) for a, b in zip(states, before))
        slots.plan.close()
    finally:
        close(ctxs)


def test_inside_an_outer_graph_with_captured_copies(cb, pool):
    import torch
    modes = [68, 4]
    n, K, R = 6, 2, 4
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    ctxs, stream = stream_contexts(cb, modes, n)
    refs, _ = stream_contexts(cb, modes, n)
    try:
        entries = entry_states(R, 3)
        states = [cb.receiver_states(entries) for _ in modes]
        ref_states = [s.clone() for s in states]
        slots = Slots(cb, ctxs, n, bounds_of(pool), states, flags)
        staged = [torch.zeros((n, 40), dtype=torch.uint8, device="cuda"), torch.zeros(n, dtype=torch.int32, device="cuda"),
                  torch.zeros(n, dtype=torch.int32, device="cuda")]
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=stream):
            slots.d_pics.copy_(staged[0])
            slots.cand.copy_(staged[1])
            slots.of.copy_(staged[2])
            slots.plan.launch()
        rng = np.random.default_rng(21)
        for k in range(3):
            pics = [pool[i] for i in rng.permutation(len(pool))[:n]]
            made = [as_tensor(p, KINDS[int(rng.integers(len(KINDS)))]) for p in pics]
            ts, orders = [t for t, _ in made], [o for _, o in made]
            slots.keep.append(ts)
            cand = rng.integers(0, 4, n)
            of = rng.integers(-1, R, n)
            staged[0].copy_(torch.from_numpy(cb.picture_descriptors(ts, orders)))
            staged[1].copy_(torch.from_numpy(cand.astype(np.int32)))
            staged[2].copy_(torch.from_numpy(of.astype(np.int32)))
            torch.cuda.synchronize()
            g.replay()
            torch.cuda.synchronize()
            check(cb, slots.records(), refs, ts, orders, cand, of, R, np.zeros(n, bool), ref_states, flags)
            assert all(torch.equal(a, b) for a, b in zip(states, ref_states)), k
        del g
        slots.plan.close()
    finally:
        close(ctxs, refs)


def test_freezing_and_null_candidates(cb, pool):
    import torch
    modes = [68, 4]
    n, R = 4, 3
    ctxs, stream = stream_contexts(cb, modes, 2 * n)
    try:
        states = [cb.receiver_states(entry_states(R, 1)) for _ in modes]
        bounds = bounds_of(pool)
        slots = Slots(cb, ctxs, n, bounds, states, 0, null_candidates=True)
        made = [as_tensor(p, "rgb") for p in pool[:n]]
        with torch.cuda.stream(stream):
            slots.write([t for t, _ in made], [o for _, o in made], np.zeros(n), np.zeros(n))   # candidates unbound: every mode
        slots.plan.launch()
        ctxs[0].sync()
        assert (slots.records()[2] != cb.EXTRACT_EMPTY).all()
        with pytest.raises(cb.Cb200Error, match="would grow"):
            Slots(cb, ctxs, n, (bounds[0], bounds[1], bounds[2] + 300), states, 0)
        with pytest.raises(cb.Cb200Error, match="would grow"):
            Slots(cb, ctxs, 2 * n, bounds, states, 0)
        slots.plan.close()
        Slots(cb, ctxs, 2 * n, bounds, states, 0).plan.close()
    finally:
        close(ctxs)
