"""Camera plans (cb200_camera_plan_*): the enqueue-only camera call captured once in a CUDA graph.  A sequence of launches, with new
pictures written into the bound buffer in stream order before each, must give bit for bit what the same sequence of direct
enqueue-only calls gives on another context: records, masks, frame flags, statuses, the transforms and the CCM -- also when plan
launches, direct calls and cb200_set_ccm interleave, when the plan runs inside an outer graph, and with two plans double-buffered.
A launch (and a create once the buffers are sized) returns while the stream is still busy, and a live plan freezes the buffers its
graph uses.

cb200_get_frame_ccms is compared where the direct call's route is fixed (CC_FIT in mode B: every call fits).  Elsewhere the direct
call takes the matrix from the host or, while a CCM is still on its way, from the device; the plan always takes the device route."""
import time

import cv2
import numpy as np
import pytest

from oracle_lib import load_sample
from ragged_samples import GLOB, sample

pytestmark = pytest.mark.gpu

K = 6


@pytest.fixture(scope="module")
def cb():
    import libcimbar_b200 as cb
    return cb


def radius(w, h):
    """Scanner's blur radius (Scanner.h:93-103), as tests/test_gpu_scan_ragged.py restates it"""
    v = (int(min(w, h) * 0.002) - 1) & 0xFFFFFFFF
    for s in (1, 2, 4, 8, 16):
        v |= v >> s
    return max((v + 2) & 0xFFFFFFFF, 3) // 2


def pad(rgb, top, bottom, left, right):
    return cv2.copyMakeBorder(rgb, top, bottom, left, right, cv2.BORDER_CONSTANT, value=(0, 0, 0))


def ragged_4c():
    """the ragged sample batch of test_gpu_scan_ragged.py (cli_batch) and a 1.7x upscale (5 taps)"""
    pics = [sample(s) for s in GLOB]
    pics.append(pad(sample("6bit/4_30_f0_627.jpg"), 120, 150, 100, 160))
    pics.append(np.random.default_rng(47).integers(0, 256, (900, 1200, 3), dtype=np.uint8))
    pics.append(pad(sample("6bit/4_30_f1_360.jpg"), 90, 70, 200, 140))
    pics.append(sample("6bit/4_30_f2_734.jpg"))
    pics.append(cv2.resize(sample("6bit/4_30_f2_734.jpg"), None, fx=1.7, fy=1.7))
    return pics


def uniform_4c():
    land = [sample(s) for s in ("6bit/4_30_f0_627.jpg", "6bit/4_30_f2_246.jpg", "6bit/4_30_802.jpg")]
    padded = pad(cv2.resize(sample("6bit/4_30_f1_360.jpg"), (720, 960)), 0, 0, 280, 280)
    return [land[0], padded, np.random.default_rng(43).integers(0, 256, land[0].shape, dtype=np.uint8), land[1], land[2]]


def ragged_b():
    a, b = load_sample("b/ex2434.jpg"), load_sample("b/ex380.jpg")
    noise = np.random.default_rng(53).integers(0, 256, (800, 1000, 3), dtype=np.uint8)
    return [a, pad(b, 200, 160, 240, 300), noise, cv2.resize(a, None, fx=1.3, fy=1.3), b, pad(a, 60, 40, 80, 21)]


def uniform_b():
    a, b = load_sample("b/ex2434.jpg"), load_sample("b/ex380.jpg")
    size = (b.shape[1], b.shape[0])
    return [b, cv2.resize(a, size), pad(cv2.resize(b, (size[0] - 200, size[1] - 160)), 80, 80, 100, 100), b[::-1, ::-1].copy()]


BATCHES = {"4c_ragged": (4, ragged_4c), "4c_uniform": (4, uniform_4c), "b_ragged": (68, ragged_b), "b_uniform": (68, uniform_b)}


def variant(pics, k):
    """batch k of a sequence: the same sizes, other pixels"""
    f = [lambda p: p, lambda p: p[::-1, ::-1], lambda p: (p.astype(np.uint16) * 3 // 4).astype(np.uint8), lambda p: p[:, ::-1]][k % 4]
    return [np.ascontiguousarray(f(p)) for p in pics]


def host_packed(pics):
    import torch
    return torch.cat([torch.from_numpy(np.ascontiguousarray(p).reshape(-1)) for p in pics]).pin_memory()


def sizes(pics):
    return np.array([(p.shape[1], p.shape[0]) for p in pics], np.int32).reshape(-1, 2)


class Out:
    """the bound output buffers of one call / plan and its records copied out after each launch"""

    def __init__(self, ctx, n):
        import torch
        self.n, self.db = n, ctx.info.data_bytes
        self.chunks = torch.full((n * self.db,), 0xA5, dtype=torch.uint8, device="cuda")
        self.mask = torch.full((n,), -1, dtype=torch.int32, device="cuda")
        self.status = torch.full((n,), 7, dtype=torch.int32, device="cuda")
        self.flags = torch.full((n,), 0xEE, dtype=torch.uint8, device="cuda")
        self.saved = []

    def ptrs(self):
        return self.chunks.data_ptr(), self.mask.data_ptr(), self.flags.data_ptr(), self.status.data_ptr()

    def direct(self, ctx, d, wh, flags):
        ctx.scan_extract_decode_chunks_dev(d.data_ptr(), wh, self.chunks.data_ptr(), self.mask.data_ptr(), self.status.data_ptr(),
                                           self.flags.data_ptr(), flags=flags)

    def plan(self, ctx, d, wh, flags):
        return ctx.camera_plan(wh, flags, d.data_ptr(), self.chunks.data_ptr(), self.mask.data_ptr(), self.flags.data_ptr(),
                               self.status.data_ptr())

    def save(self):
        """copies of the records, in the current stream's order"""
        self.saved.append((self.chunks.clone(), self.mask.clone(), self.status.clone(), self.flags.clone()))

    def host(self):
        return [tuple(t.cpu().numpy() for t in s) for s in self.saved]


def same_ccm(a, b):
    return (a is None) == (b is None) and (a is None or np.array_equal(a, b))


def direct_sequence(cb, mode_val, batches, flags_seq, between=None):
    """the direct enqueue-only calls, one per batch, on a fresh context: records per call, transforms, CCM, frame CCMs"""
    import torch
    n = len(batches[0])
    ctx = cb.Context(mode_val, max_frames=n)
    wh = sizes(batches[0])
    d = torch.empty(sum(p.nbytes for p in batches[0]), dtype=torch.uint8, device="cuda")
    out = Out(ctx, n)
    for k, (b, f) in enumerate(zip(batches, flags_seq)):
        if between:
            between(ctx, k)
        d.copy_(host_packed(b))
        torch.cuda.synchronize()
        out.direct(ctx, d, wh, f)
        ctx.sync()
        out.save()
    try:
        fc = ctx.frame_ccms(n)
    except cb.Cb200Error:                                          # no call of the sequence took the fitted-CCM route
        fc = None
    res = out.host(), ctx.camera_transforms(n), ctx.get_ccm(), fc
    ctx.close()
    return res


def check_records(got, want, what):
    assert len(got) == len(want), what
    for k, (g, w) in enumerate(zip(got, want)):
        for a, b in zip(g, w):
            assert np.array_equal(a, b), (what, k)


@pytest.mark.parametrize("flagname", ["0", "SHARPEN", "SHARPEN_IF_NEEDED|CC_FIT", "CC_SIMPLE"])
@pytest.mark.parametrize("batch", list(BATCHES))
def test_replay_equals_the_direct_sequence(cb, batch, flagname):
    import torch
    mode_val, make = BATCHES[batch]
    pics = make()
    flags = 0
    for name in flagname.split("|"):
        flags |= getattr(cb, "FLAG_" + name) if name != "0" else 0
    batches = [variant(pics, k) for k in range(K)]
    want_rec, want_tr, want_ccm, want_fc = direct_sequence(cb, mode_val, batches, [flags] * K)
    n = len(pics)
    ctx = cb.Context(mode_val, max_frames=n)
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    wh = sizes(pics)
    d = torch.empty(sum(p.nbytes for p in pics), dtype=torch.uint8, device="cuda")
    out = Out(ctx, n)
    host = [host_packed(b) for b in batches]
    torch.cuda.synchronize()
    plan = out.plan(ctx, d, wh, flags)
    with torch.cuda.stream(stream):
        for k in range(K):
            d.copy_(host[k], non_blocking=True)
            plan.launch()
            out.save()
    ctx.sync()
    torch.cuda.synchronize()
    got = out.host()
    check_records(got, want_rec, (batch, flagname))
    assert np.array_equal(ctx.camera_transforms(n), want_tr)
    assert same_ccm(ctx.get_ccm(), want_ccm), (batch, flagname)
    if mode_val == 68 and flags & cb.FLAG_CC_FIT:
        assert np.array_equal(np.nan_to_num(ctx.frame_ccms(n), nan=-1), np.nan_to_num(want_fc, nan=-1))
    plan.close()
    ctx.close()


def test_premise_of_the_replay_test(cb):
    """the batches above take the 3-, 5- and 9-tap blurs, a picture on the per-pixel path, both K1 lists (plain and sharpened
    frames in one batch) and the exact walk on frames of both kinds"""
    import torch
    radii, per_pixel, kinds = set(), False, set()
    for name, (mode_val, make) in BATCHES.items():
        pics = make()
        radii |= {radius(p.shape[1], p.shape[0]) for p in pics}
        off = 0
        for p in pics:
            per_pixel |= p.shape[1] % 4 != 0 or off % 4 != 0
            off += p.shape[0] * p.shape[1]
        (rec,), _, _, _ = direct_sequence(cb, mode_val, [pics], [cb.FLAG_SHARPEN_IF_NEEDED])
        _, _, status, fflags = rec
        kinds |= {int(s) for s, f in zip(status, fflags) if s > 0 and f & cb.FRAME_FALLBACK}
        if name == "4c_ragged":
            assert {1, 2} <= set(status.tolist())                 # plain and sharpened frames in one batch
    assert {1, 2, 4} <= radii
    assert per_pixel
    assert kinds == {1, 2}, kinds                                   # walked frames, plain and sharpened
    torch.cuda.synchronize()


def test_ccm_carry_interleaved_with_direct_calls(cb):
    """plan launches, direct calls and cb200_set_ccm between them equal the same sequence of direct calls"""
    import torch
    pics = ragged_b()
    n = len(pics)
    fit = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    m9 = np.array([[1.05, 0.02, 0], [0, 0.95, 0.01], [0.01, 0, 1.0]], np.float32)
    # step k: (plan launch?, flags); set_ccm before steps 2 (m9) and 4 (None)
    steps = [(True, fit), (False, cb.FLAG_SHARPEN_IF_NEEDED), (True, fit), (False, 0), (True, fit), (False, fit)]
    sets = {2: m9, 4: None}
    batches = [variant(pics, k) for k in range(len(steps))]

    def between(ctx, k):
        if k in sets:
            ctx.set_ccm(sets[k])
    want_rec, want_tr, want_ccm, want_fc = direct_sequence(cb, 68, batches, [f for _, f in steps], between)
    ctx = cb.Context(68, max_frames=n)
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    wh = sizes(pics)
    d = torch.empty(sum(p.nbytes for p in pics), dtype=torch.uint8, device="cuda")
    out = Out(ctx, n)
    host = [host_packed(b) for b in batches]
    torch.cuda.synchronize()
    plan = out.plan(ctx, d, wh, fit)
    with torch.cuda.stream(stream):
        for k, (use_plan, f) in enumerate(steps):
            between(ctx, k)
            d.copy_(host[k], non_blocking=True)
            if use_plan:
                plan.launch()
            else:
                out.direct(ctx, d, wh, f)
            out.save()
    ctx.sync()
    check_records(out.host(), want_rec, "interleaved")
    assert np.array_equal(ctx.camera_transforms(n), want_tr)
    assert same_ccm(ctx.get_ccm(), want_ccm) and want_ccm is not None
    assert np.array_equal(np.nan_to_num(ctx.frame_ccms(n), nan=-1), np.nan_to_num(want_fc, nan=-1))
    plan.close()
    ctx.close()


def test_plan_inside_an_outer_graph(cb):
    """launch() inside a torch.cuda.graph capture adds the plan as a child node: replays of the outer graph give the direct records"""
    import torch
    pics = uniform_4c()
    n = len(pics)
    flags = cb.FLAG_SHARPEN_IF_NEEDED
    batches = [variant(pics, k) for k in range(3)]
    want_rec, _, _, _ = direct_sequence(cb, 4, batches, [flags] * 3)
    ctx = cb.Context(4, max_frames=n)
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    wh = sizes(pics)
    d = torch.empty(sum(p.nbytes for p in pics), dtype=torch.uint8, device="cuda")
    staged = torch.empty_like(d)
    out = Out(ctx, n)
    torch.cuda.synchronize()
    plan = out.plan(ctx, d, wh, flags)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=stream):
        d.copy_(staged)
        plan.launch()
        outs = tuple(t.clone() for t in (out.chunks, out.mask, out.status, out.flags))
    got = []
    for b in batches:
        staged.copy_(host_packed(b))
        torch.cuda.synchronize()
        g.replay()
        torch.cuda.synchronize()
        got.append(tuple(t.cpu().numpy() for t in outs))
    check_records(got, want_rec, "outer graph")
    del g
    plan.close()
    ctx.close()


def test_launch_and_create_only_enqueue(cb):
    import torch
    pics = ragged_b()
    n = len(pics)
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    ctx = cb.Context(68, max_frames=n)
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    wh = sizes(pics)
    d = torch.from_numpy(host_packed(pics).numpy()).cuda()
    out = Out(ctx, n)
    torch.cuda.synchronize()
    plan = out.plan(ctx, d, wh, flags)
    plan.launch()
    ctx.sync()
    before = cb.launch_count()
    plan.launch()
    ctx.sync()
    per_launch = cb.launch_count() - before
    assert per_launch >= 15, per_launch                            # the graph's kernels, counted once per launch
    with torch.cuda.stream(stream):
        torch.cuda._sleep(int(1.5e9))
    t0 = time.perf_counter()
    plan.launch()
    second = out.plan(ctx, d, wh, flags)                           # the buffers are sized: no wait
    second.launch()
    spent = time.perf_counter() - t0
    busy = not stream.query()
    ctx.sync()
    assert busy, "the stream finished before the calls returned"
    assert spent < 0.25, spent
    second.close()
    plan.close()
    ctx.close()


def test_two_plans_double_buffered(cb):
    """two plans on one context, each bound to its own picture buffer, fed by a copy stream one batch ahead"""
    import torch
    pics = ragged_4c()
    n = len(pics)
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    batches = [variant(pics, k) for k in range(4)]
    want_rec, _, want_ccm, _ = direct_sequence(cb, 4, batches, [flags] * 4)
    ctx = cb.Context(4, max_frames=n)
    compute, copy = torch.cuda.Stream(), torch.cuda.Stream()
    ctx.set_stream(compute.cuda_stream)
    wh = sizes(pics)
    nbytes = sum(p.nbytes for p in pics)
    d = [torch.empty(nbytes, dtype=torch.uint8, device="cuda") for _ in range(2)]
    outs = [Out(ctx, n) for _ in range(2)]
    host = [host_packed(b) for b in batches]
    torch.cuda.synchronize()
    plans = [outs[i].plan(ctx, d[i], wh, flags) for i in range(2)]
    copied = [torch.cuda.Event() for _ in range(2)]
    consumed = [torch.cuda.Event() for _ in range(2)]

    def h2d(k):
        with torch.cuda.stream(copy):
            if k >= 2:
                copy.wait_event(consumed[k % 2])
            d[k % 2].copy_(host[k], non_blocking=True)
            copied[k % 2].record(copy)
    h2d(0)
    order = []
    for k in range(len(batches)):
        compute.wait_event(copied[k % 2])
        plans[k % 2].launch()
        with torch.cuda.stream(compute):
            outs[k % 2].save()
        consumed[k % 2].record(compute)
        order.append(k % 2)
        if k + 1 < len(batches):
            h2d(k + 1)
    ctx.sync()
    torch.cuda.synchronize()
    recs = [o.host() for o in outs]
    got = [recs[i].pop(0) for i in order]
    check_records(got, want_rec, "double-buffered")
    assert same_ccm(ctx.get_ccm(), want_ccm)
    for p in plans:
        p.close()
    ctx.close()


def test_live_plan_freezes_its_buffers(cb):
    import torch
    pics = uniform_4c()
    small, large = pics[:2], pics
    ctx = cb.Context(4, max_frames=len(large))
    d_small = torch.from_numpy(host_packed(small).numpy()).cuda()
    d_large = torch.from_numpy(host_packed(large).numpy()).cuda()
    out = Out(ctx, len(large))
    torch.cuda.synchronize()
    plan = out.plan(ctx, d_small, sizes(small), 0)
    plan.launch()
    out.direct(ctx, d_small, sizes(small), 0)                     # the same size grows nothing
    ctx.sync()
    with pytest.raises(cb.Cb200Error, match="camera plan"):
        out.direct(ctx, d_large, sizes(large), 0)
    with pytest.raises(cb.Cb200Error, match="would grow"):
        ctx.camera_plan(sizes(large), 0, d_large.data_ptr(), *out.ptrs())
    plan.close()
    out.direct(ctx, d_large, sizes(large), 0)
    ctx.sync()
    ctx.close()
