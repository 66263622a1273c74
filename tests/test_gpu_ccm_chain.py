"""The CC_FIT colour correction chained across ranks (csrc/chain.cu, dist.CameraExchange): ranks run as separate processes spawned
here (all on one H100 -- CUDA IPC works between processes on one device -- and one per GPU where there are two or more), each decoding
its contiguous stripe of every step's batch.  What rank 0 collects, and the CCM every rank holds after each step, must equal one
context's decode of the whole stream bit for bit; each test asserts its premise (without the chain the split changes the result)."""
import os
import subprocess
import sys
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)

import chain_batches as CB  # noqa: E402
from gpu_support import cb  # noqa: F401  (fixtures)


def _gpus():
    import torch
    return torch.cuda.device_count()


_port = [29611]


def spawn(scenario, world, tmp_path, per_gpu=False):
    """runs ccm_chain_worker.py on `world` processes (joined before returning); returns each rank's saved results"""
    _port[0] += 1
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world), "--master-addr", "127.0.0.1",
           "--master-port", str(_port[0]), os.path.join(HERE, "ccm_chain_worker.py"), scenario, str(tmp_path)]
    if per_gpu:
        cmd.append("--per-gpu")
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-4000:]
    return [dict(np.load(os.path.join(tmp_path, f"rank{r}.npz"))) for r in range(world)]


def ccm_or_nan(ctx):
    m = ctx.get_ccm()
    return np.full((3, 3), np.nan, np.float32) if m is None else m


def same(a, b):
    return np.array_equal(a, b, equal_nan=True)


# ------------------------------------------------------------------------------------------------ references (one context)
def frames_reference(cb, frames_list, chained_split=None):
    """one context's decode of the steps' frame batches (chained_split = (rank, world, per): only that rank's stripes, on a context of
    its own, unchained -- what every rank computed before the chain); per step (chunks, masks, CCM after the step)"""
    import torch
    from libcimbar_b200.dist import stripe
    per_max = max(len(f) for f in frames_list)
    ctx = cb.Context(68, max_frames=per_max)
    d_chunks = torch.zeros((per_max, ctx.info.data_bytes), dtype=torch.uint8, device="cuda")
    d_mask = torch.zeros(per_max, dtype=torch.int32, device="cuda")
    out = []
    for frames in frames_list:
        if chained_split:
            a, b = stripe(len(frames), chained_split[0], chained_split[2])
            frames = frames[a:b]
        d_fr = torch.from_numpy(np.ascontiguousarray(frames)).cuda()
        torch.cuda.synchronize()
        ctx.decode_chunks_dev(d_fr.data_ptr(), len(frames), d_chunks.data_ptr(), d_mask.data_ptr(), flags=cb.FLAG_CC_FIT)
        ctx.sync()
        out.append((d_chunks[:len(frames)].cpu().numpy(), d_mask[:len(frames)].cpu().numpy(), ccm_or_nan(ctx), ctx.frame_ccms(len(frames))))
    ctx.close()
    return out


def camera_reference(cb, mode_val, batches, jpeg=False, split=None):
    """one context's scan_extract_decode_chunks_ragged_dev (or the JPEG form) over every step's whole batch; split = (rank, per): only
    that rank's stripes, on a context of its own, unchained.  Per step (chunks, masks, statuses, CCM after the step, the matrices of
    the frames -- mode B only)"""
    import torch
    from libcimbar_b200.dist import stripe
    if split:
        batches = [b[slice(*stripe(len(b), split[0], split[1]))] for b in batches]
    n_max = max(max(len(b) for b in batches), 1)
    ctx = cb.Context(mode_val, max_frames=n_max)
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    d_chunks = torch.zeros((n_max, ctx.info.data_bytes), dtype=torch.uint8, device="cuda")
    d_mask = torch.zeros(n_max, dtype=torch.int32, device="cuda")
    d_status = torch.zeros(n_max, dtype=torch.int32, device="cuda")
    out = []
    for batch in batches:
        n = len(batch)
        if n == 0:
            out.append((np.zeros((0, ctx.info.data_bytes), np.uint8), np.zeros(0, np.uint32), np.zeros(0, np.int32), ccm_or_nan(ctx), None))
            continue
        if jpeg:
            ctx.jpeg_scan_extract_decode_chunks_dev(batch, d_chunks.data_ptr(), d_mask.data_ptr(), d_status.data_ptr(), flags=flags)
        else:
            d = torch.cat([torch.from_numpy(p.reshape(-1)) for p in batch]).cuda()
            wh = np.array([(p.shape[1], p.shape[0]) for p in batch], np.int32)
            torch.cuda.synchronize()
            ctx.scan_extract_decode_chunks_dev(d.data_ptr(), wh, d_chunks.data_ptr(), d_mask.data_ptr(), d_status.data_ptr(), flags=flags)
        ctx.sync()
        out.append((d_chunks[:n].cpu().numpy(), d_mask[:n].cpu().numpy().astype(np.uint32), d_status[:n].cpu().numpy(), ccm_or_nan(ctx),
                    ctx.frame_ccms(n) if mode_val == 68 else None))
    ctx.close()
    return out


# ------------------------------------------------------------------------------------------------ crafted fountain frames
@pytest.mark.parametrize("world,per_gpu", [(2, False), (3, False), (2, True)])
def test_frames_equal_one_context(cb, tmp_path, world, per_gpu):
    if per_gpu and _gpus() < 2:
        pytest.skip("needs two GPUs")
    steps, per = CB.frame_steps(world)
    want = frames_reference(cb, steps)
    # premise: decoded on their own (no chain), the stripes give other records than one context on at least one frame
    alone = [frames_reference(cb, steps, (r, world, per)) for r in range(world)]
    assert any(not np.array_equal(np.concatenate([alone[r][s][0] for r in range(world)]), want[s][0]) or
               not np.array_equal(np.concatenate([alone[r][s][1] for r in range(world)]), want[s][1]) for s in range(len(steps)))
    assert not np.isnan(want[0][2]).any()                        # premise: step 1 fits
    got = spawn("frames", world, tmp_path, per_gpu)
    for s, (wc, wm, wccm, wf) in enumerate(want, start=1):
        cat_c = np.concatenate([got[r][f"chunks{s}"] for r in range(world)])
        cat_m = np.concatenate([got[r][f"mask{s}"] for r in range(world)])
        assert np.array_equal(cat_c, wc) and np.array_equal(cat_m, wm), s
        assert same(np.concatenate([got[r][f"fccm{s}"] for r in range(world)]), wf), s       # every frame's matrix
        for r in range(world):
            assert same(got[r][f"ccm{s}"], wccm), (s, r)


def unchained_differs(cb, mode_val, steps, world, per, jpeg=False):
    """the stripes decoded on their own, each rank's in order on a context of its own: other records than one context's?"""
    alone = [camera_reference(cb, mode_val, steps, jpeg=jpeg, split=(r, per)) for r in range(world)]
    want = camera_reference(cb, mode_val, steps, jpeg=jpeg)
    for s in range(len(steps)):
        for k in (0, 1):
            if not np.array_equal(np.concatenate([alone[r][s][k] for r in range(world)]), want[s][k]):
                return True
    return False


# ------------------------------------------------------------------------------------------------ camera batches
@pytest.mark.parametrize("world,kind,mode_val,per_gpu", [(2, "window", 68, False), (3, "direct", 68, False), (3, "window", 68, False),
                                                         (2, "direct", 68, False), (2, "window", 68, True), (2, "window", 4, False)])
def test_camera_batches_equal_one_context(cb, tmp_path, world, kind, mode_val, per_gpu):
    """mode B: fits carried across stripe boundaries.  Mode 4C is a legacy mode, which never fits a CCM: there the case only shows
    that a linked context changes nothing"""
    if per_gpu and _gpus() < 2:
        pytest.skip("needs two GPUs")
    steps, per = CB.camera_steps(world) if mode_val == 68 else CB.legacy_steps(world)
    want = camera_reference(cb, mode_val, steps)
    st = set(np.concatenate([w[2] for w in want]).tolist())
    assert 0 in st and st & {1, 2}                                   # premise: failed and extracted pictures
    assert (want[0][1] != 0).sum() >= 3                              # premise: chunks decode
    if mode_val == 68:
        assert unchained_differs(cb, mode_val, steps, world, per)    # premise: without the chain the split changes the records
    got = spawn(f"camera-{kind}-{mode_val}", world, tmp_path, per_gpu)
    for s, (wc, wm, wst, wccm, wf) in enumerate(want, start=1):
        assert np.array_equal(got[0][f"status{s}"], wst), s
        assert np.array_equal(got[0][f"mask{s}"], wm), s
        assert np.array_equal(got[0][f"chunks{s}"], wc), s
        if mode_val == 68:
            assert same(np.concatenate([got[r][f"fccm{s}"] for r in range(world)]), wf), s
        for r in range(world):
            assert same(got[r][f"ccm{s}"], wccm), (s, r)


def test_jpeg_files_equal_one_context(cb, tmp_path):
    steps, per = CB.jpeg_steps(3)
    want = camera_reference(cb, 68, steps, jpeg=True)
    assert (want[0][1] != 0).sum() >= 3
    assert unchained_differs(cb, 68, steps, 3, per, jpeg=True)
    got = spawn("jpeg-window", 3, tmp_path)
    wc, wm, wst, wccm, wf = want[0]
    assert np.array_equal(got[0]["status1"], wst) and np.array_equal(got[0]["mask1"], wm) and np.array_equal(got[0]["chunks1"], wc)
    assert same(np.concatenate([got[r]["fccm1"] for r in range(3)]), wf)
    for r in range(3):
        assert same(got[r]["ccm1"], wccm), r


# ------------------------------------------------------------------------------------------------ one process: a chain of one rank
def linked(cb, mode_val, n):
    ctx = cb.Context(mode_val, max_frames=n)
    ctx.ccm_chain_root_create(1)
    ctx.ccm_chain_attach(0, 1)
    return ctx


def test_launch_counts_and_refused_mixes(cb):
    """an unattached context launches what it always did; a linked one three more kernels per CC_FIT call (publish, link, settle)
    and the same records; the host-CCM calls, a CC_FIT call without a step and a second step are refused before any CUDA call"""
    import torch
    steps, _ = CB.frame_steps(3)
    frames = steps[0]
    n = len(frames)
    d_fr = torch.from_numpy(np.ascontiguousarray(frames)).cuda()
    outs = []
    counts = []
    for attach in (False, True):
        ctx = linked(cb, 68, n) if attach else cb.Context(68, max_frames=n)
        d_c = torch.zeros((n, ctx.info.data_bytes), dtype=torch.uint8, device="cuda")
        d_m = torch.zeros(n, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        per_call = []
        for s in (1, 2):
            if attach:
                ctx.ccm_chain_step(s)
            k0 = cb.launch_count()
            ctx.decode_chunks_dev(d_fr.data_ptr(), n, d_c.data_ptr(), d_m.data_ptr(), flags=cb.FLAG_CC_FIT)
            per_call.append(cb.launch_count() - k0)
            ctx.sync()
        k0 = cb.launch_count()
        ctx.decode_chunks_dev(d_fr.data_ptr(), n, d_c.data_ptr(), d_m.data_ptr(), flags=0)          # not chained
        per_call.append(cb.launch_count() - k0)
        ctx.sync()
        counts.append(per_call)
        outs.append((d_c.cpu().numpy(), d_m.cpu().numpy(), ccm_or_nan(ctx)))
        if attach:
            k0 = cb.launch_count()
            stream = torch.cuda.Stream()                             # refused calls neither wait for the stream nor add to it
            ctx.set_stream(stream.cuda_stream)
            with torch.cuda.stream(stream):
                torch.cuda._sleep(int(1e9))
            t0 = time.perf_counter()
            for call in (lambda: ctx.set_ccm(None), lambda: ctx.set_ccm(np.eye(3)),
                         lambda: ctx.fit_ccm(frames[0], np.zeros(6, np.uint8), 0),
                         lambda: ctx.decode_chunks_dev(d_fr.data_ptr(), n, d_c.data_ptr(), d_m.data_ptr(), flags=cb.FLAG_CC_FIT)):
                with pytest.raises(cb.Cb200Error, match="CCM chain"):
                    call()
            ctx.ccm_chain_step(3)
            with pytest.raises(cb.Cb200Error, match="not been decoded"):
                ctx.ccm_chain_step(4)
            spent = time.perf_counter() - t0
            assert not stream.query() and spent < 0.1, spent
            assert cb.launch_count() == k0
            ctx.sync()
            ctx.ccm_chain_status()
        ctx.close()
    plain, chained = counts
    # an unlinked context launches exactly what the implementation without the chain did for these calls (counted on it: 11 per
    # CC_FIT call of these nine mode-B frames, 7 without colour correction)
    assert plain == [11, 11, 7], plain
    assert chained[0] == plain[0] + 3 and chained[1] == plain[1] + 3 and chained[2] == plain[2], counts
    for a, b in zip(outs[0], outs[1]):
        assert same(a, b)
    unlinked = cb.Context(68, max_frames=n)
    with pytest.raises(cb.Cb200Error, match="not linked"):
        unlinked.ccm_chain_step(1)
    with pytest.raises(cb.Cb200Error, match="differ"):
        unlinked.ccm_chain_root_create(2)
        unlinked.ccm_chain_attach(1, 3)
    unlinked.close()


def test_chained_calls_only_enqueue(cb):
    """chained camera calls queued behind a sleeping stream return at once, and equal one unlinked context's calls"""
    import torch
    pics = CB.camera_pictures()
    batches = [pics[0:4], pics[4:8], pics[8:12]]
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    want = camera_reference(cb, 68, batches * 2)
    assert any(not np.isnan(w[4]).all() for w in want)               # premise: fits, carried from call to call on the device
    ctx = linked(cb, 68, 4)
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    dev = []
    for b in batches:
        dev.append((torch.cat([torch.from_numpy(p.reshape(-1)) for p in b]).cuda(), np.array([(p.shape[1], p.shape[0]) for p in b], np.int32)))
    outs = [(torch.zeros((4, ctx.info.data_bytes), dtype=torch.uint8, device="cuda"), torch.zeros(4, dtype=torch.int32, device="cuda"),
             torch.zeros(4, dtype=torch.int32, device="cuda")) for _ in range(6)]
    torch.cuda.synchronize()

    def call(s):
        d, wh = dev[(s - 1) % 3]
        c, m, st = outs[s - 1]
        ctx.ccm_chain_step(s)
        ctx.scan_extract_decode_chunks_dev(d.data_ptr(), wh, c.data_ptr(), m.data_ptr(), st.data_ptr(), flags=flags)
    for s in (1, 2, 3):                                              # warm-up: every buffer at its size
        call(s)
    ctx.sync()
    with torch.cuda.stream(stream):
        torch.cuda._sleep(int(1.5e9))
    t0 = time.perf_counter()
    for s in (4, 5, 6):
        call(s)
    spent = time.perf_counter() - t0
    busy = not stream.query()
    ctx.sync()
    ctx.ccm_chain_status()
    assert busy, "the stream finished before the third call returned"
    assert spent < 0.25, spent
    for (c, m, st), (wc, wm, wst, _, _) in zip(outs, want):
        assert np.array_equal(c.cpu().numpy(), wc) and np.array_equal(m.cpu().numpy().astype(np.uint32), wm) and np.array_equal(st.cpu().numpy(), wst)
    assert same(ccm_or_nan(ctx), want[-1][3])
    ctx.close()
