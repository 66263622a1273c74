"""The exact flood walk (K1x) at the batch sizes the benchmark's camera and noise workloads run (pytest -m gpu).

flood_launch runs the walk in one of three regimes, chosen by batch size.  A batch of at most a few walks per SM keeps the
whole heap in shared memory.  A larger batch keeps only the top ten levels there and the deeper ones in a per-walk spill area
in L2, so one sift-down round may read children from both.  A batch with more flagged frames than walk slots makes every
walking warp take further frames, reusing the previous frame's priority bytes, bitmap and spill area.  The tests here build
such batches on the device from a pool of distinct frames and compare every frame with the CPU oracle's result for its pool
entry, bit for bit.  Each test asserts its own premise: the batch size against the SM count, the number of frames the walk
takes, and the oracle's heap peaks of the pool frames."""
import ctypes as C

import numpy as np
import pytest

from oracle_lib import load_sample
from gpu_support import cb  # noqa: F401  (fixtures)
from gpu_support import ORA, synth_frames

pytestmark = pytest.mark.gpu

HEAP_SMEM = 1023                # heap entries a walk keeps in shared memory when the batch is larger than one wave
HEAP_SMEM_FEW = 8191            # ... and when it is not
POOL_FLAGGED = 26               # the pool: 2 photographs + 12 frames with 1 % and 12 with 8 % noise tiles ...
POOL_CLEAN = 3                  # ... + 3 clean frames = 29, a prime, so that neighbours in a batch never repeat with a short period


@pytest.fixture(scope="module")
def torch():
    import torch
    return torch


def _heap_peak():
    return C.c_int.in_dll(ORA.lib, "cbo_dbg_max_heap")


def _oracle(m, rgb, sharpen, want_cells=False):
    """the oracle's raw bytes (and cells), RS data, chunk mask and the peak size of its walk's heap for one frame"""
    peak = _heap_peak()
    peak.value = 0
    raw = ORA.decode_raw(m, rgb, sharpen=sharpen, want_cells=want_cells)
    heap = peak.value
    data, _ = ORA.decode(m, rgb, sharpen=sharpen)
    _, _, mask = ORA.decode_fountain(m, rgb, sharpen=sharpen)
    raw, cells = raw if want_cells else (raw, None)
    return raw, cells, data, mask, heap


class Pool:
    """29 distinct mode-68 frames (flagged ones first) and the oracle's results for each, with and without sharpen"""

    def __init__(self):
        m = self.m = ORA.mode(68)
        frames = [load_sample("b/ex2434.jpg"), load_sample("b/ex380.jpg")]
        for k in range(6):
            frames += list(synth_frames(68, 2, seed=500 + k, error_rate=0.01, noise_tiles=True)[2])
            frames += list(synth_frames(68, 2, seed=600 + k, error_rate=0.08, noise_tiles=True)[2])
        frames += list(synth_frames(68, POOL_CLEAN, seed=700)[2])
        self.frames = np.stack(frames)
        assert len(self.frames) == POOL_FLAGGED + POOL_CLEAN
        self.want = {}
        for sharpen in (False, True):
            res = [_oracle(m, fr, sharpen, want_cells=not sharpen) for fr in self.frames]
            self.want[sharpen] = dict(raw=np.stack([r[0] for r in res]), data=np.stack([r[2] for r in res]),
                                      mask=np.array([r[3] for r in res], np.uint32), heap=np.array([r[4] for r in res]))
            if not sharpen:
                self.cells = np.stack([r[1] for r in res])

    def flags(self, cb, sharpen):
        """the frame flags of the pool itself, decoded as one small batch"""
        ctx = cb.Context(68, max_frames=len(self.frames))
        _, ff = ctx.decode_raw(self.frames, flags=cb.FLAG_SHARPEN if sharpen else 0)
        ctx.close()
        return ff


@pytest.fixture(scope="module")
def pool(cb):
    p = Pool()
    for sharpen in (False, True):
        ff = p.flags(cb, sharpen)
        heap = p.want[sharpen]["heap"]
        # premise: the flagged pool frames take the walk, the clean ones do not, and every walk's heap outgrows the shared-memory
        # part of the throughput regime; without sharpen, some outgrow even the one-wave regime's (sharpened frames peak lower)
        assert (ff[:POOL_FLAGGED] & cb.FRAME_FALLBACK).all() and not ff[POOL_FLAGGED:].any(), (sharpen, ff.tolist())
        assert (heap[:POOL_FLAGGED] > HEAP_SMEM).all(), (sharpen, heap.tolist())
        if not sharpen:
            assert heap[:POOL_FLAGGED].max() > HEAP_SMEM_FEW, heap.tolist()
        p.want[sharpen]["flags"] = ff
    return p


def _batch_index(n, clean_every):
    """pool indices of an n-frame batch: flagged entries in turn, with a clean entry at every `clean_every`-th position, so that
    the work list of flagged frames has non-trivial offsets"""
    idx = np.empty(n, np.int64)
    clean = np.arange(n) % clean_every == clean_every - 1
    idx[~clean] = np.arange(int((~clean).sum())) % POOL_FLAGGED
    idx[clean] = POOL_FLAGGED + np.arange(int(clean.sum())) % POOL_CLEAN
    return idx


def _check_raw(pool, sharpen, idx, raw, ff, cb):
    want = pool.want[sharpen]
    bad = np.flatnonzero((raw != want["raw"][idx]).any(axis=1))
    assert bad.size == 0, f"{bad.size} frames differ from the oracle, first {bad[:8].tolist()} (pool {idx[bad[:8]].tolist()})"
    assert np.array_equal(ff, want["flags"][idx])
    return int(((ff & cb.FRAME_FALLBACK) != 0).sum())


def _sm_count(cb):
    ctx = cb.Context(68, max_frames=1)
    sms = ctx.info.sm_count
    ctx.close()
    return sms


def _stream(torch, ctx):
    """a stream of its own for the test's torch work and the library's launches, so that the decode is ordered after the
    batch is assembled and the batch's memory is not handed back to the allocator before the decode has read it"""
    s = torch.cuda.Stream()
    ctx.set_stream(s.cuda_stream)
    return s


def test_walk_throughput_regime_past_4_gib(cb, torch, pool):
    """12 x SMs frames (5 GB on an H100): more than one wave of walks, so every walk keeps 1 023 heap entries in shared memory
    and the rest in L2; frames beyond the first 4 GiB of the batch.  Raw bytes, frame flags, RS data and chunk masks, without
    and with sharpen (the second call reuses the workspace)."""
    sms = _sm_count(cb)
    n = 12 * sms
    frame_bytes = pool.frames[0].nbytes
    idx = _batch_index(n, clean_every=7)
    assert n > 8 * sms                                  # the one-wave regime holds at most 6 walks per SM
    assert (n - 1) * frame_bytes >= 1 << 32 and (idx[(1 << 32) // frame_bytes + 1:] < POOL_FLAGGED).any()
    ctx = cb.Context(68, max_frames=n)
    m = ctx.info
    try:
        with torch.cuda.stream(_stream(torch, ctx)):
            d_rgb = torch.from_numpy(pool.frames).cuda()[torch.from_numpy(idx).cuda()]
            d_raw = torch.empty((n, m.raw_bytes), dtype=torch.uint8, device="cuda")
            d_data = torch.empty((n, m.data_bytes), dtype=torch.uint8, device="cuda")
            d_mask = torch.empty(n, dtype=torch.int32, device="cuda")
            d_flags = torch.empty(n, dtype=torch.uint8, device="cuda")
            d_flags2 = torch.empty(n, dtype=torch.uint8, device="cuda")
            for sharpen in (False, True):
                flags = cb.FLAG_SHARPEN if sharpen else 0
                ctx.decode_raw_dev(d_rgb.data_ptr(), n, d_raw.data_ptr(), d_flags.data_ptr(), flags=flags)
                ctx.decode_chunks_dev(d_rgb.data_ptr(), n, d_data.data_ptr(), d_mask.data_ptr(), d_flags2.data_ptr(), flags=flags)
                ff = d_flags.cpu().numpy()
                walked = _check_raw(pool, sharpen, idx, d_raw.cpu().numpy(), ff, cb)
                assert walked > 8 * sms, walked
                assert np.array_equal(d_flags2.cpu().numpy(), ff)
                want = pool.want[sharpen]
                assert np.array_equal(d_mask.cpu().numpy().astype(np.uint32), want["mask"][idx])
                bad = np.flatnonzero((d_data.cpu().numpy() != want["data"][idx]).any(axis=1))
                assert bad.size == 0, f"{bad.size} frames' RS data differ, first {bad[:8].tolist()}"
    finally:
        torch.cuda.synchronize()
        ctx.close()
        d_rgb = d_raw = d_data = d_mask = d_flags = d_flags2 = None
        torch.cuda.empty_cache()


def test_walk_cell_trace_in_the_throughput_regime(cb, pool):
    """the walk forced on more than one wave of frames (decode_cells): every frame's trace and cells against the oracle.  The
    order of equal priorities in the heap levels spilled to L2 shows in the trace even where the bytes agree."""
    sms = _sm_count(cb)
    n = 8 * sms + 1
    idx = _batch_index(n, clean_every=5)
    ctx = cb.Context(68, max_frames=n)
    try:
        cells, trace = ctx.decode_cells(pool.frames[idx])
    finally:
        ctx.close()
    want = pool.cells[idx]
    for k in ("order", "x", "y", "drift_offset", "distance"):
        bad = np.flatnonzero((trace[k] != want[k]).any(axis=1))
        assert bad.size == 0, f"{k}: {bad.size} frames differ, first {bad[:8].tolist()} (pool {idx[bad[:8]].tolist()})"
    assert np.array_equal(cells & 15, want["symbol"]) and np.array_equal((cells >> 4) & 7, want["color"])


def test_walk_warp_reuse(cb, torch, pool):
    """40 x SMs frames (17 GB on an H100) of which more than 33 x SMs take the walk: more walks than walk slots (at most 32 per
    SM), so warps take further frames from the work counter and reuse the previous frame's priority bytes, bitmap and spill
    area.  Raw bytes and flags against the pool; then the reversed batch in a second call."""
    sms = _sm_count(cb)
    n = 40 * sms
    idx = _batch_index(n, clean_every=11)
    ctx = cb.Context(68, max_frames=n)
    try:
        with torch.cuda.stream(_stream(torch, ctx)):
            d_pool = torch.from_numpy(pool.frames).cuda()
            d_raw = torch.empty((n, ctx.info.raw_bytes), dtype=torch.uint8, device="cuda")
            d_flags = torch.empty(n, dtype=torch.uint8, device="cuda")
            for order in (idx, idx[::-1].copy()):
                d_rgb = d_pool[torch.from_numpy(order).cuda()]
                ctx.decode_raw_dev(d_rgb.data_ptr(), n, d_raw.data_ptr(), d_flags.data_ptr())
                raw, ff = d_raw.cpu().numpy(), d_flags.cpu().numpy()     # (waits for the decode before d_rgb can go)
                d_rgb = None
                walked = _check_raw(pool, False, order, raw, ff, cb)
                assert walked > 33 * sms, walked
    finally:
        torch.cuda.synchronize()
        ctx.close()
        d_pool = d_rgb = d_raw = d_flags = None
        torch.cuda.empty_cache()
