"""The context's buffers and uploads (csrc/ctx.cuh): the `_dev` entry points only enqueue work on the context's stream (their
host-built tables go through pinned slots, so nothing waits for the stream), and destroying a context returns every buffer it
grew, whichever entry points grew them."""
import numpy as np
import pytest

from ragged_samples import GLOB, sample
from gpu_support import cb  # noqa: F401  (fixtures)
from gpu_support import POOL, check_dense, dense, frame_pool, oracle
from cpu_support import camera_view

pytestmark = pytest.mark.gpu


def test_dev_entry_points_only_enqueue(cb):
    """behind a spin kernel on the stream, cb200_deskew_dev and cb200_decode_chunks_sharpen_dev return while it still spins, and
    their results are those of the host-pointer deskew and of the oracle"""
    import cv2
    import torch
    n = 4
    m, frames = frame_pool(68)
    idx = np.arange(n) % POOL
    sel = np.array([1, 0, 0, 1], np.uint8)
    quads = [[[210, 130], [1480, 190], [160, 1350], [1530, 1290]], [[40, 60], [1500, 20], [80, 1360], [1540, 1430]]] * 2
    cams = np.stack([camera_view(frames[i], q, (1700, 1500)) for i, q in zip(idx, quads)])
    dst = np.float32([[30, 30], [994, 30], [30, 994], [994, 994]])
    m9 = np.stack([cv2.getPerspectiveTransform(np.float32(q), dst) for q in quads]).astype(np.float64)
    ctx = cb.Context(68, max_frames=n)
    want = ctx.deskew(cams, m9)
    dev = torch.device("cuda")
    d_cams = torch.from_numpy(cams).to(dev)
    d_frames = torch.from_numpy(frames[idx]).to(dev)
    d_warped = torch.zeros((n, 1024, 1024, 3), dtype=torch.uint8, device=dev)
    chunks = torch.zeros((n, ctx.info.data_bytes), dtype=torch.uint8, device=dev)
    mask = torch.zeros(n, dtype=torch.int32, device=dev)
    ff = torch.zeros(n, dtype=torch.uint8, device=dev)
    torch.cuda.synchronize()        # the context's own stream does not wait for torch's
    arg = sel.copy()

    def deskew_dev():
        cb._check(ctx.lib.cb200_deskew_dev(ctx._h, d_cams.data_ptr(), 1700, 1500, n, m9.ctypes.data, d_warped.data_ptr()))

    def decode_dev():
        cb._check(ctx.lib.cb200_decode_chunks_sharpen_dev(ctx._h, d_frames.data_ptr(), n, 0, arg.ctypes.data, chunks.data_ptr(),
                                                          mask.data_ptr(), ff.data_ptr()))

    for _ in range(3):              # every buffer and upload slot at its size: growing one would synchronise
        deskew_dev()
        decode_dev()
    ctx.sync()
    d_warped.zero_()
    chunks.zero_()
    torch.cuda.synchronize()
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    slept = torch.cuda.Event()
    with torch.cuda.stream(stream):
        torch.cuda._sleep(1_000_000_000)
        slept.record()
    deskew_dev()
    assert not slept.query() and not stream.query()
    decode_dev()
    arg[:] = 1 - arg                # the caller may reuse its selection at once
    assert not slept.query() and not stream.query()
    stream.synchronize()
    ctx.set_stream(None)
    assert np.array_equal(d_warped.cpu().numpy(), want)
    got, masks = chunks.cpu().numpy(), mask.cpu().numpy().astype(np.uint32)
    for f in range(n):
        cnt, rows = dense(m, got[f], masks[f])
        check_dense(m, rows, cnt, masks[f], oracle(68, int(idx[f]), sel[f], 0), f)
    ctx.close()


def _device_bytes_of_this_process():
    """NVML's device memory of this process on the current device, or None when NVML cannot tell it apart: in a PID namespace
    NVML lists the process under another PID, which identifies it only while it is the one process on the card"""
    import os
    import pynvml
    import torch
    p = torch.cuda.get_device_properties(torch.cuda.current_device())
    pynvml.nvmlInit()
    try:
        dev = pynvml.nvmlDeviceGetHandleByPciBusId(f"{p.pci_domain_id:08X}:{p.pci_bus_id:02X}:{p.pci_device_id:02X}.0")
        procs = pynvml.nvmlDeviceGetComputeRunningProcesses(dev)
        mine = [q for q in procs if q.pid == os.getpid()] or (procs if len(procs) == 1 else [])
        return mine[0].usedGpuMemory if len(mine) == 1 else None
    finally:
        pynvml.nvmlShutdown()


def test_destroy_returns_every_buffer(cb):
    """five contexts, each driven through every lazily grown buffer, then destroyed: the process's device memory (NVML, per
    process -- other jobs share the card) ends where it started"""
    n = 6
    m, frames = frame_pool(68)
    batch = frames[np.arange(n) % POOL]
    sel = np.arange(n) % 2 == 1
    pictures = [sample(s) for s in GLOB[:n]]
    quad = [[210, 130], [1480, 190], [160, 1350], [1530, 1290]]
    cam = camera_view(frames[0], quad, (1700, 1500))
    corners = np.float32(quad)
    dst = np.float32([[30, 30], [994, 30], [30, 994], [994, 994]])
    m9 = cb.perspective_transform(corners, dst)

    def lifetime():
        ctx = cb.Context(68, max_frames=n)
        ctx.decode_fountain(batch, flags=cb.FLAG_CC_FIT)
        ctx.decode_fountain(batch, flags=cb.FLAG_CC_SIMPLE)
        ctx.decode_fountain(batch, sharpen=sel)
        ctx.decode_cells_means(batch[:2], flags=cb.FLAG_CC_SIMPLE)
        ctx.decode(batch, flags=cb.FLAG_NO_INTERLEAVE)
        ctx.scan_extract_decode_fountain_ragged(pictures, flags=cb.FLAG_SHARPEN_IF_NEEDED)
        ctx.deskew(cam, m9)
        ctx.extract_decode_fountain(cam, corners)
        ctx.fit_ccm(None, np.arange(6, dtype=np.uint8), 0)
        ctx.close()

    lifetime()                      # the CUDA context and the lazily loaded kernels stay for the process
    start = _device_bytes_of_this_process()
    for k in range(5):
        lifetime()
        now = _device_bytes_of_this_process()
        if start is None or now is None:
            pytest.skip("NVML cannot tell this process's device memory apart from other processes on the card")
        assert now == start, (k, now - start)
