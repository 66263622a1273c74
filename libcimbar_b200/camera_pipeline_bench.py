"""Camera pictures from host memory, decoded with and without copy/compute overlap.

    python -m libcimbar_b200.camera_pipeline_bench [--pictures B] [--batches K] [--rounds R]

Workload: the reference's samples/6bit/*.jpg (tests/golden/, as ragged_bench.py loads them: every size differs from the next, one
picture is a 3584 x 2688 upscale standing in for 4_30_f0_big.jpg) replicated into K batches of B pictures, packed in pinned host
memory, mode 4C, SHARPEN_IF_NEEDED | CC_FIT (the CLI's defaults).  Three runs, timed in turn with CUDA events for R rounds:
  (a) `sync`:      cb200_scan_extract_decode_fountain_ragged per batch (host pictures in, dense chunks out, one synchronise a call);
  (b) `pipelined`: cb200_scan_extract_decode_chunks_ragged_dev per batch, the H2D of batch k+1 on a copy stream (double-buffered
                   device pictures, ordered by events) overlapping the decode of batch k, the fixed-slot records copied back;
  (c) device-resident pictures (no copy): the enqueue-only call (`dev_enqueue`) next to cb200_scan_ragged_dev +
                   cb200_extract_decode_fountain_ragged_dev (`dev_two_calls`).
Prints one JSON line: pictures/s and ms per batch of each run, the H2D time of a batch against the decode time of (c), the card's
name and power limit, and whether (a) and (b) returned the same records."""
import argparse
import json

import numpy as np

from libcimbar_b200.bench_support import card, load_pictures


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pictures", type=int, default=64)
    ap.add_argument("--batches", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    import torch
    import libcimbar_b200 as cb
    torch.cuda.set_device(0)
    B, K = args.pictures, args.batches
    pool = load_pictures()
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    # two distinct host batches (the pool in two rotations), used alternately: batch k is host batch k % 2
    host, whs, lists = [], [], []
    for r in range(2):
        pics = [pool[(r * 3 + i) % len(pool)] for i in range(B)]
        wh = np.array([(p.shape[1], p.shape[0]) for p in pics], np.int32)
        buf = torch.empty(sum(p.nbytes for p in pics), dtype=torch.uint8).pin_memory()
        at, views = 0, []
        for p in pics:
            buf[at:at + p.nbytes] = torch.from_numpy(p.reshape(-1))
            views.append(buf[at:at + p.nbytes].numpy().reshape(p.shape))
            at += p.nbytes
        host.append(buf); whs.append(wh); lists.append(views)
    nbytes = max(h.numel() for h in host)
    ctx = cb.Context(4, max_frames=B)
    db, cpf, cs = ctx.info.data_bytes, ctx.info.chunks_per_frame, ctx.info.chunk_size
    compute, copy = torch.cuda.Stream(), torch.cuda.Stream()
    ctx.set_stream(compute.cuda_stream)
    d_pics = [torch.empty(nbytes, dtype=torch.uint8, device="cuda") for _ in range(2)]
    d_chunks = torch.empty((B, db), dtype=torch.uint8, device="cuda")
    d_mask = torch.empty(B, dtype=torch.int32, device="cuda")
    d_status = torch.empty(B, dtype=torch.int32, device="cuda")
    h_chunks = torch.empty((K, B, db), dtype=torch.uint8).pin_memory()
    h_mask = torch.empty((K, B), dtype=torch.int32).pin_memory()
    h_status = torch.empty((K, B), dtype=torch.int32).pin_memory()

    def ev():
        return torch.cuda.Event(enable_timing=True)

    def run_sync():
        ctx.set_ccm(None)
        out = []
        t0, t1 = ev(), ev()
        t0.record(compute)
        for k in range(K):
            out.append(ctx.scan_extract_decode_fountain_ragged(lists[k % 2], flags=flags))
        t1.record(compute)
        t1.synchronize()
        return t0.elapsed_time(t1), out

    def run_pipelined():
        ctx.set_ccm(None)
        copied = [torch.cuda.Event() for _ in range(2)]
        consumed = [torch.cuda.Event() for _ in range(2)]
        t0, t1 = ev(), ev()
        t0.record(compute)
        copy.wait_event(t0)

        def h2d(k):
            with torch.cuda.stream(copy):
                if k >= 2:
                    copy.wait_event(consumed[k % 2])       # the decode of batch k - 2 has read this buffer
                d_pics[k % 2][:host[k % 2].numel()].copy_(host[k % 2], non_blocking=True)
                copied[k % 2].record(copy)
        h2d(0)
        for k in range(K):
            compute.wait_event(copied[k % 2])
            ctx.scan_extract_decode_chunks_dev(d_pics[k % 2].data_ptr(), whs[k % 2], d_chunks.data_ptr(), d_mask.data_ptr(),
                                               d_status.data_ptr(), flags=flags)
            consumed[k % 2].record(compute)
            # the next batch's copy is enqueued after the call: the call's own picture-table upload goes through the same
            # host-to-device copy engine, and queued behind a whole batch of pictures it would hold back this batch's decode
            if k + 1 < K:
                h2d(k + 1)
            with torch.cuda.stream(compute):
                h_chunks[k].copy_(d_chunks, non_blocking=True)
                h_mask[k].copy_(d_mask, non_blocking=True)
                h_status[k].copy_(d_status, non_blocking=True)
        t1.record(compute)
        t1.synchronize()
        return t0.elapsed_time(t1)

    def resident(which):
        ctx.set_ccm(None)
        t0, t1 = ev(), ev()
        t0.record(compute)
        for k in range(K):
            d, wh = d_pics[k % 2], whs[k % 2]
            if which == "enqueue":
                ctx.scan_extract_decode_chunks_dev(d.data_ptr(), wh, d_chunks.data_ptr(), d_mask.data_ptr(), d_status.data_ptr(), flags=flags)
            else:
                anchors, count, cutoff = np.zeros((B, 4, 4), np.int32), np.zeros(B, np.int32), np.zeros(B, np.uint32)
                cb._check(ctx.lib.cb200_scan_ragged_dev(ctx._h, d.data_ptr(), wh.ctypes.data, B, anchors.ctypes.data, count.ctypes.data,
                                                        cutoff.ctypes.data))
                corners = np.stack([(anchors[:, :, 0] + anchors[:, :, 1]) // 2, (anchors[:, :, 2] + anchors[:, :, 3]) // 2], axis=2)
                corners = np.ascontiguousarray(corners.astype(np.float32).reshape(B, 8))
                ch = np.zeros((B, cpf, cs), np.uint8)
                cnt, mk, fl = np.zeros(B, np.uint32), np.zeros(B, np.uint32), np.zeros(B, np.uint8)
                cb._check(ctx.lib.cb200_extract_decode_fountain_ragged_dev(ctx._h, d.data_ptr(), wh.ctypes.data, B, corners.ctypes.data, flags,
                                                                            ch.ctypes.data, cnt.ctypes.data, mk.ctypes.data, fl.ctypes.data))
        t1.record(compute)
        t1.synchronize()
        return t0.elapsed_time(t1)

    def h2d_only():
        t0, t1 = ev(), ev()
        t0.record(copy)
        for k in range(K):
            with torch.cuda.stream(copy):
                d_pics[k % 2][:host[k % 2].numel()].copy_(host[k % 2], non_blocking=True)
        t1.record(copy)
        t1.synchronize()
        return t0.elapsed_time(t1)

    # warm-up: every shape and buffer once
    h2d_only()
    run_sync(); run_pipelined(); resident("enqueue"); resident("two_calls")
    times = {"sync": [], "pipelined": [], "dev_enqueue": [], "dev_two_calls": [], "h2d": []}
    same = True
    for _ in range(args.rounds):
        ms, ref = run_sync(); times["sync"].append(ms)
        times["pipelined"].append(run_pipelined())
        for k in range(K):
            chunks, count, mask, _, status = ref[k]
            same &= np.array_equal(status, h_status[k].numpy()) and np.array_equal(mask, h_mask[k].numpy().view(np.uint32))
            slots = h_chunks[k].numpy().reshape(B, cpf, cs)
            for i in range(B):
                keep = [q for q in range(cpf) if int(mask[i]) >> q & 1]
                same &= len(keep) == count[i] and np.array_equal(chunks[i, :count[i]], slots[i, keep])
        times["h2d"].append(h2d_only())
        times["dev_enqueue"].append(resident("enqueue"))
        times["dev_two_calls"].append(resident("two_calls"))
    name, power = card()
    best = {k: min(v) for k, v in times.items()}
    res = {"metric": "camera_pipeline", "pictures_per_batch": B, "batches": K, "rounds": args.rounds, "mode": "4C",
           "flags": "SHARPEN_IF_NEEDED|CC_FIT", "bytes_per_batch": [int(h.numel()) for h in host]}
    for k in ("sync", "pipelined", "dev_enqueue", "dev_two_calls"):
        res[k] = {"pictures_per_s": round(B * K / (best[k] / 1e3), 1), "ms_per_batch": round(best[k] / K, 3),
                  "ms_per_batch_all_rounds": [round(t / K, 3) for t in times[k]]}
    res["h2d_ms_per_batch"] = round(best["h2d"] / K, 3)
    res["decode_ms_per_batch"] = res["dev_enqueue"]["ms_per_batch"]
    res["pipelined_speedup_over_sync"] = round(best["sync"] / best["pipelined"], 3)
    res["sync_and_pipelined_same_records"] = bool(same)
    res["gpu"] = name
    res["power_limit"] = power
    print(json.dumps(res))
    ctx.close()


if __name__ == "__main__":
    main()
