"""Camera pictures across GPUs, with the CC_FIT colour correction chained between ranks.

    torchrun --nproc-per-node N -m libcimbar_b200.camera_multi_bench [--per-rank P] [--steps K] [--warmup W] [--kind window|window-direct]

Workload: the sample photographs of camera_pipeline_bench (ragged_bench.load_pictures), P per rank, resident in HBM, mode 4C,
SHARPEN_IF_NEEDED | CC_FIT.  Every step the batch of N * P pictures is cut into contiguous stripes, rank r decodes stripe r on a
context linked to the CCM chain (dist.CameraExchange), and the records reach rank 0's window.  All ranks use GPU LOCAL_RANK modulo
the GPUs present, so N ranks on one GPU share it.  Prints one JSON line on rank 0: pictures/s over the K timed steps (slowest rank),
each rank's mean decode time per step (CUDA events around its call), the chain's link-kernel time per rank (its wait for the lower
ranks' fits), the card's name and power limit, the GPU count, and whether rank 0's records of the first step equal one context's
decode of the same batch."""
import argparse
import json
import os
import time

import numpy as np


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--per-rank", type=int, default=16)
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--kind", default="window", choices=["window", "window-direct"])
    args = ap.parse_args()
    import torch
    import torch.distributed as dist
    import libcimbar_b200 as cb
    from libcimbar_b200.dist import CameraExchange, stripe
    from libcimbar_b200.ragged_bench import card, load_pictures
    dist.init_process_group("gloo")
    rank, world = dist.get_rank(), dist.get_world_size()
    dev_index = int(os.environ.get("LOCAL_RANK", rank)) % torch.cuda.device_count()
    torch.cuda.set_device(dev_index)
    P = args.per_rank
    pool = load_pictures()
    batch = [pool[i % len(pool)] for i in range(P * world)]
    a, b = stripe(len(batch), rank, P)
    mine = batch[a:b]
    d_pics = torch.cat([torch.from_numpy(p.reshape(-1)) for p in mine]).cuda()
    wh = np.array([(p.shape[1], p.shape[0]) for p in mine], np.int32)
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    ctx = cb.Context(4, max_frames=P, device=dev_index)
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    ctx.set_timing(True)
    ex = CameraExchange(ctx, args.kind, P, flags=flags)
    torch.cuda.synchronize()

    # step 1: records to rank 0 and the check against one context
    ex.decode(1, ("rgb", d_pics.data_ptr(), wh))
    got = ex.collect(1)
    equal = None
    if rank == 0:
        one = cb.Context(4, max_frames=len(batch), device=dev_index)
        d_all = torch.cat([torch.from_numpy(p.reshape(-1)) for p in batch]).cuda()
        wh_all = np.array([(p.shape[1], p.shape[0]) for p in batch], np.int32)
        n = len(batch)
        c = torch.zeros((n, ctx.info.data_bytes), dtype=torch.uint8, device="cuda")
        m = torch.zeros(n, dtype=torch.int32, device="cuda")
        s = torch.zeros(n, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        one.scan_extract_decode_chunks_dev(d_all.data_ptr(), wh_all, c.data_ptr(), m.data_ptr(), s.data_ptr(), flags=flags)
        one.sync()
        equal = (np.array_equal(got[0], c.cpu().numpy()) and np.array_equal(got[1], m.cpu().numpy().astype(np.uint32))
                 and np.array_equal(got[2], s.cpu().numpy()))
        one.close()
        del d_all

    def step(sn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        ex.decode(sn, ("rgb", d_pics.data_ptr(), wh))
        e1.record(stream)
        ex.counts.pop(sn)
        if rank == 0:                        # rank 0 takes every step's records in its window (device-side wait) and lets go of them
            ex.records.collect(sn)
            ex.records.release(sn)
        return e0, e1

    sn = 1
    for _ in range(args.warmup):
        sn += 1
        step(sn)
    ctx.sync()
    dist.barrier()
    t0 = time.perf_counter()
    evs = []
    for _ in range(args.steps):
        sn += 1
        evs.append(step(sn))
    ctx.sync()
    wall = time.perf_counter() - t0
    dec_ms = float(np.mean([e0.elapsed_time(e1) for e0, e1 in evs]))
    # the link kernel's time, in steps of their own after the timed ones (reading it waits for it)
    links = []
    for _ in range(max(2, args.steps // 2)):
        sn += 1
        step(sn)
        links.append(ctx.ccm_chain_link_ms())
    ctx.sync()
    ctx.ccm_chain_status()
    link_ms = float(np.mean(links))
    rows = [None] * world if rank == 0 else None
    dist.gather_object((wall, dec_ms, link_ms), rows, dst=0)
    if rank == 0:
        ctx.gather_status()
        wall = max(r[0] for r in rows)
        name, power = card()
        print(json.dumps({
            "bench": "camera_multi", "ranks": world, "gpus": torch.cuda.device_count(), "ranks_per_gpu": -(-world // torch.cuda.device_count()),
            "card": name, "power_limit_w": power, "mode": "4C", "flags": "SHARPEN_IF_NEEDED|CC_FIT", "exchange": args.kind,
            "pictures_per_rank": P, "steps": args.steps, "pictures_per_s": round(P * world * args.steps / wall, 1),
            "decode_ms_per_step": [round(r[1], 3) for r in rows], "chain_link_ms_per_step": [round(r[2], 4) for r in rows],
            "records_equal_one_context": bool(equal)}))
    dist.barrier()
    ctx.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
