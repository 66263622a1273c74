"""One rank of the multi-process CCM-chain tests (tests/test_gpu_ccm_chain.py), started by torch.distributed.run; test infrastructure
only.  Every rank decodes its contiguous stripe of each step's batch on a context linked to the chain and saves what it got to
<out>/rank<r>.npz; the test compares them with one context's decode of the whole stream.

    python -m torch.distributed.run --nproc-per-node N tests/ccm_chain_worker.py <scenario> <out> [--per-gpu]

scenario: "frames"            crafted mode-B fountain frames through cb200_decode_chunks_dev, three steps
          "camera-<kind>-<m>" the ragged camera batch of chain_batches.py through dist.CameraExchange(kind) in mode m, three steps
          "jpeg-<kind>"       mode-B JPEG files through the same exchange, mode B, one step"""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))          # the package, from the repository tree


def main():
    scenario, out = sys.argv[1], sys.argv[2]
    per_gpu = "--per-gpu" in sys.argv
    dist.init_process_group("gloo")
    rank, world = dist.get_rank(), dist.get_world_size()
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)) % torch.cuda.device_count() if per_gpu else 0)
    import libcimbar_b200 as cb
    from libcimbar_b200.dist import CameraExchange, stripe
    import chain_batches as CB
    res = {}
    if scenario == "frames":
        steps, per = CB.frame_steps(world)
        ctx = cb.Context(68, max_frames=per, device=torch.cuda.current_device())
        h = [ctx.ccm_chain_root_create(world) if rank == 0 else None]
        dist.broadcast_object_list(h, src=0)
        if rank:
            ctx.ccm_chain_peer_open(world, rank, h[0])
        ctx.ccm_chain_attach(rank, world)
        rec = ctx.info.data_bytes
        d_chunks = torch.zeros((per, rec), dtype=torch.uint8, device="cuda")
        d_mask = torch.zeros(per, dtype=torch.int32, device="cuda")
        for s, frames in enumerate(steps, start=1):
            a, b = stripe(len(frames), rank, per)
            d_fr = torch.from_numpy(np.ascontiguousarray(frames[a:b])).cuda()
            torch.cuda.synchronize()
            ctx.ccm_chain_step(s)
            ctx.decode_chunks_dev(d_fr.data_ptr(), b - a, d_chunks.data_ptr(), d_mask.data_ptr(), flags=cb.FLAG_CC_FIT)
            ctx.sync()
            ctx.ccm_chain_status()
            res[f"chunks{s}"] = d_chunks[:b - a].cpu().numpy()
            res[f"mask{s}"] = d_mask[:b - a].cpu().numpy()
            res[f"fccm{s}"] = ctx.frame_ccms(b - a)
            ccm = ctx.get_ccm()
            res[f"ccm{s}"] = np.full((3, 3), np.nan, np.float32) if ccm is None else ccm
            dist.barrier()
    else:
        parts = scenario.split("-")
        kind = parts[1] if parts[1] == "window" else "window-direct"
        mode = int(parts[2]) if parts[0] == "camera" else 68
        if parts[0] == "jpeg":
            steps, per = CB.jpeg_steps(world)
        else:
            steps, per = CB.camera_steps(world) if mode == 68 else CB.legacy_steps(world)
        flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
        ctx = cb.Context(mode, max_frames=per, device=torch.cuda.current_device())
        ex = CameraExchange(ctx, kind, per, flags=flags)
        for s, batch in enumerate(steps, start=1):
            a, b = stripe(len(batch), rank, per)
            mine = batch[a:b]
            if parts[0] == "camera":
                d_pics = torch.cat([torch.from_numpy(p.reshape(-1)) for p in mine]).cuda() if mine else None
                wh = np.array([(p.shape[1], p.shape[0]) for p in mine], np.int32).reshape(-1, 2)
                torch.cuda.synchronize()
                ex.decode(s, ("rgb", d_pics.data_ptr() if mine else 0, wh))
            else:
                ex.decode(s, ("jpeg", mine))
            got = ex.collect(s)
            if rank == 0:
                res[f"chunks{s}"], res[f"mask{s}"], res[f"status{s}"] = got
            if mode == 68:
                res[f"fccm{s}"] = ctx.frame_ccms(b - a)
            ccm = ctx.get_ccm()
            res[f"ccm{s}"] = np.full((3, 3), np.nan, np.float32) if ccm is None else ccm
            dist.barrier()
    np.savez(os.path.join(out, f"rank{rank}.npz"), **res)
    dist.barrier()
    ctx.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
