"""The enqueue-only camera call against its camera plan (one CUDA graph launch per batch), on device-resident pictures.

    python -m libcimbar_b200.camera_plan_bench [--pictures B[,B...]] [--rounds R]

Workload: camera_pipeline_bench's pool (the reference's samples/6bit/*.jpg from tests/golden/, one a 3584 x 2688 upscale) rotated
into a batch of B pictures in HBM, mode 4C, SHARPEN_IF_NEEDED | CC_FIT (the CLI's defaults); B = 1, 8 and 64 by default.  For the
direct call and for the plan, per batch size:
  host_us:   perf_counter around the enqueue (the direct call's host work, or cudaGraphLaunch), median of R calls, each made with the
             stream idle so that no call waits on an earlier one;
  gpu_ms:    CUDA events around the call on the stream, median of R;
  idle_ms:   the time inside the batch's span -- first kernel start to last kernel end -- during which no kernel of the batch ran,
             from a torch.profiler trace of one call (run separately from the timed calls);
  same_records: the plan's chunks, masks, statuses and frame flags equal the direct call's.
Prints one JSON line with the card's name and power limit."""
import argparse
import json
import statistics
import time

import numpy as np

from libcimbar_b200.ragged_bench import card, load_pictures


def idle_ms(torch, fn):
    """span and idle time of the kernels one call of fn runs, from a CUDA-activity trace"""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    ks = sorted((e.time_range.start, e.time_range.end) for e in prof.events()
                if e.device_type.name == "CUDA" and not e.name.startswith(("Memcpy", "Memset", "cudaMem")))
    if not ks:
        return None
    busy, cur_s, cur_e = 0.0, ks[0][0], ks[0][1]
    for s, e in ks[1:]:
        if s > cur_e:
            busy += cur_e - cur_s
            cur_s, cur_e = s, e
        else:
            cur_e = max(cur_e, e)
    busy += cur_e - cur_s
    span = ks[-1][1] - ks[0][0]
    return {"kernels": len(ks), "span_ms": round(span / 1e3, 4), "idle_ms": round((span - busy) / 1e3, 4)}


def one_size(torch, cb, pool, B, rounds):
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    pics = [pool[i % len(pool)] for i in range(B)]
    wh = np.array([(p.shape[1], p.shape[0]) for p in pics], np.int32)
    d = torch.cat([torch.from_numpy(p.reshape(-1)) for p in pics]).cuda()
    ctx = cb.Context(4, max_frames=B)
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    db = ctx.info.data_bytes
    outs = {k: (torch.empty((B, db), dtype=torch.uint8, device="cuda"), torch.empty(B, dtype=torch.int32, device="cuda"),
                torch.empty(B, dtype=torch.int32, device="cuda"), torch.empty(B, dtype=torch.uint8, device="cuda")) for k in ("direct", "plan")}
    oc, om, os_, of = outs["direct"]

    def direct():
        ctx.scan_extract_decode_chunks_dev(d.data_ptr(), wh, oc.data_ptr(), om.data_ptr(), os_.data_ptr(), of.data_ptr(), flags=flags)
    direct()                                           # every buffer at this size before the plan freezes them
    ctx.sync()
    pc, pm, ps, pf = outs["plan"]
    plan = ctx.camera_plan(wh, flags, d.data_ptr(), pc.data_ptr(), pm.data_ptr(), pf.data_ptr(), ps.data_ptr())
    calls = {"direct": direct, "plan": plan.launch}
    res = {}
    for name, fn in calls.items():
        for _ in range(2):                             # warm-up
            fn()
        ctx.sync()
        host, gpu = [], []
        for _ in range(rounds):
            ctx.set_ccm(None)
            ctx.sync()
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record(stream)
            a = time.perf_counter()
            fn()
            b = time.perf_counter()
            t1.record(stream)
            t1.synchronize()
            host.append((b - a) * 1e6)
            gpu.append(t0.elapsed_time(t1))
        ctx.set_ccm(None)
        ctx.sync()
        res[name] = {"host_us": round(statistics.median(host), 1), "gpu_ms": round(statistics.median(gpu), 3),
                     "host_us_all": [round(h, 1) for h in host]}
        ctx.set_ccm(None)
        ctx.sync()
        res[name]["trace"] = idle_ms(torch, fn)
    ctx.sync()
    res["same_records"] = all(torch.equal(x, y) for x, y in zip(outs["direct"], outs["plan"]))
    res["pictures"] = B
    plan.close()
    ctx.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pictures", default="1,8,64")
    ap.add_argument("--rounds", type=int, default=20)
    args = ap.parse_args()
    import torch
    import libcimbar_b200 as cb
    torch.cuda.set_device(0)
    pool = load_pictures()
    sizes = [int(b) for b in str(args.pictures).split(",")]
    out = {"metric": "camera_plan", "mode": "4C", "flags": "SHARPEN_IF_NEEDED|CC_FIT", "rounds": args.rounds,
           "batches": [one_size(torch, cb, pool, B, args.rounds) for B in sizes]}
    out["gpu"], out["power_limit"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
