"""Receivers camera plans against the direct receivers call, on the workload of receivers_bench.

    python -m libcimbar_b200.receivers_plan_bench [--rounds R] [--batches B]

Workload (receivers_bench's): D receivers x k pictures (D in 16, 64, 256; k in 1, 4), picture i drawn round-robin from the
camera_pipeline_bench pool plus the two mode-B photographs, all in device memory; mode B, SHARPEN_IF_NEEDED | CC_FIT, every receiver
starting from a distinct active matrix.  Each batch has a fresh receiver map (batch b: picture i belongs to receiver (i + b) % D).
Two arms on one context and stream, B batches back to back per round, R rounds each:
  (a) `direct`: one cb200_scan_extract_decode_chunks_receivers_dev call per batch (the map from host memory);
  (e) `plan`: one receivers camera plan, created once; per batch the map is copied to its bound d_receiver_of on the stream (from
      pinned memory), then one cb200_camera_plan_launch.
Prints one JSON line: per shape, the host time to issue one batch (wall time of issuing the B batches, divided by B), the GPU time
per batch (CUDA events around the B batches, divided by B), and whether (a) and (e) gave identical records and states over the same
B batches from the same states; the card's name and power limit."""
import argparse
import json
import time

import numpy as np

from libcimbar_b200.bench_support import card, entry_states, load_pictures, photographs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batches", type=int, default=4)
    ap.add_argument("--receivers", type=int, nargs="*", default=[16, 64, 256])
    ap.add_argument("--per", type=int, nargs="*", default=[1, 4])
    args = ap.parse_args()
    import torch
    import libcimbar_b200 as cb
    torch.cuda.set_device(0)
    pool = [torch.from_numpy(p).cuda() for p in load_pictures() + photographs()]
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    stream = torch.cuda.Stream()
    B = args.batches

    def timed(fn):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        h0 = time.perf_counter()
        t0.record(stream)
        for b in range(B):
            fn(b)
        t1.record(stream)
        host = time.perf_counter() - h0
        t1.synchronize()
        return t0.elapsed_time(t1) / B, host * 1e6 / B

    results = []
    for D in args.receivers:
        for k in args.per:
            n = D * k
            pics = [pool[i % len(pool)] for i in range(n)]
            maps = [((np.arange(n) + b) % D).astype(np.int32) for b in range(B)]
            pinned = [torch.from_numpy(m).pin_memory() for m in maps]
            master = cb.receiver_states(entry_states(D))
            ctx = cb.Context(68, max_frames=n)
            ctx.set_stream(stream.cuda_stream)
            db = ctx.info.data_bytes
            outs = {arm: (torch.zeros((n, db), dtype=torch.uint8, device="cuda"), torch.zeros(n, dtype=torch.int32, device="cuda"),
                          torch.zeros(n, dtype=torch.int32, device="cuda")) for arm in ("a", "e")}
            states = {arm: master.clone() for arm in ("a", "e")}
            d_of = torch.zeros(n, dtype=torch.int32, device="cuda")

            def run_a(b):
                c, m, s = outs["a"]
                ctx.scan_extract_decode_chunks_receivers_dev(pics, maps[b], states["a"], c.data_ptr(), m.data_ptr(), s.data_ptr(), flags=flags)

            ce, me, se = outs["e"]
            torch.cuda.synchronize()
            plan = ctx.receivers_camera_plan(pics, d_of, states["e"], ce.data_ptr(), me.data_ptr(), se.data_ptr(), flags=flags)

            def run_e(b):
                with torch.cuda.stream(stream):
                    d_of.copy_(pinned[b], non_blocking=True)
                plan.launch()

            # the same B batches from the same states, once each, for the comparison (and as warm-up)
            for arm, fn in (("a", run_a), ("e", run_e)):
                states[arm].copy_(master)
                torch.cuda.synchronize()
                for b in range(B):
                    fn(b)
                torch.cuda.synchronize()
            same = all(torch.equal(x, y) for x, y in zip(outs["a"], outs["e"])) and torch.equal(states["a"], states["e"])
            ta = [timed(run_a) for _ in range(args.rounds)]
            te = [timed(run_e) for _ in range(args.rounds)]
            entry = {"receivers": D, "per_receiver": k, "pictures": n, "records_and_states_agree": bool(same),
                     "decoded_pictures": int((outs["a"][1] != 0).sum())}
            for name, t in (("direct", ta), ("plan", te)):
                entry[name] = {"gpu_ms_per_batch": [round(x[0], 3) for x in t], "host_us_per_batch": [round(x[1], 1) for x in t]}
            results.append(entry)
            plan.close()
            ctx.close()
            del outs, states, d_of
            torch.cuda.empty_cache()
    name, power = card()
    print(json.dumps({"bench": "receivers_plan", "mode": 68, "flags": "SHARPEN_IF_NEEDED|CC_FIT", "rounds": args.rounds, "batches": B,
                      "results": results, "card": name, "power_limit": power}))


if __name__ == "__main__":
    main()
