"""Receivers batches whose sessions differ in their flags: one call with a receiver flags table against one existing call per flag set.

    python -m libcimbar_b200.receiver_flags_bench [--rounds R] [--batches B]

Workload: receivers_pictures_plan_bench's pool (the camera_pipeline_bench pictures plus the two mode-B photographs, in device memory),
mode B, D receivers x k pictures, every receiver starting from a distinct active matrix, batch b mapping picture i to receiver
(i + b) % D.  Half the sessions are web-like (SHARPEN | CC_FIT, even receivers), half CLI-like (SHARPEN_IF_NEEDED | CC_FIT, odd
receivers).  Arms:
  two_calls:  two cb200_scan_extract_decode_chunks_receivers_dev per batch, one per flag set, on that set's pictures;
  flags_call: one cb200_scan_extract_decode_chunks_receivers_flags_dev per batch with the flags table;
  flags_plan: the plan over device descriptors with the table (cb200_camera_plan_create_receivers_pictures_flags_dev): the map and the
              n x 40 descriptor bytes copied from pinned memory on the plan's stream, one launch.
And a uniform batch (every session SHARPEN_IF_NEEDED | CC_FIT): `uniform_existing` (the existing call with those flags) against
`uniform_flags` (the flags call with a uniform table): what always taking the fitted-CCM route costs.
Prints one JSON line: per shape, each arm's host time to issue one batch and GPU time per batch (CUDA events around B batches back to
back, divided by B), whether the arms gave identical records, masks, statuses and states over the same B batches from the same
states; the card's name and power limit."""
import argparse
import json
import time

import numpy as np

from libcimbar_b200.bench_support import card, entry_states, load_pictures, photographs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batches", type=int, default=4)
    ap.add_argument("--receivers", type=int, nargs="*", default=[16, 64])
    ap.add_argument("--per", type=int, nargs="*", default=[1, 4])
    args = ap.parse_args()
    import torch
    import libcimbar_b200 as cb
    torch.cuda.set_device(0)
    pool = [torch.from_numpy(p).cuda() for p in load_pictures() + photographs()]
    shorts = [min(p.shape[:2]) for p in pool]
    bounds = (min(shorts), max(shorts), max(max(p.shape[:2]) for p in pool))
    web, cli = cb.FLAG_SHARPEN | cb.FLAG_CC_FIT, cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
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
            batch = [pool[i % len(pool)] for i in range(n)]
            maps = [((np.arange(n) + b) % D).astype(np.int32) for b in range(B)]
            pin_of = [torch.from_numpy(m).pin_memory() for m in maps]
            pin_desc = torch.from_numpy(cb.picture_descriptors(batch)).pin_memory()
            # per batch and flag set: the pictures of that set's receivers, in batch order
            groups = [[np.flatnonzero(m % 2 == g) for g in (0, 1)] for m in maps]
            words = torch.tensor([web if r % 2 == 0 else cli for r in range(D)], dtype=torch.int32, device="cuda")
            uniform = torch.full((D,), cli, dtype=torch.int32, device="cuda")
            master = cb.receiver_states(entry_states(D))
            ctx = cb.Context(68, max_frames=n)
            ctx.set_stream(stream.cuda_stream)
            db = ctx.info.data_bytes
            arms = ["two_calls", "flags_call", "flags_plan", "uniform_existing", "uniform_flags"]
            outs = {a: (torch.zeros((n, db), dtype=torch.uint8, device="cuda"), torch.zeros(n, dtype=torch.int32, device="cuda"),
                        torch.zeros(n, dtype=torch.int32, device="cuda")) for a in arms}
            part = [(torch.zeros((n, db), dtype=torch.uint8, device="cuda"), torch.zeros(n, dtype=torch.int32, device="cuda"),
                     torch.zeros(n, dtype=torch.int32, device="cuda")) for _ in (0, 1)]
            states = {a: master.clone() for a in arms}
            d_of = torch.zeros(n, dtype=torch.int32, device="cuda")
            d_pics = torch.zeros((n, 40), dtype=torch.uint8, device="cuda")
            torch.cuda.synchronize()
            c, m, s = outs["flags_plan"]
            plan = ctx.receivers_camera_plan_pictures_dev(d_pics, bounds, d_of, states["flags_plan"], c.data_ptr(), m.data_ptr(), s.data_ptr(),
                                                          receiver_flags=words)

            def run(arm):
                def step(b):
                    c, m, s = outs[arm]
                    if arm == "two_calls":
                        for g, fl in ((0, web), (1, cli)):
                            idx = groups[b][g]
                            pc, pm, ps = part[g]
                            ctx.scan_extract_decode_chunks_receivers_dev([batch[i] for i in idx], maps[b][idx], states[arm], pc.data_ptr(),
                                                                         pm.data_ptr(), ps.data_ptr(), flags=fl)
                    elif arm == "flags_call":
                        ctx.scan_extract_decode_chunks_receivers_dev(batch, maps[b], states[arm], c.data_ptr(), m.data_ptr(), s.data_ptr(),
                                                                     receiver_flags=words)
                    elif arm == "uniform_existing":
                        ctx.scan_extract_decode_chunks_receivers_dev(batch, maps[b], states[arm], c.data_ptr(), m.data_ptr(), s.data_ptr(),
                                                                     flags=cli)
                    elif arm == "uniform_flags":
                        ctx.scan_extract_decode_chunks_receivers_dev(batch, maps[b], states[arm], c.data_ptr(), m.data_ptr(), s.data_ptr(),
                                                                     receiver_flags=uniform)
                    else:
                        with torch.cuda.stream(stream):
                            d_of.copy_(pin_of[b], non_blocking=True)
                            d_pics.copy_(pin_desc, non_blocking=True)
                        plan.launch()
                return step

            # the same B batches from the same states, once per arm, for the comparison (and as warm-up)
            same = {}
            for a in arms:
                states[a].copy_(master)
                torch.cuda.synchronize()
                for b in range(B):
                    run(a)(b)
                    if a == "two_calls":          # the groups' records back in batch order, for the comparison
                        torch.cuda.synchronize()
                        for g in (0, 1):
                            idx = torch.from_numpy(groups[b][g]).cuda()
                            for x, y in zip(outs[a], part[g]):
                                x[idx] = y[:len(idx)]
                torch.cuda.synchronize()
            for a, ref in (("flags_call", "two_calls"), ("flags_plan", "two_calls"), ("uniform_flags", "uniform_existing")):
                same[a] = all(torch.equal(x, y) for x, y in zip(outs[ref], outs[a])) and torch.equal(states[ref], states[a])
            times = {a: [timed(run(a)) for _ in range(args.rounds)] for a in arms}
            entry = {"receivers": D, "per_receiver": k, "pictures": n, "agree_with_existing": {a: bool(v) for a, v in same.items()},
                     "decoded_pictures": int((outs["two_calls"][1] != 0).sum())}
            for a in arms:
                entry[a] = {"gpu_ms_per_batch": [round(x[0], 3) for x in times[a]], "host_us_per_batch": [round(x[1], 1) for x in times[a]]}
            results.append(entry)
            plan.close()
            ctx.close()
            del outs, part, states, d_of, d_pics
            torch.cuda.empty_cache()
    name, power = card()
    print(json.dumps({"bench": "receiver_flags", "mode": 68, "flags": {"web": "SHARPEN|CC_FIT", "cli": "SHARPEN_IF_NEEDED|CC_FIT"},
                      "bounds": bounds, "rounds": args.rounds, "batches": B, "results": results, "card": name, "power_limit": power}))


if __name__ == "__main__":
    main()
