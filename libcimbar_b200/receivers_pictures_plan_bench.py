"""Receivers camera plans over device descriptors against the fixed receivers plan and the direct receivers call.

    python -m libcimbar_b200.receivers_pictures_plan_bench [--rounds R] [--batches B]

Workload: receivers_plan_bench's pool (the camera_pipeline_bench pictures plus the two mode-B photographs, in device memory), mode B,
SHARPEN_IF_NEEDED | CC_FIT, D receivers x k pictures, every receiver starting from a distinct active matrix, batch b mapping picture
i to receiver (i + b) % D.  Two workloads:
  uniform: receivers_plan_bench's batches -- slot i always holds pool picture i % len(pool).  Arms: `direct` (one
           cb200_scan_extract_decode_chunks_receivers_dev per batch), `plan` (the fixed receivers plan: the map copied, one launch),
           `pictures_plan` (the plan over device descriptors: the map and the n x 40 descriptor bytes copied, one launch).
  mixed:   the pool reshuffled across the slots every batch, so each slot's size and layout change.  Arms: `direct` and
           `pictures_plan` (the fixed plan cannot take these batches).
  mixed_detect: the mixed batches under detect_receivers_plan_bench's candidate modes, every session in auto mode (`auto`) or a
           mix of auto and locked sessions (`mixed`).  Arms: `direct` (cb200_detect_scan_extract_decode_chunks_receivers_dev) and
           `pictures_plan` (the detect plan over device descriptors: descriptors, candidates and map copied, one launch).
The copies come from pinned memory on the plan's stream.  Prints one JSON line: per workload and shape, each arm's host time to issue
one batch and GPU time per batch (CUDA events around B batches back to back, divided by B), whether every arm gave identical
records, masks, statuses and states over the same B batches from the same states; the card's name and power limit."""
import argparse
import json
import time

import numpy as np

from libcimbar_b200.bench_support import MODES, candidates, card, entry_states, load_pictures, photographs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batches", type=int, default=4)
    ap.add_argument("--receivers", type=int, nargs="*", default=[16, 64])
    ap.add_argument("--per", type=int, nargs="*", default=[1, 4])
    ap.add_argument("--mixes", nargs="*", default=["auto", "mixed"])
    args = ap.parse_args()
    import torch
    import libcimbar_b200 as cb
    torch.cuda.set_device(0)
    pool = [torch.from_numpy(p).cuda() for p in load_pictures() + photographs()]
    shorts = [min(p.shape[:2]) for p in pool]
    bounds = (min(shorts), max(shorts), max(max(p.shape[:2]) for p in pool))
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    stream = torch.cuda.Stream()
    B = args.batches
    rng = np.random.default_rng(0)

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
    for workload in ("uniform", "mixed"):
        for D in args.receivers:
            for k in args.per:
                n = D * k
                if workload == "uniform":
                    batches = [[pool[i % len(pool)] for i in range(n)]] * B
                else:
                    batches = [[pool[j % len(pool)] for j in rng.permutation(max(n, len(pool)))[:n]] for _ in range(B)]
                maps = [((np.arange(n) + b) % D).astype(np.int32) for b in range(B)]
                pin_of = [torch.from_numpy(m).pin_memory() for m in maps]
                pin_desc = [torch.from_numpy(cb.picture_descriptors(p)).pin_memory() for p in batches]
                master = cb.receiver_states(entry_states(D))
                ctx = cb.Context(68, max_frames=n)
                ctx.set_stream(stream.cuda_stream)
                db = ctx.info.data_bytes
                arms = ["direct", "plan", "pictures_plan"] if workload == "uniform" else ["direct", "pictures_plan"]
                outs = {a: (torch.zeros((n, db), dtype=torch.uint8, device="cuda"), torch.zeros(n, dtype=torch.int32, device="cuda"),
                            torch.zeros(n, dtype=torch.int32, device="cuda")) for a in arms}
                states = {a: master.clone() for a in arms}
                d_of = {a: torch.zeros(n, dtype=torch.int32, device="cuda") for a in arms}
                d_pics = torch.zeros((n, 40), dtype=torch.uint8, device="cuda")
                torch.cuda.synchronize()
                plans = {}
                c, m, s = outs["pictures_plan"]
                plans["pictures_plan"] = ctx.receivers_camera_plan_pictures_dev(d_pics, bounds, d_of["pictures_plan"], states["pictures_plan"],
                                                                                c.data_ptr(), m.data_ptr(), s.data_ptr(), flags=flags)
                if "plan" in arms:
                    c, m, s = outs["plan"]
                    plans["plan"] = ctx.receivers_camera_plan(batches[0], d_of["plan"], states["plan"], c.data_ptr(), m.data_ptr(), s.data_ptr(),
                                                              flags=flags)

                def run(arm):
                    def step(b):
                        if arm == "direct":
                            c, m, s = outs[arm]
                            ctx.scan_extract_decode_chunks_receivers_dev(batches[b], maps[b], states[arm], c.data_ptr(), m.data_ptr(), s.data_ptr(),
                                                                         flags=flags)
                            return
                        with torch.cuda.stream(stream):
                            d_of[arm].copy_(pin_of[b], non_blocking=True)
                            if arm == "pictures_plan":
                                d_pics.copy_(pin_desc[b], non_blocking=True)
                        plans[arm].launch()
                    return step

                # the same B batches from the same states, once per arm, for the comparison (and as warm-up)
                for a in arms:
                    states[a].copy_(master)
                    torch.cuda.synchronize()
                    for b in range(B):
                        run(a)(b)
                    torch.cuda.synchronize()
                same = all(all(torch.equal(x, y) for x, y in zip(outs["direct"], outs[a])) and torch.equal(states["direct"], states[a])
                           for a in arms[1:])
                times = {a: [timed(run(a)) for _ in range(args.rounds)] for a in arms}
                entry = {"workload": workload, "receivers": D, "per_receiver": k, "pictures": n, "records_and_states_agree": bool(same),
                         "decoded_pictures": int((outs["direct"][1] != 0).sum())}
                for a in arms:
                    entry[a] = {"gpu_ms_per_batch": [round(x[0], 3) for x in times[a]], "host_us_per_batch": [round(x[1], 1) for x in times[a]]}
                results.append(entry)
                for p in plans.values():
                    p.close()
                ctx.close()
                del outs, states, d_of, d_pics
                torch.cuda.empty_cache()
    # the detect variant on mixed batches: candidate contexts MODES (detect_receivers_plan_bench's), every session in auto mode or a mix
    # of auto and locked sessions, against the direct detect receivers call
    K = len(MODES)
    for mix in args.mixes:
        for D in args.receivers:
            for k in args.per:
                n = D * k
                batches = [[pool[j % len(pool)] for j in rng.permutation(max(n, len(pool)))[:n]] for _ in range(B)]
                maps = [((np.arange(n) + b) % D).astype(np.int32) for b in range(B)]
                per_receiver = np.array(candidates(mix, D), np.uint32)
                cands = [per_receiver[m] for m in maps]
                pin_of = [torch.from_numpy(m).pin_memory() for m in maps]
                pin_cand = [torch.from_numpy(c.view(np.int32)).pin_memory() for c in cands]
                pin_desc = [torch.from_numpy(cb.picture_descriptors(p)).pin_memory() for p in batches]
                master = cb.receiver_states(entry_states(D))
                arms = {}
                for a in ("direct", "pictures_plan"):
                    ctxs = [cb.Context(m, max_frames=n) for m in MODES]
                    for c in ctxs:
                        c.set_stream(stream.cuda_stream)
                    slot = max(c.info.data_bytes for c in ctxs)
                    arms[a] = {"ctxs": ctxs, "states": [master.clone() for _ in MODES],
                               "out": [torch.zeros((n, slot), dtype=torch.uint8, device="cuda")] +
                                      [torch.zeros(n * w, dtype=torch.int32, device="cuda") for w in (1, 1, 1, K)]}
                d_pics = torch.zeros((n, 40), dtype=torch.uint8, device="cuda")
                d_cand = torch.zeros(n, dtype=torch.int32, device="cuda")
                d_of = torch.zeros(n, dtype=torch.int32, device="cuda")
                e = arms["pictures_plan"]
                torch.cuda.synchronize()
                plan = cb.detect_receivers_camera_plan_pictures_dev(e["ctxs"], d_pics, bounds, d_cand, d_of, e["states"],
                                                                    *[t.data_ptr() for t in e["out"]], flags=flags)

                def detect_step(arm):
                    def step(b):
                        if arm == "direct":
                            a = arms[arm]
                            cb.detect_scan_extract_decode_chunks_receivers_dev(a["ctxs"], batches[b], maps[b], a["states"],
                                                                               *[t.data_ptr() for t in a["out"][:4]], candidates=cands[b],
                                                                               d_mode_masks=a["out"][4].data_ptr(), flags=flags)
                            return
                        with torch.cuda.stream(stream):
                            d_pics.copy_(pin_desc[b], non_blocking=True)
                            d_cand.copy_(pin_cand[b], non_blocking=True)
                            d_of.copy_(pin_of[b], non_blocking=True)
                        plan.launch()
                    return step

                for a in arms:
                    for st in arms[a]["states"]:
                        st.copy_(master)
                    torch.cuda.synchronize()
                    for b in range(B):
                        detect_step(a)(b)
                    torch.cuda.synchronize()
                same = all(torch.equal(x, y) for x, y in zip(arms["direct"]["out"], e["out"])) and \
                    all(torch.equal(x, y) for x, y in zip(arms["direct"]["states"], e["states"]))
                times = {a: [timed(detect_step(a)) for _ in range(args.rounds)] for a in arms}
                entry = {"workload": "mixed_detect", "mix": mix, "modes": MODES, "receivers": D, "per_receiver": k, "pictures": n,
                         "records_and_states_agree": bool(same)}
                for a in arms:
                    entry[a] = {"gpu_ms_per_batch": [round(x[0], 3) for x in times[a]], "host_us_per_batch": [round(x[1], 1) for x in times[a]]}
                results.append(entry)
                plan.close()
                for arm in arms.values():
                    for c in arm["ctxs"]:
                        c.close()
                del arms, e, d_pics, d_cand, d_of
                torch.cuda.empty_cache()
    name, power = card()
    print(json.dumps({"bench": "receivers_pictures_plan", "mode": 68, "flags": "SHARPEN_IF_NEEDED|CC_FIT", "bounds": bounds, "rounds": args.rounds,
                      "batches": B, "results": results, "card": name, "power_limit": power}))


if __name__ == "__main__":
    main()
