"""The auto mode for receivers replayed from a graph (a detect receivers camera plan), against the direct call.

    python -m libcimbar_b200.detect_receivers_plan_bench [--rounds R] [--batches B]

Workload: detect_receivers_bench's pool, shapes (D receivers x k pictures: 16 x 4 and 64 x 4), candidates [66, 68, 67, 4] and
flags (SHARPEN_IF_NEEDED | CC_FIT), and its three session mixes (auto, locked: even receivers to 68 and odd ones to 4, mixed: every
tenth receiver in auto mode).  Each batch has a fresh map (the pictures dealt to the receivers in a new random order) and so fresh
candidates; B batches run back to back, the states carrying from one to the next.  Two arms, timed in turn with CUDA events:
  (a) `direct`: one cb200_detect_scan_extract_decode_chunks_receivers_dev call per batch, from the host map and candidates;
  (e) `plan`:   per batch, the candidates and the map copied from pinned host memory into the plan's bound buffers on the stream,
                then one launch of a plan made once per shape and mix (cb200_camera_plan_create_detect_receivers).
Prints one JSON line: per shape and mix, for each arm host us and GPU ms per batch (each round's), kernel launches per batch; whether
(a) and (e) gave identical records, masks, statuses, modes, mode masks and states over the B batches; the card and its power limit."""
import argparse
import json
import time

import numpy as np

from libcimbar_b200.bench_support import MODES, candidates, card, load_pictures, photographs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batches", type=int, default=4)
    ap.add_argument("--shapes", nargs="*", default=["16x4", "64x4"])
    ap.add_argument("--mixes", nargs="*", default=["auto", "locked", "mixed"])
    args = ap.parse_args()
    import torch
    import libcimbar_b200 as cb
    torch.cuda.set_device(0)
    pool = [torch.from_numpy(p).cuda() for p in load_pictures() + photographs()]
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    stream = torch.cuda.Stream()
    K, B = len(MODES), args.batches

    def timed(fn):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        h0 = time.perf_counter()
        t0.record(stream)
        fn()
        t1.record(stream)
        host = time.perf_counter() - h0
        t1.synchronize()
        return t0.elapsed_time(t1) / B, host * 1e6 / B

    results = []
    for shape in args.shapes:
        D, k = (int(x) for x in shape.split("x"))
        n = D * k
        pics = [pool[i % len(pool)] for i in range(n)]
        ents = [np.diag([1.0 + 0.002 * (r % 50), 1.0, 0.999 - 0.002 * (r % 50)]).astype(np.float32) for r in range(D)]
        master = cb.receiver_states(ents)
        arms = {}
        for name in ("direct", "plan"):
            ctxs = [cb.Context(m, max_frames=n) for m in MODES]
            for c in ctxs:
                c.set_stream(stream.cuda_stream)
            slot = max(c.info.data_bytes for c in ctxs)
            arms[name] = {"ctxs": ctxs, "states": [master.clone() for _ in MODES],
                          "out": [torch.zeros((n, slot), dtype=torch.uint8, device="cuda")] +
                                 [torch.zeros(n * w, dtype=torch.int32, device="cuda") for w in (1, 1, 1, K)]}
        e = arms["plan"]
        d_cand = torch.zeros(n, dtype=torch.int32, device="cuda")
        d_of = torch.zeros(n, dtype=torch.int32, device="cuda")
        h_cand = torch.zeros((B, n), dtype=torch.int32).pin_memory()
        h_of = torch.zeros((B, n), dtype=torch.int32).pin_memory()
        rng = np.random.default_rng(D * 1000 + k)
        for mix in args.mixes:
            per_receiver = np.array(candidates(mix, D), np.uint32)
            ofs = [rng.permutation(n).astype(np.int32) % D for _ in range(B)]       # fresh maps, so fresh candidates
            cands = [per_receiver[of] for of in ofs]
            for b in range(B):
                h_of[b].copy_(torch.from_numpy(ofs[b]))
                h_cand[b].copy_(torch.from_numpy(cands[b].view(np.int32)))
            torch.cuda.synchronize()
            plan = cb.detect_receivers_camera_plan(e["ctxs"], pics, d_cand, d_of, e["states"], *[t.data_ptr() for t in e["out"]], flags=flags)

            def reset(arm):
                with torch.cuda.stream(stream):
                    for s in arm["states"]:
                        s.copy_(master)

            def batch_a(b):
                a = arms["direct"]
                cb.detect_scan_extract_decode_chunks_receivers_dev(a["ctxs"], pics, ofs[b], a["states"], *[t.data_ptr() for t in a["out"][:4]],
                                                                   candidates=cands[b], d_mode_masks=a["out"][4].data_ptr(), flags=flags)

            def batch_e(b):
                with torch.cuda.stream(stream):
                    d_cand.copy_(h_cand[b], non_blocking=True)
                    d_of.copy_(h_of[b], non_blocking=True)
                plan.launch()

            def run(arm, fn):
                reset(arm)
                for b in range(B):
                    fn(b)

            # exactness: every batch's outputs and the final states
            seen = {}
            for name, fn in (("direct", batch_a), ("plan", batch_e)):
                reset(arms[name])
                outs = []
                for b in range(B):
                    fn(b)
                    torch.cuda.synchronize()
                    outs.append([t.cpu().numpy().copy() for t in arms[name]["out"]])
                seen[name] = (outs, [s.cpu().numpy().copy() for s in arms[name]["states"]])
            same = all(np.array_equal(x, y) for ba, be in zip(seen["direct"][0], seen["plan"][0]) for x, y in zip(ba, be)) and \
                all(np.array_equal(x, y) for x, y in zip(seen["direct"][1], seen["plan"][1]))
            entry = {"receivers": D, "per_receiver": k, "pictures": n, "mix": mix, "batches": B, "a_equals_e": bool(same),
                     "decoded_pictures": int(sum((o[3] >= 0).sum() for o in seen["direct"][0]))}
            ta, te = [], []
            for _ in range(args.rounds):                   # alternated, so that both see the same state of the card
                ta.append(timed(lambda: run(arms["direct"], batch_a)))
                te.append(timed(lambda: run(e, batch_e)))
            for name, t, fn in (("direct", ta, batch_a), ("plan", te, batch_e)):
                torch.cuda.synchronize()
                before = cb.launch_count()
                fn(0)
                count = cb.launch_count() - before
                torch.cuda.synchronize()
                entry[name] = {"gpu_ms_per_batch": [round(x[0], 2) for x in t], "host_us_per_batch": [round(x[1]) for x in t], "launches": count}
            results.append(entry)
            plan.close()
        for arm in arms.values():
            for c in arm["ctxs"]:
                c.close()
        del arms, e
        torch.cuda.empty_cache()
    name, power = card()
    print(json.dumps({"bench": "detect_receivers_plan", "modes": MODES, "flags": "SHARPEN_IF_NEEDED|CC_FIT", "rounds": args.rounds,
                      "results": results, "card": name, "power_limit": power}))


if __name__ == "__main__":
    main()
