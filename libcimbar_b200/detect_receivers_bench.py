"""The auto mode for receivers in one call, against what a decode service must do without it to get the same results.

    python -m libcimbar_b200.detect_receivers_bench [--rounds R]

Workload: receivers_bench's pool (the reference's samples/6bit/*.jpg with its 3584 x 2688 upscale, mode 4C, and the two mode-B
photographs tests/golden/b__ex*.jpg), D receivers x k pictures (16 x 4 and 64 x 4), picture i drawn round-robin from the pool and
belonging to receiver i % D.  Candidates [66, 68, 67, 4] (the reference web receiver's order), SHARPEN_IF_NEEDED | CC_FIT (the
CLI's defaults), every receiver starting from a distinct active matrix in every mode's table.  Three session mixes:
  auto    every receiver in auto mode: every picture under all four modes;
  locked  every receiver locked: even receivers to 68, odd ones to 4;
  mixed   90 % locked as above, every tenth receiver in auto mode.
Two runs per shape and mix, timed in turn with CUDA events, R rounds each:
  (a) `detect_receivers`: one cb200_detect_scan_extract_decode_chunks_receivers_dev call;
  (b) `per_mode`: per mode with pictures, one cb200_scan_extract_decode_chunks_receivers_dev on those pictures with that mode's
      table, back to back on one stream, then the same selection (first mode with a chunk) in torch on the device.
Prints one JSON line: per shape and mix, for each run pictures/s, GPU ms per batch, host us to issue it, kernel launches and exact
walk launches (k_flood_walk, counted with torch.profiler in a separate run); whether (a) and (b) gave identical records, masks,
statuses, modes and states; the card's name and power limit."""
import argparse
import json
import time

import numpy as np

from libcimbar_b200.bench_support import MODES, candidates, card, load_pictures, photographs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--shapes", nargs="*", default=["16x4", "64x4"])
    ap.add_argument("--mixes", nargs="*", default=["auto", "locked", "mixed"])
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    import libcimbar_b200 as cb
    torch.cuda.set_device(0)
    pool = [torch.from_numpy(p).cuda() for p in load_pictures() + photographs()]
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    stream = torch.cuda.Stream()
    K = len(MODES)

    def timed(fn):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        h0 = time.perf_counter()
        t0.record(stream)
        fn()
        t1.record(stream)
        host = time.perf_counter() - h0
        t1.synchronize()
        return t0.elapsed_time(t1), host * 1e6

    def launches(fn):
        torch.cuda.synchronize()
        before = cb.launch_count()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        walks = sum("k_flood_walk" in e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)
        return cb.launch_count() - before, walks

    results = []
    for shape in args.shapes:
        D, k = (int(x) for x in shape.split("x"))
        n = D * k
        pics = [pool[i % len(pool)] for i in range(n)]
        of = np.arange(n, dtype=np.int32) % D
        ents = [np.diag([1.0 + 0.002 * (r % 50), 1.0, 0.999 - 0.002 * (r % 50)]).astype(np.float32) for r in range(D)]
        master = cb.receiver_states(ents)
        ctxs = [cb.Context(m, max_frames=n) for m in MODES]
        for c in ctxs:
            c.set_stream(stream.cuda_stream)
        slot = max(c.info.data_bytes for c in ctxs)
        states = [master.clone() for _ in MODES]
        chunks = torch.zeros((n, slot), dtype=torch.uint8, device="cuda")
        mask = torch.zeros(n, dtype=torch.int32, device="cuda")
        status = torch.zeros(n, dtype=torch.int32, device="cuda")
        mode = torch.zeros(n, dtype=torch.int32, device="cuda")
        # (b)'s per-mode outputs and its selection's
        pc = [torch.zeros((n, c.info.data_bytes), dtype=torch.uint8, device="cuda") for c in ctxs]
        pm = [torch.zeros(n, dtype=torch.int32, device="cuda") for _ in MODES]
        ps = [torch.zeros(n, dtype=torch.int32, device="cuda") for _ in MODES]
        b_chunks, b_mask, b_status, b_mode = (torch.zeros_like(t) for t in (chunks, mask, status, mode))
        rows = torch.arange(n, device="cuda")
        for mix in args.mixes:
            per_receiver = candidates(mix, D)
            cand = np.array([per_receiver[r] for r in of], np.uint32)
            subsets = [np.flatnonzero(cand >> np.uint32(j) & np.uint32(1)) for j in range(K)]
            idx = [torch.from_numpy(s).cuda() for s in subsets]

            def reset():
                with torch.cuda.stream(stream):
                    for s in states:
                        s.copy_(master)

            def run_a():
                reset()
                cb.detect_scan_extract_decode_chunks_receivers_dev(ctxs, pics, of, states, chunks.data_ptr(), mask.data_ptr(), status.data_ptr(),
                                                                   mode.data_ptr(), candidates=cand, flags=flags)

            def run_b():
                reset()
                for j, c in enumerate(ctxs):
                    if len(subsets[j]):
                        c.scan_extract_decode_chunks_receivers_dev([pics[i] for i in subsets[j]], of[subsets[j]], states[j], pc[j].data_ptr(),
                                                                   pm[j].data_ptr(), ps[j].data_ptr(), flags=flags)
                with torch.cuda.stream(stream):            # the selection, in stream order behind the calls
                    M = torch.zeros((n, K), dtype=torch.int64, device="cuda")
                    S = torch.zeros((n, K), dtype=torch.int32, device="cuda")
                    have = torch.zeros((n, K), dtype=torch.bool, device="cuda")
                    for j in range(K):
                        m = len(subsets[j])
                        if m:
                            M[idx[j], j] = pm[j][:m].to(torch.int64) & 0xFFFFFFFF
                            S[idx[j], j] = ps[j][:m]
                            have[idx[j], j] = True
                    nz = M != 0
                    sel = torch.where(nz.any(1), nz.to(torch.int32).argmax(1), -1)
                    first = have.to(torch.int32).argmax(1)
                    b_mode.copy_(sel)
                    b_mask.copy_(torch.where(sel >= 0, M[rows, sel.clamp(min=0)], 0).to(torch.int32))
                    b_status.copy_(S[rows, torch.where(sel >= 0, sel, first)])
                    b_chunks.zero_()
                    for j in range(K):
                        m = len(subsets[j])
                        if m:
                            db = ctxs[j].info.data_bytes       # no boolean indexing: it would wait for the device
                            take = (sel[idx[j]] == j)[:, None]
                            b_chunks[idx[j], :db] = torch.where(take, pc[j][:m], b_chunks[idx[j], :db])

            entry = {"receivers": D, "per_receiver": k, "pictures": n, "mix": mix, "auto_receivers": sum(c == (1 << K) - 1 for c in per_receiver),
                     "pictures_per_mode": {str(m): len(s) for m, s in zip(MODES, subsets)}}
            run_a()
            torch.cuda.synchronize()
            a_out = [t.cpu().numpy().copy() for t in (chunks, mask, status, mode)] + [s.cpu().numpy().copy() for s in states]
            run_b()
            torch.cuda.synchronize()
            b_out = [t.cpu().numpy().copy() for t in (b_chunks, b_mask, b_status, b_mode)] + [s.cpu().numpy().copy() for s in states]
            entry["a_equals_b"] = all(np.array_equal(x, y) for x, y in zip(a_out, b_out))
            entry["decoded_pictures"] = int((a_out[3] >= 0).sum())
            entry["detected"] = {str(m): int((a_out[3] == j).sum()) for j, m in enumerate(MODES)}
            ta, tb = [], []
            for _ in range(args.rounds):                   # alternated, so that both see the same state of the card
                ta.append(timed(run_a))
                tb.append(timed(run_b))
            for name, t, fn in (("detect_receivers", ta, run_a), ("per_mode", tb, run_b)):
                count, walks = launches(fn)
                entry[name] = {"pictures_per_s": round(n / (min(x[0] for x in t) / 1e3), 1), "gpu_ms": [round(x[0], 2) for x in t],
                               "host_us": [round(x[1]) for x in t], "launches": count, "walk_launches": walks}
            entry["gpu_ratio"] = round(min(x[0] for x in ta) / min(x[0] for x in tb), 3)
            results.append(entry)
        for c in ctxs:
            c.close()
        del chunks, mask, status, mode, pc, pm, ps, states
        torch.cuda.empty_cache()
    name, power = card()
    print(json.dumps({"bench": "detect_receivers", "modes": MODES, "flags": "SHARPEN_IF_NEEDED|CC_FIT", "rounds": args.rounds,
                      "results": results, "card": name, "power_limit": power}))


if __name__ == "__main__":
    main()
