"""The auto-mode call (cb200_detect_scan_extract_decode_chunks_dev) against decoding the same batch once per candidate mode.

    python -m libcimbar_b200.detect_bench [--pictures B[,B...]] [--rounds R]

Workload: the mode-B photographs of tests/golden/ alternating with camera_plan_bench's pool (the reference's samples/6bit/*.jpg, one a
3584 x 2688 upscale), B pictures in HBM, SHARPEN_IF_NEEDED | CC_FIT, the reference receiver's candidates [66, 68, 67, 4], all
contexts on one stream; B = 1, 8 and 64 by default.  Per batch size, median of R calls (each started with the stream idle and every
context's CCM reset):
  a_detect:   the detect call;
  b_four:     the four direct scan_extract_decode_chunks_dev calls, one per candidate, one after another;
  c_one:      the one direct call of mode 68 (the mode of the batch's B pictures);
each as gpu_ms (CUDA events around the calls on the stream) and host_us (perf_counter around the enqueue).  Also: the walk launches of
one detect call and of the four direct calls, and whether the detect call's walks overlap in time (torch.profiler trace), and
same_as_b: the detect call's modes, records, masks and statuses equal the selection over the four direct calls' results.
Prints one JSON line with the card's name and power limit."""
import argparse
import json
import os
import statistics
import time

import numpy as np

from libcimbar_b200.bench_support import ROOT, card, load_pictures

CANDIDATES = [66, 68, 67, 4]


def load_pool():
    import cv2

    def load(name):
        img = cv2.imread(os.path.join(ROOT, "tests", "golden", name), cv2.IMREAD_COLOR)
        return np.ascontiguousarray(cv2.cvtColor(img, cv2.COLOR_BGR2RGB))
    b = [load("b__ex2434.jpg"), load("b__ex380.jpg")]
    c = load_pictures()
    pool = []
    for i in range(max(len(b), len(c))):
        pool += ([b[i % len(b)]] if i < 2 * len(b) else []) + [c[i]]
    return pool


def walk_trace(torch, fn):
    """(walk launches, their spans overlap) of one call of fn"""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    w = [(e.time_range.start, e.time_range.end) for e in prof.events() if e.device_type.name == "CUDA" and "k_flood_walk" in e.name]
    overlap = len(w) > 1 and max(s for s, _ in w) < min(e for _, e in w)
    return len(w), overlap, [[round((s - w[0][0]) / 1e3, 3), round((e - w[0][0]) / 1e3, 3)] for s, e in sorted(w)] if w else []


def one_size(torch, cb, pool, B, rounds):
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    pics = [pool[i % len(pool)] for i in range(B)]
    wh = np.array([(p.shape[1], p.shape[0]) for p in pics], np.int32)
    d = torch.cat([torch.from_numpy(p.reshape(-1)) for p in pics]).cuda()
    stream = torch.cuda.Stream()
    det = [cb.Context(m, max_frames=B) for m in CANDIDATES]
    ref = [cb.Context(m, max_frames=B) for m in CANDIDATES]
    for c in det + ref:
        c.set_stream(stream.cuda_stream)
    slot = max(c.info.data_bytes for c in det)
    a_out = (torch.zeros(B * slot, dtype=torch.uint8, device="cuda"), torch.zeros(B, dtype=torch.int32, device="cuda"),
             torch.zeros(B, dtype=torch.int32, device="cuda"), torch.zeros(B, dtype=torch.int32, device="cuda"),
             torch.zeros(B * len(det), dtype=torch.int32, device="cuda"))
    b_out = [(torch.zeros((B, c.info.data_bytes), dtype=torch.uint8, device="cuda"), torch.zeros(B, dtype=torch.int32, device="cuda"),
              torch.zeros(B, dtype=torch.int32, device="cuda")) for c in ref]
    right = CANDIDATES.index(68)

    def a():
        cb.detect_scan_extract_decode_chunks_dev(det, d.data_ptr(), wh, *[t.data_ptr() for t in a_out], flags=flags)

    def b():
        for c, (oc, om, os_) in zip(ref, b_out):
            c.scan_extract_decode_chunks_dev(d.data_ptr(), wh, oc.data_ptr(), om.data_ptr(), os_.data_ptr(), flags=flags)

    def c1():
        oc, om, os_ = b_out[right]
        ref[right].scan_extract_decode_chunks_dev(d.data_ptr(), wh, oc.data_ptr(), om.data_ptr(), os_.data_ptr(), flags=flags)

    def reset():
        for c in det + ref:
            c.set_ccm(None)
        torch.cuda.synchronize()

    res = {"pictures": B}
    for name, fn in (("a_detect", a), ("b_four", b), ("c_one", c1)):
        for _ in range(2):                             # warm-up: buffers grown, side streams created
            reset()
            fn()
        host, gpu = [], []
        for _ in range(rounds):
            reset()
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record(stream)
            s = time.perf_counter()
            fn()
            e = time.perf_counter()
            t1.record(stream)
            t1.synchronize()
            host.append((e - s) * 1e6)
            gpu.append(t0.elapsed_time(t1))
        res[name] = {"gpu_ms": round(statistics.median(gpu), 3), "host_us": round(statistics.median(host), 1)}
    res["a_over_b"] = round(res["a_detect"]["gpu_ms"] / res["b_four"]["gpu_ms"], 3)
    res["a_over_c"] = round(res["a_detect"]["gpu_ms"] / res["c_one"]["gpu_ms"], 3)
    reset()
    res["walks_a"], res["walks_overlap_a"], res["walk_spans_ms_a"] = walk_trace(torch, a)
    reset()
    res["walks_b"] = walk_trace(torch, b)[0]
    # the same state on both sides, then one call each: the detect outputs against the selection over the direct results
    reset()
    a()
    b()
    torch.cuda.synchronize()
    chunks, mask, status, mode, mm = [t.cpu().numpy() for t in a_out]
    chunks = chunks.reshape(B, slot)
    mm = mm.view(np.uint32).reshape(B, len(det))
    want = [(o[0].cpu().numpy(), o[1].cpu().numpy().view(np.uint32), o[2].cpu().numpy()) for o in b_out]
    same = True
    for i in range(B):
        masks = [int(w[1][i]) for w in want]
        k = next((j for j, v in enumerate(masks) if v), -1)
        db = det[k].info.data_bytes if k >= 0 else 0
        same &= mm[i].tolist() == masks and mode[i] == k and status[i] == want[max(k, 0)][2][i]
        same &= (k < 0 and not chunks[i].any()) or (k >= 0 and np.array_equal(chunks[i, :db], want[k][0][i]) and not chunks[i, db:].any())
    res["same_as_b"] = bool(same)
    res["detected"] = {str(CANDIDATES[k] if k >= 0 else -1): int((mode == k).sum()) for k in range(-1, len(det))}
    for c in det + ref:
        c.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pictures", default="1,8,64")
    ap.add_argument("--rounds", type=int, default=10)
    args = ap.parse_args()
    import torch
    import libcimbar_b200 as cb
    torch.cuda.set_device(0)
    pool = load_pool()
    sizes = [int(b) for b in str(args.pictures).split(",")]
    out = {"metric": "detect", "candidates": CANDIDATES, "flags": "SHARPEN_IF_NEEDED|CC_FIT", "rounds": args.rounds,
           "batches": [one_size(torch, cb, pool, B, args.rounds) for B in sizes]}
    out["gpu"], out["power_limit"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
