"""Ragged camera batches: the reference CLI's decode loop (`cimbar -m 4C samples/6bit/*.jpg`) as one call.

    python -m libcimbar_b200.ragged_bench [--pictures B] [--rounds R]

One step = B camera pictures (the reference's samples/6bit/*.jpg, tests/golden/, in glob order -- the shape changes at every step --
replicated; 4_30_f0_big.jpg, 3052 x 2704, is not kept in the repository and stands in as a 2.8x upscale of 4_30_f1_360.jpg,
3584 x 2688, portrait and 9-tap like it), resident in HBM, scanned, deskewed and decoded with SHARPEN_IF_NEEDED | CC_FIT (the CLI's defaults).  Three ways, timed
alternately for R rounds with CUDA events around the step:
  (a) `ragged`:    one cb200_scan_ragged_dev + one cb200_extract_decode_fountain_ragged_dev call for the whole batch;
  (b) `per_run`:   what an order-preserving caller does with the uniform entry points: one cb200_scan_dev +
                   cb200_extract_decode_fountain_dev call per run of equal shapes -- here one per picture;
  (c) `per_shape`: one uniform call per shape (pictures grouped by shape).  This reorders the CC_FIT carry, so it is NOT the
                   CLI's result: a timing reference only.
Prints one JSON line: pictures/s and ms per step of each, the scan / decode kernel split of (a) from cb200_get_timing, the card's
name and power limit, and whether (a) and (b) returned the same chunks."""
import argparse
import json
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GLOB = ["4_30_802", "4_30_f0_177_ccm", "4_30_f0_627", "4_30_f0_627_extract", None, "4_30_f1_360", "4_30_f2_246", "4_30_f2_734"]


def load_pictures():
    import cv2

    def load(name):
        img = cv2.imread(os.path.join(ROOT, "tests", "golden", "6bit__%s.jpg" % name), cv2.IMREAD_COLOR)
        return np.ascontiguousarray(cv2.cvtColor(img, cv2.COLOR_BGR2RGB))
    return [load(n) if n else cv2.resize(load("4_30_f1_360"), None, fx=2.8, fy=2.8) for n in GLOB]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in q.split(",")]
        return name, power
    except Exception as e:          # the numbers are reported without it, never estimated
        return "unknown (%s)" % e, "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pictures", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    import torch
    import libcimbar_b200 as cb
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    B = args.pictures
    pool = load_pictures()
    idx = [i % len(pool) for i in range(B)]
    pics = [pool[i] for i in idx]
    wh = np.array([(p.shape[1], p.shape[0]) for p in pics], np.int32)
    sizes = [p.nbytes for p in pics]
    starts = np.cumsum([0] + sizes)
    d_batch = torch.cat([torch.from_numpy(p.reshape(-1)) for p in pics]).to(dev)
    base = d_batch.data_ptr()
    ctx = cb.Context(4, max_frames=B)
    ctx.set_stream(torch.cuda.current_stream().cuda_stream)
    lib, hnd, info = ctx.lib, ctx._h, ctx.info
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    anchors, count, cutoff = np.zeros((B, 4, 4), np.int32), np.zeros(B, np.int32), np.zeros(B, np.uint32)
    chunks = np.zeros((B, info.chunks_per_frame, info.chunk_size), np.uint8)
    ccount, cmask, ff = np.zeros(B, np.uint32), np.zeros(B, np.uint32), np.zeros(B, np.uint8)

    def corners(a):
        c = np.stack([(a[:, :, 0] + a[:, :, 1]) // 2, (a[:, :, 2] + a[:, :, 3]) // 2], axis=2)
        return np.ascontiguousarray(c.astype(np.float32).reshape(-1, 8))

    def ragged():
        cb._check(lib.cb200_scan_ragged_dev(hnd, base, wh.ctypes.data, B, anchors.ctypes.data, count.ctypes.data, cutoff.ctypes.data))
        cr = corners(anchors)
        cb._check(lib.cb200_extract_decode_fountain_ragged_dev(hnd, base, wh.ctypes.data, B, cr.ctypes.data, flags, chunks.ctypes.data,
                                                                ccount.ctypes.data, cmask.ctypes.data, ff.ctypes.data))

    def uniform(group):
        """one uniform call pair for the pictures `group` (equal shapes, consecutive in memory, or copied so)"""
        k = len(group)
        w, h = int(wh[group[0], 0]), int(wh[group[0], 1])
        if all(group[j + 1] == group[j] + 1 for j in range(k - 1)):
            ptr, keep = base + int(starts[group[0]]), None
        else:
            keep = torch.cat([d_batch[int(starts[i]):int(starts[i + 1])] for i in group])
            ptr = keep.data_ptr()
        a, c, cut = np.zeros((k, 4, 4), np.int32), np.zeros(k, np.int32), np.zeros(k, np.uint32)
        cb._check(lib.cb200_scan_dev(hnd, ptr, w, h, k, a.ctypes.data, c.ctypes.data, cut.ctypes.data))
        cr = corners(a)
        ch, n1, m1, f1 = (np.zeros((k, info.chunks_per_frame, info.chunk_size), np.uint8), np.zeros(k, np.uint32), np.zeros(k, np.uint32),
                          np.zeros(k, np.uint8))
        cb._check(lib.cb200_extract_decode_fountain_dev(hnd, ptr, w, h, k, cr.ctypes.data, flags, ch.ctypes.data, n1.ctypes.data,
                                                        m1.ctypes.data, f1.ctypes.data))
        return group, ch, n1, m1

    runs, shapes = [], {}
    for i in range(B):
        if runs and tuple(wh[i]) == tuple(wh[runs[-1][-1]]):
            runs[-1].append(i)
        else:
            runs.append([i])
        shapes.setdefault(tuple(wh[i]), []).append(i)
    # the per-shape groups are copied together once, outside the timed region (a caller holding them grouped has them so)
    grouped = {s: torch.cat([d_batch[int(starts[i]):int(starts[i + 1])] for i in g]) for s, g in shapes.items()}

    def per_run():
        ctx.set_ccm(None)
        return [uniform(g) for g in runs]

    def per_shape():
        ctx.set_ccm(None)
        for s, g in shapes.items():
            k, w, h = len(g), s[0], s[1]
            a, c, cut = np.zeros((k, 4, 4), np.int32), np.zeros(k, np.int32), np.zeros(k, np.uint32)
            cb._check(lib.cb200_scan_dev(hnd, grouped[s].data_ptr(), w, h, k, a.ctypes.data, c.ctypes.data, cut.ctypes.data))
            cr = corners(a)
            cb._check(lib.cb200_extract_decode_fountain_dev(hnd, grouped[s].data_ptr(), w, h, k, cr.ctypes.data, flags, chunks.ctypes.data,
                                                            ccount.ctypes.data, cmask.ctypes.data, ff.ctypes.data))

    def run_ragged():
        ctx.set_ccm(None)
        ragged()

    # warm-up of every shape, and the parity check of (a) against (b)
    run_ragged()
    torch.cuda.synchronize()
    assert (count == 4).all(), "the scan did not find four anchors in every sample photograph"
    got = (chunks.copy(), ccount.copy(), cmask.copy())
    ref = per_run()
    same = True
    for g, ch, n1, m1 in ref:
        for j, i in enumerate(g):
            same = same and ccount[i] == n1[j] and cmask[i] == m1[j] and np.array_equal(got[0][i], ch[j])
    per_shape()
    torch.cuda.synchronize()
    ms = {"ragged": [], "per_run": [], "per_shape": []}
    split = []
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(args.rounds):
        for name, fn in (("ragged", run_ragged), ("per_run", per_run), ("per_shape", per_shape)):
            if name == "ragged":
                ctx.set_timing(True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ms[name].append(e0.elapsed_time(e1))
            if name == "ragged":
                scan_t, dec_t = ctx.get_timing(1), ctx.get_timing(0)
                split.append({"blur": scan_t[0], "otsu": scan_t[1], "anchors": scan_t[2], "K1": dec_t[0], "K1x": dec_t[1]})
                ctx.set_timing(False)
    name, power = card()
    best = {k: min(v) for k, v in ms.items()}
    out = {
        "metric": "camera pictures/s through scan + extract + decode of a ragged batch (mode 4C, SHARPEN_IF_NEEDED | CC_FIT)",
        "pictures_per_step": B, "shapes": len(shapes), "shape_changes": sum(1 for i in range(1, B) if tuple(wh[i]) != tuple(wh[i - 1])),
        "input_bytes_per_step": int(starts[-1]), "rounds": args.rounds,
        "ragged": {"pictures_per_s": B / (best["ragged"] * 1e-3), "ms_per_step": ms["ragged"], "calls": 2},
        "per_run": {"pictures_per_s": B / (best["per_run"] * 1e-3), "ms_per_step": ms["per_run"], "calls": 2 * len(runs)},
        "per_shape": {"pictures_per_s": B / (best["per_shape"] * 1e-3), "ms_per_step": ms["per_shape"], "calls": 2 * len(shapes),
                      "note": "reorders the CC_FIT carry: not the CLI's result, timing reference only"},
        "ragged_kernel_ms": {k: float(np.mean([s[k] for s in split])) for k in split[0]},
        "ragged_equals_per_run": bool(same),
        "card": name, "power_limit": power,
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
