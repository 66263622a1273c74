"""Cost of finding the pictures of one frame on the device: cb200_scan_extract_decode_chunks_grouped_dev next to the combined call given
the same groups and the pictures call, on the same batch.

    python -m libcimbar_b200.group_bench [--frames 64 256] [--per 4] [--iters 10] [--warmup 3]

The batch is mode 4 (4C): `per` synthetic captures (tests/group_fixtures.py: 8 % noise tiles and a perspective warp each) of each of
`frames` distinct frames, the oracle's renderings of seeded payloads, in a seeded order.  combine_bench's batch shows one encoder frame,
which the grouping would put into groups of 16; distinct frames are what a camera loop sees.  The three calls alternate, each timed
with CUDA events around it after warm-up, and the result is the median per call.  A separate run under torch.profiler gives the
pairing and assignment kernels' own times.  The groups the call finds must be exactly the planted frames.  The card's name and power
limit are read in the same run.  Without a CUDA device it fails."""
import argparse
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tests"))

from libcimbar_b200.bench_support import card  # noqa: E402


def bench(cb, torch, frames, per, iters, warmup):
    from group_fixtures import frame_captures
    pics, frame_of = frame_captures(4, [per] * frames, seed=2024)
    order = np.random.default_rng(frames).permutation(len(pics))
    pics, frame_of = [pics[i] for i in order], [frame_of[i] for i in order]
    n, slots = len(pics), len(pics) // 2
    d = [torch.from_numpy(np.ascontiguousarray(p)).cuda() for p in pics]
    ctx = cb.Context(4, max_frames=n)
    db = ctx.info.data_bytes
    z = lambda *shape, dt=torch.int32: torch.zeros(shape, dtype=dt, device="cuda")
    chunks, mask, status = z(n, db, dt=torch.uint8), z(n), z(n)
    gchunks, gmask, gused, gof, count = z(slots, db, dt=torch.uint8), z(slots), z(slots), z(n), z(1)
    flags = cb.FLAG_SHARPEN_IF_NEEDED
    grouped = lambda: ctx.scan_extract_decode_chunks_grouped_dev(d, chunks.data_ptr(), mask.data_ptr(), status.data_ptr(), gof.data_ptr(),
                                                                 count.data_ptr(), gchunks.data_ptr(), gmask.data_ptr(), gused.data_ptr(),
                                                                 flags=flags)
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    grouped()
    ctx.sync()
    of, m, st = gof.cpu().numpy().copy(), int(count[0]), status.cpu().numpy()
    # the planted frames: one group per frame, and no group with pictures of two frames.  A picture may stay alone (-1): one that
    # failed extraction, or one whose cells agree with no other picture's
    part = np.isin(st, (1, 2))
    found = [{int(of[i]) for i in range(n) if frame_of[i] == f} - {-1} for f in range(frames)]
    planted = m == frames and all(len(g) == 1 for g in found) and len(set().union(*found)) == frames
    assert planted, f"{m} groups for {frames} planted frames: {[sorted(g) for g in found if len(g) != 1]}"
    calls = {
        "grouped": grouped,
        "combined": lambda: ctx.scan_extract_decode_chunks_combined_dev(d, of, m, chunks.data_ptr(), mask.data_ptr(), status.data_ptr(),
                                                                        gchunks.data_ptr(), gmask.data_ptr(), gused.data_ptr(), flags=flags),
        "pictures": lambda: ctx.scan_extract_decode_chunks_pictures_dev(d, chunks.data_ptr(), mask.data_ptr(), status.data_ptr(), flags=flags),
    }
    times = {k: [] for k in calls}
    for it in range(warmup + iters):
        for k, f in calls.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            f()
            e1.record(stream)
            e1.synchronize()
            if it >= warmup:
                times[k].append(e0.elapsed_time(e1))
    # the new kernels' own times, in a run of their own under the profiler
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            grouped()
        ctx.sync()
    kern = {}
    for e in prof.key_averages():
        for name in ("k_pair_match", "k_assign_groups"):
            if name in e.key:
                kern[name] = round(e.device_time_total / max(1, e.count) / 1000.0, 4)
    ctx.close()
    med = {k: float(np.median(v)) for k, v in times.items()}
    return {"pictures": n, "frames": frames, "per_frame": per, "groups_found": m, "planted_frames_found": bool(planted),
            "pictures_not_extracted": int((~part).sum()), "extracted_pictures_alone": int((part & (of < 0)).sum()),
            **{f"{k}_call_ms": round(v, 3) for k, v in med.items()},
            "grouped_minus_combined_ms": round(med["grouped"] - med["combined"], 3),
            "spread_ms": {k: [round(min(v), 3), round(max(v), 3)] for k, v in times.items()},
            "kernel_ms": kern, "pairs": n * (n - 1) // 2}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, nargs="+", default=[64, 256])
    ap.add_argument("--per", type=int, default=4)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("group_bench: no CUDA device")
    import libcimbar_b200 as cb
    name, power = card()
    runs = [bench(cb, torch, f, a.per, a.iters, a.warmup) for f in a.frames]
    print(json.dumps({"card": name, "power_limit": power, "mode": 4, "flags": "SHARPEN_IF_NEEDED", "runs": runs}))


if __name__ == "__main__":
    main()
