"""Cost of finding the pictures of one frame within each receiver of a receivers batch: cb200_scan_extract_decode_chunks_grouped_receivers_dev
next to the receivers call and to one grouped call per receiver (the CCM set on the host before each), on the same batch.

    python -m libcimbar_b200.grouped_receivers_bench [--receivers 16 64] [--frames 4] [--per 4] [--iters 10] [--warmup 3]

The batch is mode 4 (4C): each receiver holds `per` synthetic captures (tests/group_fixtures.py: 8 % noise tiles and a perspective warp
each) of each of `frames` frames, the oracle's renderings of seeded payloads.  Receivers 2k and 2k + 1 receive the same file, so they
hold captures of the same frames.  The batch is in a seeded order, and every receiver has its own active entry state.  The three ways
alternate, each timed with CUDA events around it after warm-up, and the result is the median per way.  A separate run under
torch.profiler gives the pairing and assignment kernels' own times for the grouped receivers call and for the per-receiver calls.
The groups the call finds must be exactly the planted (receiver, frame) pairs.  The card's name and power limit are read in the same
run.  Without a CUDA device it fails."""
import argparse
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tests"))

from libcimbar_b200.bench_support import card, entry_states  # noqa: E402


def batch(receivers, frames, per):
    from group_fixtures import capture_of, seeded_frame
    pics, of, frame_of = [], [], []
    rendered = {}
    for r in range(receivers):
        for f in range(frames):
            key = (r // 2) * frames + f                            # receivers 2k and 2k + 1 show the same frames
            if key not in rendered:
                rendered[key] = seeded_frame(4, 5000 + key)
            for s in range(per):
                pics.append(capture_of(4, rendered[key], [r, f, s]))
                of.append(r)
                frame_of.append(key)
    order = np.random.default_rng(receivers).permutation(len(pics))
    return [pics[i] for i in order], np.array([of[i] for i in order], np.int32), [frame_of[i] for i in order]


def bench(cb, torch, receivers, frames, per, iters, warmup):
    pics, of, frame_of = batch(receivers, frames, per)
    n, slots = len(pics), len(pics) // 2
    d = [torch.from_numpy(np.ascontiguousarray(p)).cuda() for p in pics]
    ccms = entry_states(receivers)
    states = cb.receiver_states(ccms)
    ctx = cb.Context(4, max_frames=n)
    db = ctx.info.data_bytes
    z = lambda *shape, dt=torch.int32: torch.zeros(shape, dtype=dt, device="cuda")
    chunks, mask, status = z(n, db, dt=torch.uint8), z(n), z(n)
    gchunks, gmask, gused, gof, count, grec = z(slots, db, dt=torch.uint8), z(slots), z(slots), z(n), z(1), z(slots)
    flags = cb.FLAG_SHARPEN_IF_NEEDED                              # no CC flag: the states pass through, every iteration is alike
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    mine = [np.flatnonzero(of == r) for r in range(receivers)]

    def grouped_receivers():
        ctx.scan_extract_decode_chunks_grouped_receivers_dev(d, of, states, chunks.data_ptr(), mask.data_ptr(), status.data_ptr(),
                                                             gof.data_ptr(), count.data_ptr(), gchunks.data_ptr(), gmask.data_ptr(),
                                                             gused.data_ptr(), grec.data_ptr(), flags=flags)

    def per_receiver():
        for r in range(receivers):
            ctx.set_ccm(ccms[r])
            ctx.scan_extract_decode_chunks_grouped_dev([d[i] for i in mine[r]], chunks.data_ptr(), mask.data_ptr(), status.data_ptr(),
                                                       gof.data_ptr(), count.data_ptr(), gchunks.data_ptr(), gmask.data_ptr(),
                                                       gused.data_ptr(), flags=flags)

    grouped_receivers()
    ctx.sync()
    g, m, rec, st = gof.cpu().numpy().copy(), int(count[0]), grec.cpu().numpy(), status.cpu().numpy()
    # the planted (receiver, frame) pairs: one group each, and no group with pictures of two frames or two receivers
    found = {}
    for i in range(n):
        if g[i] >= 0:
            found.setdefault((int(of[i]), frame_of[i]), set()).add(int(g[i]))
    planted = m == receivers * frames and len(found) == m and all(len(v) == 1 for v in found.values()) and \
        len(set().union(*found.values())) == m and all(int(rec[next(iter(v))]) == r for (r, _), v in found.items())
    assert planted, f"{m} groups for {receivers * frames} planted (receiver, frame) pairs"
    calls = {
        "receivers": lambda: ctx.scan_extract_decode_chunks_receivers_dev(d, of, states, chunks.data_ptr(), mask.data_ptr(),
                                                                          status.data_ptr(), flags=flags),
        "grouped_receivers": grouped_receivers,
        "grouped_per_receiver": per_receiver,
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
    # the pairing and assignment kernels' own times, in runs of their own under the profiler: per call, and per batch for the
    # per-receiver way (the sum over its calls)
    from torch.profiler import ProfilerActivity, profile
    kern = {}
    for way, fn in (("grouped_receivers", grouped_receivers), ("grouped_per_receiver", per_receiver)):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(iters):
                fn()
            ctx.sync()
        kern[way] = {}
        for e in prof.key_averages():
            for name in ("k_pair_match", "k_assign_groups"):
                if name in e.key:
                    kern[way][name] = round(e.device_time_total / iters / 1000.0, 4)
    ctx.close()
    med = {k: float(np.median(v)) for k, v in times.items()}
    sizes = np.bincount(of, minlength=receivers)
    return {"pictures": n, "receivers": receivers, "frames_per_receiver": frames, "per_frame": per, "groups_found": m,
            "planted_pairs_found": bool(planted), "pictures_not_extracted": int((~np.isin(st, (1, 2))).sum()),
            **{f"{k}_ms": round(v, 3) for k, v in med.items()},
            "grouped_receivers_minus_receivers_ms": round(med["grouped_receivers"] - med["receivers"], 3),
            "spread_ms": {k: [round(min(v), 3), round(max(v), 3)] for k, v in times.items()},
            "kernel_ms_per_batch": kern, "same_receiver_pairs": int((sizes * (sizes - 1) // 2).sum()), "all_pairs": n * (n - 1) // 2}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--receivers", type=int, nargs="+", default=[16, 64])
    ap.add_argument("--frames", type=int, default=4)
    ap.add_argument("--per", type=int, default=4)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("grouped_receivers_bench: no CUDA device")
    import libcimbar_b200 as cb
    name, power = card()
    runs = [bench(cb, torch, r, a.frames, a.per, a.iters, a.warmup) for r in a.receivers]
    print(json.dumps({"card": name, "power_limit": power, "mode": 4, "flags": "SHARPEN_IF_NEEDED", "runs": runs}))


if __name__ == "__main__":
    main()
