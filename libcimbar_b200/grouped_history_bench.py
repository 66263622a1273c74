"""Cost and payoff of grouping across calls: cb200_scan_extract_decode_chunks_grouped_history_dev next to the grouped call and the
pictures call, in a camera loop.

    python -m libcimbar_b200.grouped_history_bench [--frames 32] [--per 3] [--batches 1 4 16] [--capacity 32] [--passes 3]

The loop is mode 4 (4C): `per` synthetic captures (tests/group_fixtures.py: 8 % noise tiles and a perspective warp each) of each of
`frames` distinct frames, the oracle's renderings of seeded payloads, in sender order (a frame's captures one after another), handed
over in batches of b pictures.  Each call kind runs the whole loop on its own context, `passes` times (the history reset before each
pass); every call is timed with CUDA events, the first pass is warm-up, and the result is the median per call.  A frame is recovered
when a record of it (a picture's own, or a group record whose batch members show it) has every chunk; the counts come from the first
pass and are deterministic.  A separate pass under torch.profiler gives the history call's kernels their own times.  The card's name
and power limit are read in the same run.  Without a CUDA device it fails."""
import argparse
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tests"))

from libcimbar_b200.bench_support import card  # noqa: E402

KINDS = ("history", "grouped", "pictures")
KERNELS = ("k_pair_match", "k_assign_groups", "k_history_groups", "k_history_keep", "k_history_copy", "k_combine")


def loop(cb, torch, d, frame_of, b, capacity, passes):
    n_all = len(d)
    batches = [list(range(s, min(s + b, n_all))) for s in range(0, n_all, b)]
    flags = cb.FLAG_SHARPEN_IF_NEEDED
    out, times, recovered = {}, {}, {}
    for kind in KINDS:
        ctx = cb.Context(4, max_frames=b)
        hist = ctx.group_history(capacity) if kind == "history" else None
        db, full = ctx.info.data_bytes, (1 << ctx.info.chunks_per_frame) - 1
        z = lambda *shape, dt=torch.int32: torch.zeros(shape, dtype=dt, device="cuda")
        chunks, mask, status = z(b, db, dt=torch.uint8), z(b), z(b)
        gchunks, gmask, gused, gof, count = z(b, db, dt=torch.uint8), z(b), z(b), z(b), z(1)
        stream = torch.cuda.Stream()
        ctx.set_stream(stream.cuda_stream)
        torch.cuda.synchronize()

        def call(idx):
            pics = [d[i] for i in idx]
            if kind == "history":
                ctx.scan_extract_decode_chunks_grouped_history_dev(pics, hist, chunks.data_ptr(), mask.data_ptr(), status.data_ptr(),
                                                                   gof.data_ptr(), count.data_ptr(), gchunks.data_ptr(), gmask.data_ptr(),
                                                                   gused.data_ptr(), flags=flags)
            elif kind == "grouped":
                ctx.scan_extract_decode_chunks_grouped_dev(pics, chunks.data_ptr(), mask.data_ptr(), status.data_ptr(), gof.data_ptr(),
                                                           count.data_ptr(), gchunks.data_ptr(), gmask.data_ptr(), gused.data_ptr(),
                                                           flags=flags)
            else:
                ctx.scan_extract_decode_chunks_pictures_dev(pics, chunks.data_ptr(), mask.data_ptr(), status.data_ptr(), flags=flags)

        # the first pass: warm-up, and the frames recovered
        got, ms = set(), []
        for idx in batches:
            call(idx)
            ctx.sync()
            m, groups, gm = mask[:len(idx)].cpu().numpy(), gof[:len(idx)].cpu().numpy(), gmask.cpu().numpy()
            got |= {frame_of[i] for i, mm in zip(idx, m) if int(mm) == full}
            if kind != "pictures" and len(idx) >= (1 if kind == "history" else 2):
                got |= {frame_of[i] for i, g in zip(idx, groups) if g >= 0 and int(gm[g]) == full}
        # timed passes: every call between two events on the context's stream
        for p in range(passes):
            if hist is not None:
                hist.reset()
            for idx in batches:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                call(idx)
                e1.record(stream)
                e1.synchronize()
                ms.append(e0.elapsed_time(e1))
        if kind == "history":
            from torch.profiler import ProfilerActivity, profile
            hist.reset()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for idx in batches:
                    call(idx)
                ctx.sync()
            kern = {}
            for e in prof.key_averages():
                for name in KERNELS:
                    if name in e.key:
                        kern[name] = round(e.device_time_total / max(1, e.count) / 1000.0, 4)
            out["history_kernel_ms"] = kern
            hist.close()
        ctx.close()
        times[kind] = ms
        recovered[kind] = len(got)
    med = {k: float(np.median(v)) for k, v in times.items()}
    return {"batch": b, "calls_per_pass": len(batches), **{f"{k}_call_ms": round(v, 3) for k, v in med.items()},
            "spread_ms": {k: [round(min(v), 3), round(max(v), 3)] for k, v in times.items()},
            "frames_recovered": recovered, **out}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=32)
    ap.add_argument("--per", type=int, default=3)
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 4, 16])
    ap.add_argument("--capacity", type=int, default=32)
    ap.add_argument("--passes", type=int, default=3)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("grouped_history_bench: no CUDA device")
    import libcimbar_b200 as cb
    from group_fixtures import frame_captures
    name, power = card()
    pics, frame_of = frame_captures(4, [a.per] * a.frames, seed=2026)
    d = [torch.from_numpy(np.ascontiguousarray(p)).cuda() for p in pics]
    runs = [loop(cb, torch, d, frame_of, b, a.capacity, a.passes) for b in a.batches]
    print(json.dumps({"card": name, "power_limit": power, "mode": 4, "flags": "SHARPEN_IF_NEEDED", "frames": a.frames, "per_frame": a.per,
                      "capacity": a.capacity, "runs": runs}))


if __name__ == "__main__":
    main()
