"""Cost of decoding groups of pictures of one frame: cb200_scan_extract_decode_chunks_combined_dev next to
cb200_scan_extract_decode_chunks_pictures_dev on the same batch.

    python -m libcimbar_b200.combine_bench [--groups 64] [--per 4] [--iters 10] [--warmup 3]

The batch is mode 4 (4C): groups of `per` pictures of one frame.  All but two groups are synthetic captures (tests/combine_fixtures.py:
the encoder frame with 8 % noise tiles per capture and its own perspective warp); the last two hold the sample photographs' two pairs
of one frame, each pair twice.  Each call is timed with CUDA events around it, after warm-up, the two calls alternating; the result
is the median per call and the combined call's increment, with the card's name and power limit read in the same run.  It also prints
the chunk counts (the device's masks) and the Reed-Solomon block counts per picture and per group on the synthetic groups; the call
reports no block flags, so the block counts come from the CPU oracle on the same pictures, whose chunk masks must equal the device's.
Without a CUDA device it fails."""
import argparse
import json
import os
import sys

import numpy as np

from libcimbar_b200.bench_support import card

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tests"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--groups", type=int, default=64)
    ap.add_argument("--per", type=int, default=4)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("combine_bench: no CUDA device")
    import libcimbar_b200 as cb
    from combine_fixtures import capture
    from ragged_samples import sample

    pics, of = [], []
    real = [("6bit/4_30_f0_627.jpg", "6bit/4_30_f0_177_ccm.jpg"), ("6bit/4_30_f2_246.jpg", "6bit/4_30_f2_734.jpg")]
    synth = a.groups - len(real)
    for g in range(synth):
        for k in range(a.per):
            pics.append(capture(4, 100000 + a.per * g + k))
            of.append(g)
    for r, pair in enumerate(real):
        for k in range(a.per):
            pics.append(sample(pair[k % 2]))
            of.append(synth + r)
    n, m = len(pics), a.groups
    d = [torch.from_numpy(np.ascontiguousarray(p)).cuda() for p in pics]
    ctx = cb.Context(4, max_frames=max(n, m))
    db = ctx.info.data_bytes
    chunks = torch.zeros((n, db), dtype=torch.uint8, device="cuda")
    mask = torch.zeros(n, dtype=torch.int32, device="cuda")
    status = torch.zeros(n, dtype=torch.int32, device="cuda")
    gchunks = torch.zeros((m, db), dtype=torch.uint8, device="cuda")
    gmask = torch.zeros(m, dtype=torch.int32, device="cuda")
    gused = torch.zeros(m, dtype=torch.int32, device="cuda")
    flags = cb.FLAG_SHARPEN_IF_NEEDED
    calls = {
        "pictures": lambda: ctx.scan_extract_decode_chunks_pictures_dev(d, chunks.data_ptr(), mask.data_ptr(), status.data_ptr(), flags=flags),
        "combined": lambda: ctx.scan_extract_decode_chunks_combined_dev(d, of, m, chunks.data_ptr(), mask.data_ptr(), status.data_ptr(),
                                                                        gchunks.data_ptr(), gmask.data_ptr(), gused.data_ptr(), flags=flags),
    }
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    times = {k: [] for k in calls}
    for it in range(a.warmup + a.iters):
        for k, f in calls.items():
            ctx.set_ccm(None)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            f()
            e1.record(stream)
            e1.synchronize()
            if it >= a.warmup:
                times[k].append(e0.elapsed_time(e1))
    ctx.sync()
    full = (1 << ctx.info.chunks_per_frame) - 1
    pm = mask.cpu().numpy().view(np.uint32)
    gm = gmask.cpu().numpy().view(np.uint32)
    pop = np.vectorize(lambda x: bin(int(x)).count("1"))
    synth_pics = synth * a.per
    # blocks: the call reports chunk masks only, so the Reed-Solomon block counts of the same pictures and groups come from the CPU
    # oracle (combine_fixtures: the reference CLI's extraction and decode, the vote, the oracle's RS); its chunk masks are checked
    # against the device's on the way
    from combine_fixtures import cells_record, picture_cells, vote
    per = [picture_cells(4, pics[i], "needed") for i in range(synth_pics)]
    pic_blocks, pic_masks = [], []
    for st, v, _ in per:
        if v is None:
            pic_blocks.append(0); pic_masks.append(0)
            continue
        _, _, mk, ok = cells_record(4, v)
        pic_blocks.append(int(ok.sum())); pic_masks.append(mk)
    grp_blocks, grp_masks = [], []
    for g in range(synth):
        part = [per[i] for i in range(synth_pics) if of[i] == g and per[i][0] in (1, 2)]
        if not part:
            grp_blocks.append(0); grp_masks.append(0)
            continue
        _, _, mk, ok = cells_record(4, vote(np.stack([p[1] for p in part]), np.stack([p[2] for p in part])))
        grp_blocks.append(int(ok.sum())); grp_masks.append(mk)
    oracle_agrees = pic_masks == [int(x) for x in pm[:synth_pics]] and grp_masks == [int(x) for x in gm[:synth]]
    name, power = card()
    med = {k: float(np.median(v)) for k, v in times.items()}
    print(json.dumps({
        "card": name, "power_limit": power, "mode": 4, "pictures": n, "groups": m, "per_group": a.per, "flags": "SHARPEN_IF_NEEDED",
        "pictures_call_ms": round(med["pictures"], 3), "combined_call_ms": round(med["combined"], 3),
        "increment_ms": round(med["combined"] - med["pictures"], 3),
        "spread_ms": {k: [round(min(v), 3), round(max(v), 3)] for k, v in times.items()},
        "synthetic": {"chunks_per_frame": ctx.info.chunks_per_frame,
                      "pictures_full": int((pm[:synth_pics] == full).sum()), "pictures_chunks_mean": float(pop(pm[:synth_pics]).mean()),
                      "groups_full": int((gm[:synth] == full).sum()), "groups_chunks_mean": float(pop(gm[:synth]).mean()),
                      "of_pictures": synth_pics, "of_groups": synth, "blocks_per_frame": ctx.info.rs_blocks,
                      "picture_blocks_mean": float(np.mean(pic_blocks)), "picture_blocks_range": [min(pic_blocks), max(pic_blocks)],
                      "group_blocks_mean": float(np.mean(grp_blocks)), "group_blocks_range": [min(grp_blocks), max(grp_blocks)],
                      "blocks_source": "CPU oracle on the same pictures and flags", "oracle_masks_equal_device": oracle_agrees},
        "real_pairs": {"picture_chunks": pop(pm[synth_pics:]).tolist(), "group_chunks": pop(gm[synth:]).tolist(),
                       "group_used": gused[synth:].cpu().tolist()},
    }))
    ctx.close()


if __name__ == "__main__":
    main()
