"""Per-frame sharpen choice on one GPU: a batch of synthetic frames in HBM of which a fixed, seeded half is decoded with
should_preprocess = true (cb200_decode_chunks_sharpen_dev, the batch the reference CLI's --preprocess -1 makes of a mixed camera
batch), next to the same batch decoded plain and sharpened throughout.

    python -m libcimbar_b200.sharpen_bench [--frames 10000] [--steps 20] [--warmup 5] [--mode 68]

The three runs take turns for two rounds of `steps` steps each, so drift of a shared host or of the clocks hits all three alike.
Prints one JSON line: frames/s, ms per step and the K1 / K1x times (CUDA events recorded by the library around its launches) of
each run, the card's name and power limit, and whether every decoded chunk equals the payload."""
import argparse
import json

import numpy as np

import libcimbar_b200 as cb


def device_card():
    """the card as NVML gives it: name, enforced power limit in W as a number, maximum SM clock"""
    import torch
    out = {"name": torch.cuda.get_device_name(), "power_limit_w": None}
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(torch.cuda.current_device())
        out["power_limit_w"] = pynvml.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0
        out["sm_max_mhz"] = pynvml.nvmlDeviceGetMaxClockInfo(h, pynvml.NVML_CLOCK_SM)
    except Exception:
        pass
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=10000)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--mode", type=int, default=68, choices=[68, 67, 66, 4, 8])
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("sharpen_bench: no CUDA device (the decode path has no CPU fallback)")
    dev = torch.device("cuda", 0)
    B, K, W = args.frames, max(args.steps, 1), max(args.warmup, 1)
    ctx = cb.Context(args.mode, max_frames=B)
    info = ctx.info
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(stream)
    ctx.set_stream(stream.cuda_stream)

    # synthetic input on the device: payload -> RS -> interleaved cells -> RGB8 frames (as bench.py's clean workload)
    g = torch.Generator(device=dev)
    g.manual_seed(0xC1B4)
    payload = torch.randint(0, 256, (B, info.data_bytes), dtype=torch.uint8, device=dev, generator=g)
    cells = torch.empty((B, info.total_cells), dtype=torch.uint8, device=dev)
    ctx.encode_cells_dev(payload.data_ptr(), B, cells.data_ptr())
    frames = torch.empty((B, info.image_size_y, info.image_size_x, 3), dtype=torch.uint8, device=dev)
    ctx.render_frames_dev(cells.data_ptr(), B, frames.data_ptr())
    del cells
    chunks = torch.empty((B, info.data_bytes), dtype=torch.uint8, device=dev)
    mask = torch.empty(B, dtype=torch.int32, device=dev)
    fflags = torch.empty(B, dtype=torch.uint8, device=dev)
    sel = np.zeros(B, np.uint8)
    sel[np.random.default_rng(0x5A).permutation(B)[:B // 2]] = 1

    runs = {"mixed": (0, sel), "plain": (0, None), "sharpen": (cb.FLAG_SHARPEN, None)}
    full = (1 << info.chunks_per_frame) - 1

    def decode(flags, s):
        ctx.decode_chunks_dev(frames.data_ptr(), B, chunks.data_ptr(), mask.data_ptr(), fflags.data_ptr(), flags=flags, sharpen=s)

    acc = {k: {"ms": [], "k1": [], "k1x": [], "exact": True} for k in runs}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ctx.set_timing(True)
    for _ in range(2):
        for name, (flags, s) in runs.items():
            for _ in range(W):
                decode(flags, s)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(K):
                decode(flags, s)
            e1.record()
            torch.cuda.synchronize()
            acc[name]["ms"].append(e0.elapsed_time(e1) / K)
            per = [ctx.get_timing(i) for i in range(min(K, 64))]
            acc[name]["k1"] += [r[0] for r in per]
            acc[name]["k1x"] += [r[1] for r in per]
            acc[name]["exact"] &= bool((mask == full).all().item()) and bool(torch.equal(chunks, payload))
    ctx.set_timing(False)

    out = {"metric": "decoded cimbar frames/sec with a per-frame sharpen choice (mode %d)" % args.mode, "unit": "frames/s",
           "frames_per_step": B, "steps_per_round": K, "rounds": 2, "warmup": W,
           "pattern": "seeded permutation: %d of %d frames sharpened" % (int(sel.sum()), B), "card": device_card()}
    for name, a in acc.items():
        ms = sum(a["ms"]) / len(a["ms"])
        out[name] = {"value": B / (ms * 1e-3), "ms_per_step": ms, "ms_per_step_rounds": a["ms"],
                     "k1_ms": sum(a["k1"]) / len(a["k1"]), "k1x_ms": sum(a["k1x"]) / len(a["k1x"]),
                     "parity": "all chunks == payload" if a["exact"] else "MISMATCH"}
    out["value"] = out["mixed"]["value"]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
