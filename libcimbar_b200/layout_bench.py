"""Camera pictures in the caller's layout: what taking BGR, RGBA, BGRA and planar pictures directly saves over converting them.

    python -m libcimbar_b200.layout_bench [--pictures B] [--rounds R]

One step = B camera pictures at ragged_bench's batch shapes (the reference's samples/6bit/*.jpg from tests/golden/, in glob order,
with the 2.8x upscale of 4_30_f1_360.jpg standing in for the largest one, replicated), one tensor per picture, resident in HBM,
decoded in mode 4C with SHARPEN_IF_NEEDED | CC_FIT (the CLI's defaults) by the enqueue-only camera calls.  For each layout:
  (a) `convert`:  torch converts every picture to packed RGB into one batch buffer (one copy kernel per picture: a channel flip,
                  the alpha dropped, or the planes interleaved), then cb200_scan_extract_decode_chunks_ragged_dev;
  (b) `direct`:   cb200_scan_extract_decode_chunks_pictures_dev on the pictures as they are.
And for packed RGB pictures in one buffer: the existing ragged call against the new call given one descriptor per picture.
The C calls get their host inputs prebuilt (wh, the descriptor arrays), as a C caller holds them; `rgb/pictures_python` times the
Python wrapper instead, which builds the descriptors from the tensors inside the step (its host time shows in the step).
Each variant is timed with CUDA events around its step (ms, from the first enqueue until the stream has run it), after a warm-up,
in R rounds that alternate all variants; every (b) is checked to give (a)'s chunks, masks and statuses.  Prints one JSON line
with every round's time, the median and the spread per variant, the card's name and its power limit."""
import argparse
import ctypes as C
import json

import numpy as np

from libcimbar_b200.bench_support import card, load_pictures

LAYOUTS = ["bgr", "rgba", "bgra", "planar"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pictures", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=7)
    args = ap.parse_args()
    import torch
    import libcimbar_b200 as cb
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    B = args.pictures
    pool = load_pictures()
    pics = [pool[i % len(pool)] for i in range(B)]
    wh = np.array([(p.shape[1], p.shape[0]) for p in pics], np.int32)
    starts = np.cumsum([0] + [p.nbytes for p in pics])
    packed = torch.cat([torch.from_numpy(p.reshape(-1)) for p in pics]).to(dev)
    views = [packed[int(starts[i]):int(starts[i + 1])].view(p.shape) for i, p in enumerate(pics)]
    inputs = {
        "bgr": [v.flip(2).contiguous() for v in views],
        "rgba": [torch.cat([v, torch.full(v.shape[:2] + (1,), 255, dtype=torch.uint8, device=dev)], 2) for v in views],
        "bgra": [torch.cat([v.flip(2), torch.full(v.shape[:2] + (1,), 255, dtype=torch.uint8, device=dev)], 2) for v in views],
        "planar": [v.permute(2, 0, 1).contiguous() for v in views],
    }
    order = {"bgr": "bgr", "rgba": "rgb", "bgra": "bgr", "planar": "rgb"}
    convert = {"bgr": lambda t: t.flip(2), "rgba": lambda t: t[:, :, :3], "bgra": lambda t: t[:, :, :3].flip(2),
               "planar": lambda t: t.permute(1, 2, 0)}
    staging = torch.empty_like(packed)
    stage_views = [staging[int(starts[i]):int(starts[i + 1])].view(p.shape) for i, p in enumerate(pics)]
    stream = torch.cuda.Stream()                                    # the context's stream: every step and its events run on it
    ctx = cb.Context(4, max_frames=B)
    ctx.set_stream(stream.cuda_stream)
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    db = ctx.info.data_bytes
    outs = {}

    def buffers(name):
        if name not in outs:
            outs[name] = (torch.zeros(B * db, dtype=torch.uint8, device=dev), torch.zeros(B, dtype=torch.int32, device=dev),
                          torch.zeros(B, dtype=torch.int32, device=dev))
        return outs[name]

    def ragged(name, base):
        ch, mk, st = buffers(name)
        ctx.set_ccm(None)
        ctx.scan_extract_decode_chunks_dev(base, wh, ch.data_ptr(), mk.data_ptr(), st.data_ptr(), flags=flags)

    descs = {}

    def direct(name, tensors, o):
        ch, mk, st = buffers(name)
        if name not in descs:
            descs[name] = (cb.Picture * B)(*[cb.picture(t, o) for t in tensors])
        ctx.set_ccm(None)
        cb._check(ctx.lib.cb200_scan_extract_decode_chunks_pictures_dev(ctx._h, C.cast(descs[name], C.c_void_p), B, flags, ch.data_ptr(),
                                                                         mk.data_ptr(), None, st.data_ptr()))

    def python_wrapper(name, tensors, o):
        ch, mk, st = buffers(name)
        ctx.set_ccm(None)
        ctx.scan_extract_decode_chunks_pictures_dev(tensors, ch.data_ptr(), mk.data_ptr(), st.data_ptr(), flags=flags, order=o)

    def conv_step(lay):
        def step():
            for src, dst in zip(inputs[lay], stage_views):
                dst.copy_(convert[lay](src))
            ragged(lay + "/convert", staging.data_ptr())
        return step

    variants = {"rgb/ragged": lambda: ragged("rgb/ragged", packed.data_ptr()),
                "rgb/pictures": lambda: direct("rgb/pictures", views, "rgb"),
                "rgb/pictures_python": lambda: python_wrapper("rgb/pictures_python", views, "rgb")}
    for lay in LAYOUTS:
        variants[lay + "/convert"] = conv_step(lay)
        variants[lay + "/direct"] = (lambda lay=lay: direct(lay + "/direct", inputs[lay], order[lay]))
    torch.cuda.synchronize()
    with torch.cuda.stream(stream):
        for fn in variants.values():                                # warm-up: every buffer at its size, every kernel loaded
            fn()
    torch.cuda.synchronize()
    ref = [t.cpu() for t in outs["rgb/ragged"]]
    equal = {k: all(torch.equal(a.cpu(), b) for a, b in zip(v, ref)) for k, v in outs.items()}
    ms = {k: [] for k in variants}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    names = list(variants)
    with torch.cuda.stream(stream):
        for r in range(args.rounds):
            for k in (names if r % 2 == 0 else names[::-1]):        # alternate the order from round to round
                torch.cuda.synchronize()
                e0.record(stream)
                variants[k]()
                e1.record(stream)
                torch.cuda.synchronize()
                ms[k].append(e0.elapsed_time(e1))
    name, power = card()
    summary = {k: {"median_ms": float(np.median(v)), "min_ms": float(np.min(v)), "max_ms": float(np.max(v)), "ms": v} for k, v in ms.items()}
    out = {
        "metric": "ms per step of B camera pictures through scan + extract + decode (mode 4C, SHARPEN_IF_NEEDED | CC_FIT), by input layout",
        "pictures_per_step": B, "rgb_bytes_per_step": int(starts[-1]), "rounds": args.rounds,
        "variants": summary,
        "direct_minus_convert_median_ms": {lay: summary[lay + "/direct"]["median_ms"] - summary[lay + "/convert"]["median_ms"] for lay in LAYOUTS},
        "pictures_minus_ragged_median_ms": summary["rgb/pictures"]["median_ms"] - summary["rgb/ragged"]["median_ms"],
        "outputs_equal_the_ragged_call": equal,
        "card": name, "power_limit": power,
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
