"""PNG files in, pictures and chunks out: the device PNG decode in front of the camera and frame paths.

    python -m libcimbar_b200.png_bench [--rounds R]

Input: the five golden PNG frames (tests/golden/) and cv2-written RGB8 PNG copies of the golden sample photographs, replicated to
B = 256 and 1024 files in host memory.  Timed with CUDA events (best of R rounds):
  (a) cb200_png_decode_dev alone: pictures/s, compressed MB/s and its kernel split (CRC + inflate, unfilter, expand);
  (b) the frame files (mode B: tr_0..3, mode 4C: the 4-colour fountain frame) through cb200_png_decode_dev + cb200_decode_chunks_dev,
      and whether the records equal cb200_decode_chunks_dev on cv2's frames;
  (c) cv2.imdecode of the (a) files on all usable host cores;
  (d) the latency of one file (b__tr_1.png, 1024 x 1024 RGB8 with the Sub filter; cb200_png_decode_dev, n = 1).
Prints one JSON line with the card's name and power limit."""
import argparse
import glob
import json
import os
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from libcimbar_b200.ragged_bench import ROOT, card

GOLDEN = os.path.join(ROOT, "tests", "golden")
FRAMES = {68: ["b__tr_0.png", "b__tr_1.png", "b__tr_2.png", "b__tr_3.png"], 4: ["6bit__4color_ecc30_fountain_0.png"]}


def load_files():
    import cv2
    out = [open(os.path.join(GOLDEN, n), "rb").read() for n in FRAMES[68] + FRAMES[4]]
    for f in sorted(glob.glob(os.path.join(GOLDEN, "*.jpg"))):
        ok, buf = cv2.imencode(".png", cv2.imread(f, cv2.IMREAD_COLOR))
        out.append(buf.tobytes())
    return out


def timed(fn, rounds, stream):
    """best and all of `rounds` runs of fn, CUDA events on the context's stream around it (host work inside the call included)"""
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms = []
    for _ in range(rounds):
        torch.cuda.synchronize()
        e0.record(stream)
        fn()
        e1.record(stream)
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return min(ms), ms


def rgb_of(data):
    import cv2
    return cv2.cvtColor(cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_COLOR), cv2.COLOR_BGR2RGB)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import cv2
    import torch
    import libcimbar_b200 as cb
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    pool = load_files()
    out = {"metric": "PNG files decoded on the device", "rounds": args.rounds, "pool": len(pool)}
    ctx = cb.Context(68, max_frames=1024)
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    for B in (256, 1024):
        files = [pool[i % len(pool)] for i in range(B)]
        mb = sum(len(f) for f in files) / 1e6
        shapes = [cb.png_info(f) for f in files]
        rgb = torch.empty(sum(3 * w * h for w, h in shapes), dtype=torch.uint8, device=dev)
        status = torch.empty(B, dtype=torch.int32, device=dev)

        def dec():
            ctx.png_decode_dev(files, rgb.data_ptr(), status.data_ptr())

        dec()                                                          # warm-up: every buffer at its size
        torch.cuda.synchronize()
        assert (status.cpu().numpy() == 0).all()
        a_ms, a_all = timed(dec, args.rounds, stream)
        ctx.set_timing(True)
        dec()
        torch.cuda.synchronize()
        split = ctx.get_timing(0)
        ctx.set_timing(False)
        out["a_B%d" % B] = {"compressed_MB": round(mb, 2), "ms": a_ms, "all_ms": a_all, "pictures_per_s": B / (a_ms * 1e-3),
                            "compressed_MB_per_s": mb / (a_ms * 1e-3),
                            "split_ms": {"crc_inflate": split[0], "unfilter": split[1], "expand": split[2]}}
        del rgb
    # (b) the frame path
    for mode_val, names in FRAMES.items():
        fctx = cb.Context(mode_val, max_frames=256)
        fctx.set_stream(stream.cuda_stream)
        one = [open(os.path.join(GOLDEN, n), "rb").read() for n in names]
        files = [one[i % len(one)] for i in range(256)]
        n = len(files)
        w, h = cb.png_info(files[0])
        d_rgb = torch.empty(n * 3 * w * h, dtype=torch.uint8, device=dev)
        ref = torch.from_numpy(np.stack([rgb_of(f) for f in files]).reshape(-1)).to(dev)
        chunks = [torch.empty(n * fctx.info.data_bytes, dtype=torch.uint8, device=dev) for _ in range(2)]
        masks = [torch.empty(n, dtype=torch.int32, device=dev) for _ in range(2)]

        def frames():
            fctx.png_decode_dev(files, d_rgb.data_ptr())
            fctx.decode_chunks_dev(d_rgb.data_ptr(), n, chunks[0].data_ptr(), masks[0].data_ptr())

        frames()
        fctx.decode_chunks_dev(ref.data_ptr(), n, chunks[1].data_ptr(), masks[1].data_ptr())
        torch.cuda.synchronize()
        same = torch.equal(chunks[0], chunks[1]) and torch.equal(masks[0], masks[1])
        b_ms, _ = timed(frames, args.rounds, stream)
        r_ms, _ = timed(lambda: fctx.decode_chunks_dev(ref.data_ptr(), n, chunks[1].data_ptr(), masks[1].data_ptr()), args.rounds, stream)
        out["b_frames_mode%d" % mode_val] = {"frames": n, "ms": b_ms, "frames_per_s": n / (b_ms * 1e-3),
                                              "decode_chunks_only_ms": r_ms, "records_equal_rgb_call": bool(same)}
        fctx.close()
    # (c) the CPU leg on the B = 256 files
    files = [pool[i % len(pool)] for i in range(256)]
    cores = len(os.sched_getaffinity(0))
    cv2.setNumThreads(1)
    with ThreadPoolExecutor(cores) as ex:
        list(ex.map(lambda f: cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_COLOR), files))
        t0 = time.perf_counter()
        list(ex.map(lambda f: cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_COLOR), files))
        c_s = time.perf_counter() - t0
    out["c_cpu_imdecode_all_cores"] = {"cores": cores, "pictures": 256, "ms": c_s * 1e3, "pictures_per_s": 256 / c_s}
    # (d) one file
    one = [open(os.path.join(GOLDEN, "b__tr_1.png"), "rb").read()]
    w, h = cb.png_info(one[0])
    rgb1 = torch.empty(3 * w * h, dtype=torch.uint8, device=dev)
    ctx.png_decode_dev(one, rgb1.data_ptr())
    d_ms, _ = timed(lambda: ctx.png_decode_dev(one, rgb1.data_ptr()), max(args.rounds, 5), stream)
    out["d_latency_one_b__tr_1_ms"] = d_ms
    name, power = card()
    out["card"], out["power_limit"] = name, power
    ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
