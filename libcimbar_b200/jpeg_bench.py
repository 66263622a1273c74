"""JPEG files in, chunks out: the device JPEG decode in front of the camera path.

    python -m libcimbar_b200.jpeg_bench [--rounds R]

The input is ragged_bench's sample photographs as compressed files in host memory (tests/golden/, in glob order; the stand-in for
4_30_f0_big.jpg is ragged_bench's 2.8x upscale encoded by cv2 as a progressive JPEG), replicated to B = 64 and 256 pictures.  Timed
with CUDA events (best of R rounds):
  (a) cb200_jpeg_decode_dev alone: pictures/s, compressed MB/s, and its kernel split (unstuffing, entropy decode, IDCT, upsampling + colour);
  (b) cb200_jpeg_scan_extract_decode_chunks_dev (mode 4C, SHARPEN_IF_NEEDED | CC_FIT) against
  (c) cb200_scan_extract_decode_chunks_ragged_dev on the same pictures already decoded and resident in HBM;
  (d) the latency of one 1280 x 960 progressive picture (cb200_jpeg_decode_dev, n = 1);
  (e) the CPU leg: cv2.imdecode of the same files on all usable host cores.
Prints one JSON line with the card's name and power limit, and whether (b) and (c) returned identical records."""
import argparse
import json
import os
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from libcimbar_b200.bench_support import GLOB, ROOT, card, timed


def load_files():
    import cv2
    out = []
    for n in GLOB:
        if n:
            out.append(open(os.path.join(ROOT, "tests", "golden", "6bit__%s.jpg" % n), "rb").read())
        else:
            img = cv2.imread(os.path.join(ROOT, "tests", "golden", "6bit__4_30_f1_360.jpg"), cv2.IMREAD_COLOR)
            big = cv2.resize(cv2.cvtColor(img, cv2.COLOR_BGR2RGB), None, fx=2.8, fy=2.8)
            ok, buf = cv2.imencode(".jpg", cv2.cvtColor(big, cv2.COLOR_RGB2BGR), [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])
            out.append(buf.tobytes())
    return out


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
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    out = {"metric": "JPEG camera pictures decoded on the device (mode 4C, SHARPEN_IF_NEEDED | CC_FIT)", "rounds": args.rounds}
    ctx = cb.Context(4, max_frames=256)
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    for B in (64, 256):
        files = [pool[i % len(pool)] for i in range(B)]
        mb = sum(len(f) for f in files) / 1e6
        shapes = [cb.jpeg_info(f) for f in files]
        rgb = torch.empty(sum(3 * w * h for w, h in shapes), dtype=torch.uint8, device=dev)
        wh = np.array(shapes, np.int32)
        status = torch.empty(B, dtype=torch.int32, device=dev)
        chunks = [torch.empty(B * ctx.info.data_bytes, dtype=torch.uint8, device=dev) for _ in range(2)]
        masks = [torch.empty(B, dtype=torch.int32, device=dev) for _ in range(2)]
        stats = [torch.empty(B, dtype=torch.int32, device=dev) for _ in range(2)]
        ff = [torch.empty(B, dtype=torch.uint8, device=dev) for _ in range(2)]

        def dec():
            ctx.jpeg_decode_dev(files, rgb.data_ptr(), status.data_ptr())

        def jcam():
            ctx.set_ccm(None)
            ctx.jpeg_scan_extract_decode_chunks_dev(files, chunks[0].data_ptr(), masks[0].data_ptr(), stats[0].data_ptr(), ff[0].data_ptr(), flags)

        def rcam():
            ctx.set_ccm(None)
            ctx.scan_extract_decode_chunks_dev(rgb.data_ptr(), wh, chunks[1].data_ptr(), masks[1].data_ptr(), stats[1].data_ptr(), ff[1].data_ptr(),
                                               flags)

        dec(); jcam(); rcam()                                         # warm-up: every buffer at its size
        torch.cuda.synchronize()
        assert (status.cpu().numpy() == 0).all()
        a_ms, a_all = timed(dec, args.rounds, stream)
        ctx.set_timing(True)
        dec()
        torch.cuda.synchronize()
        split = ctx.get_timing(0)
        ctx.set_timing(False)
        b_ms, _ = timed(jcam, args.rounds, stream)
        c_ms, _ = timed(rcam, args.rounds, stream)
        same = all(torch.equal(x[0], x[1]) for x in (chunks, masks, stats, ff))
        out["B%d" % B] = {
            "compressed_MB": round(mb, 2),
            "a_jpeg_decode": {"ms": a_ms, "pictures_per_s": B / (a_ms * 1e-3), "compressed_MB_per_s": mb / (a_ms * 1e-3),
                              "split_ms": {"unstuff": split[0], "entropy_decode": split[1], "idct": split[2],
                                                                                     "upsample_colour": split[3]}},
            "b_jpeg_camera_call": {"ms": b_ms, "pictures_per_s": B / (b_ms * 1e-3)},
            "c_rgb_camera_call_resident": {"ms": c_ms, "pictures_per_s": B / (c_ms * 1e-3)},
            "b_equals_c": bool(same),
        }
    one = [pool[0]]
    w, h = cb.jpeg_info(one[0])
    rgb1 = torch.empty(3 * w * h, dtype=torch.uint8, device=dev)
    ctx.jpeg_decode_dev(one, rgb1.data_ptr())
    d_ms, _ = timed(lambda: ctx.jpeg_decode_dev(one, rgb1.data_ptr()), max(args.rounds, 5), stream)
    out["d_latency_one_1280x960_progressive_ms"] = d_ms
    # (e) the CPU leg on the B = 64 files
    files = [pool[i % len(pool)] for i in range(64)]
    cores = len(os.sched_getaffinity(0))
    cv2.setNumThreads(1)
    with ThreadPoolExecutor(cores) as ex:
        list(ex.map(lambda f: cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_COLOR), files))
        t0 = time.perf_counter()
        list(ex.map(lambda f: cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_COLOR), files))
        e_s = time.perf_counter() - t0
    out["e_cpu_imdecode_all_cores"] = {"cores": cores, "pictures": 64, "ms": e_s * 1e3, "pictures_per_s": 64 / e_s}
    name, power = card()
    out["card"], out["power_limit"] = name, power
    ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
