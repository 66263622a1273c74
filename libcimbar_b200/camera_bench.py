"""The camera path: photographs in, fountain chunks out (SURVEY.md 8f-2: the extractor in front of the decode).

    python bench.py --camera [--frames B] [--steps K] [--warmup W]

One step = B camera pictures (the reference's own sample photographs of mode-4C codes, 960 x 1280, tests/golden/, replicated)
through what the reference's facade does per picture (cimbar_recv_js.cpp:152-189): Scanner::scan -> Corners -> Deskewer::deskew
-> Decoder::decode_fountain(should_preprocess = true):
  * `value`: pictures/s with the pictures resident in HBM -- cb200_scan_dev + cb200_extract_decode_fountain_dev, CUDA events,
    incl. the one host round trip of 64 B of anchors per picture between scan and deskew;
  * `e2e`: the same through cb200_scan_extract_decode_fountain with pinned HOST pictures (H2D of 3.7 MB per picture inside);
  * `roofline`: k_scan_blur4 (gray + Gaussian + histogram), algorithmic 4 B per pixel (3 read, 1 written);
  * `cpu_baseline`: the same per-picture pipeline on one host core (the restatement's scan, cv2's deskew, the oracle's decode).
Photographs need the exact flood walk (K1x), so the decode leg is the walk's throughput, not K1's."""
import json
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def load_pictures():
    import cv2
    out = []
    for name in ("6bit__4_30_f0_627.jpg", "6bit__4_30_f2_246.jpg"):
        img = cv2.imread(os.path.join(ROOT, "tests", "golden", name), cv2.IMREAD_COLOR)
        out.append(np.ascontiguousarray(cv2.cvtColor(img, cv2.COLOR_BGR2RGB)))
    return out


def cpu_pipeline(pics, reps=6):
    """the same path on ONE host core, a bounded sample: the CPU restatement of the scan (oracle/scan_oracle.c), OpenCV's own
    getPerspectiveTransform + warpPerspective (what Deskewer calls), the oracle's decode_fountain with should_preprocess = true"""
    import cv2
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import oracle_lib as ol
    from scan_oracle_lib import ScanOracle
    so, ora = ScanOracle(), ol.Oracle()
    m = ora.mode(4)
    W, H, an = m.image_size_x, m.image_size_y, 30
    dst = np.array([[an, an], [W - an, an], [an, H - an], [W - an, H - an]], np.float32)
    t_scan = t_warp = t_dec = 0.0
    good = 0
    for i in range(reps):
        rgb = pics[i % len(pics)]
        t0 = time.perf_counter()
        anchors, _ = so.scan(rgb)
        t1 = time.perf_counter()
        assert len(anchors) == 4
        src = np.array(so.corners(anchors), np.float32).reshape(4, 2)
        frame = cv2.warpPerspective(rgb, cv2.getPerspectiveTransform(src, dst), (W, H), flags=cv2.INTER_LINEAR)
        t2 = time.perf_counter()
        g, _, _ = ora.decode_fountain(m, frame, sharpen=True)
        t3 = time.perf_counter()
        good += g
        t_scan += t1 - t0; t_warp += t2 - t1; t_dec += t3 - t2
    total = t_scan + t_warp + t_dec
    # ... and on all usable cores: one picture stream per thread (the oracle keeps its decoder state per thread; ctypes and cv2
    # release the GIL), a bounded sample
    from concurrent.futures import ThreadPoolExecutor
    threads = max(1, min(len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1), 16))
    cv2.setNumThreads(1)

    def worker(k):
        done = 0
        for i in range(reps):
            rgb = pics[(k + i) % len(pics)]
            a, _ = so.scan(rgb)
            srcp = np.array(so.corners(a), np.float32).reshape(4, 2)
            fr = cv2.warpPerspective(rgb, cv2.getPerspectiveTransform(srcp, dst), (W, H), flags=cv2.INTER_LINEAR)
            done += ora.decode_fountain(m, fr, sharpen=True)[0] > 0
        return done

    t0 = time.perf_counter()
    with ThreadPoolExecutor(max_workers=threads) as ex:
        ok_pics = sum(ex.map(worker, range(threads)))
    t_all = time.perf_counter() - t0
    return {"value": reps / total, "unit": "pictures/s (scan + deskew + decode)", "cores": 1, "kind": "port",
            "all_cores": {"threads": threads, "pictures_per_s": threads * reps / t_all, "decoded": int(ok_pics)},
            "sample": "%d of the sample photographs on one thread: oracle scan, cv2 warpPerspective, oracle decode_fountain with sharpen" % reps,
            "stages_ms_per_picture": {"scan": 1e3 * t_scan / reps, "deskew_cv2": 1e3 * t_warp / reps, "decode": 1e3 * t_dec / reps},
            "scan_only_pictures_per_s": reps / t_scan, "good_bytes_per_picture": good / reps}


def run(args, ClockSampler, measured_peak_gbs):
    import torch
    import libcimbar_b200 as cb
    import ctypes as C
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    # photographs go through the exact walk (one warp per frame, ~50 ms each): throughput needs thousands of them in flight
    B = min(args.frames, 4096)
    E = min(B, 2 * args.e2e_frames)                       # pictures per call of the end-to-end leg (pinned host memory)
    K, W = args.steps, max(args.warmup, 3)
    pics = load_pictures()
    h, w = pics[0].shape[:2]
    host = torch.from_numpy(np.stack([pics[i % len(pics)] for i in range(E)])).pin_memory()
    d_small = host.to(dev)
    d_pics = torch.empty((B, h, w, 3), dtype=torch.uint8, device=dev)
    for i in range(0, B, E):
        d_pics[i:i + E] = d_small[:min(E, B - i)]
    del d_small
    ctx = cb.Context(4, max_frames=B)
    info = ctx.info
    stream = torch.cuda.current_stream()
    ctx.set_stream(stream.cuda_stream)
    anchors = np.zeros((B, 4, 4), np.int32); count = np.zeros(B, np.int32); cutoff = np.zeros(B, np.uint32)
    chunks = np.zeros((B, info.chunks_per_frame, info.chunk_size), np.uint8)
    ccount = np.zeros(B, np.uint32); cmask = np.zeros(B, np.uint32); ff = np.zeros(B, np.uint8); status = np.zeros(B, np.int32)
    flags = cb.FLAG_SHARPEN
    lib, hnd = ctx.lib, ctx._h

    def step_dev():
        cb._check(lib.cb200_scan_dev(hnd, d_pics.data_ptr(), w, h, B, anchors.ctypes.data, count.ctypes.data, cutoff.ctypes.data))
        corners = ((anchors[:, :, 0] + anchors[:, :, 1]) // 2, (anchors[:, :, 2] + anchors[:, :, 3]) // 2)
        cr = np.ascontiguousarray(np.stack(corners, axis=2).astype(np.float32).reshape(B, 8))
        cb._check(lib.cb200_extract_decode_fountain_dev(hnd, d_pics.data_ptr(), w, h, B, cr.ctypes.data, flags, chunks.ctypes.data,
                                                        ccount.ctypes.data, cmask.ctypes.data, ff.ctypes.data))

    def step_e2e(n=None):
        cb._check(lib.cb200_scan_extract_decode_fountain(hnd, host.data_ptr(), w, h, E if n is None else n, flags, chunks.ctypes.data, ccount.ctypes.data,
                                                         cmask.ctypes.data, ff.ctypes.data, status.ctypes.data))

    for _ in range(W):
        step_dev()
    torch.cuda.synchronize()
    assert (count == 4).all(), "scan did not find four anchors in every sample photograph"
    sampler = ClockSampler(0)
    sampler.start()
    ctx.set_timing(True)
    launches0 = cb.launch_count()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    scan_ms = []
    for _ in range(K):
        step_dev()
        scan_ms.append(ctx.get_timing(1))           # the scan's event set (the decode's is the latest)
    e1.record()
    torch.cuda.synchronize()
    launches = cb.launch_count() - launches0
    dev_ms = e0.elapsed_time(e1)
    ctx.set_timing(False)
    good_chunks = int(ccount.sum())
    for _ in range(2):
        step_e2e()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(K):
        step_e2e()
    torch.cuda.synchronize()
    e2e_s = time.perf_counter() - t0
    sampler.stop_flag = True
    sampler.join(timeout=1.0)
    assert (status[:E] > 0).all()
    # the facade's call shape: ONE picture per call (cimbard_scan_extract_decode); the exact walk is one warp per frame
    lat = []
    for _ in range(12):
        t0 = time.perf_counter()
        step_e2e(1)
        lat.append((time.perf_counter() - t0) * 1e3)
    lat.sort()

    blur_ms = sum(r[0] for r in scan_ms) / len(scan_ms)
    otsu_ms = sum(r[1] for r in scan_ms) / len(scan_ms)
    anch_ms = sum(r[2] for r in scan_ms) / len(scan_ms)
    peak, peak_src = measured_peak_gbs()
    algo = B * w * h * 4
    achieved = algo / (blur_ms * 1e-3) / 1e9

    cpu = cpu_pipeline(pics) if not args.no_cpu_baseline else None
    if cpu:
        cpu["gpu_scan_pictures_per_s"] = B / ((blur_ms + otsu_ms + anch_ms) * 1e-3)
    out = {
        "metric": "camera pictures/s through scan + extract + decode (mode 4C photographs, should_preprocess = true)",
        "value": B * K / (dev_ms * 1e-3), "unit": "pictures/s", "n_gpus": 1, "steps": K, "warmup": W, "ms_per_step": dev_ms / K,
        "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "u8 (integer; double only in Otsu and the perspective transform, bit-exact vs OpenCV)",
        "data": "the reference's sample photographs 6bit/4_30_f0_627.jpg and 4_30_f2_246.jpg (960 x 1280), replicated",
        "config": {"workload": "camera path (SURVEY 8f-2): %d photographs of %d x %d per step: Scanner::scan (k_scan_blur, k_scan_otsu, "
                               "k_scan_anchors) -> corners -> k_deskew -> decode (K1 sharpen + exact walk K1x + RS)" % (B, w, h),
                   "mode": "4C (4)", "pictures_per_step": B, "l2": "input %.2f GB per step >> 50 MB L2" % (B * w * h * 3 / 1e9)},
        "parity": "%d of %d chunks decoded per step (tests/test_gpu_scan.py checks the bytes against the CPU pipeline)" % (good_chunks, B * info.chunks_per_frame),
        "gpu_launches": launches,
        "kernel_ms_per_step": {"scan_blur_hist": blur_ms, "scan_otsu": otsu_ms, "scan_anchors": anch_ms},
        "roofline": {"kernel": "k_scan_blur4", "bound": "hbm", "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak,
                     "peak_source": peak_src, "algorithmic_bytes_per_launch": algo, "traffic": None,
                     "note": "3 bytes read + 1 written per pixel; the tile halo re-reads (2R per 128 x 32 tile) hit L2"},
        "e2e": {"value": E * K / e2e_s, "unit": "pictures/s", "h2d_bytes_per_step": int(E * w * h * 3),
                "d2h_bytes_per_step": int(E * (info.chunks_per_frame * info.chunk_size + 4 + 4 + 1 + 64 + 12)),
                "note": "cb200_scan_extract_decode_fountain from pinned host pictures, %d per call, wall clock around K calls" % E},
        "e2e_single_picture": {"median_ms": lat[len(lat) // 2], "p90_ms": lat[int(len(lat) * 0.9)],
                               "note": "one photograph per call (the facade's call shape): scan + deskew + K1 + the exact walk (one warp per "
                                       "frame: the latency of a 12 400-step serial chain) + RS"},
        "clocks": sampler.summary(),
    }
    if cpu:
        out["cpu_baseline"] = cpu
    print(json.dumps(out))
