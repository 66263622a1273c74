"""GPU parity of the device anchor scan (libcimbar_b200/csrc/scan.cu) through the C ABI: against the CPU restatement
(oracle/scan_oracle.c, pinned to cv2 and to ScannerTest's golden strings in tests/test_scan_oracle.py) and against those
golden strings directly; Extractor::extract + decode as one call against its parts."""
import cv2
import numpy as np
import pytest

import oracle_lib as ol
from scan_oracle_lib import ScanOracle, join
from test_scan_core_host import pictures

pytestmark = pytest.mark.gpu

SO = ScanOracle()


@pytest.fixture(scope="module")
def cb():
    import libcimbar_b200 as cb
    return cb


def _check(ctx, pics):
    """pics: list of same-sized pictures; device blur / threshold / anchors / cutoff == oracle for each"""
    batch = np.stack(pics)
    n, h, w, _ = batch.shape
    anchors, count, cutoff = ctx.scan(batch)
    blurred, thr = ctx.scan_blurred(n, h, w)
    for i, rgb in enumerate(pics):
        t, bin_, bl = SO.preprocess(rgb)
        assert np.array_equal(blurred[i], bl), i
        assert thr[i] == t, i
        want, want_cutoff = SO.scan(rgb)
        got = [tuple(int(v) for v in anchors[i, k]) for k in range(max(count[i], 0))]
        assert count[i] == len(want) and got == want, (i, join(got), join(want))
        assert cutoff[i] == want_cutoff, i
        assert not anchors[i, len(want):].any()


@pytest.mark.parametrize("name,rgb", pictures(), ids=[p[0] for p in pictures()])
def test_scan_matches_oracle(cb, name, rgb):
    ctx = cb.Context(68, max_frames=1)
    _check(ctx, [rgb])
    ctx.close()


def test_scan_goldens_on_gpu(cb):
    # extractor/test/ScannerTest.cpp:54-176: the strings the reference's own tests expect, from the device
    ctx = cb.Context(4, max_frames=1)
    for g in ol.manifest()["scan_goldens"]:
        anchors, count, cutoff = ctx.scan(ol.load_sample(g["sample"]))
        assert count[0] == 4
        assert join([tuple(a) for a in anchors[0]]) == g["scan"], g["source"]
        if "cutoff" in g:
            assert cutoff[0] == g["cutoff"]
    ctx.close()


def test_scan_batches(cb):
    # many pictures per call (one CTA each), two picture shapes through one context, workspace reuse and growth
    ctx = cb.Context(4, max_frames=1)
    land = [ol.load_sample(s) for s in ("6bit/4_30_f0_627.jpg", "6bit/4_30_f2_246.jpg")]           # 960 x 1280
    port = [ol.load_sample(s) for s in ("6bit/4_30_f2_734.jpg", "6bit/4_30_f1_360.jpg")]           # 1280 x 960
    rng = np.random.default_rng(8)
    noisy = [np.clip(p.astype(np.int16) + rng.integers(-25, 26, p.shape), 0, 255).astype(np.uint8) for p in land]
    _check(ctx, land)
    _check(ctx, port + port[::-1] + port)
    _check(ctx, (land + noisy) * 6 + [np.zeros_like(land[0])])
    ctx.close()


def test_scan_nine_tap_blur(cb):
    big = cv2.resize(ol.load_sample("6bit/4_30_f0_627.jpg"), None, fx=3, fy=3, interpolation=cv2.INTER_LINEAR)   # 2880 x 3840
    ctx = cb.Context(4, max_frames=1)
    _check(ctx, [big])
    mid = cv2.resize(ol.load_sample("6bit/4_30_f2_734.jpg"), None, fx=2.2, fy=2.2)                                # 7-tap does not occur; 5-tap here
    _check(ctx, [mid])
    ctx.close()


def test_scan_rejects_what_is_not_restated(cb):
    ctx = cb.Context(68, max_frames=1)
    with pytest.raises(cb.Cb200Error):
        ctx.scan(np.zeros((4500, 4600, 3), np.uint8))       # 17-tap Gaussian
    with pytest.raises(cb.Cb200Error):
        ctx.scan(np.zeros((50, 400, 3), np.uint8))          # Scanner's row step would be 0
    ctx.close()


def test_scan_extract_decode_is_its_parts(cb):
    """cb200_scan_extract_decode_fountain == Scanner (oracle) -> Corners -> cb200_extract_decode_fountain (pinned to cv2 in
    tests/test_deskew.py), with Extractor::extract's status per picture (Extractor.h:30-46)"""
    m = ol.Oracle().mode(4)
    cam = ol.load_sample("6bit/4_30_f0_627.jpg")                       # mode 4C photograph, 960 x 1280: upscaled by the deskew
    cam2 = ol.load_sample("6bit/4_30_f2_246.jpg")
    rng = np.random.default_rng(5)
    junk = rng.integers(0, 256, cam.shape, dtype=np.uint8)
    big = cv2.resize(cam, None, fx=1.5, fy=1.5)                        # 1440 x 1920: every side longer than 1024 -> SUCCESS
    for batch in ([cam, junk, cam2], [big]):
        pics = np.stack(batch)
        ctx = cb.Context(4, max_frames=len(batch))
        for flags in (0, cb.FLAG_SHARPEN):
            chunks, count, mask, ff, status = ctx.scan_extract_decode_fountain(pics, flags=flags)
            for i, rgb in enumerate(batch):
                anchors, _ = SO.scan(rgb)
                if len(anchors) < 4:
                    assert status[i] == 0 and count[i] == 0 and mask[i] == 0
                    continue
                xy = SO.corners(anchors)
                assert status[i] == (1 if SO.is_granular_scale(xy, m.image_size_x, m.image_size_y) else 2)
                c1, n1, m1, f1 = ctx.extract_decode_fountain(rgb, np.array(xy, np.float32), flags=flags)
                assert count[i] == n1[0] and mask[i] == m1[0] and np.array_equal(chunks[i], c1[0]), (i, flags)
        ctx.close()
    # end to end against the CPU pipeline: oracle scan -> cv2 getPerspectiveTransform / warpPerspective (what Deskewer calls) ->
    # oracle decode_fountain, with the reference facade's setting should_preprocess = true (cimbar_recv_js.cpp:171-186)
    ctx = cb.Context(4, max_frames=1)
    O = ol.Oracle()
    for rgb in (cam, cam2):
        chunks, count, mask, ff, status = ctx.scan_extract_decode_fountain(rgb, flags=cb.FLAG_SHARPEN)
        anchors, _ = SO.scan(rgb)
        src = np.array(SO.corners(anchors), np.float32).reshape(4, 2)
        an, W, H = 30, m.image_size_x, m.image_size_y
        dst = np.array([[an, an], [W - an, an], [an, H - an], [W - an, H - an]], np.float32)
        frame = cv2.warpPerspective(rgb, cv2.getPerspectiveTransform(src, dst), (W, H), flags=cv2.INTER_LINEAR)
        good, ochunks, omask = O.decode_fountain(m, frame, sharpen=True)
        assert status[0] == 2 and mask[0] == omask and np.array_equal(chunks[0], ochunks)
        assert good > 0
    ctx.close()


def test_cpp_extractor_mirrors_rerun_reference_tests(cb, tmp_path):
    """libcimbar_b200/host/Extractor.h keeps the reference's Scanner / Anchor / Extractor names; tests/cpp/extractor_test.cpp runs
    ScannerTest/testExampleScan's and ExtractorTest's call shapes through them: golden anchor strings, Extractor's status, the
    extracted frame == what Deskewer's two OpenCV calls give for those corners, and its decode == the oracle's."""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / "extractor_test")
    libdir = os.path.join(root, "libcimbar_b200", "lib")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-o", exe, os.path.join(root, "tests", "cpp", "extractor_test.cpp"),
                           "-L" + libdir, "-lcb200", "-Wl,-rpath," + libdir])
    O = ol.Oracle()
    m = O.mode(4)
    for g in ol.manifest()["scan_goldens"]:
        rgb = ol.load_sample(g["sample"])
        h, w = rgb.shape[:2]
        fpath, prefix = str(tmp_path / "picture.rgb"), str(tmp_path / "out")
        rgb.tofile(fpath)
        res = subprocess.run([exe, "4", str(w), str(h), fpath, prefix], capture_output=True, text=True)
        assert res.returncode == 0, res.stdout + res.stderr
        assert open(prefix + ".anchors").read() == g["scan"], g["source"]
        anchors, _ = SO.scan(rgb)
        xy = SO.corners(anchors)
        assert int(open(prefix + ".status").read()) == (1 if SO.is_granular_scale(xy, 1024, 1024) else 2)
        src = np.array(xy, np.float32).reshape(4, 2)
        dst = np.array([[30, 30], [994, 30], [30, 994], [994, 994]], np.float32)
        want = cv2.warpPerspective(rgb, cv2.getPerspectiveTransform(src, dst), (1024, 1024), flags=cv2.INTER_LINEAR)
        frame = np.fromfile(prefix + ".frame", dtype=np.uint8).reshape(1024, 1024, 3)
        assert np.array_equal(frame, want), g["sample"]
        odata, ook = O.decode(m, want, use_ecc=True, sharpen=True)
        assert np.array_equal(np.fromfile(prefix + ".ecc", dtype=np.uint8), odata), g["sample"]


def test_scan_blur_on_aligned_and_unaligned_widths(cb):
    """k_scan_blur4 (four pixels per thread: aligned word loads, IDP.2A gray, IDP.4A taps; single pixels where rows are not word
    aligned) against the oracle, on aligned and unaligned widths and all three kernel sizes the scanner uses"""
    ctx = cb.Context(68, max_frames=1)
    cam = ol.load_sample("6bit/4_30_f2_734.jpg")
    for rgb in (cam, np.ascontiguousarray(cam[:, 3:958]), cv2.resize(cam, None, fx=1.7, fy=1.7), cv2.resize(cam, None, fx=2.9, fy=2.9)[:, :2781]):
        _check(ctx, [rgb])
    ctx.close()
