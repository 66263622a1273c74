"""The enqueue-only camera entry point (cb200_scan_extract_decode_chunks_ragged_dev): scan, Extractor::extract, deskew and decode on
the device with no host round trip.  Every picture must come out as the reference CLI's decode loop gives it (scan, Corners, warp,
decode, one decoder state in order), the transforms must be getPerspectiveTransform's bit for bit, and the call must return while
the device is still busy -- with three calls in flight giving what one call over the three batches gives."""
import time

import cv2
import numpy as np
import pytest

from oracle_lib import load_sample
from ragged_samples import GLOB, sample
from scan_oracle_lib import ScanOracle
from test_gpu_sharpen_select import ORA, dense

pytestmark = pytest.mark.gpu

SO = ScanOracle()


@pytest.fixture(scope="module")
def cb():
    import libcimbar_b200 as cb
    return cb


def pad(rgb, top, bottom, left, right):
    return cv2.copyMakeBorder(rgb, top, bottom, left, right, cv2.BORDER_CONSTANT, value=(0, 0, 0))


def batch_4c():
    """the sample directory, padded photographs of two further sizes and a noise picture (test_gpu_scan_ragged's cli_batch)"""
    pics = [sample(s) for s in GLOB]
    pics.append(pad(sample("6bit/4_30_f0_627.jpg"), 120, 150, 100, 160))
    pics.append(np.random.default_rng(47).integers(0, 256, (900, 1200, 3), dtype=np.uint8))
    pics.append(pad(sample("6bit/4_30_f1_360.jpg"), 90, 70, 200, 140))
    pics.append(sample("6bit/4_30_f2_734.jpg"))
    return pics


def batch_b():
    """the two mode-B photographs, a zero-padded and an upscaled variant of each, and a noise picture"""
    a, b = load_sample("b/ex2434.jpg"), load_sample("b/ex380.jpg")
    noise = np.random.default_rng(53).integers(0, 256, (800, 1000, 3), dtype=np.uint8)
    return [a, pad(b, 200, 160, 240, 300), noise, cv2.resize(a, None, fx=1.3, fy=1.3), b, pad(a, 60, 40, 80, 20),
            cv2.resize(b, None, fx=1.6, fy=1.6)]


_loops = {}


def cli_loop(mode_val, name, pics, cc, sharpen):
    """the reference CLI's loop: sharpen = 'no' / 'all' / 'needed' (--preprocess 0 / 1 / -1); FAILURE pictures are skipped.  Returns
    per picture (status, corners, (good, dense chunks, mask)) and the decoder's CCM at the end"""
    key = (mode_val, name, cc, sharpen)
    if key in _loops:
        return _loops[key]
    m = ORA.mode(mode_val)
    an, W, H = 30, m.image_size_x, m.image_size_y
    dst = np.array([[an, an], [W - an, an], [an, H - an], [W - an, H - an]], np.float32)
    out = []
    ORA.set_ccm(None)
    try:
        for rgb in pics:
            anchors, _ = SO.scan(rgb)
            if anchors is None or len(anchors) < 4:
                out.append((0, None, None))
                continue
            xy = SO.corners(anchors)
            status = 1 if SO.is_granular_scale(xy, W, H) else 2
            frame = cv2.warpPerspective(rgb, cv2.getPerspectiveTransform(np.array(xy, np.float32).reshape(4, 2), dst), (W, H),
                                        flags=cv2.INTER_LINEAR)
            sh = {"no": False, "all": True, "needed": status == 2}[sharpen]
            good, chunks, mask = ORA.decode_fountain(m, frame, sharpen=sh, color_correction=cc)
            out.append((status, xy, (good, chunks.copy(), mask)))
        ccm = ORA.get_ccm()
    finally:
        ORA.set_ccm(None)
    _loops[key] = (out, ccm)
    return _loops[key]


def packed(pics):
    import torch
    d = torch.cat([torch.from_numpy(np.ascontiguousarray(p).reshape(-1)) for p in pics]).cuda()
    wh = np.array([(p.shape[1], p.shape[0]) for p in pics], np.int32).reshape(-1, 2)
    return d, wh


class Outputs:
    """device output buffers of one call, each starting `offset` bytes into its allocation (the byte-sized ones)"""

    def __init__(self, ctx, n, offset=0):
        import torch
        self.n, self.offset, self.db = n, offset, ctx.info.data_bytes
        self.chunks = torch.full((n * self.db + offset,), 0xA5, dtype=torch.uint8, device="cuda")
        self.mask = torch.full((n,), -1, dtype=torch.int32, device="cuda")
        self.status = torch.full((n,), 7, dtype=torch.int32, device="cuda")
        self.flags = torch.full((n + offset,), 0xEE, dtype=torch.uint8, device="cuda")

    def call(self, ctx, d, wh, flags):
        ctx.scan_extract_decode_chunks_dev(d.data_ptr(), wh, self.chunks.data_ptr() + self.offset, self.mask.data_ptr(),
                                           self.status.data_ptr(), self.flags.data_ptr() + self.offset, flags=flags)

    def host(self):
        o = self.offset
        return (self.chunks[o:].cpu().numpy().reshape(self.n, self.db), self.mask.cpu().numpy().view(np.uint32),
                self.status.cpu().numpy(), self.flags[o:].cpu().numpy())


def run(cb, ctx, pics, flags, offset=0):
    import torch
    d, wh = packed(pics)
    out = Outputs(ctx, len(pics), offset)
    torch.cuda.synchronize()
    out.call(ctx, d, wh, flags)
    ctx.sync()
    return out.host()


def check_against_loop(m, got, want, what):
    chunks, mask, status, _ = got
    assert status.tolist() == [w[0] for w in want], what
    for i, (st, xy, wd) in enumerate(want):
        if st == 0:
            assert mask[i] == 0, (what, i)
            continue
        good, wchunks, wmask = wd
        cnt, rows = dense(m, chunks[i], int(mask[i]))
        assert mask[i] == wmask and cnt * m.chunk_size == good, (what, i)
        assert np.array_equal(rows, wchunks[:cnt]), (what, i)


def same_ccm(a, b):
    return (a is None) == (b is None) and (a is None or np.array_equal(a, b))


FLAGS = [("no", 0, 0), ("all", "SHARPEN", 0), ("needed", "SHARPEN_IF_NEEDED", 0), ("needed", "SHARPEN_IF_NEEDED", "CC_SIMPLE"),
         ("needed", "SHARPEN_IF_NEEDED", "CC_FIT")]


@pytest.mark.parametrize("mode_val", [4, 68])
@pytest.mark.parametrize("sharpen,sflag,ccflag", FLAGS)
def test_matches_the_cli_loop(cb, mode_val, sharpen, sflag, ccflag):
    pics = batch_4c() if mode_val == 4 else batch_b()
    name = "4c" if mode_val == 4 else "b"
    cc = {0: 0, "CC_SIMPLE": 1, "CC_FIT": 2}[ccflag]
    flags = (getattr(cb, "FLAG_" + sflag) if sflag else 0) | (getattr(cb, "FLAG_" + ccflag) if ccflag else 0)
    m = ORA.mode(mode_val)
    want, want_ccm = cli_loop(mode_val, name, pics, cc, sharpen)
    statuses = {w[0] for w in want}
    if mode_val == 4:
        assert statuses == {0, 1, 2}                                    # premise
    assert any(w[0] > 0 and w[2][0] > 0 for w in want)
    ctx = cb.Context(mode_val, max_frames=len(pics))
    for offset in (0, 1):
        ctx.set_ccm(None)
        got = run(cb, ctx, pics, flags, offset)
        check_against_loop(m, got, want, (mode_val, flags, offset))
        assert same_ccm(ctx.get_ccm(), want_ccm), (mode_val, flags, offset)
    ctx.close()


def test_transforms_are_get_perspective_transform(cb):
    pics = batch_4c()
    m = ORA.mode(4)
    an, W, H = 30, m.image_size_x, m.image_size_y
    outp = np.array([[an, an], [W - an, an], [an, H - an], [W - an, H - an]], np.float32)
    ctx = cb.Context(4, max_frames=len(pics))
    _, _, status, _ = run(cb, ctx, pics, cb.FLAG_SHARPEN_IF_NEEDED)
    got = ctx.camera_transforms(len(pics))
    anchors, count, _ = ctx.scan_ragged(pics)
    ok = 0
    for i in range(len(pics)):
        if status[i] <= 0:
            want = cb.perspective_transform(outp, outp)
        else:
            xy = np.stack([(anchors[i, :, 0] + anchors[i, :, 1]) // 2, (anchors[i, :, 2] + anchors[i, :, 3]) // 2], axis=1).astype(np.float32)
            want = cb.perspective_transform(xy, outp)
            assert np.array_equal(cv2.getPerspectiveTransform(xy, outp), want), i
            ok += 1
        assert np.array_equal(got[i], want), i
    assert ok >= 5
    with pytest.raises(cb.Cb200Error, match="last camera call"):
        ctx.camera_transforms(len(pics) + 1)
    ctx.close()


def test_calls_only_enqueue(cb):
    """three calls queued behind a sleeping stream return at once and equal one call over the three batches, CCM carry included"""
    import torch
    pics = batch_b()
    batches = [pics[0:3], pics[3:5], pics[5:7]]
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    n = len(pics)
    ref = cb.Context(68, max_frames=n)
    want = run(cb, ref, pics, flags)
    want_ccm = ref.get_ccm()
    assert want_ccm is not None and (want[1] != 0).sum() >= 3          # premise: fits happen, chunks decode
    ctx = cb.Context(68, max_frames=n)
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    dev = [packed(b) for b in batches]
    outs = [Outputs(ctx, len(b)) for b in batches]
    torch.cuda.synchronize()
    for (d, wh), o in zip(dev, outs):                                # warm-up: every buffer at its size, then the same state again
        o.call(ctx, d, wh, flags)
    ctx.sync()
    ctx.set_ccm(None)
    torch.cuda.synchronize()
    with torch.cuda.stream(stream):
        torch.cuda._sleep(int(1.5e9))                                # about a second at the H100's clock
    t0 = time.perf_counter()
    for (d, wh), o in zip(dev, outs):
        o.call(ctx, d, wh, flags)
    spent = time.perf_counter() - t0
    busy = not stream.query()
    ctx.sync()
    assert busy, "the stream finished before the third call returned"
    assert spent < 0.25, spent
    got = [o.host() for o in outs]
    at = 0
    for g in got:
        k = g[0].shape[0]
        for a, b in zip(g, want):
            assert np.array_equal(a, b[at:at + k])
        at += k
    assert same_ccm(ctx.get_ccm(), want_ccm)
    ref.close()
    ctx.close()


def test_uniform_wrapper_and_small_batches(cb):
    import torch
    pics = [sample("6bit/4_30_f0_627.jpg"), sample("6bit/4_30_f2_246.jpg"), cv2.resize(sample("6bit/4_30_f1_360.jpg"), (1280, 960))]
    n = len(pics)
    flags = cb.FLAG_SHARPEN_IF_NEEDED
    ctx = cb.Context(4, max_frames=n)
    want = run(cb, ctx, pics, flags)
    d = torch.from_numpy(np.stack(pics)).cuda()
    out = Outputs(ctx, n)
    torch.cuda.synchronize()
    cb._check(ctx.lib.cb200_scan_extract_decode_chunks_dev(ctx._h, d.data_ptr(), 1280, 960, n, flags, out.chunks.data_ptr(),
                                                           out.mask.data_ptr(), out.flags.data_ptr(), out.status.data_ptr()))
    ctx.sync()
    for a, b in zip(out.host(), want):
        assert np.array_equal(a, b)
    # n = 1, and n = 0 (nothing to do: no work, no error)
    one = run(cb, ctx, pics[:1], flags)
    for a, b in zip(one, want):
        assert np.array_equal(a, b[:1])
    wh0 = np.zeros((0, 2), np.int32)
    cb._check(ctx.lib.cb200_scan_extract_decode_chunks_ragged_dev(ctx._h, d.data_ptr(), wh0.ctypes.data, 0, flags, out.chunks.data_ptr(),
                                                                  out.mask.data_ptr(), None, out.status.data_ptr()))
    # more pictures than the context holds: refused before any work
    small = cb.Context(4, max_frames=1)
    dd, wh = packed(pics[:2])
    rc = small.lib.cb200_scan_extract_decode_chunks_ragged_dev(small._h, dd.data_ptr(), wh.ctypes.data, 2, flags, out.chunks.data_ptr(),
                                                               out.mask.data_ptr(), None, out.status.data_ptr())
    assert rc == -1 and b"max_frames" in small.lib.cb200_last_error()
    ctx.close()
    small.close()


@pytest.mark.parametrize("mode_val,ccflag", [(68, "CC_FIT"), (4, "CC_SIMPLE")])
def test_carried_ccm_into_batches_without_colour_correction(cb, mode_val, ccflag):
    """a batch without colour correction enqueued behind one that changes the CCM (still running) reads that CCM on the device: the
    same results as the three calls made one at a time, each after the previous one finished"""
    import torch
    pics = batch_b() if mode_val == 68 else batch_4c()[:6]
    batches = [pics[0:3], pics[3:5], pics[5:]]
    ccf = getattr(cb, "FLAG_" + ccflag)
    seq = [cb.FLAG_SHARPEN_IF_NEEDED | ccf, 0, cb.FLAG_SHARPEN_IF_NEEDED]
    n = max(len(b) for b in batches)
    ref, ctx = cb.Context(mode_val, max_frames=n), cb.Context(mode_val, max_frames=n)
    want = [run(cb, ref, b, f) for b, f in zip(batches, seq)]
    want_ccm = ref.get_ccm()
    assert want_ccm is not None
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    dev = [packed(b) for b in batches]
    outs = [Outputs(ctx, len(b)) for b in batches]
    torch.cuda.synchronize()
    for (d, wh), o, f in zip(dev, outs, seq):                        # warm-up
        o.call(ctx, d, wh, f)
    ctx.sync()
    ctx.set_ccm(None)
    with torch.cuda.stream(stream):
        torch.cuda._sleep(int(2e8))
    for (d, wh), o, f in zip(dev, outs, seq):
        o.call(ctx, d, wh, f)
    ctx.sync()
    for o, w in zip(outs, want):
        for a, b in zip(o.host(), w):
            assert np.array_equal(a, b)
    assert same_ccm(ctx.get_ccm(), want_ccm)
    ref.close()
    ctx.close()
