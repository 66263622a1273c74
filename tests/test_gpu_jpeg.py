"""JPEG files decoded on the device (cb200_jpeg_decode_dev) and run through the camera path
(cb200_jpeg_scan_extract_decode_chunks_dev): every picture must be cv2.imread + cvtColor(BGR2RGB)'s bytes, and the camera call must
give exactly what cb200_scan_extract_decode_chunks_ragged_dev gives on cv2's pictures -- in every mode and flag set, across calls in
flight, with corrupt files reported as status -2 and without the call waiting for the device."""
import time

import numpy as np
import pytest

from jpeg_matrix import cv2_rgb, golden_files, matrix, photo_files

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cb():
    import libcimbar_b200 as cb
    return cb


def decode_dev(cb, ctx, files):
    """[(rgb, status)] of one cb200_jpeg_decode_dev call"""
    import torch
    shapes = [cb.jpeg_info(f) for f in files]
    total = sum(3 * w * h for w, h in shapes)
    out = torch.full((total,), 0xA5, dtype=torch.uint8, device="cuda")
    status = torch.full((len(files),), 7, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    ctx.jpeg_decode_dev(files, out.data_ptr(), status.data_ptr())
    ctx.sync()
    host, st = out.cpu().numpy(), status.cpu().numpy()
    res, at = [], 0
    for (w, h), s in zip(shapes, st):
        res.append((host[at:at + 3 * w * h].reshape(h, w, 3), int(s)))
        at += 3 * w * h
    return res


def test_decode_matches_cv2(cb):
    files = golden_files() + matrix()
    ctx = cb.Context(4, max_frames=1)
    got = decode_dev(cb, ctx, [d for _, d in files])
    for (name, data), (rgb, st) in zip(files, got):
        assert st == 0, name
        want = cv2_rgb(data)
        assert rgb.shape == want.shape and np.array_equal(rgb, want), (name, int(np.count_nonzero(rgb != want)))
    ctx.close()


class Outputs:
    def __init__(self, ctx, n):
        import torch
        self.n, self.db = n, ctx.info.data_bytes
        self.chunks = torch.full((n * self.db,), 0xA5, dtype=torch.uint8, device="cuda")
        self.mask = torch.full((n,), -1, dtype=torch.int32, device="cuda")
        self.status = torch.full((n,), 7, dtype=torch.int32, device="cuda")
        self.flags = torch.full((n,), 0xEE, dtype=torch.uint8, device="cuda")

    def rgb_call(self, ctx, d, wh, flags):
        ctx.scan_extract_decode_chunks_dev(d.data_ptr(), wh, self.chunks.data_ptr(), self.mask.data_ptr(), self.status.data_ptr(),
                                           self.flags.data_ptr(), flags=flags)

    def jpeg_call(self, ctx, files, flags):
        ctx.jpeg_scan_extract_decode_chunks_dev(files, self.chunks.data_ptr(), self.mask.data_ptr(), self.status.data_ptr(),
                                                self.flags.data_ptr(), flags=flags)

    def host(self):
        return (self.chunks.cpu().numpy().reshape(self.n, self.db), self.mask.cpu().numpy().view(np.uint32), self.status.cpu().numpy(),
                self.flags.cpu().numpy())


def packed(pics):
    import torch
    d = torch.cat([torch.from_numpy(np.ascontiguousarray(p).reshape(-1)) for p in pics]).cuda()
    wh = np.array([(p.shape[1], p.shape[0]) for p in pics], np.int32).reshape(-1, 2)
    return d, wh


def batches_of(mode_val):
    """three batches of golden photographs of the mode (each photograph once, the B ones twice)"""
    files = [d for _, d in photo_files("6bit" if mode_val == 4 else "b")]
    if mode_val == 68:
        files = files + files[::-1] + files
    k = len(files)
    return [files[: k // 3], files[k // 3: 2 * k // 3], files[2 * k // 3:]]


def reference(cb, mode_val, batches, flags, pics_of=None):
    """the RGB camera call on cv2's pictures, one batch after the other; outputs and the final CCM"""
    ref = cb.Context(mode_val, max_frames=max(len(b) for b in batches))
    ref.set_ccm(None)
    out = []
    for b in batches:
        pics = [cv2_rgb(f) if pics_of is None else pics_of(f) for f in b]
        d, wh = packed(pics)
        o = Outputs(ref, len(b))
        import torch
        torch.cuda.synchronize()
        o.rgb_call(ref, d, wh, flags)
        ref.sync()
        out.append(o.host())
    ccm = ref.get_ccm()
    ref.close()
    return out, ccm


def same_ccm(a, b):
    return (a is None) == (b is None) and (a is None or np.array_equal(a, b))


@pytest.mark.parametrize("mode_val", [4, 68])
@pytest.mark.parametrize("flagset", ["SHARPEN_IF_NEEDED|CC_FIT", "none"])
def test_camera_call_matches_rgb_call(cb, mode_val, flagset):
    flags = (cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT) if flagset != "none" else 0
    batches = batches_of(mode_val)
    want, want_ccm = reference(cb, mode_val, batches, flags)
    assert any((w[1] != 0).any() for w in want)                       # premise: chunks decode
    ctx = cb.Context(mode_val, max_frames=max(len(b) for b in batches))
    ctx.set_ccm(None)
    outs = [Outputs(ctx, len(b)) for b in batches]
    import torch
    torch.cuda.synchronize()
    for b, o in zip(batches, outs):                                   # three calls in flight
        o.jpeg_call(ctx, b, flags)
    ctx.sync()
    for o, w in zip(outs, want):
        for a, b in zip(o.host(), w):
            assert np.array_equal(a, b), (mode_val, flagset)
    assert same_ccm(ctx.get_ccm(), want_ccm)
    ctx.close()


def all_ones(data):
    """a copy of `data` with 8 bytes in the middle of its first scan's data replaced by FF 00 FF 00 FF 00 FF 00: 32 one bits after
    unstuffing, which no Huffman code and no extra bits can span (no code is all ones), so the data cannot decode"""
    sos = data.index(b"\xff\xda")
    mid = sos + (len(data) - sos) // 2
    while data[mid - 1] == 0xFF:                                      # not the stuffing byte of an FF 00 pair
        mid += 1
    return data[:mid] + b"\xff\x00" * 4 + data[mid + 8:]


def test_corrupt_files_get_status_minus_2(cb):
    good = [d for _, d in photo_files("6bit")]
    ctx = cb.Context(4, max_frames=len(good))
    flipped = all_ones(good[2])
    truncated = good[4][: len(good[4]) * 2 // 3]
    files = list(good)
    files[2], files[4] = flipped, truncated
    # the other pictures are as in the RGB call where the corrupt ones are black pictures of their sizes
    black = {flipped: np.zeros_like(cv2_rgb(good[2])), truncated: np.zeros_like(cv2_rgb(good[4]))}
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    (want,), _ = reference(cb, 4, [files], flags, pics_of=lambda f: black[f] if f in black else cv2_rgb(f))
    got = decode_dev(cb, ctx, files)
    assert [s for _, s in got] == [0, 0, -2, 0, -2, 0, 0]
    o = Outputs(ctx, len(files))
    ctx.set_ccm(None)
    o.jpeg_call(ctx, files, flags)
    ctx.sync()
    chunks, mask, status, fflags = o.host()
    assert status[2] == -2 and status[4] == -2 and mask[2] == 0 and mask[4] == 0
    assert status.tolist() == [s if i not in (2, 4) else -2 for i, s in enumerate(want[2].tolist())]
    keep = [i for i in range(len(files)) if i not in (2, 4)]
    assert np.array_equal(chunks[keep], want[0][keep]) and np.array_equal(mask[keep], want[1][keep])
    assert np.array_equal(fflags, want[3])
    ctx.close()


def test_calls_only_enqueue(cb):
    """three calls queued behind a sleeping stream return at once and give what the same calls give one at a time"""
    import torch
    files = [d for _, d in photo_files("b")]
    batches = [files, files[::-1], files]
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    ctx = cb.Context(68, max_frames=len(files))
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    outs = [Outputs(ctx, len(b)) for b in batches]
    torch.cuda.synchronize()
    want = []
    for b, o in zip(batches, outs):                                   # warm-up, one at a time: every buffer at its size
        o.jpeg_call(ctx, b, flags)
        ctx.sync()
        want.append(o.host())
    want_ccm = ctx.get_ccm()
    ctx.set_ccm(None)
    with torch.cuda.stream(stream):
        torch.cuda._sleep(int(1.5e9))
    t0 = time.perf_counter()
    for b, o in zip(batches, outs):
        o.jpeg_call(ctx, b, flags)
    spent = time.perf_counter() - t0
    busy = not stream.query()
    ctx.sync()
    assert busy, "the stream finished before the third call returned"
    assert spent < 0.25, spent
    for o, w in zip(outs, want):
        for a, b in zip(o.host(), w):
            assert np.array_equal(a, b)
    assert same_ccm(ctx.get_ccm(), want_ccm)
    ctx.close()
