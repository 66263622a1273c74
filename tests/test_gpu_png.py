"""PNG files decoded on the device (cb200_png_decode_dev) and run through the camera path (cb200_png_scan_extract_decode_chunks_dev)
and the frame path (cb200_png_decode_dev -> cb200_decode_chunks_dev, the CLI's --no-deskew): every picture must be
cv2.imread + cvtColor(BGR2RGB)'s bytes, the camera call must give exactly what cb200_scan_extract_decode_chunks_ragged_dev gives on
cv2's pictures, the golden frames must reproduce the reference's SHA-256 goldens, and corrupt files are reported as status -2 without
the call waiting for the device."""
import hashlib
import struct
import time

import cv2
import numpy as np
import pytest

import png_matrix as pm
from jpeg_matrix import photo_files
from oracle_lib import manifest
from gpu_support import cb  # noqa: F401  (fixtures)
from gpu_support import packed, same_ccm
from png_corpus import ACCEPTED, CORRUPT

pytestmark = pytest.mark.gpu


def decode_dev(cb, ctx, files):
    """[(rgb, status)] of one cb200_png_decode_dev call"""
    import torch
    shapes = [cb.png_info(f) for f in files]
    total = sum(3 * w * h for w, h in shapes)
    out = torch.full((total,), 0xA5, dtype=torch.uint8, device="cuda")
    status = torch.full((len(files),), 7, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    ctx.png_decode_dev(files, out.data_ptr(), status.data_ptr())
    ctx.sync()
    host, st = out.cpu().numpy(), status.cpu().numpy()
    res, at = [], 0
    for (w, h), s in zip(shapes, st):
        res.append((host[at:at + 3 * w * h].reshape(h, w, 3), int(s)))
        at += 3 * w * h
    return res


def camera_sized(files):
    return [(n, d) for n, d in files if min(pm.cv2_rgb(d).shape[:2]) >= 60]


def test_decode_matches_cv2(cb):
    files = camera_sized(pm.golden_files() + pm.matrix() + [(n, d) for n, d in ACCEPTED])
    assert len(files) > 150
    ctx = cb.Context(4, max_frames=1)
    got = decode_dev(cb, ctx, [d for _, d in files])
    for (name, data), (rgb, st) in zip(files, got):
        assert st == 0, name
        want = pm.cv2_rgb(data)
        assert rgb.shape == want.shape and np.array_equal(rgb, want), (name, int(np.count_nonzero(rgb != want)))
    ctx.close()


def test_corrupt_files_get_status_minus_2_and_black(cb):
    good = [d for _, d in pm.golden_files()]
    corrupt = [d for _, d in CORRUPT if min(struct.unpack(">II", d[16:24])) >= 60]
    assert len(corrupt) >= 10
    files, expect = [], []
    for k, bad in enumerate(corrupt):                                 # each corrupt file between two good ones
        files += [good[k % len(good)], bad]
        expect += [0, -2]
    files.append(good[0])
    expect.append(0)
    ctx = cb.Context(4, max_frames=1)
    got = decode_dev(cb, ctx, files)
    assert [s for _, s in got] == expect
    for f, (rgb, s) in zip(files, got):
        if s == -2:
            assert not rgb.any()
        else:
            assert np.array_equal(rgb, pm.cv2_rgb(f))
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

    def png_call(self, ctx, files, flags):
        ctx.png_scan_extract_decode_chunks_dev(files, self.chunks.data_ptr(), self.mask.data_ptr(), self.status.data_ptr(),
                                               self.flags.data_ptr(), flags=flags)

    def host(self):
        return (self.chunks.cpu().numpy().reshape(self.n, self.db), self.mask.cpu().numpy().view(np.uint32), self.status.cpu().numpy(),
                self.flags.cpu().numpy())


def as_png(jpeg_bytes):
    ok, buf = cv2.imencode(".png", cv2.imdecode(np.frombuffer(jpeg_bytes, np.uint8), cv2.IMREAD_COLOR))
    assert ok
    return buf.tobytes()


def batches_of(mode_val):
    """three batches of golden photographs of the mode saved as PNG (each photograph once, the B ones three times)"""
    files = [as_png(d) for _, d in photo_files("6bit" if mode_val == 4 else "b")]
    if mode_val == 68:
        files = files + files[::-1] + files
    k = len(files)
    return [files[: k // 3], files[k // 3: 2 * k // 3], files[2 * k // 3:]]


def reference(cb, mode_val, batches, flags):
    """the RGB camera call on cv2's pictures, one batch after the other; outputs and the final CCM"""
    import torch
    ref = cb.Context(mode_val, max_frames=max(len(b) for b in batches))
    ref.set_ccm(None)
    out = []
    for b in batches:
        d, wh = packed([pm.cv2_rgb(f) for f in b])
        o = Outputs(ref, len(b))
        torch.cuda.synchronize()
        o.rgb_call(ref, d, wh, flags)
        ref.sync()
        out.append(o.host())
    ccm = ref.get_ccm()
    ref.close()
    return out, ccm


@pytest.mark.parametrize("mode_val", [4, 68])
@pytest.mark.parametrize("flagset", ["SHARPEN_IF_NEEDED|CC_FIT", "none"])
def test_camera_call_matches_rgb_call(cb, mode_val, flagset):
    import torch
    flags = (cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT) if flagset != "none" else 0
    batches = batches_of(mode_val)
    want, want_ccm = reference(cb, mode_val, batches, flags)
    assert any((w[1] != 0).any() for w in want)                       # premise: chunks decode
    ctx = cb.Context(mode_val, max_frames=max(len(b) for b in batches))
    ctx.set_ccm(None)
    outs = [Outputs(ctx, len(b)) for b in batches]
    torch.cuda.synchronize()
    for b, o in zip(batches, outs):                                   # three calls in flight
        o.png_call(ctx, b, flags)
    ctx.sync()
    for o, w in zip(outs, want):
        for a, b in zip(o.host(), w):
            assert np.array_equal(a, b), (mode_val, flagset)
    assert same_ccm(ctx.get_ccm(), want_ccm)
    ctx.close()


FRAMES = {68: ["b__tr_0.png", "b__tr_1.png", "b__tr_2.png", "b__tr_3.png"], 4: ["6bit__4color_ecc30_fountain_0.png"]}


@pytest.mark.parametrize("mode_val", [68, 4])
def test_frames_through_decode_chunks_equal_rgb_call(cb, mode_val):
    """the CLI's --no-deskew on the device: png_decode_dev -> decode_chunks_dev equals decode_chunks_dev on cv2's frames"""
    import torch
    g = dict(pm.golden_files())
    files = [g[n] for n in FRAMES[mode_val]]
    n = len(files)
    ctx = cb.Context(mode_val, max_frames=n)
    w, h = cb.png_info(files[0])
    d_rgb = torch.empty((n * h * w * 3,), dtype=torch.uint8, device="cuda")
    status = torch.full((n,), 7, dtype=torch.int32, device="cuda")
    out = [torch.full((n * ctx.info.data_bytes,), 0xA5, dtype=torch.uint8, device="cuda") for _ in range(2)]
    mask = [torch.full((n,), -1, dtype=torch.int32, device="cuda") for _ in range(2)]
    torch.cuda.synchronize()
    ctx.png_decode_dev(files, d_rgb.data_ptr(), status.data_ptr())
    ctx.decode_chunks_dev(d_rgb.data_ptr(), n, out[0].data_ptr(), mask[0].data_ptr())
    ref = torch.from_numpy(np.stack([pm.cv2_rgb(f) for f in files]).reshape(-1)).cuda()
    ctx.decode_chunks_dev(ref.data_ptr(), n, out[1].data_ptr(), mask[1].data_ptr())
    ctx.sync()
    assert status.cpu().tolist() == [0] * n
    assert np.array_equal(out[0].cpu().numpy(), out[1].cpu().numpy()) and np.array_equal(mask[0].cpu().numpy(), mask[1].cpu().numpy())
    if mode_val == 68:
        assert (mask[0].cpu().numpy().view(np.uint32) == 0xFFF).all()
    ctx.close()


@pytest.mark.parametrize("g", [g for g in manifest()["goldens"] if g["sample"].endswith(".png")],
                         ids=lambda g: f"{g['sample']}-m{g['mode']}-ecc{int(g['ecc'])}")
def test_reference_sha256_goldens_from_device_png(cb, g):
    name = g["sample"].replace("/", "__")
    data = dict(pm.golden_files())[name]
    ctx = cb.Context(g["mode"], max_frames=1)
    (rgb, st), = decode_dev(cb, ctx, [data])
    assert st == 0
    if g["ecc"]:
        out = ctx.decode(rgb)[0][0]
    else:
        out = ctx.decode_raw(rgb)[0][0]
    assert out.size == g["bytes"]
    assert hashlib.sha256(np.ascontiguousarray(out).tobytes()).hexdigest() == g["sha256"], g["source"]
    ctx.close()


def test_sample_stream_reassembles_from_png_files(cb):
    from oracle_lib import Ref
    try:
        ref = Ref()
    except (FileNotFoundError, OSError) as e:                        # pragma: no cover
        pytest.skip(f"oracle/_ref not available: {e}")
    import torch
    g = dict(pm.golden_files())
    files = [g[n] for n in FRAMES[68]]
    ctx = cb.Context(68, max_frames=4)
    d_rgb = torch.empty((4 * 1024 * 1024 * 3,), dtype=torch.uint8, device="cuda")
    d_chunks = torch.empty((4 * ctx.info.data_bytes,), dtype=torch.uint8, device="cuda")
    d_mask = torch.empty(4, dtype=torch.int32, device="cuda")
    ctx.png_decode_dev(files, d_rgb.data_ptr())
    ctx.decode_chunks_dev(d_rgb.data_ptr(), 4, d_chunks.data_ptr(), d_mask.data_ptr())
    ctx.sync()
    m = ctx.info
    sink = cb.FountainSink(m.chunk_size, ref.lib)
    fid = sink.ingest(d_chunks.cpu().numpy().reshape(4, -1), d_mask.cpu().numpy().astype(np.uint32))
    assert fid > 0
    assert sink.file(fid).size == 23586
    sink.close()
    ctx.close()


def test_calls_only_enqueue(cb):
    """three calls queued behind a sleeping stream return at once and give what the same calls give one at a time"""
    import torch
    files = batches_of(68)[0]
    batches = [files, files[::-1], files]
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    ctx = cb.Context(68, max_frames=len(files))
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    outs = [Outputs(ctx, len(b)) for b in batches]
    torch.cuda.synchronize()
    want = []
    for b, o in zip(batches, outs):                                   # warm-up, one at a time: every buffer at its size
        o.png_call(ctx, b, flags)
        ctx.sync()
        want.append(o.host())
    want_ccm = ctx.get_ccm()
    ctx.set_ccm(None)
    with torch.cuda.stream(stream):
        torch.cuda._sleep(int(1.5e9))
    t0 = time.perf_counter()
    for b, o in zip(batches, outs):
        o.png_call(ctx, b, flags)
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


def test_four_calls_in_flight_equal_one_at_a_time(cb):
    import torch
    files = camera_sized(pm.golden_files() + pm.matrix())
    groups = [[d for _, d in files[k::4]] for k in range(4)]
    ctx = cb.Context(4, max_frames=1)
    want = [decode_dev(cb, ctx, g) for g in groups]
    outs = []
    for g in groups:
        total = sum(3 * w * h for w, h in (cb.png_info(f) for f in g))
        outs.append((torch.full((total,), 0xA5, dtype=torch.uint8, device="cuda"), torch.full((len(g),), 7, dtype=torch.int32, device="cuda")))
    torch.cuda.synchronize()
    for g, (o, s) in zip(groups, outs):
        ctx.png_decode_dev(g, o.data_ptr(), s.data_ptr())
    ctx.sync()
    for w, (o, s) in zip(want, outs):
        assert np.array_equal(o.cpu().numpy(), np.concatenate([r.reshape(-1) for r, _ in w]))
        assert s.cpu().tolist() == [st for _, st in w]
    ctx.close()
