"""k_deskew (libcimbar_b200/csrc/deskew.cu) against cv2.warpPerspective(INTER_LINEAR) pixel for pixel, on the corpus of
deskew_corpus.py: camera-like quads, turns and a mirror, exact ties, tiny and large sources, the horizon inside the frame, w == 0,
coordinates past the short and int ranges, and the scan's own transforms -- in every frame geometry (modes 68, 67, 66), through
the host, device and picture-descriptor entry points, in batches whose frames each have their own picture and transform, and in
every picture layout with padded rows, offset bases and canary bytes around the pictures.  A failure names the first bad pixel
with the kernel's, cv2's and the contract model's values (tests/test_deskew_contract.py pins the model to cv2 on the CPU).

Not reached here: the grid-stride loop over more than 32 768 frames, and the last-bit slips of a missing block origin or FMA
contraction, which change no pixel of any transform tried (the __dmul_rn / __dadd_rn code guards those)."""
import cv2
import numpy as np
import pytest

import deskew_corpus as dc

pytestmark = pytest.mark.gpu

MODES = [68, 67, 66]
KINDS = ["rgb", "bgr", "rgba", "bgra", "planar"]
CH = {"rgb": 3, "bgr": 3, "rgba": 4, "bgra": 4}


@pytest.fixture(scope="module")
def ctxs():
    import libcimbar_b200 as cb
    out = {m: cb.Context(m, max_frames=48) for m in MODES}
    yield out
    for c in out.values():
        c.close()


def geometry(ctx):
    return ctx.info.image_size_x, ctx.info.image_size_y


def check(got, want, src, M, what):
    assert got.shape == want.shape and np.array_equal(got, want), f"{what}: {dc.first_mismatch(got, want, src, M)}"


def frames_dev(ctx, n):
    """n frames of the context's mode in device memory, filled with a value no deskew writes everywhere"""
    import torch
    W, H = geometry(ctx)
    return torch.full((n, H, W, 3), 0xA5, dtype=torch.uint8, device="cuda")


def settled():
    """wait for torch's stream: the context's own stream does not, so the pictures and output frames torch wrote are complete
    before a library call reads or writes them"""
    import torch
    torch.cuda.synchronize()


def deskew_dev(ctx, srcs, ms):
    """cb200_deskew_dev of n pictures of one size (n, h, w, 3) with n transforms -> the frames on the host"""
    import torch
    import libcimbar_b200 as cb
    n, h, w, _ = srcs.shape
    d_src = torch.from_numpy(np.ascontiguousarray(srcs)).cuda()
    d_dst = frames_dev(ctx, n)
    m = np.ascontiguousarray(ms, np.float64).reshape(n, 9)
    settled()
    cb._check(ctx.lib.cb200_deskew_dev(ctx._h, d_src.data_ptr(), w, h, n, m.ctypes.data, d_dst.data_ptr()))
    ctx.sync()
    return d_dst.cpu().numpy()


def place(p, kind, pad, off, fill, rng):
    """picture p (h, w, 3 RGB) in its own buffer as a `kind` tensor: rows padded by `pad` bytes, `off` bytes into the buffer, the
    planes `pad` x 7 + 5 bytes apart, and every byte that is not a pixel (padding, gaps, before and after) = fill.  Alpha is random.
    Returns (tensor, order)"""
    import torch
    h, w, _ = p.shape
    t = torch.from_numpy(np.ascontiguousarray(p))
    if kind == "planar":
        pitch = w + pad
        plane = h * pitch + 7 * pad + 5
        buf = torch.full((off + 2 * plane + h * pitch + 16,), fill, dtype=torch.uint8)
        view = torch.as_strided(buf, (3, h, w), (plane, pitch, 1), off)
        view.copy_(t.permute(2, 0, 1))
        return torch.as_strided(buf.cuda(), (3, h, w), (plane, pitch, 1), off), "rgb"
    ch = CH[kind]
    if kind in ("bgr", "bgra"):
        t = t.flip(2)
    if ch == 4:
        t = torch.cat([t, torch.from_numpy(rng.integers(0, 256, (h, w, 1), dtype=np.uint8))], 2)
    pitch = w * ch + pad
    buf = torch.full((off + h * pitch + 16,), fill, dtype=torch.uint8)
    torch.as_strided(buf, (h, w, ch), (pitch, ch, 1), off).copy_(t)
    return torch.as_strided(buf.cuda(), (h, w, ch), (pitch, ch, 1), off), kind


def deskew_pictures(ctx, pics, ms, kinds, fill, seed=0):
    """cb200_deskew_pictures_dev of the pictures, picture i in layout kinds[i] with row padding i % 14 and base offset i % 4"""
    rng = np.random.default_rng(seed)
    placed = [place(p, k, i % 14, i % 4, fill, rng) for i, (p, k) in enumerate(zip(pics, kinds))]
    d_dst = frames_dev(ctx, len(pics))
    settled()
    ctx.deskew_pictures_dev([t for t, _ in placed], ms, d_dst.data_ptr(), order=[o for _, o in placed])
    ctx.sync()
    return d_dst.cpu().numpy()


@pytest.mark.parametrize("mode", MODES)
def test_corpus_host_and_dev(ctxs, mode):
    ctx = ctxs[mode]
    W, H = geometry(ctx)
    for c in dc.cases(W, H):
        want = dc.cv2_warp(c.src, c.M, W, H)
        check(ctx.deskew(c.src, c.M)[0], want, c.src, c.M, f"cb200_deskew {c.name}")
        check(deskew_dev(ctx, c.src[None], c.M[None])[0], want, c.src, c.M, f"cb200_deskew_dev {c.name}")


def pictures_cases(W, H):
    """the corpus cases whose pictures the pictures call takes (short side 60 .. 4499)"""
    return [c for c in dc.cases(W, H) if 60 <= min(c.src.shape[:2]) <= 4499]


@pytest.mark.parametrize("mode", MODES)
def test_corpus_pictures_in_every_layout_with_canaries(ctxs, mode):
    """the corpus in one batch of mixed sizes and layouts, twice: with 0x00 and with 0xFF in every byte around the pictures"""
    ctx = ctxs[mode]
    W, H = geometry(ctx)
    cs = pictures_cases(W, H)
    assert len(cs) >= 20
    kinds = [KINDS[(i + mode) % len(KINDS)] for i in range(len(cs))]          # each case meets another layout in each mode
    ms = np.stack([c.M for c in cs])
    zeros = deskew_pictures(ctx, [c.src for c in cs], ms, kinds, 0x00)
    ones = deskew_pictures(ctx, [c.src for c in cs], ms, kinds, 0xFF)
    for f, c in enumerate(cs):
        want = dc.cv2_warp(c.src, c.M, W, H)
        check(zeros[f], want, c.src, c.M, f"pictures {kinds[f]} {c.name} (canary 0x00)")
        check(ones[f], want, c.src, c.M, f"pictures {kinds[f]} {c.name} (canary 0xFF)")


@pytest.mark.parametrize("mode", MODES)
def test_corpus_pictures_packed_rgb(ctxs, mode):
    """every descriptor packed RGB (row pitch 3 w): the kernel without the layout code, at base offsets 0 .. 3"""
    import torch
    ctx = ctxs[mode]
    W, H = geometry(ctx)
    cs = pictures_cases(W, H)
    bufs = []
    for i, c in enumerate(cs):
        off = i % 4
        flat = torch.full((off + c.src.size + 16,), 0xFF, dtype=torch.uint8)
        flat[off:off + c.src.size] = torch.from_numpy(c.src.reshape(-1))
        h, w, _ = c.src.shape
        bufs.append(torch.as_strided(flat.cuda(), (h, w, 3), (3 * w, 3, 1), off))
    d_dst = frames_dev(ctx, len(cs))
    settled()
    ctx.deskew_pictures_dev(bufs, np.stack([c.M for c in cs]), d_dst.data_ptr())
    ctx.sync()
    got = d_dst.cpu().numpy()
    for f, c in enumerate(cs):
        check(got[f], dc.cv2_warp(c.src, c.M, W, H), c.src, c.M, f"pictures packed {c.name}")


def distinct_batch(n, W, H, seed):
    """n pictures of 1100 x 900, each its own noise, and n distinct camera-like transforms"""
    rng = np.random.default_rng(seed)
    srcs = rng.integers(0, 256, (n, 900, 1100, 3), dtype=np.uint8)
    ms = np.stack([cv2.getPerspectiveTransform(dc.camera_quad(rng, 1100, 900, i % 2 == 1), dc.output_points(W, H)) for i in range(n)])
    return srcs, ms


@pytest.mark.parametrize("n", [1, 5, 48])
def test_batches_of_distinct_transforms(ctxs, n):
    """frame f is picture f under transform f, through every entry point"""
    ctx = ctxs[68]
    W, H = geometry(ctx)
    srcs, ms = distinct_batch(n, W, H, n)
    host = ctx.deskew(srcs, ms)
    dev = deskew_dev(ctx, srcs, ms)
    pics = deskew_pictures(ctx, list(srcs), ms, [KINDS[f % len(KINDS)] for f in range(n)], 0x00, seed=n)
    for f in range(n):
        want = dc.cv2_warp(srcs[f], ms[f], W, H)
        for name, got in (("cb200_deskew", host), ("cb200_deskew_dev", dev), ("cb200_deskew_pictures_dev", pics)):
            check(got[f], want, srcs[f], ms[f], f"{name} frame {f} of {n}")


def test_mixed_sizes_in_one_launch(ctxs):
    """48 pictures of 48 sizes, landscape and portrait, in one call: frame f reads picture f's size, pitch and layout"""
    ctx = ctxs[66]
    W, H = geometry(ctx)
    rng = np.random.default_rng(48)
    pics, ms = [], []
    for f in range(48):
        w, h = int(rng.integers(60, 1500)), int(rng.integers(60, 1500))
        pics.append(rng.integers(0, 256, (h, w, 3), dtype=np.uint8))
        ms.append(cv2.getPerspectiveTransform(dc.camera_quad(rng, w, h, f % 3 == 0), dc.output_points(W, H)))
    got = deskew_pictures(ctx, pics, np.stack(ms), [KINDS[f % len(KINDS)] for f in range(48)], 0xFF, seed=1)
    for f in range(48):
        check(got[f], dc.cv2_warp(pics[f], ms[f], W, H), pics[f], ms[f], f"frame {f} ({pics[f].shape[1]} x {pics[f].shape[0]})")


def test_the_camera_paths_transforms(ctxs):
    """the transforms a pictures camera call reports (cb200_camera_transforms), fed back to the pictures deskew, give cv2's frames"""
    import torch
    from gpu_support import as_tensor
    from oracle_lib import load_sample
    ctx = ctxs[68]
    W, H = geometry(ctx)
    names = ["b/ex2434.jpg", "b/ex380.jpg", "6bit/4_30_f0_627.jpg", "6bit/4_30_f2_734.jpg", "6bit/4_30_f1_360.jpg", "b/tr_0.png"]
    pics = [load_sample(s) for s in names]
    pics.append(np.ascontiguousarray(np.rot90(pics[0])))
    kinds = ["rgb", "bgr", "planar", "pitched", "rgba", "bgra", "rgb"]
    placed = [as_tensor(p, k) for p, k in zip(pics, kinds)]
    ts, orders = [t for t, _ in placed], [o for _, o in placed]
    n = len(ts)
    chunks = torch.zeros((n, ctx.info.data_bytes), dtype=torch.uint8, device="cuda")
    mask = torch.zeros(n, dtype=torch.int32, device="cuda")
    status = torch.zeros(n, dtype=torch.int32, device="cuda")
    settled()
    ctx.scan_extract_decode_chunks_pictures_dev(ts, chunks.data_ptr(), mask.data_ptr(), status.data_ptr(), order=orders)
    ctx.sync()
    ms = ctx.camera_transforms(n)
    st = status.cpu().numpy()
    assert (st[:len(names)] >= 1).all(), st                       # every sample photograph extracts: its own transform, not a fallback
    d_dst = frames_dev(ctx, n)
    settled()
    ctx.deskew_pictures_dev(ts, ms, d_dst.data_ptr(), order=orders)
    ctx.sync()
    got = d_dst.cpu().numpy()
    for f in range(n):
        check(got[f], dc.cv2_warp(pics[f], ms[f], W, H), pics[f], ms[f], f"camera transform of {names[f] if f < len(names) else 'rot90'}")


def test_pictures_call_refusals_with_a_context(ctxs):
    import torch
    import libcimbar_b200 as cb
    ctx = ctxs[68]
    t = torch.zeros((100, 120, 3), dtype=torch.uint8, device="cuda")
    d_dst = frames_dev(ctx, 2)
    settled()
    with pytest.raises(cb.Cb200Error, match="singular perspective transform"):
        ctx.deskew_pictures_dev([t, t], np.stack([np.eye(3), np.zeros((3, 3))]), d_dst.data_ptr())
    with pytest.raises(cb.Cb200Error, match="1 transforms for 2 pictures"):
        ctx.deskew_pictures_dev([t, t], np.eye(3), d_dst.data_ptr())
    ctx.deskew_pictures_dev([], np.zeros((0, 9)), d_dst.data_ptr())          # n = 0: nothing to do
    ctx.sync()
    assert (d_dst.cpu().numpy() == 0xA5).all()
