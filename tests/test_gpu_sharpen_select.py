"""Per-frame sharpen selection inside one batch (cb200_decode_chunks_sharpen_dev / cb200_decode_fountain_sharpen and
CB200_FLAG_SHARPEN_IF_NEEDED on the camera entry points): every frame must decode exactly as the oracle decodes it with its own
should_preprocess, in batch order for the CCM carry of color_correction 2, and the camera path must equal the reference CLI's
default `--preprocess -1` loop (scan, warp, decode with sharpen iff Extractor::extract said NEEDS_SHARPEN)."""
import cv2
import numpy as np
import pytest

from oracle_lib import load_sample
from scan_oracle_lib import ScanOracle
from test_gpu_parity import ORA, synth_frames

pytestmark = pytest.mark.gpu

MODES = [68, 4, 8, 67, 66]
POOL = 12                  # per mode: 4 clean frames, 4 with 1 % noise tiles (exact walk), 4 blurred (sigma 1.6) + noise
_pools, _oracle = {}, {}


@pytest.fixture(scope="module")
def cb():
    import libcimbar_b200 as cb
    return cb


def pool(mode_val):
    if mode_val not in _pools:
        m, _, clean = synth_frames(mode_val, 4, seed=700 + mode_val)
        noisy = synth_frames(mode_val, 4, seed=710 + mode_val, error_rate=0.01, noise_tiles=True)[2]
        base = synth_frames(mode_val, 4, seed=720 + mode_val)[2]
        rng = np.random.default_rng(730 + mode_val)
        blurred = []
        for b in base:
            b = cv2.GaussianBlur(b, (0, 0), 1.6).astype(np.int16) + np.rint(rng.normal(0, 6, b.shape)).astype(np.int16)
            blurred.append(np.clip(b, 0, 255).astype(np.uint8))
        _pools[mode_val] = (m, np.concatenate([clean, noisy, np.stack(blurred)]))
    return _pools[mode_val]


def oracle(mode_val, p, sharpen, cc):
    """Decoder::decode_fountain of pool frame p by a fresh reference decoder: (good bytes, dense chunks, chunk mask)"""
    key = (mode_val, p, bool(sharpen), cc)
    if key not in _oracle:
        m, frames = pool(mode_val)
        ORA.set_ccm(None)
        try:
            good, chunks, mask = ORA.decode_fountain(m, frames[p], sharpen=bool(sharpen), color_correction=cc)
        finally:
            ORA.set_ccm(None)
        _oracle[key] = (good, chunks.copy(), mask)
    return _oracle[key]


def selection(mode_val, n, seed):
    """a seeded batch over the pool (every pool frame at least twice) and an irregular sharpen choice"""
    rng = np.random.default_rng(seed + mode_val)
    idx = np.concatenate([np.arange(POOL), np.arange(POOL), rng.integers(0, POOL, n - 2 * POOL)])
    rng.shuffle(idx)
    return idx, rng.random(n) < 0.5


def differs(mode_val, p, cc=0):
    a, b = oracle(mode_val, p, False, cc), oracle(mode_val, p, True, cc)
    return a[2] != b[2] or not np.array_equal(a[1], b[1])


def check_dense(m, chunks, count, mask, want, what):
    good, wchunks, wmask = want
    assert mask == wmask and count * m.chunk_size == good, what
    assert np.array_equal(chunks[:count], wchunks[:count]), what


def dense(m, slots, mask):
    """the fixed-slot records of cb200_decode_chunks_dev as escrow_buffer_writer's dense order"""
    rows = slots.reshape(m.chunks_per_frame, m.chunk_size)
    keep = [q for q in range(m.chunks_per_frame) if mask >> q & 1]
    return len(keep), rows[keep]


def premise(mode_val, idx, sel):
    # some frames of each kind decode differently under the other choice
    assert any(differs(mode_val, int(p)) for p, s in zip(idx, sel) if s)
    assert any(differs(mode_val, int(p)) for p, s in zip(idx, sel) if not s)


# ------------------------------------------------------------------------------------------------ frame level
@pytest.mark.parametrize("mode_val", MODES)
def test_mixed_selection_matches_oracle_every_mode(cb, mode_val):
    """a 40-frame batch (both kinds in K1's band schedule) with an irregular selection, colour correction 0 and 1 and, where the
    reference fits a CCM, 2 against the oracle decoding the batch in order with one decoder state"""
    m, frames = pool(mode_val)
    n = 40
    idx, sel = selection(mode_val, n, 11)
    batch = frames[idx]
    premise(mode_val, idx, sel)
    ctx = cb.Context(mode_val, max_frames=n)
    assert (~sel).sum() < ctx.info.sm_count * 4 and sel.sum() < ctx.info.sm_count * 3          # both lists run in bands
    for cc, ccf in ((0, 0), (1, cb.FLAG_CC_SIMPLE)):
        chunks, count, mask, ff = ctx.decode_fountain(batch, flags=ccf, sharpen=sel)
        for f in range(n):
            check_dense(m, chunks[f], count[f], mask[f], oracle(mode_val, int(idx[f]), sel[f], cc), (cc, f))
        if cc == 0:
            # frame flags: those of the uniform call of the frame's own kind; both exact-walk rasters had frames
            ff0 = ctx.decode_fountain(batch, flags=ccf)[3]
            ff1 = ctx.decode_fountain(batch, flags=ccf | cb.FLAG_SHARPEN)[3]
            assert np.array_equal(ff, np.where(sel, ff1, ff0))
            assert (ff[sel] & cb.FRAME_FALLBACK).any() and (ff[~sel] & cb.FRAME_FALLBACK).any()
    if mode_val in (68, 67, 66):
        ctx.set_ccm(None)
        chunks, count, mask, ff = ctx.decode_fountain(batch, flags=cb.FLAG_CC_FIT, sharpen=sel)
        ORA.set_ccm(None)
        try:
            for f in range(n):
                want = ORA.decode_fountain(m, batch[f], sharpen=bool(sel[f]), color_correction=2)
                check_dense(m, chunks[f], count[f], mask[f], want, (2, f))
            last = ORA.get_ccm()
        finally:
            ORA.set_ccm(None)
        got = ctx.get_ccm()
        assert (got is None) == (last is None) and (last is None or np.array_equal(got, last))
    ctx.close()


def _device_batch(mode_val, idx):
    import torch
    m, frames = pool(mode_val)
    dev = torch.device("cuda")
    return m, torch.from_numpy(frames).to(dev)[torch.from_numpy(idx).to(dev)].contiguous()


def _decode_dev(ctx, d_frames, n, flags=0, sharpen=None):
    import torch
    chunks = torch.empty((n, ctx.info.data_bytes), dtype=torch.uint8, device=d_frames.device)
    mask = torch.empty(n, dtype=torch.int32, device=d_frames.device)
    ff = torch.empty(n, dtype=torch.uint8, device=d_frames.device)
    ctx.decode_chunks_dev(d_frames.data_ptr(), n, chunks.data_ptr(), mask.data_ptr(), ff.data_ptr(), flags=flags, sharpen=sharpen)
    ctx.sync()
    return chunks.cpu().numpy(), mask.cpu().numpy().astype(np.uint32), ff.cpu().numpy()


def test_mixed_selection_in_the_whole_frame_schedule(cb):
    """both lists long enough for K1's whole-frame schedule (length >= SMs x CTAs per SM of their kind), through the enqueue-only
    device entry point; the selection array is overwritten right after the call returns"""
    sm = cb.Context(68, max_frames=1).info.sm_count
    n = 9 * sm
    idx, _ = selection(68, n, 23)
    sel = np.zeros(n, bool)
    sel[np.random.default_rng(29).permutation(n)[:n // 2]] = True
    assert (~sel).sum() >= sm * 4 and sel.sum() >= sm * 3
    premise(68, idx, sel)
    m, d_frames = _device_batch(68, idx)
    ctx = cb.Context(68, max_frames=n)
    import torch
    chunks = torch.empty((n, ctx.info.data_bytes), dtype=torch.uint8, device=d_frames.device)
    mask = torch.empty(n, dtype=torch.int32, device=d_frames.device)
    ff = torch.empty(n, dtype=torch.uint8, device=d_frames.device)
    arg = sel.astype(np.uint8)
    ctx.lib.cb200_decode_chunks_sharpen_dev(ctx._h, d_frames.data_ptr(), n, 0, arg.ctypes.data, chunks.data_ptr(), mask.data_ptr(), ff.data_ptr())
    arg[:] = 1 - arg                                                      # the caller may reuse its array at once
    ctx.sync()
    chunks, mask, ff = chunks.cpu().numpy(), mask.cpu().numpy().astype(np.uint32), ff.cpu().numpy()
    for f in range(n):
        cnt, rows = dense(m, chunks[f], mask[f])
        check_dense(m, rows, cnt, mask[f], oracle(68, int(idx[f]), sel[f], 0), f)
    assert (ff[sel] & cb.FRAME_FALLBACK).any() and (ff[~sel] & cb.FRAME_FALLBACK).any()
    ctx.close()


@pytest.mark.parametrize("few", [True, False], ids=["bands", "whole-frames"])
def test_degenerate_selections_are_the_uniform_calls(cb, few):
    """all zero == the call without CB200_FLAG_SHARPEN, all one == the call with it, bit for bit, in each K1 schedule"""
    sm = cb.Context(68, max_frames=1).info.sm_count
    n = 30 if few else 5 * sm
    idx, _ = selection(68, n, 31)
    m, d_frames = _device_batch(68, idx)
    ctx = cb.Context(68, max_frames=n)
    for bit, flags in ((0, 0), (1, cb.FLAG_SHARPEN)):
        want = _decode_dev(ctx, d_frames, n, flags=flags)
        got = _decode_dev(ctx, d_frames, n, sharpen=np.full(n, bit, np.uint8))
        for w, g in zip(want, got):
            assert np.array_equal(w, g), bit
        assert (got[2] & cb.FRAME_FALLBACK).any()
    ctx.close()


# ------------------------------------------------------------------------------------------------ camera path
def _camera_batch():
    """1440 x 1920 pictures: 1.5x upscales of the landscape sample photographs (SUCCESS), the same photographs zero-padded to that
    size (NEEDS_SHARPEN) and a noise picture (FAILURE)"""
    cams = [load_sample(s) for s in ("6bit/4_30_f0_627.jpg", "6bit/4_30_f2_246.jpg")]      # 960 x 1280
    pics = []
    for cam in cams:
        h, w = cam.shape[:2]
        pics.append(cv2.resize(cam, None, fx=1.5, fy=1.5))
        pics.append(cv2.copyMakeBorder(cam, h // 4, h // 2 - h // 4, w // 4, w // 2 - w // 4, cv2.BORDER_CONSTANT, value=(0, 0, 0)))
    noise = np.random.default_rng(3).integers(0, 256, pics[0].shape, dtype=np.uint8)
    return np.stack([pics[0], pics[1], noise, pics[3], pics[2]])


def _cli_loop(m, pics, cc):
    """the reference CLI's decode loop with --preprocess -1: scan, Corners, warp, decode with sharpen iff NEEDS_SHARPEN, one
    decoder state in picture order; FAILURE pictures are skipped"""
    so = ScanOracle()
    an, W, H = 30, m.image_size_x, m.image_size_y
    dst = np.array([[an, an], [W - an, an], [an, H - an], [W - an, H - an]], np.float32)
    out = []
    ORA.set_ccm(None)
    try:
        for rgb in pics:
            anchors, _ = so.scan(rgb)
            if anchors is None or len(anchors) < 4:
                out.append((0, None, None))
                continue
            xy = so.corners(anchors)
            status = 1 if so.is_granular_scale(xy, W, H) else 2
            frame = cv2.warpPerspective(rgb, cv2.getPerspectiveTransform(np.array(xy, np.float32).reshape(4, 2), dst), (W, H),
                                        flags=cv2.INTER_LINEAR)
            good, chunks, mask = ORA.decode_fountain(m, frame, sharpen=status == 2, color_correction=cc)
            out.append((status, xy, (good, chunks.copy(), mask)))
    finally:
        ORA.set_ccm(None)
    return out


def test_camera_batch_matches_the_cli_loop(cb):
    import torch
    pics = _camera_batch()
    n = len(pics)
    m = ORA.mode(4)
    for cc, ccf in ((0, 0), (2, cb.FLAG_CC_FIT)):
        want = _cli_loop(m, pics, cc)
        assert sorted({w[0] for w in want}) == [0, 1, 2]
        assert any(w[0] == 2 and w[2][0] > 0 for w in want)
        ctx = cb.Context(4, max_frames=n)
        chunks, count, mask, ff, status = ctx.scan_extract_decode_fountain(pics, flags=cb.FLAG_SHARPEN_IF_NEEDED | ccf)
        assert status.tolist() == [w[0] for w in want]
        for i, (st, xy, wd) in enumerate(want):
            if st == 0:
                assert count[i] == 0 and mask[i] == 0
            else:
                check_dense(m, chunks[i], count[i], mask[i], wd, (cc, i))
        # the corner-taking device entry point decides from the corners it is given (the oracle's) -- the same batch minus the
        # picture without anchors
        keep = [i for i, w in enumerate(want) if w[0]]
        d_src = torch.from_numpy(pics[keep]).cuda()
        corners = np.array([want[i][1] for i in keep], np.float32)
        k = len(keep)
        ch = np.zeros((k, m.chunks_per_frame, m.chunk_size), np.uint8)
        cnt, mk, fl = np.zeros(k, np.uint32), np.zeros(k, np.uint32), np.zeros(k, np.uint8)
        ctx2 = cb.Context(4, max_frames=n)
        rc = ctx2.lib.cb200_extract_decode_fountain_dev(ctx2._h, d_src.data_ptr(), pics.shape[2], pics.shape[1], k, corners.ctypes.data,
                                                        cb.FLAG_SHARPEN_IF_NEEDED | ccf, ch.ctypes.data, cnt.ctypes.data,
                                                        mk.ctypes.data, fl.ctypes.data)
        assert rc == 0, ctx2.lib.cb200_last_error()
        for j, i in enumerate(keep):
            check_dense(m, ch[j], cnt[j], mk[j], want[i][2], (cc, i))
        ctx.close()
        ctx2.close()


# ------------------------------------------------------------------------------------------------ C++ mirror
def test_cpp_decoder_per_frame_overload(cb, tmp_path):
    """tests/cpp/decoder_sharpen_test.cpp: Decoder::decode_fountain(imgs, n, stream, const bool* should_preprocess, cc) equals
    single-frame calls on one Decoder (with and without ECC, color_correction 0 / 1 / 2); its chunks under color_correction 2
    equal the oracle decoding the frames in order with one decoder state, each with its own should_preprocess"""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / "decoder_sharpen_test")
    libdir = os.path.join(root, "libcimbar_b200", "lib")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-o", exe, os.path.join(root, "tests", "cpp", "decoder_sharpen_test.cpp"),
                           "-L" + libdir, "-lcb200", "-Wl,-rpath," + libdir])
    m, frames = pool(68)
    batch = np.stack([load_sample("b/tr_0.png"), load_sample("b/ex2434.jpg"), frames[8], load_sample("b/ex380.jpg"),
                      load_sample("b/tr_1.png"), frames[4], frames[9]])
    pattern = "0110101"
    sel = [c == "1" for c in pattern]
    assert differs(68, 8) and differs(68, 9)                              # the blurred frames decode differently either way
    batch.tofile(str(tmp_path / "frames.rgb"))
    prefix = str(tmp_path / "out")
    res = subprocess.run([exe, "68", str(tmp_path / "frames.rgb"), pattern, prefix], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    want = []
    ORA.set_ccm(None)
    try:
        for fr, s in zip(batch, sel):
            good, chunks, _ = ORA.decode_fountain(m, fr, sharpen=s, color_correction=2)
            want.append(chunks.reshape(-1)[:good])
    finally:
        ORA.set_ccm(None)
    assert np.array_equal(np.fromfile(prefix + ".chunks_cc2", dtype=np.uint8), np.concatenate(want))
