"""GPU parity tests (run on an H100: pytest -m gpu).  Everything goes through the C ABI of libcb200.so and is
compared bit for bit with the CPU oracle (itself pinned to the reference's goldens, tests/test_oracle_goldens.py),
with the reference's SHA-256 goldens directly, and with size-independent round-trip properties."""
import ctypes as C
import hashlib

import numpy as np
import pytest

from oracle_lib import load_sample, manifest, _ptr
from gpu_support import cb  # noqa: F401  (fixtures)
from gpu_support import ORA, synth_frames, tint

pytestmark = pytest.mark.gpu


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


# ------------------------------------------------------------------------------------------------ goldens
@pytest.mark.parametrize("g", [g for g in manifest()["goldens"] if g["sample"] != "b/scan2434.jpg"],
                         ids=lambda g: f"{g['sample']}-m{g['mode']}-ecc{int(g['ecc'])}")
def test_reference_sha256_goldens_on_gpu(cb, g):
    # src/lib/encoder/test/DecoderTest.cpp:26-106, including the camera JPEG that needs the exact flood walk
    ctx = cb.Context(g["mode"], max_frames=1)
    rgb = load_sample(g["sample"])
    if g["ecc"]:
        data, ok, ff = ctx.decode(rgb)
        out = data[0]
    else:
        raw, ff = ctx.decode_raw(rgb)
        out = raw[0]
    assert out.size == g["bytes"]
    assert sha(out) == g["sha256"], g["source"]
    if g["sample"].endswith(".jpg"):
        assert ff[0] & cb.FRAME_FALLBACK
    ctx.close()


def test_camera_frame_mode_b_matches_oracle(cb):
    ctx = cb.Context(68, max_frames=1)
    rgb = load_sample("b/ex2434.jpg")
    raw, ff = ctx.decode_raw(rgb)
    assert ff[0] & cb.FRAME_FALLBACK
    assert np.array_equal(raw[0], ORA.decode_raw(ORA.mode(68), rgb))
    data, ok, _ = ctx.decode(rgb)
    odata, ook = ORA.decode(ORA.mode(68), rgb)
    assert np.array_equal(data[0], odata) and np.array_equal(ok[0], ook)
    ctx.close()


def test_sharpen_flag_matches_oracle(cb):
    ctx = cb.Context(68, max_frames=1)
    for name in ("b/ex2434.jpg", "b/tr_0.png"):
        rgb = load_sample(name)
        raw, ff = ctx.decode_raw(rgb, flags=cb.FLAG_SHARPEN)
        assert np.array_equal(raw[0], ORA.decode_raw(ORA.mode(68), rgb, sharpen=True)), name
    ctx.close()


def test_sample_stream_chunks(cb):
    # samples/b/tr_0..3.png: every chunk decodes; headers carry encode_id 0, size 23586, distinct block ids
    ctx = cb.Context(68, max_frames=4)
    frames = np.stack([load_sample(f"b/tr_{k}.png") for k in range(4)])
    chunks, count, mask, ff = ctx.decode_fountain(frames)
    assert count.tolist() == [12] * 4 and mask.tolist() == [0xFFF] * 4 and not ff.any()
    m = ORA.mode(68)
    for k in range(4):
        good, ochunks, omask = ORA.decode_fountain(m, frames[k])
        assert good == 7500 and np.array_equal(chunks[k], ochunks)
    ids = sorted(int(c[4]) << 8 | int(c[5]) for c in chunks.reshape(-1, 625))
    assert len(set(ids)) == 48
    ctx.close()


# ------------------------------------------------------------------------------------------------ synthetic frames
@pytest.mark.parametrize("mode_val", [68, 4, 8, 67, 66])
def test_clean_synthetic_frames_all_modes(cb, mode_val):
    m, payloads, frames = synth_frames(mode_val, 3, seed=mode_val)
    ctx = cb.Context(mode_val, max_frames=3)
    raw, ff = ctx.decode_raw(frames)
    assert not ff.any()
    for f in range(3):
        assert np.array_equal(raw[f], ORA.decode_raw(m, frames[f])), (mode_val, f)
    data, ok, _ = ctx.decode(frames)
    assert ok.all() and np.array_equal(data, payloads)
    ctx.close()


@pytest.mark.parametrize("n", [1, 2, 7, 200])
def test_band_splitting_is_invisible(cb, n):
    # few frames are split into bands of cell rows, many frames are processed whole: same bits either way
    m, payloads, frames = synth_frames(68, min(n, 8), seed=100 + n)
    reps = (n + frames.shape[0] - 1) // frames.shape[0]
    big = np.concatenate([frames] * reps)[:n]
    ctx = cb.Context(68, max_frames=n)
    raw, ff = ctx.decode_raw(big)
    assert not ff.any()
    want = np.stack([ORA.decode_raw(m, fr) for fr in frames])
    for f in range(n):
        assert np.array_equal(raw[f], want[f % frames.shape[0]]), f
    ctx.close()


@pytest.mark.parametrize("mode_val", [68, 4, 8, 66, 67])
def test_whole_frame_schedule_every_mode(cb, mode_val):
    """n >= 4 x SMs switches K1 from band-split CTAs to the persistent whole-frame schedule the bench runs in (api.cu
    run_cells); every mode -- incl. the non-1024x1024 geometries 66 (736x637) and 67 (1024x720) and the legacy coupled
    layouts 4C / 8C (Decoder.h:121-161, GridConf.h:144-189) -- must give the same bits there as the oracle."""
    m, payloads, frames = synth_frames(mode_val, 5, seed=200 + mode_val)
    n = 640                                                     # > 4 x 132 CTAs (H100)
    big = np.concatenate([frames] * (n // 5))
    ctx = cb.Context(mode_val, max_frames=n)
    assert n >= 4 * ctx.info.sm_count, "test sized for <= 160 SMs"
    raw, ff = ctx.decode_raw(big)
    assert not ff.any()
    want = np.stack([ORA.decode_raw(m, fr) for fr in frames])
    assert np.array_equal(raw.reshape(n // 5, 5, -1), np.broadcast_to(want, (n // 5,) + want.shape))
    data, ok, _ = ctx.decode(big)
    assert ok.all() and np.array_equal(data.reshape(n // 5, 5, -1), np.broadcast_to(payloads, (n // 5,) + payloads.shape))
    ctx.close()


def test_config3_256_frames_match_oracle(cb):
    """BASELINE configs[2] at a size where a systematic slip would show: 256 distinct frames with 1 % wrong (valid) tiles,
    raw bits, RS-corrected bytes and per-block ok flags against the oracle frame by frame"""
    n = 256
    m, payloads, frames = synth_frames(68, n, seed=77, error_rate=0.01)
    ctx = cb.Context(68, max_frames=n)
    raw, ff = ctx.decode_raw(frames)
    data, ok, _ = ctx.decode(frames)
    chunks, count, mask, _ = ctx.decode_fountain(frames)
    assert not ff.any()                                          # valid tiles keep the drift-0 proof intact
    for f in range(n):
        assert np.array_equal(raw[f], ORA.decode_raw(m, frames[f])), f
        odata, ook = ORA.decode(m, frames[f])
        assert np.array_equal(ok[f], ook) and np.array_equal(data[f], odata), f
    assert ok.all() and np.array_equal(data, payloads) and (mask == 0xFFF).all() and (count == 12).all()
    ctx.close()


@pytest.mark.parametrize("mode_val,rate", [(4, 0.01), (4, 0.045), (8, 0.01), (67, 0.01), (66, 0.01)])
def test_other_modes_with_tile_errors_match_oracle(cb, mode_val, rate):
    """BASELINE configs[4] (legacy 4C: coupled 6-bit layout, 10 chunks x 750 B, one RS stream) and the other modes with
    wrong tiles: RS repairs (1 %) or gives up on some blocks (4.5 %) exactly where libcorrect does"""
    n = 48
    m, payloads, frames = synth_frames(mode_val, n, seed=90 + mode_val, error_rate=rate)
    ctx = cb.Context(mode_val, max_frames=n)
    raw, ff = ctx.decode_raw(frames)
    data, ok, _ = ctx.decode(frames)
    chunks, count, mask, _ = ctx.decode_fountain(frames)
    nfail = 0
    for f in range(n):
        assert np.array_equal(raw[f], ORA.decode_raw(m, frames[f])), f
        odata, ook = ORA.decode(m, frames[f])
        assert np.array_equal(ok[f], ook) and np.array_equal(data[f], odata), f
        good, ochunks, omask = ORA.decode_fountain(m, frames[f])
        assert mask[f] == omask and count[f] * m.chunk_size == good, f
        assert np.array_equal(chunks[f][:count[f]], ochunks[:count[f]]), f
        nfail += int((ook == 0).sum())
    if rate <= 0.01:
        assert ok.all() and np.array_equal(data, payloads)
    else:
        assert nfail > 0
    ctx.close()


def test_one_percent_tile_errors_config3(cb):
    # BASELINE config 3: 1 % of cells replaced by a different valid tile -> RS repairs everything
    m, payloads, frames = synth_frames(68, 6, seed=7, error_rate=0.01)
    ctx = cb.Context(68, max_frames=6)
    raw, ff = ctx.decode_raw(frames)
    data, ok, _ = ctx.decode(frames)
    for f in range(6):
        assert np.array_equal(raw[f], ORA.decode_raw(m, frames[f]))
        odata, ook = ORA.decode(m, frames[f])
        assert np.array_equal(data[f], odata) and np.array_equal(ok[f], ook)
    assert ok.all() and np.array_equal(data, payloads)
    ctx.close()


@pytest.mark.parametrize("rate,mode_val", [pytest.param(r, mv, id=str(r) if mv == 68 else f"{r}-m{mv}")
                                            for mv in (68, 4, 8, 66, 67) for r in (0.01, 0.08)])
def test_noise_tiles_and_rs_failures_match_oracle(cb, mode_val, rate):
    """noise tiles break the centre-wins proof (-> exact walk, k_flood_raster_fast on every geometry, k_flood_colour with every
    palette) and, at 8 %, overwhelm RS: good/bad masks must match; then colour correction 1 (one matrix per frame) on the walk"""
    m, payloads, frames = synth_frames(mode_val, 4, seed=11, error_rate=rate, noise_tiles=True)
    ctx = cb.Context(mode_val, max_frames=4)
    raw, ff = ctx.decode_raw(frames)
    assert all(int(x) & cb.FRAME_FALLBACK for x in ff)
    data, ok, _ = ctx.decode(frames)
    chunks, count, mask, _ = ctx.decode_fountain(frames)
    for f in range(4):
        assert np.array_equal(raw[f], ORA.decode_raw(m, frames[f])), f
        odata, ook = ORA.decode(m, frames[f])
        assert np.array_equal(ok[f], ook) and np.array_equal(data[f], odata)
        good, ochunks, omask = ORA.decode_fountain(m, frames[f])
        assert mask[f] == omask and count[f] * m.chunk_size == good
        assert np.array_equal(chunks[f][:count[f]], ochunks[:count[f]])
    tinted = tint(frames, (0.75, 1.0, 0.85))
    raw1, ff1 = ctx.decode_raw(tinted, flags=cb.FLAG_CC_SIMPLE)
    assert all(int(x) & cb.FRAME_FALLBACK for x in ff1)
    try:
        for f in range(4):
            assert np.array_equal(raw1[f], ORA.decode_raw(m, tinted[f], color_correction=1)), f
    finally:
        ORA.set_ccm(None)
    ctx.close()


def test_large_batch_round_trip_property(cb):
    # size-independent property at scale: encode -> render on device -> decode == payload for every frame
    import torch
    n = 1024
    m = ORA.mode(68)
    rng = np.random.default_rng(5)
    payloads = rng.integers(0, 256, (n, 7500), dtype=np.uint8)
    cells = np.stack([ORA.payload_to_cells(m, p) for p in payloads])
    ctx = cb.Context(68, max_frames=n)
    d_cells = torch.from_numpy(cells).cuda()
    d_rgb = torch.empty((n, 1024, 1024, 3), dtype=torch.uint8, device="cuda")
    d_chunks = torch.empty((n, 7500), dtype=torch.uint8, device="cuda")
    d_mask = torch.empty(n, dtype=torch.int32, device="cuda")
    d_flags = torch.empty(n, dtype=torch.uint8, device="cuda")
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    ctx.set_stream(stream.cuda_stream)
    ctx.render_frames_dev(d_cells.data_ptr(), n, d_rgb.data_ptr())
    ctx.decode_chunks_dev(d_rgb.data_ptr(), n, d_chunks.data_ptr(), d_mask.data_ptr(), d_flags.data_ptr())
    torch.cuda.synchronize()
    assert (d_mask.cpu().numpy() == 0xFFF).all() and not d_flags.cpu().numpy().any()
    assert np.array_equal(d_chunks.cpu().numpy(), payloads)
    # the device renderer is the oracle's renderer
    assert np.array_equal(d_rgb[3].cpu().numpy(), ORA.render_frame(m, cells[3]))
    ctx.close()


# ------------------------------------------------------------------------------------------------ Reed-Solomon
@pytest.mark.parametrize("mode_val", [68, 4, 67, 66])
def test_rs_kernel_matches_libcorrect_semantics(cb, mode_val):
    import torch
    m = ORA.mode(mode_val)
    rng = np.random.default_rng(mode_val + 1)
    cap, block, parity = ORA.capacity(m), m.ecc_block_size, m.ecc_bytes
    msg, nblocks = block - parity, ORA.capacity(m) // m.ecc_block_size
    n = 24
    raws = np.zeros((n, cap), np.uint8)
    rs = ORA.lib.cbo_rs_create(parity)
    enc = np.zeros(255, np.uint8)
    t = parity // 2
    for f in range(n):
        for b in range(nblocks):
            p = rng.integers(0, 256, msg, dtype=np.uint8)
            ORA.lib.cbo_rs_encode(rs, _ptr(p), msg, _ptr(enc))
            blk = enc[:block].copy()
            kind = (f * nblocks + b) % 7
            nerr = [0, 1, t, t + 1, int(rng.integers(0, parity + 6)), t - 1, int(rng.integers(0, 4))][kind]
            pos = rng.choice(block, nerr, replace=False)
            blk[pos] ^= rng.integers(1, 256, nerr, dtype=np.uint8)
            if (f * nblocks + b) % 53 == 0:
                blk = rng.integers(0, 256, block, dtype=np.uint8)
            raws[f, b * block:(b + 1) * block] = blk
    ORA.lib.cbo_rs_destroy(rs)
    ctx = cb.Context(mode_val, max_frames=n)
    d_raw = torch.from_numpy(raws).cuda()
    d_data = torch.zeros((n, nblocks * msg), dtype=torch.uint8, device="cuda")
    d_ok = torch.zeros((n, nblocks), dtype=torch.uint8, device="cuda")
    ctx.rs_correct_dev(d_raw.data_ptr(), n, d_data.data_ptr(), d_ok.data_ptr())
    ctx.sync()
    data, ok = d_data.cpu().numpy(), d_ok.cpu().numpy()
    nfail = 0
    for f in range(n):
        if m.legacy_mode:
            odata, ook = ORA.rs_stream(parity, block, raws[f])
        else:
            cs = ORA.capacity(m, m.symbol_bits)
            o1, k1 = ORA.rs_stream(parity, block, raws[f, :cs])
            o2, k2 = ORA.rs_stream(parity, block, raws[f, cs:])
            odata, ook = np.concatenate([o1, o2]), np.concatenate([k1, k2])
        assert np.array_equal(ok[f], ook), f
        assert np.array_equal(data[f], odata), f
        nfail += int((ook == 0).sum())
    assert nfail > 0
    ctx.close()


# ------------------------------------------------------------------------------------------------ single-cell API
def test_decode_symbols_matches_oracle(cb):
    rng = np.random.default_rng(3)
    n = 4000
    windows = rng.integers(0, 1024, (n, 10), dtype=np.uint16)
    # half of the windows: exact tiles embedded with a random drift, the rest pure noise
    ORA.lib.cbo_tile_hashes.restype = C.POINTER(C.c_uint64)
    T = ORA.lib.cbo_tile_hashes()
    for i in range(0, n, 2):
        t = int(T[int(rng.integers(0, 16))])
        dx, dy = int(rng.integers(0, 3)), int(rng.integers(0, 3))
        rows = [int(rng.integers(0, 1024)) for _ in range(10)]
        for r in range(8):
            byte = (t >> (8 * (7 - r))) & 0xFF
            rows[dy + r] = (rows[dy + r] & ~(0xFF << (2 - dx))) | (byte << (2 - dx))
        windows[i] = rows
    cooldown = rng.choice(np.array([0xFF, 0xFE, 1, 3, 4, 5, 7], dtype=np.uint8), n)
    ctx = cb.Context(68, max_frames=1)
    sym, off, dist = ctx.decode_symbols(windows, cooldown)
    hashes = (C.c_uint64 * 9)()
    doff, ddist = C.c_uint(0), C.c_uint(0)
    for i in range(n):
        # build a 10x10 MSB-first bit buffer (row pitch 16 bits) and run the oracle's fuzzy_ahash + best_symbol
        buf = np.zeros(24, np.uint8)
        for r in range(10):
            v = int(windows[i, r]) << 6
            buf[2 * r], buf[2 * r + 1] = v >> 8, v & 0xFF
        all_ = int(cooldown[i] == 0xFE)
        ORA.lib.cbo_fuzzy_ahash(_ptr(buf), 16, 0, 0, all_, hashes)
        s = ORA.lib.cbo_best_symbol(hashes, all_, 16, int(cooldown[i]), C.byref(doff), C.byref(ddist))
        assert (sym[i], off[i], dist[i]) == (s, doff.value, ddist.value), i
    ctx.close()


def test_best_colors_matches_oracle(cb):
    rng = np.random.default_rng(4)
    means = rng.integers(0, 256, (20000, 3), dtype=np.uint8)
    for mode_val in (68, 4, 8):
        m = ORA.mode(mode_val)
        ctx = cb.Context(mode_val, max_frames=1)
        got = ctx.best_colors(means)
        want = np.array([ORA.lib.cbo_best_color(float(r), float(g), float(b), 1 << m.color_bits, m.color_mode, None)
                         for r, g, b in means], dtype=np.uint8)
        assert np.array_equal(got, want), mode_val
        ctx.close()


# ------------------------------------------------------------------------------------------------ errors
def test_argument_errors(cb):
    ctx = cb.Context(68, max_frames=2)
    with pytest.raises(cb.Cb200Error):
        ctx.decode_raw(np.zeros((3, 1024, 1024, 3), np.uint8))      # n > max_frames
    with pytest.raises(cb.Cb200Error):
        ctx.decode_raw(np.zeros((1, 512, 512, 3), np.uint8))        # wrong geometry
    with pytest.raises(cb.Cb200Error):
        cb.Context(12345, max_frames=1)                             # unknown mode
    ctx.close()


# ------------------------------------------------------------------------------------------------ C++ shims
def test_cpp_shims_rerun_reference_unit_tests(cb, tmp_path):
    """libcimbar_b200/host/{Decoder,CimbReader,CimbDecoder}.h keep the reference's class/method names; tests/cpp/shim_test.cpp
    re-runs the reference's DecoderTest / CimbReaderTest / CimbDecoderTest cases through them (and so through the kernels)."""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / "shim_test")
    libdir = os.path.join(root, "libcimbar_b200", "lib")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-o", exe, os.path.join(root, "tests", "cpp", "shim_test.cpp"),
                           "-L" + libdir, "-lcb200", "-Wl,-rpath," + libdir])
    golden = {(g["sample"], g["mode"], g["ecc"]): g["sha256"] for g in manifest()["goldens"]}
    first22 = {
        ("6bit/4color_ecc30_fountain_0.png", 4): ("0=0 99=8 11680=3 11681=32 11900=28 11901=25 11904=12 11995=2 11996=8 11998=6 "
                                                  "11999=54 12001=29 12004=6 12099=2 12195=57 12196=1 12200=5 12201=0 12298=32 "
                                                  "12299=34 12300=30 12399=15"),     # CimbReaderTest.cpp:80-83 (colour mode 0)
        ("6bit/4color_ecc30_fountain_0.png", 68): ("0=16 99=24 11680=19 11681=48 11900=44 11901=41 11904=28 11995=18 11996=24 "
                                                   "11998=22 11999=6 12001=45 12004=22 12099=18 12195=9 12196=17 12200=21 12201=16 "
                                                   "12298=48 12299=50 12300=46 12399=31"),  # CimbReaderTest.cpp:116-118 (colour mode 1)
        ("6bit/4_30_f0_627_extract.jpg", 68): ("0=16 1=44 99=24 100=44 600=49 601=54 711=46 712=9 11464=5 11576=48 11577=60 "
                                               "11687=57 11688=7 11689=48 11690=0 11798=31 11799=41 12297=62 12298=48 12299=50 "
                                               "12300=46 12399=31"),                  # CimbReaderTest.cpp:153-155
    }
    for sample, mode in [("b/tr_0.png", 68), ("6bit/4color_ecc30_fountain_0.png", 4), ("6bit/4color_ecc30_fountain_0.png", 68),
                         ("6bit/4_30_f0_627_extract.jpg", 4), ("6bit/4_30_f0_627_extract.jpg", 68)]:
        rgb = load_sample(sample)
        fpath = str(tmp_path / "frame.rgb")
        rgb.tofile(fpath)
        prefix = str(tmp_path / "out")
        res = subprocess.run([exe, str(mode), fpath, prefix], capture_output=True, text=True)
        assert res.returncode == 0, res.stdout + res.stderr
        raw = np.fromfile(prefix + ".raw", dtype=np.uint8)
        ecc = np.fromfile(prefix + ".ecc", dtype=np.uint8)
        if (sample, mode, False) in golden:
            assert sha(raw) == golden[(sample, mode, False)]
        if (sample, mode, True) in golden:
            assert sha(ecc) == golden[(sample, mode, True)]
        m = ORA.mode(mode)
        assert np.array_equal(raw, ORA.decode_raw(m, rgb))
        good, ochunks, omask = ORA.decode_fountain(m, rgb)
        chunks = np.fromfile(prefix + ".chunks", dtype=np.uint8)
        assert chunks.size == good and np.array_equal(chunks, ochunks.reshape(-1)[:good])
        # colour correction through the mirrors: 2 (decode_fountain's default) and 1, against one fresh reference decoder each
        for cc in (2, 1):
            ORA.set_ccm(None)
            try:
                good_cc, ochunks_cc, _ = ORA.decode_fountain(m, rgb, color_correction=cc)
                want_ccm = ORA.get_ccm()
            finally:
                ORA.set_ccm(None)
            got = np.fromfile(prefix + ".chunks_cc%d" % cc, dtype=np.uint8)
            assert got.size == good_cc and np.array_equal(got, ochunks_cc.reshape(-1)[:good_cc]), (sample, mode, cc)
            if cc == 2:
                if want_ccm is None:
                    assert not os.path.exists(prefix + ".ccm")
                else:
                    assert np.array_equal(np.fromfile(prefix + ".ccm", dtype=np.float32).reshape(3, 3), want_ccm)
        # Decoder(false, interleave=false): cells in linear order
        import copy
        mlin = copy.copy(m)
        mlin.interleave_blocks = 0
        assert np.array_equal(np.fromfile(prefix + ".raw_nointerleave", dtype=np.uint8), ORA.decode_raw(mlin, rgb)), (sample, mode)
        # do_decode restated on the CimbReader / CimbDecoder mirrors with color_correction 2 (read, update_metadata, init_ccm,
        # read_color): the colours and the fitted matrix of one fresh reference decoder
        if os.path.exists(prefix + ".cells_cc2"):
            ORA.set_ccm(None)
            try:
                raw_cc2 = np.zeros(ORA.capacity(m), np.uint8)
                ORA.decode_fountain(m, rgb, color_correction=2)
                want_ccm2 = ORA.get_ccm()
                # colours per cell under that matrix == what decode_raw gives with the matrix active
                _, ocells = ORA.decode_raw(m, rgb, want_cells=True)
            finally:
                ORA.set_ccm(None)
            got_cols = np.fromfile(prefix + ".cells_cc2", dtype=np.uint8)
            assert np.array_equal(got_cols, ocells["color"]), (sample, mode)
            if want_ccm2 is None:
                assert not os.path.exists(prefix + ".ccm_reader")
            else:
                assert np.array_equal(np.fromfile(prefix + ".ccm_reader", dtype=np.float32).reshape(3, 3), want_ccm2)
        for ext in (".cells_cc2", ".ccm_reader"):
            if os.path.exists(prefix + ext):
                os.remove(prefix + ext)
        lines = open(prefix + ".first22").read().split("\n")
        if (sample, mode) in first22:
            assert lines[0] == first22[(sample, mode)]
        if sample == "6bit/4color_ecc30_fountain_0.png":
            assert lines[1] == "0 62 8"                                   # CimbReaderTest.cpp:37-58: first read


# ------------------------------------------------------------------------------------------------ edge cases
def test_degenerate_frames_match_oracle(cb):
    """all-black, all-white, pure noise, a vertical gradient: no valid tiles anywhere, every path still has to agree"""
    m = ORA.mode(68)
    rng = np.random.default_rng(9)
    frames = np.zeros((4, 1024, 1024, 3), np.uint8)
    frames[1] = 255
    frames[2] = rng.integers(0, 256, (1024, 1024, 3), dtype=np.uint8)
    frames[3] = (np.arange(1024, dtype=np.uint32)[:, None, None] // 4).astype(np.uint8)
    ctx = cb.Context(68, max_frames=4)
    raw, ff = ctx.decode_raw(frames)
    data, ok, _ = ctx.decode(frames)
    chunks, count, mask, _ = ctx.decode_fountain(frames)
    for f in range(4):
        assert np.array_equal(raw[f], ORA.decode_raw(m, frames[f])), f
        odata, ook = ORA.decode(m, frames[f])
        assert np.array_equal(ok[f], ook) and np.array_equal(data[f], odata), f
        good, ochunks, omask = ORA.decode_fountain(m, frames[f])
        assert mask[f] == omask and count[f] * m.chunk_size == good
    ctx.close()


def test_cell_trace_matches_oracle_walk(cb):
    """cb200_decode_cells == the reference's CimbReader loop: same walk order, positions, drift offsets and distances; on
    photographs, a clean sample frame and frames with noise tiles in the 8-colour mode and the two smaller geometries"""
    cases = [(sample, mode, load_sample(sample)) for sample, mode in
             (("b/ex2434.jpg", 68), ("6bit/4_30_f0_627_extract.jpg", 4), ("b/tr_1.png", 68))]
    for mode, rate in ((8, 0.01), (66, 0.08), (67, 0.01)):
        cases.append((f"noise tiles {rate:.0%}", mode, synth_frames(mode, 1, seed=450 + mode, error_rate=rate, noise_tiles=True)[2][0]))
    for sample, mode, rgb in cases:
        m = ORA.mode(mode)
        ctx = cb.Context(mode, max_frames=1)
        cells, trace = ctx.decode_cells(rgb)
        _, ocells = ORA.decode_raw(m, rgb, want_cells=True)
        assert np.array_equal(trace[0]["order"], ocells["order"]), (sample, mode)
        assert np.array_equal(trace[0]["x"], ocells["x"]) and np.array_equal(trace[0]["y"], ocells["y"]), (sample, mode)
        assert np.array_equal(trace[0]["drift_offset"], ocells["drift_offset"]), (sample, mode)
        assert np.array_equal(trace[0]["distance"], ocells["distance"]), (sample, mode)
        sb = m.symbol_bits
        assert np.array_equal(cells[0] & ((1 << sb) - 1), ocells["symbol"]), (sample, mode)
        assert np.array_equal((cells[0] >> sb) & ((1 << m.color_bits) - 1), ocells["color"]), (sample, mode)
        ctx.close()


def test_batch_mixing_clean_and_dirty_frames(cb):
    """a batch where only some frames need the exact walk: flags identify exactly those, every frame is bit-exact"""
    m, payloads, frames = synth_frames(68, 6, seed=21)
    cam = load_sample("b/ex2434.jpg")
    batch = np.stack([frames[0], cam, frames[1], frames[2], cam, frames[3]])
    ctx = cb.Context(68, max_frames=6)
    raw, ff = ctx.decode_raw(batch)
    assert [int(x & cb.FRAME_FALLBACK) for x in ff] == [0, 1, 0, 0, 1, 0]
    for f in range(6):
        assert np.array_equal(raw[f], ORA.decode_raw(m, batch[f])), f
    # NO_FALLBACK: dirty frames are reported, not silently wrong
    raw2, ff2 = ctx.decode_raw(batch, flags=cb.FLAG_NO_FALLBACK)
    assert [int(x) for x in ff2] == [0, cb.FRAME_INEXACT, 0, 0, cb.FRAME_INEXACT, 0]
    ctx.close()


def test_two_contexts_and_modes_coexist(cb):
    """tables are per context / per launch: interleaving a mode-B and a legacy 4C context must not cross-contaminate"""
    mb, pb, fb = synth_frames(68, 2, seed=31)
    m4, p4, f4 = synth_frames(4, 2, seed=32)
    cb_b, cb_4 = cb.Context(68, max_frames=2), cb.Context(4, max_frames=2)
    for _ in range(2):
        d4, ok4, _ = cb_4.decode(f4)
        db, okb, _ = cb_b.decode(fb)
        assert ok4.all() and okb.all() and np.array_equal(d4, p4) and np.array_equal(db, pb)
    cb_b.close(); cb_4.close()


# ------------------------------------------------------------------------------------------------ BASELINE config 4 (one GPU)
def test_fountain_file_round_trip_with_frame_loss(cb):
    """file -> wirehair blocks (the reference's own codec) -> 625-byte chunks -> RS + tiles -> frames -> GPU decode ->
    rank-0 sink -> file, with a third of the frames lost and the rest fed in shuffled order (wirehair does not care)."""
    import torch
    from oracle_lib import Ref
    try:
        ref = Ref()
    except (FileNotFoundError, OSError) as e:
        pytest.skip(f"oracle/_ref not available: {e}")
    m = ORA.mode(68)
    rng = np.random.default_rng(44)
    size = 300_000
    data = rng.integers(0, 256, size, dtype=np.uint8)
    payload = m.chunk_size - 6
    enc = ref.lib.wirehair_encoder_create(None, data.ctypes.data, size, payload)
    n_frames = 66                                                 # 792 blocks for N = 485
    chunks = np.zeros((n_frames, 12, m.chunk_size), np.uint8)
    for b in range(n_frames * 12):
        ch = chunks[b // 12, b % 12]
        ORA.lib.cbo_md_pack(7, size, b, _ptr(ch))
        wrote = C.c_uint32(0)
        assert ref.lib.wirehair_encode(enc, b, ch[6:].ctypes.data, payload, C.byref(wrote)) == 0
    ref.lib.wirehair_free(enc)
    ctx = cb.Context(68, max_frames=n_frames)
    d_payload = torch.from_numpy(chunks.reshape(n_frames, -1)).cuda()
    d_cells = torch.empty((n_frames, m.total_cells), dtype=torch.uint8, device="cuda")
    d_rgb = torch.empty((n_frames, 1024, 1024, 3), dtype=torch.uint8, device="cuda")
    d_chunks = torch.empty((n_frames, 7500), dtype=torch.uint8, device="cuda")
    d_mask = torch.empty(n_frames, dtype=torch.int32, device="cuda")
    ctx.encode_cells_dev(d_payload.data_ptr(), n_frames, d_cells.data_ptr())
    ctx.render_frames_dev(d_cells.data_ptr(), n_frames, d_rgb.data_ptr())
    ctx.decode_chunks_dev(d_rgb.data_ptr(), n_frames, d_chunks.data_ptr(), d_mask.data_ptr())
    ctx.sync()
    got, masks = d_chunks.cpu().numpy(), d_mask.cpu().numpy().astype(np.uint32)
    assert (masks == 0xFFF).all() and np.array_equal(got, chunks.reshape(n_frames, -1))
    keep = rng.permutation(n_frames)[: (2 * n_frames) // 3]       # lose a third of the frames, shuffle the rest
    sink = cb.FountainSink(m.chunk_size, ref.lib)
    fid = sink.ingest(got[keep], masks[keep])
    assert fid > 0
    assert np.array_equal(sink.file(fid), data)
    sink.close()
    ctx.close()


# ------------------------------------------------------------------------------------------------ colour correction (CCM)
@pytest.mark.parametrize("idx", [0, 2])
def test_ccm_reference_goldens_on_gpu(cb, idx):
    # CimbReaderTest.cpp:181-214 / :239-272: with the printed CCM active the first six reads give colours 0,1,1,2,2,2;
    # and every cell of the camera frame must match the oracle under the same CCM
    g = manifest()["ccm_goldens"][idx]
    ctx = cb.Context(g["mode"], max_frames=1)
    rgb = load_sample(g["sample"])
    ctx.set_ccm(g["matrix"])
    assert np.array_equal(ctx.get_ccm(), np.asarray(g["matrix"], np.float32))
    cells, trace = ctx.decode_cells(rgb)
    m = ORA.mode(g["mode"])
    order = np.argsort(trace[0]["order"])
    assert (cells[0][order[:6]] >> m.symbol_bits).tolist() == g["first_colors"]
    raw, ff = ctx.decode_raw(rgb)
    ORA.set_ccm(g["matrix"])
    try:
        want = ORA.decode_raw(m, rgb)
    finally:
        ORA.set_ccm(None)
    assert np.array_equal(raw[0], want)
    ctx.set_ccm(None)
    assert ctx.get_ccm() is None
    raw0, _ = ctx.decode_raw(rgb)
    assert np.array_equal(raw0[0], ORA.decode_raw(m, rgb))
    if idx == 2:          # ex380 is the reference's "VeryNecessary" case; on ex2434 the CCM changes no colour
        assert not np.array_equal(raw0[0], raw[0])


@pytest.mark.parametrize("mode_val", [68, 8, 67])
def test_ccm_on_clean_frames_goes_through_k1(cb, mode_val):
    # tinted synthetic frames stay on the drift-0 kernel (K1's CCM variant); the matrix is an arbitrary strong one
    m, payloads, frames = synth_frames(mode_val, 3, seed=41)
    frames = tint(frames, (0.62, 0.95, 0.8))
    mat = np.array([[1.61, 0.02, -0.11], [-0.07, 1.05, 0.03], [-0.2, -0.15, 1.45]], np.float32)
    ctx = cb.Context(mode_val, max_frames=3)
    ctx.set_ccm(mat)
    raw, ff = ctx.decode_raw(frames)
    assert ff.tolist() == [0, 0, 0]
    ORA.set_ccm(mat)
    try:
        for f in range(3):
            assert np.array_equal(raw[f], ORA.decode_raw(m, frames[f])), f
    finally:
        ORA.set_ccm(None)
    # single-value entry point under the same CCM (CimbDecoder::get_best_color with an active CCM)
    rng = np.random.default_rng(5)
    means = rng.integers(0, 256, (4096, 3), dtype=np.uint8)
    got = ctx.best_colors(means)
    cm = (C.c_float * 9)(*mat.reshape(9).tolist())
    want = [ORA.lib.cbo_best_color(float(r), float(g), float(b), 1 << m.color_bits, m.color_mode, cm) for r, g, b in means]
    assert got.tolist() == want


def test_simple_color_correction_matches_oracle(cb):
    # color_correction == 1 (simpleColorCorrection, CimbReader.cpp:55-93): per-frame von Kries matrix from the anchors
    m, payloads, frames = synth_frames(68, 4, seed=43)
    frames[1] = tint(frames[1:2], (0.7, 1.0, 0.9))[0]
    frames[2] = tint(frames[2:3], (1.0, 0.55, 0.8))[0]
    frames[3] = load_sample("b/ex380.jpg")                      # camera frame: exact walk + CCM
    ctx = cb.Context(68, max_frames=4)
    raw, ff = ctx.decode_raw(frames, flags=cb.FLAG_CC_SIMPLE)
    assert ff.tolist()[:3] == [0, 0, 0] and ff[3] == cb.FRAME_FALLBACK
    try:
        for f in range(4):
            assert np.array_equal(raw[f], ORA.decode_raw(m, frames[f], color_correction=1)), f
        # the decoder keeps the last frame's matrix (CimbDecoder.cpp:82-85), bit for bit
        assert np.array_equal(ctx.get_ccm(), ORA.simple_ccm(m, frames[3]))
        # ... and uses it for the next call without the flag, like a reference decoder whose CCM was set earlier
        raw2, _ = ctx.decode_raw(frames[:2])
        ORA.set_ccm(ORA.simple_ccm(m, frames[3]))
        for f in range(2):
            assert np.array_equal(raw2[f], ORA.decode_raw(m, frames[f])), f
    finally:
        ORA.set_ccm(None)
    # full decode with RS under color_correction == 1 still returns the payload of the tinted frames
    ctx2 = cb.Context(68, max_frames=4)
    data, ok, _ = ctx2.decode(frames[:3], flags=cb.FLAG_CC_SIMPLE)
    assert ok.all() and np.array_equal(data, payloads[:3])


def _oracle_fountain_batch(m, frames, color_correction, initial=None):
    """frames decoded in order by ONE reference decoder: the thread-local CCM carries from frame to frame"""
    ORA.set_ccm(initial)
    out = []
    try:
        for fr in frames:
            good, chunks, mask = ORA.decode_fountain(m, fr, color_correction=color_correction)
            out.append((good, chunks.copy(), mask, ORA.get_ccm()))
    finally:
        ORA.set_ccm(None)
    return out


def test_color_correction_2_fit_matches_oracle(cb):
    # color_correction == 2 (CimbReader::init_ccm): real fountain frames (clean PNGs), a camera frame that needs both the
    # exact walk and the CCM, tinted synthetic frames whose random "headers" still predict their own colours, a frame whose
    # first symbol chunks are destroyed (header comes from a later chunk), and a frame with no decodable chunk at all
    # (keeps the previous frame's CCM)
    m, payloads, synth = synth_frames(68, 3, seed=47)
    synth[0] = tint(synth[0:1], (0.8, 0.6, 1.0))[0]
    rng = np.random.default_rng(9)
    xs, ys = np.zeros(m.total_cells, np.int32), np.zeros(m.total_cells, np.int32)
    ORA.lib.cbo_cell_positions(C.byref(m), 0, _ptr(xs, C.c_int), _ptr(ys, C.c_int))
    idx = np.zeros(m.total_cells, np.uint32)
    ORA.lib.cbo_interleave_indices(m.total_cells, m.interleave_blocks, m.interleave_partitions, _ptr(idx, C.c_uint))
    # frame 1: wreck the cells of the first two symbol chunks' RS blocks (stream slots of blocks 0..9: bytes 0..1549 -> slots 0..3099)
    for s in rng.choice(3100, 1200, replace=False):
        c = idx[s]
        synth[1][ys[c]:ys[c] + 8, xs[c]:xs[c] + 8] = rng.integers(0, 256, (8, 8, 3), dtype=np.uint8)
    # frame 2: noise everywhere -> nothing decodes
    synth[2] = rng.integers(0, 256, synth[2].shape, dtype=np.uint8)
    frames = np.stack([load_sample("b/tr_0.png"), load_sample("b/ex380.jpg"), synth[0], synth[1], synth[2], load_sample("b/tr_1.png")])
    want = _oracle_fountain_batch(m, frames, 2)
    assert want[4][3] is not None and np.array_equal(want[4][3], want[3][3])      # the scenario the carry exists for
    ctx = cb.Context(68, max_frames=len(frames))
    chunks, counts, masks, ff = ctx.decode_fountain(frames, flags=cb.FLAG_CC_FIT)
    for f, (good, wchunks, wmask, wccm) in enumerate(want):
        assert masks[f] == wmask, f
        assert counts[f] * m.chunk_size == good, f
        assert np.array_equal(chunks[f][:counts[f]], wchunks[:counts[f]]), f
    assert np.array_equal(ctx.get_ccm(), want[-1][3])                             # bit-exact fit, carried to the context
    # the block-level entry point (what the C++ Decoder mirror replays into the caller's aligned_stream) agrees
    ctx2 = cb.Context(68, max_frames=len(frames))
    data, ok, _ = ctx2.decode(frames, flags=cb.FLAG_CC_FIT)
    for f in range(len(frames)):
        for q in range(m.chunks_per_frame):
            if masks[f] >> q & 1:
                assert np.array_equal(data[f].reshape(m.chunks_per_frame, m.chunk_size)[q], chunks[f][bin(masks[f] & ((1 << q) - 1)).count("1")]), (f, q)
    # a second batch starts from the CCM the first one left, like the next frames of the same reference decoder
    again = _oracle_fountain_batch(m, frames[4:5], 2, initial=want[-1][3])
    chunks3, counts3, masks3, _ = ctx.decode_fountain(frames[4:5], flags=cb.FLAG_CC_FIT)
    assert masks3[0] == again[0][2] and np.array_equal(ctx.get_ccm(), again[0][3])


@pytest.mark.parametrize("mode_val", [8, 67])
def test_color_correction_2_other_modes(cb, mode_val):
    m, payloads, frames = synth_frames(mode_val, 3, seed=53)
    frames[1] = tint(frames[1:2], (0.9, 0.7, 0.75))[0]
    want = _oracle_fountain_batch(m, frames, 2)
    ctx = cb.Context(mode_val, max_frames=3)
    chunks, counts, masks, ff = ctx.decode_fountain(frames, flags=cb.FLAG_CC_FIT)
    for f, (good, wchunks, wmask, wccm) in enumerate(want):
        assert masks[f] == wmask and counts[f] * m.chunk_size == good, f
        assert np.array_equal(chunks[f][:counts[f]], wchunks[:counts[f]]), f
    assert np.array_equal(ctx.get_ccm(), want[-1][3])


def test_exact_walk_work_list_in_several_chunks(cb, monkeypatch):
    # the exact-walk kernels keep raster/result for at most N listed frames at a time (16 384 by default) and go through
    # longer work lists chunk by chunk; force tiny chunks so that the chunk loop, its counters and the list offsets are exercised
    monkeypatch.setenv("CB200_K1X_MAX_ENTRIES", "3")
    m, payloads, frames = synth_frames(68, 10, seed=61, error_rate=0.01, noise_tiles=True)
    clean = synth_frames(68, 3, seed=62)[2]
    batch = np.concatenate([frames[:4], clean[:2], frames[4:], clean[2:]])        # 13 frames, 10 of them need the walk
    ctx = cb.Context(68, max_frames=len(batch))
    monkeypatch.delenv("CB200_K1X_MAX_ENTRIES")
    raw, ff = ctx.decode_raw(batch)
    assert ff.tolist() == [1, 1, 1, 1, 0, 0, 1, 1, 1, 1, 1, 1, 0]
    for f in range(len(batch)):
        assert np.array_equal(raw[f], ORA.decode_raw(m, batch[f])), f
    raw2, ff2 = ctx.decode_raw(batch[::-1].copy())                                  # a second call reuses the workspace
    for f in range(len(batch)):
        assert np.array_equal(raw2[f], raw[len(batch) - 1 - f]), f


@pytest.mark.gpu
def test_exact_walk_with_the_literal_pop_forced(cb, monkeypatch):
    # K1x pops through a lane-parallel sift-down (three five-level rounds); heaps beyond 65 535 entries fall back to the literal
    # one-level-per-step __adjust_heap.  No real frame gets there, so the fallback is forced here and must give the same walk:
    # cell trace of a camera frame against the oracle's, and a noisy synthetic frame's raw bytes
    monkeypatch.setenv("CB200_K1X_SERIAL_ABOVE", "0")
    ctx = cb.Context(68, max_frames=2)
    monkeypatch.delenv("CB200_K1X_SERIAL_ABOVE")
    cam = load_sample("b/ex2434.jpg")
    m = ORA.mode(68)
    want_raw, want_cells = ORA.decode_raw(m, cam, want_cells=True)
    raw, ff = ctx.decode_raw(cam[None])
    assert (ff[0] & cb.FRAME_FALLBACK) and np.array_equal(raw[0], want_raw)
    _, _, noisy = synth_frames(68, 2, seed=77, error_rate=0.01, noise_tiles=True)
    raw2, ff2 = ctx.decode_raw(noisy)
    assert all(int(x) & cb.FRAME_FALLBACK for x in ff2)
    for f in range(2):
        assert np.array_equal(raw2[f], ORA.decode_raw(m, noisy[f]))


# ------------------------------------------------------------------------------------------------ sharpen inside K1
@pytest.mark.parametrize("mode_val,n", [(68, 3), (68, 640), (4, 5), (8, 480), (67, 4), (67, 640), (66, 7), (66, 500)])
def test_sharpen_clean_batches_stay_on_k1(cb, mode_val, n):
    """needs_sharpen preprocessing (CimbReader.cpp:17-46: filter2D 4.5-centre kernel + adaptiveThreshold block 7) runs inside
    K1 (template SH): clean frames keep their K1 result (no exact walk), in the band-split schedule (few frames) and in the
    persistent whole-frame schedule (n >= 3 x SMs), for the 1024x1024 geometry and the two others."""
    m, payloads, frames = synth_frames(mode_val, 4, seed=300 + mode_val)
    big = np.concatenate([frames] * ((n + 3) // 4))[:n]
    ctx = cb.Context(mode_val, max_frames=n)
    raw, ff = ctx.decode_raw(big, flags=cb.FLAG_SHARPEN)
    assert not ff.any()
    want = np.stack([ORA.decode_raw(m, fr, sharpen=True) for fr in frames])
    for f in range(n):
        assert np.array_equal(raw[f], want[f % 4]), f
    data, ok, _ = ctx.decode(big, flags=cb.FLAG_SHARPEN)
    assert ok.all() and np.array_equal(data[:min(n, 4)], payloads[:min(n, 4)])
    ctx.close()


def test_sharpen_mixed_batch_and_the_walk_on_every_frame(cb):
    """camera frames in a sharpened batch are flagged by K1 and re-done by the exact walk on the sharpened raster, with the
    oracle's bytes; the walk forced on every frame (decode_cells) gives the oracle's cells and trace on the clean frames too"""
    m, payloads, frames = synth_frames(68, 3, seed=331)
    batch = np.stack([frames[0], load_sample("b/ex2434.jpg"), frames[1], load_sample("b/ex380.jpg"), frames[2]])
    want = [ORA.decode_raw(m, fr, sharpen=True, want_cells=True) for fr in batch]
    ctx = cb.Context(68, max_frames=5)
    raw, ff = ctx.decode_raw(batch, flags=cb.FLAG_SHARPEN)
    assert [int(x & cb.FRAME_FALLBACK) for x in ff] == [0, 1, 0, 1, 0]
    cells, trace = ctx.decode_cells(batch, flags=cb.FLAG_SHARPEN)
    for f, (want_raw, ocells) in enumerate(want):
        assert np.array_equal(raw[f], want_raw), f
        for k in ("order", "x", "y", "drift_offset", "distance"):
            assert np.array_equal(trace[f][k], ocells[k]), (f, k)
        assert np.array_equal(cells[f] & 15, ocells["symbol"]) and np.array_equal((cells[f] >> 4) & 7, ocells["color"]), f
    ctx.close()


def test_sharpen_with_noise_tiles_and_colour_correction(cb):
    # noise tiles make some frames dirty under sharpen too; colour correction 1 goes through K1's CCM variant (CM = 1, SH)
    m, payloads, frames = synth_frames(68, 6, seed=341, error_rate=0.01, noise_tiles=True)
    clean = synth_frames(68, 2, seed=342)[2]
    batch = np.concatenate([frames[:3], clean, frames[3:]])
    ctx = cb.Context(68, max_frames=len(batch))
    raw, ff = ctx.decode_raw(batch, flags=cb.FLAG_SHARPEN)
    for f in range(len(batch)):
        assert np.array_equal(raw[f], ORA.decode_raw(m, batch[f], sharpen=True)), f
    assert not ff[3] and not ff[4]
    raw1, ff1 = ctx.decode_raw(batch, flags=cb.FLAG_SHARPEN | cb.FLAG_CC_SIMPLE)
    try:
        for f in range(len(batch)):
            assert np.array_equal(raw1[f], ORA.decode_raw(m, batch[f], sharpen=True, color_correction=1)), f
    finally:
        ORA.set_ccm(None)
    ctx.close()


@pytest.mark.parametrize("mode_val,sharpen", [pytest.param(mv, sh, id=str(mv) if sh else f"{mv}-plain")
                                              for sh in (True, False) for mv in (68, 66, 67)])
def test_sharpen_raster_of_the_exact_walk(cb, mode_val, sharpen):
    """K1x's streaming rasters against the oracle: with sharpen k_flood_raster_fast_sharpen (OpenCV's borders, reflect for the
    filter, replicate for the box sum), without it k_flood_raster_fast (replicate borders); on frames whose cells reach the
    borders' influence (noise everywhere), on the 736 x 637 geometry of mode Bu with its 61-row last band and on the 1024 x 720
    geometry of mode Bm with its 16-row last band"""
    m = ORA.mode(mode_val)
    flags = cb.FLAG_SHARPEN if sharpen else 0
    rng = np.random.default_rng(400 + mode_val)
    frames = rng.integers(0, 256, (5, m.image_size_y, m.image_size_x, 3), dtype=np.uint8)
    frames[1, :, ::3] //= 4
    frames[2] = np.repeat(np.repeat(rng.integers(0, 256, (m.image_size_y // 4 + 1, m.image_size_x // 4 + 1, 3), dtype=np.uint8), 4, 0), 4, 1)[:m.image_size_y, :m.image_size_x]
    if mode_val == 68:
        frames[3] = load_sample("b/ex2434.jpg"); frames[4] = load_sample("b/ex380.jpg")
    ctx = cb.Context(mode_val, max_frames=5)
    raw, ff = ctx.decode_raw(frames, flags=flags)
    assert all(int(x) & cb.FRAME_FALLBACK for x in ff)
    for f in range(5):
        assert np.array_equal(raw[f], ORA.decode_raw(m, frames[f], sharpen=sharpen)), f
    ctx.close()
