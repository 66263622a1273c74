"""Fixtures and helpers shared by the GPU test files.  Test infrastructure only.  pytest finds a fixture in the test module that
uses it, so a test file imports the fixtures it needs from here by name (`from gpu_support import cb, entries  # noqa: F401`)."""
import ctypes as C

import cv2
import numpy as np
import pytest

import chain_batches as CB
from oracle_lib import Oracle, _ptr, load_sample
from ragged_samples import GLOB, sample
from scan_oracle_lib import ScanOracle

ORA = Oracle()
SO = ScanOracle()
INT_MIN, INT_MAX = -2 ** 31, 2 ** 31 - 1


@pytest.fixture(scope="module")
def cb():
    import libcimbar_b200 as cb
    return cb


# ------------------------------------------------------------------------------------------------ synthetic frames and the oracle
def synth_frames(mode_val, n, seed, error_rate=0.0, noise_tiles=False):
    """payload -> RS-encoded cells -> frames, optionally replacing a fraction of cells with a different valid tile
    (keeps the drift-0 pass exact) or with random 8x8 noise (SURVEY 8d config 3)."""
    m = ORA.mode(mode_val)
    rng = np.random.default_rng(seed)
    nbytes = (ORA.capacity(m) // m.ecc_block_size) * (m.ecc_block_size - m.ecc_bytes)
    payloads = rng.integers(0, 256, (n, nbytes), dtype=np.uint8)
    frames = np.zeros((n, m.image_size_y, m.image_size_x, 3), dtype=np.uint8)
    for f in range(n):
        cells = ORA.payload_to_cells(m, payloads[f])
        k = int(round(error_rate * m.total_cells))
        bad = rng.choice(m.total_cells, k, replace=False) if k else np.zeros(0, dtype=np.int64)
        if k and not noise_tiles:
            nvals = 1 << (m.symbol_bits + m.color_bits)
            cells[bad] = (cells[bad] + rng.integers(1, nvals, k, dtype=np.uint8)) % nvals
        frames[f] = ORA.render_frame(m, cells)
        if k and noise_tiles:
            xs, ys = np.zeros(m.total_cells, np.int32), np.zeros(m.total_cells, np.int32)
            ORA.lib.cbo_cell_positions(C.byref(m), 0, _ptr(xs, C.c_int), _ptr(ys, C.c_int))
            for i in bad:
                frames[f, ys[i]:ys[i] + 8, xs[i]:xs[i] + 8] = rng.integers(0, 256, (8, 8, 3), dtype=np.uint8)
    return m, payloads, frames


def tint(frames, gains):
    """a coloured cast: per-channel gain, the kind of error a CCM exists to undo"""
    out = frames.astype(np.float32) * np.asarray(gains, np.float32)
    return np.clip(np.rint(out), 0, 255).astype(np.uint8)


POOL = 12                  # per mode: 4 clean frames, 4 with 1 % noise tiles (exact walk), 4 blurred (sigma 1.6) + noise
_pools, _oracle = {}, {}


def frame_pool(mode_val):
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
        m, frames = frame_pool(mode_val)
        ORA.set_ccm(None)
        try:
            good, chunks, mask = ORA.decode_fountain(m, frames[p], sharpen=bool(sharpen), color_correction=cc)
        finally:
            ORA.set_ccm(None)
        _oracle[key] = (good, chunks.copy(), mask)
    return _oracle[key]


def check_dense(m, chunks, count, mask, want, what):
    good, wchunks, wmask = want
    assert mask == wmask and count * m.chunk_size == good, what
    assert np.array_equal(chunks[:count], wchunks[:count]), what


def dense(m, slots, mask):
    """the fixed-slot records of cb200_decode_chunks_dev as escrow_buffer_writer's dense order"""
    rows = slots.reshape(m.chunks_per_frame, m.chunk_size)
    keep = [q for q in range(m.chunks_per_frame) if mask >> q & 1]
    return len(keep), rows[keep]


def sharpen_cli_loop(m, pics, cc):
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


# ------------------------------------------------------------------------------------------------ camera pictures and the CLI loop
def pad(rgb, top, bottom, left, right):
    return cv2.copyMakeBorder(rgb, top, bottom, left, right, cv2.BORDER_CONSTANT, value=(0, 0, 0))


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


def same_ccm(a, b):
    return (a is None) == (b is None) and (a is None or np.array_equal(a, b))


# ------------------------------------------------------------------------------------------------ receivers
@pytest.fixture(scope="module")
def frames():
    """the crafted frames under the frame cast (0, 1, 3, 4 fit their own matrix; 2 has no header), then the same five with the
    encoder's anchors pasted in and dimmed to 80 % (5 .. 9): the crafted frames have no anchor white, these have one, so CC_SIMPLE
    gives the two halves different matrices"""
    fr = np.stack(CB.crafted(CB.CAST_FRAMES))
    lit = np.stack([CB.with_anchors(f) for f in fr])
    return np.concatenate([fr, np.rint(lit * np.float32(0.8)).astype(np.uint8)])


@pytest.fixture(scope="module")
def entries(cb, frames):
    """entry states: inactive, fitted from another frame (crafted frames 0 and 4), the identity"""
    import torch
    ctx = cb.Context(68, max_frames=1)
    out = torch.zeros((1, ctx.info.data_bytes), dtype=torch.uint8, device="cuda")
    mask = torch.zeros(1, dtype=torch.int32, device="cuda")
    fits = []
    for i in (0, 4):
        ctx.set_ccm(None)
        d = torch.from_numpy(frames[i:i + 1]).cuda()
        ctx.decode_chunks_dev(d.data_ptr(), 1, out.data_ptr(), mask.data_ptr(), flags=cb.FLAG_CC_FIT)
        fits.append(ctx.get_ccm())
    assert fits[0] is not None and fits[1] is not None and not np.array_equal(fits[0], fits[1])
    return [None, fits[0], np.eye(3, dtype=np.float32), fits[1]]


def layouts(pics):
    """the pictures as CUDA tensors in mixed layouts and pitches: RGB, BGR, planar, padded RGB, RGBA, in turn"""
    import torch
    ts, orders = [], []
    for i, p in enumerate(pics):
        t = torch.from_numpy(np.ascontiguousarray(p)).cuda()
        k = i % 5
        if k == 1:
            t, o = t.flip(2).contiguous(), "bgr"
        elif k == 2:
            t, o = t.permute(2, 0, 1).contiguous(), "rgb"
        elif k == 3:
            h, w, _ = t.shape
            big = torch.zeros((h, w + 13, 3), dtype=torch.uint8, device="cuda")
            big[:, :w] = t
            t, o = big[:, :w], "rgb"
        elif k == 4:
            t, o = torch.cat([t, torch.full_like(t[:, :, :1], 77)], 2).contiguous(), "rgba"
        else:
            o = "rgb"
        ts.append(t)
        orders.append(o)
    return ts, orders


def camera_call(cb, ctx, ts, orders, flags, receiver_of=None, states=None):
    import torch
    n = len(ts)
    chunks = torch.full((n, ctx.info.data_bytes), 0xA5, dtype=torch.uint8, device="cuda")
    mask = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    status = torch.full((n,), 7, dtype=torch.int32, device="cuda")
    ff = torch.full((n,), 0xEE, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    if receiver_of is None:
        ctx.scan_extract_decode_chunks_pictures_dev(ts, chunks.data_ptr(), mask.data_ptr(), status.data_ptr(), ff.data_ptr(), flags=flags,
                                                    order=orders)
    else:
        ctx.scan_extract_decode_chunks_receivers_dev(ts, receiver_of, states, chunks.data_ptr(), mask.data_ptr(), status.data_ptr(),
                                                     ff.data_ptr(), flags=flags, order=orders)
    ctx.sync()
    return chunks.cpu().numpy(), mask.cpu().numpy(), status.cpu().numpy(), ff.cpu().numpy(), ctx.camera_transforms(n)


def graph_kernel_nodes(graph):
    cuda = C.CDLL("libcuda.so.1")
    count = C.c_size_t(0)
    assert cuda.cuGraphGetNodes(C.c_void_p(graph), None, C.byref(count)) == 0
    nodes = (C.c_void_p * count.value)()
    assert cuda.cuGraphGetNodes(C.c_void_p(graph), nodes, C.byref(count)) == 0
    kinds = []
    for nd in nodes:
        t = C.c_int(-1)
        assert cuda.cuGraphNodeGetType(C.c_void_p(nd), C.byref(t)) == 0
        kinds.append(t.value)
    return kinds.count(0)                                                  # CU_GRAPH_NODE_TYPE_KERNEL


KINDS = ["rgb", "bgr", "planar", "pitched", "rgba", "bgra"]


def resized(p, short):
    import cv2
    f = short / min(p.shape[:2])
    return cv2.resize(p, (round(p.shape[1] * f), round(p.shape[0] * f)), interpolation=cv2.INTER_LINEAR if f > 1 else cv2.INTER_AREA)


def pool(mode):
    """the golden photographs and pictures of the mode at native size (landscape and portrait), upscales to 5 and 9 taps, downscales"""
    base = CB.camera_pictures() if mode == 68 else CB.legacy_pictures()
    photo = base[0]
    s = min(photo.shape[:2])
    up5 = resized(photo, 1.7 * s if 1500 <= 1.7 * s < 2500 else 1800)
    return base + [np.ascontiguousarray(np.transpose(photo, (1, 0, 2))), up5, resized(photo, 2600), resized(base[-1], 0.6 * min(base[-1].shape[:2]))]


def as_tensor(p, kind):
    """picture p as a fresh CUDA tensor (its own allocation) in one of the layouts, and its order"""
    import torch
    t = torch.from_numpy(np.ascontiguousarray(p)).cuda()
    if kind == "bgr":
        return t.flip(2).contiguous(), "bgr"
    if kind == "planar":
        return t.permute(2, 0, 1).contiguous(), "rgb"
    if kind == "pitched":
        h, w, _ = t.shape
        big = torch.zeros((h, w + 13, 3), dtype=torch.uint8, device="cuda")
        big[:, :w] = t
        return big[:, :w], "rgb"
    if kind == "rgba":
        return torch.cat([t, torch.full_like(t[:, :, :1], 77)], 2).contiguous(), "rgba"
    if kind == "bgra":
        return torch.cat([t.flip(2), torch.full_like(t[:, :, :1], 99)], 2).contiguous(), "bgra"
    return t, "rgb"


def bounds_of(pics):
    s = [min(p.shape[:2]) for p in pics]
    return (min(s), max(s), max(max(p.shape[:2]) for p in pics))


def direct(cb, ref, ts, orders, of, states, flags):
    """the direct receivers call on ref: records, transforms, frame CCMs (nothing for an empty batch)"""
    import torch
    n = len(ts)
    if n == 0:
        return None
    chunks = torch.full((n, ref.info.data_bytes), 0xA5, dtype=torch.uint8, device="cuda")
    mask = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    status = torch.full((n,), 7, dtype=torch.int32, device="cuda")
    ff = torch.full((n,), 0xEE, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    ref.scan_extract_decode_chunks_receivers_dev(ts, np.asarray(of, np.int32), states, chunks.data_ptr(), mask.data_ptr(), status.data_ptr(),
                                                 ff.data_ptr(), flags=flags, order=orders)
    ref.sync()
    return [t.cpu().numpy() for t in (chunks, mask, status, ff)], ref.camera_transforms(n), ref.frame_ccms(n)


def fresh(pics, rng):
    """every picture in a random layout, each in a new allocation"""
    out = [as_tensor(p, KINDS[int(rng.integers(len(KINDS)))]) for p in pics]
    return [t for t, _ in out], [o for _, o in out]


# ------------------------------------------------------------------------------------------------ detect
RECV = [66, 68, 67, 4]                                  # the reference receiver's candidates, in its order
FLAGS = [("SHARPEN_IF_NEEDED", 0), (0, 0), ("SHARPEN", 0), ("SHARPEN_IF_NEEDED", "CC_SIMPLE"), ("SHARPEN_IF_NEEDED", "CC_FIT"),
         ("SHARPEN", "CC_FIT")]


def mixed_pictures():
    """the mode-B photographs (padded and upscaled variants among them) interleaved with the 4C sample photographs, and a noise
    picture; returns the pictures and their kind ('b', '4c', 'noise')"""
    b = [p for i, p in enumerate(batch_b()) if i != 2]            # batch_b's third picture is its noise picture
    c = [sample(s) for s in GLOB]
    noise = np.random.default_rng(61).integers(0, 256, (900, 1100, 3), dtype=np.uint8)
    pics, kinds = [], []
    for i in range(max(len(b), len(c))):
        if i < len(b):
            pics.append(b[i]); kinds.append("b")
        if i < len(c):
            pics.append(c[i]); kinds.append("4c")
        if i == 2:
            pics.append(noise); kinds.append("noise")
    return pics, kinds


def with_anchors(frame):
    """a rendered frame of any geometry as a camera picture: the four anchor squares of a real encoder frame pasted into its corners
    (as chain_batches.with_anchors does for 1024 x 1024; they lie outside every cell of the 8x8 modes)"""
    tr, c = load_sample("b/tr_0.png"), 62
    f = frame.copy()
    H, W = f.shape[:2]
    for ys, ts in ((slice(0, c), slice(0, c)), (slice(H - c, H), slice(1024 - c, 1024))):
        for xs, us in ((slice(0, c), slice(0, c)), (slice(W - c, W), slice(1024 - c, 1024))):
            f[ys, xs] = tr[ts, us]
    return f


_rendered = {}


def rendered(cb, mode_val):
    """two camera pictures of a random-payload frame of this mode: zero-padded, and upscaled with a perspective tilt"""
    if mode_val in _rendered:
        return _rendered[mode_val]
    import torch
    ctx = cb.Context(mode_val, max_frames=1)
    info = ctx.info
    payload = torch.from_numpy(np.random.default_rng(900 + mode_val).integers(0, 256, info.data_bytes, dtype=np.uint8)).cuda()
    cells = torch.zeros(info.total_cells, dtype=torch.uint8, device="cuda")
    ctx.encode_cells_dev(payload.data_ptr(), 1, cells.data_ptr())
    ctx.sync()
    ctx.close()
    frame = with_anchors(ORA.render_frame(ORA.mode(mode_val), cells.cpu().numpy()))
    H, W = frame.shape[:2]
    big = pad(frame, 90, 110, 120, 80)
    src = np.float32([[0, 0], [W, 0], [0, H], [W, H]])
    dst = np.float32([[40, 30], [1.3 * W + 20, 10], [10, 1.3 * H + 30], [1.3 * W + 50, 1.3 * H + 60]])
    tilt = cv2.warpPerspective(frame, cv2.getPerspectiveTransform(src, dst), (int(1.3 * W) + 100, int(1.3 * H) + 100), flags=cv2.INTER_LINEAR)
    _rendered[mode_val] = [big, tilt]
    return _rendered[mode_val]


_streams = []


def contexts(cb, modes, n):
    """candidate contexts of these modes, all on one stream (the detect call runs on the stream its contexts share)"""
    import torch
    _streams.append(torch.cuda.Stream())
    ctxs = [cb.Context(m, max_frames=n) for m in modes]
    for c in ctxs:
        c.set_stream(_streams[-1].cuda_stream)
    return ctxs


class Detect:
    """device outputs of one detect call over n pictures with these contexts"""

    def __init__(self, ctxs, n):
        import torch
        self.n, self.k = n, len(ctxs)
        self.slot = max(c.info.data_bytes for c in ctxs)
        self.chunks = torch.full((n * self.slot,), 0xA5, dtype=torch.uint8, device="cuda")
        self.mask = torch.full((n,), -7, dtype=torch.int32, device="cuda")
        self.status = torch.full((n,), 7, dtype=torch.int32, device="cuda")
        self.mode = torch.full((n,), 9, dtype=torch.int32, device="cuda")
        self.mode_masks = torch.full((n * self.k,), -7, dtype=torch.int32, device="cuda")

    def call(self, cb, ctxs, d, wh, flags):
        cb.detect_scan_extract_decode_chunks_dev(ctxs, d.data_ptr(), wh, self.chunks.data_ptr(), self.mask.data_ptr(), self.status.data_ptr(),
                                                 self.mode.data_ptr(), self.mode_masks.data_ptr(), flags=flags)

    def host(self):
        return (self.chunks.cpu().numpy().reshape(self.n, self.slot), self.mask.cpu().numpy().view(np.uint32), self.status.cpu().numpy(),
                self.mode.cpu().numpy(), self.mode_masks.cpu().numpy().view(np.uint32).reshape(self.n, self.k))


def detect(cb, ctxs, pics, flags):
    import torch
    d, wh = packed(pics)
    out = Detect(ctxs, len(pics))
    torch.cuda.synchronize()
    out.call(cb, ctxs, d, wh, flags)
    ctxs[0].sync()
    return out.host()


def exact_pictures(cb):
    pics, _ = mixed_pictures()
    return pics[:9] + rendered(cb, 66)[:1] + rendered(cb, 67)[1:] + pics[9:]


def entry_states(n_receivers, seed):
    """distinct entry states: inactive, and colour casts of different strengths"""
    rng = np.random.default_rng(seed)
    out = []
    for r in range(n_receivers):
        if r % 4 == 0:
            out.append(None)
        else:
            out.append(np.diag(rng.uniform(0.7, 1.3, 3)).astype(np.float32) + np.float32(0.01) * rng.standard_normal((3, 3)).astype(np.float32))
    return out


class Out:
    """device outputs of one call over n pictures with these contexts"""

    def __init__(self, ctxs, n):
        import torch
        self.n, self.k = n, len(ctxs)
        self.slot = max(c.info.data_bytes for c in ctxs)
        self.chunks = torch.full((n * self.slot,), 0xA5, dtype=torch.uint8, device="cuda")
        self.mask = torch.full((n,), -7, dtype=torch.int32, device="cuda")
        self.status = torch.full((n,), 7, dtype=torch.int32, device="cuda")
        self.mode = torch.full((n,), 9, dtype=torch.int32, device="cuda")
        self.mode_masks = torch.full((n * self.k,), -7, dtype=torch.int32, device="cuda")

    def call(self, cb, ctxs, ts, orders, of, states, cand, flags):
        cb.detect_scan_extract_decode_chunks_receivers_dev(ctxs, ts, of, states, self.chunks.data_ptr(), self.mask.data_ptr(), self.status.data_ptr(),
                                                           self.mode.data_ptr(), candidates=cand, d_mode_masks=self.mode_masks.data_ptr(),
                                                           flags=flags, order=orders)

    def host(self):
        return (self.chunks.cpu().numpy().reshape(self.n, self.slot), self.mask.cpu().numpy().view(np.uint32), self.status.cpu().numpy(),
                self.mode.cpu().numpy(), self.mode_masks.cpu().numpy().view(np.uint32).reshape(self.n, self.k))


def run(cb, ctxs, ts, orders, of, states, cand, flags):
    import torch
    out = Out(ctxs, len(ts))
    torch.cuda.synchronize()
    out.call(cb, ctxs, ts, orders, of, states, cand, flags)
    ctxs[0].sync()
    return out.host()


def close(*lists):
    for cs in lists:
        for c in cs:
            c.close()


def stream_contexts(cb, modes, n):
    """candidate contexts on one new stream: (contexts, stream)"""
    import torch
    stream = torch.cuda.Stream()
    ctxs = [cb.Context(m, max_frames=n) for m in modes]
    for c in ctxs:
        c.set_stream(stream.cuda_stream)
    return ctxs, stream


def nonempty(cand, of, K, R):
    return np.flatnonzero((np.asarray(of, np.int64) >= 0) & (np.asarray(of, np.int64) < R) & (np.asarray(cand, np.uint32) & np.uint32((1 << K) - 1) != 0))


def launches(n, K, R, rng, modes):
    """five launches' (candidates, map): all-auto, all locked to one mode, mixed sessions, empty slots of both kinds, random"""
    auto = (1 << K) - 1
    lock = 1 << (modes.index(68) if 68 in modes else 0)
    of = [rng.integers(0, R - 1, n) for _ in range(5)]          # receiver R - 1 never has a picture
    sess_lock = rng.integers(0, K, R)
    sess_auto = rng.random(R) < 0.3
    mixed = np.where(sess_auto[of[2]], auto, 1 << sess_lock[of[2]])
    holes = rng.integers(1, auto + 1, n)
    holes[::4] = 0                                              # no candidate
    holes[1::6] = 1 << (K + 1 + np.arange(len(holes[1::6])) % (31 - K))    # only bits at or above n_modes
    of3 = of[3].copy()
    of3[2::5] = np.array([-1, R, INT_MIN, INT_MAX, R + 7])[np.arange(len(of3[2::5])) % 5]
    rand_of = rng.integers(-2, R + 2, n)
    rand_of[rand_of == R - 1] = R                               # out of range instead: receiver R - 1 still has no picture
    rand_cand = rng.integers(0, 1 << (K + 2), n)
    return [(np.full(n, auto), of[0]), (np.full(n, lock), of[1]), (mixed, of[2]), (holes, of3), (rand_cand, rand_of)]
