"""Ragged camera batches -- n pictures, each of its own size -- through the extractor kernels (csrc/scan.cu, csrc/deskew.cu) and the
ragged entry points: every picture must come out as the CPU restatement (oracle/scan_oracle.c) and the reference CLI's decode loop
(`cimbar -m 4C samples/6bit/*.jpg`: scan, warp, decode with sharpen iff NEEDS_SHARPEN, one decoder, in order) give it, and a
batch of one shape must equal the uniform entry points bit for bit.  Each test asserts its own premise.  The sample directory is
tests/ragged_samples.py's GLOB (its largest photograph stands in as an upscale of another)."""
import cv2
import numpy as np
import pytest

from ragged_samples import BIG, GLOB, sample
from scan_oracle_lib import ScanOracle, join
from gpu_support import cb  # noqa: F401  (fixtures)
from gpu_support import ORA, check_dense, pad, sharpen_cli_loop

pytestmark = pytest.mark.gpu

SO = ScanOracle()


def radius(w, h):
    """Scanner's blur radius (Scanner.h:93-103): unit = next power of two + 1 of 0.002 x the short side, at least 3"""
    v = int(min(w, h) * 0.002) - 1
    v &= 0xFFFFFFFF
    for s in (1, 2, 4, 8, 16):
        v |= v >> s
    return max((v + 2) & 0xFFFFFFFF, 3) // 2


def word_path(pics):
    """per picture: (width a multiple of 4, its packed offset 4-byte aligned) -- the bases themselves come from cudaMalloc"""
    out, off = [], 0
    for p in pics:
        h, w = p.shape[:2]
        out.append((w % 4 == 0, off % 4 == 0))
        off += w * h
    return out


# ------------------------------------------------------------------------------------------------ scan
def scan_batch():
    rng = np.random.default_rng(41)
    pics = [sample(s) for s in GLOB]
    pics.append(cv2.resize(sample("6bit/4_30_f2_734.jpg"), None, fx=1.7, fy=1.7))           # 2176 x 1632: 5 taps
    pics.append(np.ascontiguousarray(sample("6bit/4_30_f0_627.jpg")[:637, 3:958]))         # 955 x 637: odd area
    pics.append(sample("6bit/4_30_f2_246.jpg"))                                            # width 1280 at an unaligned base
    pics.append(rng.integers(0, 256, (701, 900, 3), dtype=np.uint8))
    pics.append(np.zeros((480, 640, 3), np.uint8))
    return pics


def test_ragged_scan_matches_oracle(cb):
    pics = scan_batch()
    want = [(SO.preprocess(p), SO.scan(p)) for p in pics]
    orders = [list(range(len(pics))), list(range(len(pics)))[::-1]]
    # premise: the 3-, 5- and 9-tap blurs, and widths that are a multiple of 4 at aligned and at unaligned offsets
    assert {radius(p.shape[1], p.shape[0]) for p in pics} == {1, 2, 4}
    outcomes = {al for order in orders for m4, al in word_path([pics[i] for i in order]) if m4}
    assert outcomes == {True, False}
    ctx = cb.Context(4, max_frames=1)
    for order in orders:
        batch = [pics[i] for i in order]
        anchors, count, cutoff = ctx.scan_ragged(batch)
        blurred, thr = ctx.scan_blurred_ragged([p.shape for p in batch])
        for j, i in enumerate(order):
            (t, _, bl), (wa, wc) = want[i]
            assert np.array_equal(blurred[j], bl), (order[0], i)
            assert thr[j] == t, (order[0], i)
            got = [tuple(int(v) for v in anchors[j, k]) for k in range(max(count[j], 0))]
            assert count[j] == len(wa) and got == wa, (i, join(got), join(wa))
            assert cutoff[j] == wc, i
            assert not anchors[j, len(wa):].any()
    ctx.close()


# ------------------------------------------------------------------------------------------------ uniform batches
@pytest.mark.parametrize("n", [1, 5])
def test_one_shape_equals_the_uniform_calls(cb, n):
    rng = np.random.default_rng(43)
    land = [sample(s) for s in ("6bit/4_30_f0_627.jpg", "6bit/4_30_f2_246.jpg", "6bit/4_30_802.jpg")]        # 960 x 1280
    small = cv2.resize(sample("6bit/4_30_f1_360.jpg"), (720, 960))                                          # portrait, shrunk
    padded = pad(small, 0, 0, 280, 280)                                                                    # 960 x 1280, zero-padded
    pool = [land[0], padded, rng.integers(0, 256, land[0].shape, dtype=np.uint8), land[1], land[2]]
    pics = pool[:n]
    stack = np.stack(pics)
    u, r = cb.Context(4, max_frames=n), cb.Context(4, max_frames=n)
    a0 = u.scan(stack)
    a1 = r.scan_ragged(pics)
    for x, y in zip(a0, a1):
        assert np.array_equal(x, y)
    b0 = u.scan_blurred(n, 960, 1280)
    b1 = r.scan_blurred_ragged([p.shape for p in pics])
    assert np.array_equal(b0[0], np.stack(b1[0])) and np.array_equal(b0[1], b1[1])
    statuses = set()
    for flags in (0, cb.FLAG_SHARPEN, cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT):
        u.set_ccm(None)
        r.set_ccm(None)
        o0 = u.scan_extract_decode_fountain(stack, flags=flags)
        o1 = r.scan_extract_decode_fountain_ragged(pics, flags=flags)
        for x, y in zip(o0, o1):
            assert np.array_equal(x, y), flags
        c0, c1 = u.get_ccm(), r.get_ccm()
        assert (c0 is None) == (c1 is None) and (c0 is None or np.array_equal(c0, c1))
        statuses |= set(o0[4].tolist())
    if n == 5:
        assert {0, 2} <= statuses                                      # premise: failures and NEEDS_SHARPEN pictures in the batch
    u.close()
    r.close()


# ------------------------------------------------------------------------------------------------ the CLI loop
def cli_batch():
    """samples/6bit/*.jpg in glob order, zero-padded photographs of two further sizes and a noise picture (not last: the CLI skips a
    FAILURE picture, so the CCM after the batch is the last decoded picture's either way)"""
    pics = [sample(s) for s in GLOB]
    pics.append(pad(sample("6bit/4_30_f0_627.jpg"), 120, 150, 100, 160))                 # 1230 x 1540
    pics.append(np.random.default_rng(47).integers(0, 256, (900, 1200, 3), dtype=np.uint8))
    pics.append(pad(sample("6bit/4_30_f1_360.jpg"), 90, 70, 200, 140))                   # 1440 x 1300
    pics.append(sample("6bit/4_30_f2_734.jpg"))
    return pics


def cli_loop(m, pics, cc, monkeypatch):
    """_cli_loop, and the oracle decoder's CCM at its end (read just before its final reset)"""
    seen = {}
    set_ccm = ORA.set_ccm

    def spy(m9):
        if m9 is None:
            seen.setdefault("calls", 0)
            seen["calls"] += 1
            if seen["calls"] == 2:
                seen["ccm"] = ORA.get_ccm()
        set_ccm(m9)
    monkeypatch.setattr(ORA, "set_ccm", spy)
    out = sharpen_cli_loop(m, pics, cc)
    monkeypatch.setattr(ORA, "set_ccm", set_ccm)
    assert seen["calls"] == 2
    return out, seen["ccm"]


@pytest.mark.parametrize("cc", [0, 1, 2])
def test_ragged_batch_matches_the_cli_loop(cb, cc, monkeypatch):
    pics = cli_batch()
    n = len(pics)
    m = ORA.mode(4)
    want, last_ccm = cli_loop(m, pics, cc, monkeypatch)
    assert sorted({w[0] for w in want}) == [0, 1, 2]
    assert any(w[0] == 2 and w[2][0] > 0 for w in want) and any(w[0] == 1 and w[2][0] > 0 for w in want)
    assert sum(a.shape != b.shape for a, b in zip(pics, pics[1:])) >= 5
    ccf = {0: 0, 1: cb.FLAG_CC_SIMPLE, 2: cb.FLAG_CC_FIT}[cc]
    ctx = cb.Context(4, max_frames=n)
    chunks, count, mask, ff, status = ctx.scan_extract_decode_fountain_ragged(pics, flags=cb.FLAG_SHARPEN_IF_NEEDED | ccf)
    assert status.tolist() == [w[0] for w in want]
    for i, (st, xy, wd) in enumerate(want):
        if st == 0:
            assert count[i] == 0 and mask[i] == 0
        else:
            check_dense(m, chunks[i], count[i], mask[i], wd, (cc, i))
    got = ctx.get_ccm()
    assert (got is None) == (last_ccm is None) and (last_ccm is None or np.array_equal(got, last_ccm)), cc
    ctx.close()


def test_given_corners_equal_single_picture_calls(cb):
    """cb200_extract_decode_fountain_ragged_dev with the oracle's corners == in-order single-picture cb200_extract_decode_fountain
    calls on one context (CC_FIT carries across both)"""
    import torch
    pics = [p for p in cli_batch() if len(SO.scan(p)[0] or []) == 4]
    corners = np.array([SO.corners(SO.scan(p)[0]) for p in pics], np.float32)
    n = len(pics)
    assert len({p.shape for p in pics}) >= 5
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    one = cb.Context(4, max_frames=1)
    want = [one.extract_decode_fountain(p, c, flags=flags) for p, c in zip(pics, corners)]
    d_src = torch.cat([torch.from_numpy(p.reshape(-1)) for p in pics]).cuda()
    wh = np.array([(p.shape[1], p.shape[0]) for p in pics], np.int32)
    ctx = cb.Context(4, max_frames=n)
    ch = np.zeros((n, ctx.info.chunks_per_frame, ctx.info.chunk_size), np.uint8)
    cnt, mk, fl = np.zeros(n, np.uint32), np.zeros(n, np.uint32), np.zeros(n, np.uint8)
    cb._check(ctx.lib.cb200_extract_decode_fountain_ragged_dev(ctx._h, d_src.data_ptr(), wh.ctypes.data, n, corners.ctypes.data, flags,
                                                                ch.ctypes.data, cnt.ctypes.data, mk.ctypes.data, fl.ctypes.data))
    for i, (c1, n1, m1, f1) in enumerate(want):
        assert cnt[i] == n1[0] and mk[i] == m1[0] and fl[i] == f1[0] and np.array_equal(ch[i], c1[0]), i
    assert cnt.sum() > 0
    c0, c1 = one.get_ccm(), ctx.get_ccm()
    assert (c0 is None) == (c1 is None) and (c0 is None or np.array_equal(c0, c1))
    # more pictures than the context holds: refused before any work
    small = cb.Context(4, max_frames=1)
    rc = small.lib.cb200_extract_decode_fountain_ragged_dev(small._h, d_src.data_ptr(), wh.ctypes.data, 2, corners.ctypes.data, flags,
                                                            ch.ctypes.data, cnt.ctypes.data, mk.ctypes.data, fl.ctypes.data)
    assert rc == -1 and b"max_frames" in small.lib.cb200_last_error()
    with pytest.raises(cb.Cb200Error, match="max_frames"):
        small.scan_extract_decode_fountain_ragged(pics[:2])
    for c in (one, ctx, small):
        c.close()


# ------------------------------------------------------------------------------------------------ past 4 GiB
def test_batch_beyond_four_gib(cb):
    """a packed batch of more than 2^32 bytes whose last picture starts beyond 2^32: every output equals its pool entry's
    single-picture result, through the device entry points (batch assembled on the device) and the host entry point (n pointers into
    the pool, packed by the library)"""
    import torch
    pool = [sample(BIG),                                                                      # 3584 x 2688, 28.9 MB
            cv2.resize(sample("6bit/4_30_f0_627.jpg"), None, fx=2.5, fy=2.5),                 # 2400 x 3200
            pad(sample("6bit/4_30_f2_246.jpg"), 1, 0, 1, 0),                                  # 1281 x 961, odd area: the rest lands unaligned
            cv2.resize(sample("6bit/4_30_f2_734.jpg"), None, fx=2.3, fy=2.3)]
    flags = cb.FLAG_SHARPEN_IF_NEEDED
    one = cb.Context(4, max_frames=1)
    single = []
    for p in pool:
        a, c, cut = one.scan_ragged([p])
        _, thr = one.scan_blurred_ragged([p.shape])
        single.append(((a[0], c[0], cut[0], thr[0]), one.scan_extract_decode_fountain_ragged([p], flags=flags)))
    assert all(s[1][1][0] > 0 for s in single[:2])
    idx, off = [], 0
    while off <= 1 << 32:                       # until the next picture starts beyond 2^32, then that one
        i = len(idx) % len(pool)
        idx.append(i)
        off += pool[i].nbytes
    idx.append(0)
    starts = np.cumsum([0] + [pool[i].nbytes for i in idx])
    assert starts[-2] > 1 << 32 and starts[-1] > 1 << 32
    n = len(idx)
    d_pool = [torch.from_numpy(p.reshape(-1)).cuda() for p in pool]
    d_batch = torch.empty(int(starts[-1]), dtype=torch.uint8, device="cuda")
    for k, i in enumerate(idx):
        d_batch[int(starts[k]):int(starts[k + 1])] = d_pool[i]
    wh = np.array([(pool[i].shape[1], pool[i].shape[0]) for i in idx], np.int32)
    ctx = cb.Context(4, max_frames=n)
    anchors, count, cutoff = np.zeros((n, 4, 4), np.int32), np.zeros(n, np.int32), np.zeros(n, np.uint32)
    cb._check(ctx.lib.cb200_scan_ragged_dev(ctx._h, d_batch.data_ptr(), wh.ctypes.data, n, anchors.ctypes.data, count.ctypes.data,
                                            cutoff.ctypes.data))
    thr = np.zeros(n, np.int32)
    cb._check(ctx.lib.cb200_scan_blurred_ragged(ctx._h, None, thr.ctypes.data, wh.ctypes.data, n))
    for k, i in enumerate(idx):
        (a, c, cut, t), _ = single[i]
        assert np.array_equal(anchors[k], a) and count[k] == c and cutoff[k] == cut and thr[k] == t, (k, i)
    assert (count == 4).all()
    corners = np.stack([(anchors[:, :, 0] + anchors[:, :, 1]) // 2, (anchors[:, :, 2] + anchors[:, :, 3]) // 2], axis=2)
    corners = np.ascontiguousarray(corners.astype(np.float32).reshape(n, 8))
    ch = np.zeros((n, ctx.info.chunks_per_frame, ctx.info.chunk_size), np.uint8)
    cnt, mk, fl = np.zeros(n, np.uint32), np.zeros(n, np.uint32), np.zeros(n, np.uint8)
    cb._check(ctx.lib.cb200_extract_decode_fountain_ragged_dev(ctx._h, d_batch.data_ptr(), wh.ctypes.data, n, corners.ctypes.data, flags,
                                                                ch.ctypes.data, cnt.ctypes.data, mk.ctypes.data, fl.ctypes.data))
    del d_batch
    torch.cuda.empty_cache()
    for k, i in enumerate(idx):
        c1, n1, m1, f1, s1 = single[i][1]
        assert cnt[k] == n1[0] and mk[k] == m1[0] and fl[k] == f1[0] and np.array_equal(ch[k], c1[0]), (k, i)
    chunks, ccount, cmask, ff, status = ctx.scan_extract_decode_fountain_ragged([pool[i] for i in idx], flags=flags)
    for k, i in enumerate(idx):
        c1, n1, m1, f1, s1 = single[i][1]
        assert status[k] == s1[0] and ccount[k] == n1[0] and cmask[k] == m1[0] and ff[k] == f1[0] and np.array_equal(chunks[k], c1[0]), (k, i)
    one.close()
    ctx.close()
