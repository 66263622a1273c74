"""K2 (Reed-Solomon correction and chunk masks) on frames whose RS input is crafted byte by byte.

Every frame here starts as a raw stream: RS codewords (cbo_rs_encode), each damaged by one entry of an error catalogue.  A numpy
inverse of the P7/P10 bit packing turns the stream into cell bytes, and the oracle renders them.  The oracle's decode_raw of the
rendered frame, and the GPU's, return exactly that stream, so the RS kernels see exactly the crafted bytes.  The expected
results come from the reference's own libcorrect (one decoder per stream, in stream order) and its reed_solomon_stream ->
aligned_stream -> escrow stack.

The frames are placed so that every RS kernel meets its edges:
  - k_rs_frames (modes 68 and 4: the whole block range, 4 + 2 bits per cell, 155-byte blocks, parity <= 32, a 4-byte-aligned
    output) takes two frames per CTA and one warp per unit of four blocks: units with 0 to 4 dirty blocks, dirty blocks in
    slot 0 or slot 1 of a pair or both, an unpaired dirty last frame, and more pairs than CTAs (grid-stride loop, cp.async
    prefetch of the next pair);
  - the fused k_rs_decode (modes 8, 66, 67, the colour-correction block ranges, an unaligned output) and the unfused one
    (rs_correct_dev): in mode 8, 70 blocks per frame put blocks 68-69 of an even frame and blocks 0-1 of the next in one unit;
  - k_chunk_mask: failed blocks at every chunk boundary, and in mode 68 every single failed block and every adjacent pair.
The CPU tests (unmarked) pin the premises: the oracle's RS and chunk replay equal the reference's on every crafted block and
frame, the catalogue reaches failure, corrections, and libcorrect's alpha^0 and shortened-code successes, and the raw stream
survives render + decode in all five modes."""
import ctypes as C
import functools

import numpy as np
import pytest

from crafted_rs import ORA, cc_pool, geo, make_block, raw_to_cells
from oracle_lib import Ref, _ptr
from gpu_support import cb  # noqa: F401  (fixtures)

try:
    REF = Ref()
except (FileNotFoundError, OSError) as e:  # pragma: no cover
    REF = None
    pytestmark = pytest.mark.skip(reason=f"oracle/_ref not available: {e}")

MODES = [68, 4, 8, 66, 67]
CATALOGUE = ["clean", "zero", "e1", "t", "tpar", "t1", "many", "random", "first", "last", "short", "shortj"]
# four consecutive blocks: one unit of k_rs_frames (two units of k_rs_decode with T = 2); "fail" is a random block libcorrect rejects
UNITS = [("clean",) * 4, ("clean", "clean", "clean", "t"), ("clean", "clean", "clean", "fail"), ("fail",) * 4,
         ("t", "fail", "e1", "fail"), ("fail", "t", "fail", "tpar"), ("e1", "clean", "clean", "clean"), ("t", "t", "clean", "clean"),
         ("clean", "t", "short", "t"), ("t", "t", "t", "t"), ("fail", "clean", "clean", "clean"), ("shortj", "fail", "last", "t1")]


# ------------------------------------------------------------------------------------------------ expected values
def ref_blocks(g, raw):
    """the reference's libcorrect, one decoder per stream in stream order (reed_solomon_stream): data (zeros when failed), ok"""
    data = np.zeros(g.nblocks * g.msg, np.uint8)
    ok = np.zeros(g.nblocks, np.uint8)
    out = np.zeros(256, np.uint8)
    for lo, hi in g.streams():
        r = REF.lib.ref_rs_create(g.parity)
        for b in range(lo, hi):
            blk = np.ascontiguousarray(raw[b * g.block:(b + 1) * g.block])
            if REF.lib.ref_rs_decode2(r, _ptr(blk), g.block, _ptr(out)) > 0:
                data[b * g.msg:(b + 1) * g.msg] = out[:g.msg]
                ok[b] = 1
        REF.lib.ref_rs_destroy(r)
    return data, ok


def oracle_blocks(g, raw):
    """the same with the oracle's restatement of libcorrect (cbo_rs_decode, one decoder per stream)"""
    data = np.zeros(g.nblocks * g.msg, np.uint8)
    ok = np.zeros(g.nblocks, np.uint8)
    out = np.zeros(256, np.uint8)
    for lo, hi in g.streams():
        rs = ORA.lib.cbo_rs_create(g.parity)
        for b in range(lo, hi):
            blk = np.ascontiguousarray(raw[b * g.block:(b + 1) * g.block])
            if ORA.lib.cbo_rs_decode(rs, _ptr(blk), g.block, _ptr(out)) > 0:
                data[b * g.msg:(b + 1) * g.msg] = out[:g.msg]
                ok[b] = 1
        ORA.lib.cbo_rs_destroy(rs)
    return data, ok


def ref_chunks(g, raw):
    """the reference's stream stack on the raw stream: the good chunks (dense, escrow order) and their count"""
    chunks = np.zeros((g.cpf, g.cs), np.uint8)
    used = C.c_uint(0)
    col_len = g.cap - g.cap_sym
    good = REF.lib.ref_rs_align_escrow(g.parity, g.block, _ptr(np.ascontiguousarray(raw)), g.cap_sym, col_len, g.cs, g.cpf,
                                       _ptr(chunks), C.byref(used))
    assert good == used.value * g.cs
    return chunks, used.value


def oracle_chunks(g, data, ok):
    """the oracle's aligned_stream replay on block results: (dense chunks, chunk mask)"""
    chunks = np.zeros((g.cpf, g.cs), np.uint8)
    mask = C.c_uint32(0)
    ORA.lib.cbo_align_chunks(_ptr(np.ascontiguousarray(data)), _ptr(np.ascontiguousarray(ok)), g.nblocks, g.msg, g.cs,
                             _ptr(chunks), C.byref(mask))
    return chunks, mask.value


# ------------------------------------------------------------------------------------------------ frames
def pool_specs(g):
    """(name, kind per block) of the pool frames of one mode"""
    nb, pc = g.nblocks, g.per_chunk
    specs = [("clean", ["clean"] * nb)]
    for r in range(4):                          # every catalogue kind at every position of a unit
        specs.append((f"catalogue{r}", [CATALOGUE[(b + r) % len(CATALOGUE)] for b in range(nb)]))
    for s in (0, 5):
        specs.append((f"units{s}", [UNITS[(b // 4 + s) % len(UNITS)][b % 4] for b in range(nb)]))
    mix = np.random.default_rng(g.mode_val + 7)
    for r in range(9):
        specs.append((f"mix{r}", [str(k) for k in mix.choice(CATALOGUE + ["fail"], nb)]))
    # the straddle pair: dirty blocks 68-69 of an even frame, 0-1 of the next (one k_rs_decode unit in mode 8)
    tail = [str(k) for k in mix.choice(CATALOGUE, nb)]
    tail[-2:] = ["t", "fail"]
    specs.append(("tail", tail))
    specs.append(("head", ["fail", "t"] + ["clean"] * (nb - 2)))

    def bad(blocks, base="clean"):
        kinds = [base] * nb
        for b in blocks:
            kinds[b] = "fail"
        return kinds
    specs += [("cm_last_of_q", bad([2 * pc - 1])),                       # chunk 1 fails, chunk 2 is dropped by the carry
              ("cm_first_of_q1", bad([2 * pc])),                         # chunk 2 fails, chunk 3 is emitted
              ("cm_carry_over_good", bad([pc - 1], base="t")),           # chunk 1 corrects every block, and is still dropped
              ("cm_last_of_every", bad([q * pc + pc - 1 for q in range(g.cpf)])),
              ("cm_last_symbol", bad([g.nbs - 1 if not g.legacy else nb // 2 - 1])),
              ("cm_frame_last", bad([nb - 1])),
              ("cm_all", bad(range(nb)))]
    return specs


def pair_specs(g):
    """mode 68: every single failed block and every adjacent failed pair"""
    nb = g.nblocks
    return ([(f"bad{b}", ["fail" if k == b else "clean" for k in range(nb)]) for b in range(nb)] +
            [(f"bad{b}-{b + 1}", ["fail" if k in (b, b + 1) else "clean" for k in range(nb)]) for b in range(nb - 1)])


class Pool:
    """crafted frames of one mode: raw stream, cells, rendered frame and the reference's results per frame"""

    def __init__(self, g, specs, seed, render=True):
        rng = np.random.default_rng(seed)
        self.g, self.names = g, [s[0] for s in specs]
        self.kinds = [s[1] for s in specs]
        P = len(specs)
        self.raw = np.zeros((P, g.cap), np.uint8)
        for f, kinds in enumerate(self.kinds):
            for b, kind in enumerate(kinds):
                self.raw[f, b * g.block:(b + 1) * g.block] = make_block(g, kind, rng)
        self.data = np.zeros((P, g.nblocks * g.msg), np.uint8)
        self.ok = np.zeros((P, g.nblocks), np.uint8)
        self.chunks = np.zeros((P, g.cpf, g.cs), np.uint8)
        self.used = np.zeros(P, np.int64)
        self.mask = np.zeros(P, np.uint32)
        for f in range(P):
            self.data[f], self.ok[f] = ref_blocks(g, self.raw[f])
            self.chunks[f], self.used[f] = ref_chunks(g, self.raw[f])
            ochunks, self.mask[f] = oracle_chunks(g, self.data[f], self.ok[f])
            # the mask names the reference's chunks: same count, same bytes
            assert bin(int(self.mask[f])).count("1") == self.used[f] and np.array_equal(ochunks, self.chunks[f]), self.names[f]
            for b, kind in enumerate(self.kinds[f]):
                if kind == "fail":
                    assert self.ok[f, b] == 0, (self.names[f], b)          # libcorrect rejects every forced failure
        if render:
            self.cells = np.stack([raw_to_cells(g, r) for r in self.raw])
            self.frames = np.stack([ORA.render_frame(g.m, c) for c in self.cells])

    def index(self, name):
        return self.names.index(name)


@functools.lru_cache(maxsize=None)
def pool(mode_val):
    g = geo(mode_val)
    return Pool(g, pool_specs(g), seed=1000 + mode_val)


@functools.lru_cache(maxsize=None)
def pair_pool():
    g = geo(68)
    return Pool(g, pair_specs(g), seed=2068)


# ------------------------------------------------------------------------------------------------ launch arithmetic (k2_rs.cu)
def frames_kernel_admits(g):
    """k2_rs_fused_launch's condition for k_rs_frames, for the whole block range and a 4-byte-aligned output"""
    m = g.m
    return (m.symbol_bits == 4 and m.color_bits == 2 and (not g.legacy or g.ncells * 6 == g.cap * 8) and g.block == 155 and
            g.parity <= 32 and g.parity <= 40 and g.nblocks % 4 == 0 and 2 * (g.nblocks // 4) <= 32 and g.ncells % 16 == 0 and
            g.cap_sym % 155 == 0 and (g.nblocks * g.msg) % 4 == 0)


def frames_grid(n, sms):
    """k_rs_frames: (pair groups, CTAs)"""
    groups = (n + 1) // 2
    return groups, min(groups, 2 * sms)


def decode_grid(n, b_count, parity, sms):
    """k_rs_decode: (units, CTAs); 16 warps per CTA, one unit per warp and pass"""
    T = 1 if parity <= 32 else 2
    units = -(-n * b_count // (4 // T))
    return units, max(1, min(-(-units // 16), sms * (4 if T == 1 else 2)))


# ================================================================================================ CPU tests
@pytest.mark.parametrize("mode_val", MODES)
def test_catalogue_oracle_rs_matches_libcorrect(mode_val):
    """every crafted block: the oracle's libcorrect restatement and the reference's libcorrect agree (result and bytes), and the
    catalogue reaches failure, success with corrections, the alpha^0 success and the shortened-code success"""
    p = pool(mode_val)
    g = p.g
    seen = dict(fail=0, corrected=0, alpha0=0, shortened=0, t_ok=0)
    for f in range(len(p.names)):
        data, ok = oracle_blocks(g, p.raw[f])
        assert np.array_equal(ok, p.ok[f]) and np.array_equal(data, p.data[f]), p.names[f]
        for b, kind in enumerate(p.kinds[f]):
            sent = p.raw[f, b * g.block:b * g.block + g.msg]
            got = p.data[f, b * g.msg:(b + 1) * g.msg]
            if not p.ok[f, b]:
                seen["fail"] += 1
                assert not got.any()
                continue
            seen["corrected"] += int(not np.array_equal(got, sent))
            if kind == "last":                  # root alpha^0: location 255, outside the received polynomial
                assert np.array_equal(got, sent)
                seen["alpha0"] += 1
            if kind == "short":                 # the k corrections land in the bytes that were never sent
                assert np.array_equal(got, sent)
                seen["shortened"] += 1
            if kind in ("e1", "t", "tpar", "first", "shortj"):
                seen["t_ok"] += 1
        for b, kind in enumerate(p.kinds[f]):   # at most t errors: always decoded
            if kind in ("clean", "zero", "e1", "t", "tpar", "first", "last", "short", "shortj"):
                assert p.ok[f, b], (p.names[f], b, kind)
    assert min(seen.values()) > 0, seen


@pytest.mark.parametrize("mode_val", MODES)
def test_crafted_raw_survives_render_and_decode(mode_val):
    """raw -> cells -> rendered frame -> the oracle's decode_raw is the identity on every pool frame, and the oracle's decode and
    decode_fountain of the frame give the reference's blocks, chunks and mask"""
    p = pool(mode_val)
    g = p.g
    for f in range(len(p.names)):
        assert np.array_equal(ORA.decode_raw(g.m, p.frames[f]), p.raw[f]), p.names[f]
        data, ok = ORA.decode(g.m, p.frames[f])
        assert np.array_equal(ok, p.ok[f]) and np.array_equal(data, p.data[f]), p.names[f]
        good, chunks, mask = ORA.decode_fountain(g.m, p.frames[f])
        assert mask == p.mask[f] and good == p.used[f] * g.cs, p.names[f]
        assert np.array_equal(chunks[:p.used[f]], p.chunks[f, :p.used[f]]), p.names[f]


@pytest.mark.parametrize("mode_val", MODES)
def test_chunk_replay_matches_reference_stack(mode_val):
    """the oracle's aligned_stream replay (on the oracle's own RS results) against the reference's stream stack, for the chunk-mask
    patterns (and mode 8, which the older stream-stack test leaves out); in mode 68 also every single failed block and every
    adjacent pair"""
    pools = [pool(mode_val)] + ([pair_pool()] if mode_val == 68 else [])
    for p in pools:
        g = p.g
        for f in range(len(p.names)):
            data, ok = oracle_blocks(g, p.raw[f])
            chunks, mask = oracle_chunks(g, data, ok)
            assert mask == p.mask[f] and np.array_equal(chunks, p.chunks[f]), p.names[f]
    p = pool(mode_val)
    masks = {n: int(p.mask[p.index(n)]) for n in p.names if n.startswith("cm_") or n == "clean"}
    full, pc = (1 << p.g.cpf) - 1, p.g.per_chunk
    assert masks["clean"] == full and masks["cm_all"] == 0
    assert masks["cm_last_of_q"] == full & ~0b110 and masks["cm_first_of_q1"] == full & ~0b100
    assert masks["cm_carry_over_good"] == full & ~0b11 and masks["cm_last_of_every"] == 0
    assert masks["cm_frame_last"] == full >> 1
    i = p.index("cm_carry_over_good")
    assert not p.ok[i].all() and p.ok[i, pc:2 * pc].all()                  # chunk 1 decodes and is still dropped
    assert len(p.names) == 25
    if mode_val == 68:
        q = pair_pool()
        assert len(q.names) == 119 and (q.ok.sum(axis=1) >= 58).all()


def test_frame_pair_kernel_serves_modes_68_and_4_only():
    """the frame-pair kernel's launch condition admits exactly the 4 + 2 bit modes with 155-byte blocks: 68 (B) and 4 (4C)"""
    assert [mv for mv in MODES if frames_kernel_admits(geo(mv))] == [68, 4]


# ================================================================================================ GPU tests


@pytest.fixture(scope="module")
def torch():
    import torch
    return torch


@pytest.fixture(scope="module")
def sms(cb):
    ctx = cb.Context(68, max_frames=1)
    n = ctx.info.sm_count
    ctx.close()
    return n


@pytest.fixture(scope="module")
def premised(cb):
    """pool frames checked once per mode: the GPU's decode_raw returns the crafted stream, without the exact-walk fallback"""
    done = set()

    def check(p):
        if id(p) in done:
            return p
        ctx = cb.Context(p.g.mode_val, max_frames=len(p.names))
        try:
            raw, ff = ctx.decode_raw(p.frames)
        finally:
            ctx.close()
        bad = [p.names[f] for f in range(len(p.names)) if not np.array_equal(raw[f], p.raw[f])]
        assert not bad and not (ff & cb.FRAME_FALLBACK).any(), (bad, ff.tolist())
        done.add(id(p))
        return p
    return check


def batch_index(p, n):
    """pool indices of an n-frame batch.  Frames 0-1 are the straddle pair (tail, head); then pairs with dirty frames in slot 0
    only, slot 1 only, both, neither, in turn; an odd batch ends with the dirty tail frame, unpaired"""
    clean, tail, head = p.index("clean"), p.index("tail"), p.index("head")
    dirty = [i for i in range(len(p.names)) if i != clean]
    seq, k, r = [tail, head], 0, 0
    while len(seq) < n:
        d1, d2 = dirty[k % len(dirty)], dirty[(k + 1) % len(dirty)]
        seq += [(d1, clean), (clean, d1), (d1, d2), (clean, clean)][r % 4]
        k += (1, 1, 2, 0)[r % 4]
        r += 1
    seq = seq[:n]
    if n % 2:
        seq[-1] = tail
    return np.array(seq, np.int64)


def _stream(torch, ctx):
    s = torch.cuda.Stream()
    ctx.set_stream(s.cuda_stream)
    return s


def _rows_differ(a, b):
    return np.flatnonzero((a != b).reshape(a.shape[0], -1).any(axis=1))


def _check_batch(p, idx, data, ok=None, mask=None, what=""):
    bad = _rows_differ(data, p.data[idx])
    assert bad.size == 0, f"{what}: {bad.size} frames' data differ, first {bad[:6].tolist()} ({[p.names[i] for i in idx[bad[:6]]]})"
    if ok is not None:
        bad = _rows_differ(ok, p.ok[idx])
        assert bad.size == 0, f"{what}: block_ok differs in {bad.size} frames, first {[p.names[i] for i in idx[bad[:6]]]}"
    if mask is not None:
        bad = np.flatnonzero(mask.astype(np.uint32) != p.mask[idx])
        assert bad.size == 0, f"{what}: chunk mask differs in {bad.size} frames, first {[p.names[i] for i in idx[bad[:6]]]}"


def _run_batch(cb, torch, p, idx):
    """decode_chunks_dev into an aligned and a 1-byte-offset buffer, and rs_correct_dev on the raw streams, for the batch idx"""
    g, n = p.g, idx.size
    ctx = cb.Context(g.mode_val, max_frames=n)
    db = ctx.info.data_bytes
    try:
        with torch.cuda.stream(_stream(torch, ctx)):
            d_idx = torch.from_numpy(idx).cuda()
            d_rgb = torch.from_numpy(p.frames).cuda()[d_idx]
            d_raw = torch.from_numpy(p.raw).cuda()[d_idx]
            d_data = torch.empty((n, db), dtype=torch.uint8, device="cuda")
            d_odd = torch.empty(n * db + 16, dtype=torch.uint8, device="cuda")
            d_rs = torch.empty((n, db), dtype=torch.uint8, device="cuda")
            d_ok = torch.empty((n, g.nblocks), dtype=torch.uint8, device="cuda")
            d_mask = torch.empty(n, dtype=torch.int32, device="cuda")
            d_mask2 = torch.empty(n, dtype=torch.int32, device="cuda")
            d_flags = torch.empty(n, dtype=torch.uint8, device="cuda")
            assert d_data.data_ptr() % 4 == 0
            ctx.decode_chunks_dev(d_rgb.data_ptr(), n, d_data.data_ptr(), d_mask.data_ptr(), d_flags.data_ptr())
            ctx.decode_chunks_dev(d_rgb.data_ptr(), n, d_odd.data_ptr() + 1, d_mask2.data_ptr())
            ctx.rs_correct_dev(d_raw.data_ptr(), n, d_rs.data_ptr(), d_ok.data_ptr())
            out = dict(data=d_data.cpu().numpy(), odd=d_odd.cpu().numpy()[1:1 + n * db].reshape(n, db), mask=d_mask.cpu().numpy(),
                       mask2=d_mask2.cpu().numpy(), flags=d_flags.cpu().numpy(), rs=d_rs.cpu().numpy(), ok=d_ok.cpu().numpy())
    finally:
        torch.cuda.synchronize()
        ctx.close()
        d_rgb = d_raw = d_data = d_odd = d_rs = None
        torch.cuda.empty_cache()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 2, 3, 31, "4sms+1"])
@pytest.mark.parametrize("mode_val", MODES)
def test_crafted_batches_every_rs_kernel(cb, torch, sms, premised, mode_val, n):
    """decode_chunks_dev (aligned: k_rs_frames in modes 68 and 4, fused k_rs_decode elsewhere; offset by one byte: fused
    k_rs_decode everywhere) and rs_correct_dev (unfused k_rs_decode) against libcorrect, block for block, and the chunk masks
    against the reference's stream stack"""
    p = premised(pool(mode_val))
    g = p.g
    big = n == "4sms+1"
    n = 4 * sms + 1 if big else n
    idx = batch_index(p, n)
    dirty = p.ok[idx].min(axis=1) == 0
    clean = p.index("clean")
    if n >= 2:
        assert dirty[0] and dirty[1]                                        # the straddle pair
    if n % 2:
        assert idx[-1] == p.index("tail") and dirty[-1]                      # an unpaired dirty last frame
    if n >= 31:
        pairs = set(zip((idx[0::2] == clean).tolist(), (idx[1::2] == clean).tolist()))
        assert {(False, True), (True, False), (False, False), (True, True)} <= pairs
    if big:
        if frames_kernel_admits(g):
            groups, ctas = frames_grid(n, sms)
            # more pairs than CTAs: CTA 0 takes the unpaired last frame in its second pass, after prefetching it
            assert groups == 2 * sms + 1 and ctas == 2 * sms and (groups - 1) % ctas == 0 and n == 2 * (groups - 1) + 1
        else:
            units, ctas = decode_grid(n, g.nblocks, g.parity, sms)
            assert units > 16 * ctas, (units, ctas)                         # the persistent grid takes more than one pass
    if g.mode_val == 8:
        assert g.nblocks % 4 == 2                                           # units of four blocks straddle an even and an odd frame
    out = _run_batch(cb, torch, p, idx)
    assert not out["flags"].any()
    _check_batch(p, idx, out["data"], mask=out["mask"], what="decode_chunks_dev")
    _check_batch(p, idx, out["odd"], mask=out["mask2"], what="decode_chunks_dev, unaligned output")
    assert np.array_equal(out["odd"], out["data"]) and np.array_equal(out["mask2"], out["mask"])
    _check_batch(p, idx, out["rs"], ok=out["ok"], what="rs_correct_dev")
    if n <= 31:                                                            # the host entry points
        ctx = cb.Context(g.mode_val, max_frames=n)
        try:
            data, ok, ff = ctx.decode(p.frames[idx])
            _check_batch(p, idx, data, ok=ok, what="decode")
            chunks, count, mask, ff2 = ctx.decode_fountain(p.frames[idx])
        finally:
            ctx.close()
        assert not ff.any() and not ff2.any()
        _check_batch(p, idx, data, mask=mask, what="decode_fountain")
        for f, i in enumerate(idx):
            assert count[f] == p.used[i] and np.array_equal(chunks[f][:count[f]], p.chunks[i, :count[f]]), (f, p.names[i])


@pytest.mark.gpu
def test_chunk_masks_every_failed_block_and_pair(cb, torch, premised):
    """mode 68: one frame per single failed block (60) and per adjacent failed pair (59), in one batch and reversed"""
    p = premised(pair_pool())
    for idx in (np.arange(len(p.names)), np.arange(len(p.names))[::-1].copy()):
        out = _run_batch(cb, torch, p, idx)
        _check_batch(p, idx, out["data"], mask=out["mask"], what="decode_chunks_dev")
        _check_batch(p, idx, out["odd"], mask=out["mask2"], what="decode_chunks_dev, unaligned output")
        _check_batch(p, idx, out["rs"], ok=out["ok"], what="rs_correct_dev")


@pytest.mark.gpu
@pytest.mark.parametrize("mode_val", [68, 66, 67])
def test_colour_correction_fit_block_ranges(cb, mode_val):
    """FLAG_CC_FIT runs the fused k_rs_decode on the symbol blocks, fits each frame's matrix from the header they carry, and
    runs it again on the colour blocks.  Against the oracle's in-order decode: chunks, masks, and every frame's matrix bit for
    bit (the batch's prefixes leave each frame's matrix in the context)"""
    g, payload, raw, frames = cc_pool(mode_val)
    m = g.m
    ORA.set_ccm(None)
    want = []
    try:
        for fr in frames:
            good, chunks, mask = ORA.decode_fountain(m, fr, color_correction=2)
            want.append((good, chunks.copy(), mask, ORA.get_ccm()))
    finally:
        ORA.set_ccm(None)
    # premises: frame 1 recovers its header only through RS correction; frame 2 has none and carries frame 1's matrix
    sym1 = ORA.decode_raw(m, frames[1], color_correction=0)[:g.cap_sym]
    data1, ok1 = oracle_blocks(g, ORA.decode_raw(m, frames[1]))
    assert not np.array_equal(sym1[:6], payload[1, :6]) and ok1[0] and np.array_equal(data1[:6], payload[1, :6])
    assert want[1][3] is not None and not np.array_equal(want[1][3], want[0][3])
    _, ok2 = oracle_blocks(g, ORA.decode_raw(m, frames[2]))
    assert not ok2[:g.nbs].any() and np.array_equal(want[2][3], want[1][3])
    ctx = cb.Context(mode_val, max_frames=len(frames))
    try:
        chunks, counts, masks, ff = ctx.decode_fountain(frames, flags=cb.FLAG_CC_FIT)
        for f, (good, wchunks, wmask, _) in enumerate(want):
            assert masks[f] == wmask and counts[f] * g.cs == good, f
            assert np.array_equal(chunks[f][:counts[f]], wchunks[:counts[f]]), f
        for k in range(1, len(frames) + 1):
            ctx.set_ccm(None)
            ctx.decode_fountain(frames[:k], flags=cb.FLAG_CC_FIT)
            got = ctx.get_ccm()
            assert got is not None and np.array_equal(got, want[k - 1][3]), k
    finally:
        ctx.close()
