"""Crafted raw Reed-Solomon streams: the stream layout of each mode, an error catalogue of single RS blocks, the numpy inverse of
the bit packing that turns a raw stream into cell bytes, and the colour-correction fountain frames built from them.  Test
infrastructure only: tests/test_gpu_rs_crafted.py pins these against libcorrect, and chain_batches.py renders the fountain
frames under colour casts."""
import ctypes as C
import functools

import numpy as np

from oracle_lib import Oracle, _ptr

ORA = Oracle()


# ------------------------------------------------------------------------------------------------ geometry and packing
class Geo:
    """one mode's stream layout: RS blocks of the symbol stream, then of the colour stream (one coupled stream when legacy)"""

    def __init__(self, mode_val):
        m = self.m = ORA.mode(mode_val)
        self.mode_val = mode_val
        self.block, self.parity = m.ecc_block_size, m.ecc_bytes
        self.msg, self.t = self.block - self.parity, self.parity // 2
        self.cap = ORA.capacity(m)
        self.nblocks = self.cap // self.block
        self.legacy = bool(m.legacy_mode)
        self.cap_sym = self.cap if self.legacy else ORA.capacity(m, m.symbol_bits)
        self.nbs = self.cap_sym // self.block
        self.cs, self.cpf = m.chunk_size, m.chunks_per_frame
        self.per_chunk = self.cs // self.msg
        self.ncells = m.total_cells
        idx = np.zeros(self.ncells, np.uint32)
        ORA.lib.cbo_interleave_indices(self.ncells, m.interleave_blocks, m.interleave_partitions, _ptr(idx, C.c_uint))
        self.idx = idx.astype(np.int64)                       # interleave slot -> cell
        assert self.nblocks * self.block == self.cap and self.nbs * self.block == self.cap_sym
        assert self.per_chunk * self.msg == self.cs and self.per_chunk * self.cpf == self.nblocks
        self.rs = ORA.lib.cbo_rs_create(self.parity)

    def streams(self):
        return [(0, self.nblocks)] if self.legacy else [(0, self.nbs), (self.nbs, self.nblocks)]


def _slots(bits, width):
    v = np.zeros(bits.size // width, np.int64)
    for k in range(width):
        v = (v << 1) | bits[k::width]
    return v


def raw_to_cells(g, raw):
    """inverse of P7/P10 (Decoder.h bit packing + Interleave): cell bytes symbol | colour << symbol_bits whose decode is `raw`"""
    m = g.m
    bits = np.unpackbits(raw).astype(np.int64)
    cells = np.zeros(g.ncells, np.uint8)
    if g.legacy:                                   # one MSB-first stream of colour << symbol_bits | symbol values
        cells[g.idx] = _slots(bits, m.symbol_bits + m.color_bits)
    else:                                          # symbols (two per byte), then colours (four per byte), MSB first
        sym = _slots(bits[:8 * g.cap_sym], m.symbol_bits)
        col = _slots(bits[8 * g.cap_sym:], m.color_bits)
        cells[g.idx] = (col << m.symbol_bits) | sym
    return cells


# ------------------------------------------------------------------------------------------------ the error catalogue
def _codeword(g, rng, zero=False):
    msg = np.zeros(g.msg, np.uint8) if zero else rng.integers(0, 256, g.msg, dtype=np.uint8)
    enc = np.zeros(255, np.uint8)
    ORA.lib.cbo_rs_encode(g.rs, _ptr(msg), g.msg, _ptr(enc))
    return enc[:g.block].copy()


def _hit(blk, pos, rng):
    pos = np.asarray(pos, np.int64)
    blk[pos] ^= rng.integers(1, 256, pos.size, dtype=np.uint8)
    return blk


def _shortened(g, rng, k, j):
    """a full-length codeword (255 - parity message bytes) with k non-zero bytes among its leading 255 - block bytes, sent without
    them, plus j errors inside the block: libcorrect finds all k + j <= t, "corrects" the k outside the received word, succeeds"""
    msg = rng.integers(0, 256, 255 - g.parity, dtype=np.uint8)
    lead = 255 - g.block
    msg[:lead] = 0
    msg[rng.choice(lead, k, replace=False)] = rng.integers(1, 256, k, dtype=np.uint8)
    enc = np.zeros(255, np.uint8)
    ORA.lib.cbo_rs_encode(g.rs, _ptr(msg), 255 - g.parity, _ptr(enc))
    blk = enc[lead:].copy()
    return _hit(blk, rng.choice(g.block, j, replace=False), rng) if j else blk


def _oracle_fails(g, blk):
    out = np.zeros(256, np.uint8)
    return ORA.lib.cbo_rs_decode(g.rs, _ptr(blk), g.block, _ptr(out)) <= 0


def make_block(g, kind, rng):
    t, P, B = g.t, g.parity, g.block
    if kind == "clean":
        return _codeword(g, rng)
    if kind == "zero":
        return _codeword(g, rng, zero=True)
    if kind == "random":
        return rng.integers(0, 256, B, dtype=np.uint8)
    if kind == "fail":
        while True:
            blk = rng.integers(0, 256, B, dtype=np.uint8)
            if _oracle_fails(g, blk):
                return blk
    if kind == "short":
        return _shortened(g, rng, int(rng.integers(1, t + 1)), 0)
    if kind == "shortj":
        k = int(rng.integers(1, t))
        return _shortened(g, rng, k, int(rng.integers(1, t - k + 1)))
    blk = _codeword(g, rng)
    pos = {"e1": lambda: rng.choice(B, 1, replace=False),
           "t": lambda: rng.choice(B, t, replace=False),
           "tpar": lambda: g.msg + rng.choice(P, t, replace=False),
           "t1": lambda: rng.choice(B, t + 1, replace=False),
           "many": lambda: rng.choice(B, int(rng.integers(t + 1, P + 7)), replace=False),
           "first": lambda: [0],
           "last": lambda: [B - 1]}[kind]()
    return _hit(blk, pos, rng)


@functools.lru_cache(maxsize=None)
def geo(mode_val):
    return Geo(mode_val)


def cc_pool(mode_val):
    """fountain frames for colour correction 2: every chunk starts with a FountainMetadata header (consecutive block ids)"""
    g = geo(mode_val)
    rng = np.random.default_rng(3000 + mode_val)
    P = 5
    payload = rng.integers(0, 256, (P, g.nblocks * g.msg), dtype=np.uint8)
    hdr = np.zeros(6, np.uint8)
    for f in range(P):
        for q in range(g.cpf):
            ORA.lib.cbo_md_pack(3, 40000, 1 + f * g.cpf + q, _ptr(hdr))
            payload[f, q * g.cs:q * g.cs + 6] = hdr
    raw = np.zeros((P, g.cap), np.uint8)
    enc = np.zeros(255, np.uint8)
    for f in range(P):
        for b in range(g.nblocks):
            ORA.lib.cbo_rs_encode(g.rs, _ptr(payload[f, b * g.msg:(b + 1) * g.msg].copy()), g.msg, _ptr(enc))
            raw[f, b * g.block:(b + 1) * g.block] = enc[:g.block]
    # frame 1: the first chunk's header bytes are wrong in the received block; only RS correction brings the header back
    _hit(raw[1, :g.block], np.concatenate([np.arange(6), 6 + rng.choice(g.block - 6, g.t - 6, replace=False)]), rng)
    # frame 2: every symbol-stream block fails, so the frame has no header and keeps the previous frame's matrix
    for b in range(g.nbs):
        raw[2, b * g.block:(b + 1) * g.block] = make_block(g, "fail", rng)
    # frame 3: the first symbol chunk fails, the header comes from the second
    for b in range(g.per_chunk):
        raw[3, b * g.block:(b + 1) * g.block] = make_block(g, "fail", rng)
    frames = np.stack([ORA.render_frame(g.m, raw_to_cells(g, r)) for r in raw])
    for f, gains in ((0, (0.8, 0.6, 1.0)), (1, (0.7, 1.0, 0.85)), (2, (1.0, 0.75, 0.7)), (3, (0.85, 0.9, 0.6))):
        frames[f] = np.clip(np.rint(frames[f].astype(np.float32) * np.asarray(gains, np.float32)), 0, 255).astype(np.uint8)
    return g, payload, raw, frames
