"""Fixtures and the CPU expectation of the combined camera call (cb200_scan_extract_decode_chunks_combined_dev).

Synthetic captures: an encoder frame of the golden set (mode 68: b/tr_0.png, mode 4: 6bit/4color_ecc30_fountain_0.png; in the other
modes the oracle's rendering of a seeded payload with an encoder frame's anchors) with about
8 % of its cells, chosen per capture and away from the anchors, overwritten by 8 x 8 noise tiles, then put through its own mild
perspective warp onto a black canvas.  Each capture alone fails some Reed-Solomon blocks; two or three of them decode every block.

The expectation restates the rule of include/cb200.h on the oracle's cells: each picture as the reference CLI decodes it (scan,
Corners, warpPerspective, the oracle's walk with its per-cell symbol, colour and distance; under colour correction 2 with the
matrix its CC 2 route fits, fitted_cells), the vote per cell, and the voted cells as a clean frame (the oracle's renderer), which
the oracle decodes back to exactly those cells (asserted each time): its de-interleave, Reed-Solomon and aligned_stream chunk rule
give the group's record and mask."""
import ctypes as C

import cv2
import numpy as np

from oracle_lib import Oracle, _ptr, load_sample
from scan_oracle_lib import ScanOracle

ORA = Oracle()
SO = ScanOracle()

FRAME = {68: "b/tr_0.png", 4: "6bit/4color_ecc30_fountain_0.png"}
NOISE = 0.08
MARGIN = 70


def base_frame(mode_val):
    """the encoder frame of the golden set (modes 68 and 4), else the oracle's rendering of a seeded random payload"""
    if mode_val in FRAME:
        return load_sample(FRAME[mode_val]).copy()
    m = ORA.mode(mode_val)
    nbytes = (ORA.capacity(m) // m.ecc_block_size) * (m.ecc_block_size - m.ecc_bytes)
    payload = np.random.default_rng(mode_val).integers(0, 256, nbytes, dtype=np.uint8)
    f = ORA.render_frame(m, ORA.payload_to_cells(m, payload)).copy()
    tr, c = load_sample(FRAME[68]), 62                  # the anchor squares of an encoder frame in its corners, outside every cell
    H, W = f.shape[:2]
    for ys, ts in ((slice(0, c), slice(0, c)), (slice(H - c, H), slice(1024 - c, 1024))):
        for xs, us in ((slice(0, c), slice(0, c)), (slice(W - c, W), slice(1024 - c, 1024))):
            f[ys, xs] = tr[ts, us]
    return f


def capture(mode_val, seed, rate=NOISE):
    """one synthetic capture of the mode's encoder frame: noise tiles on `rate` of the cells, a perspective warp of up to 14 px per
    corner onto a canvas 70 px larger on each side"""
    m = ORA.mode(mode_val)
    rng = np.random.default_rng(seed)
    frame = base_frame(mode_val)
    H, W = frame.shape[:2]
    xs, ys = np.zeros(m.total_cells, np.int32), np.zeros(m.total_cells, np.int32)
    ORA.lib.cbo_cell_positions(C.byref(m), 0, _ptr(xs, C.c_int), _ptr(ys, C.c_int))
    far = np.ones(m.total_cells, bool)                   # away from the anchors: no cell within 150 px of a corner of the frame
    for cx, cy in ((0, 0), (W, 0), (0, H), (W, H)):
        far &= np.hypot(xs + 4 - cx, ys + 4 - cy) > 150
    pool = np.flatnonzero(far)
    for i in rng.choice(pool, int(round(rate * m.total_cells)), replace=False):
        frame[ys[i]:ys[i] + 8, xs[i]:xs[i] + 8] = rng.integers(0, 256, (8, 8, 3), dtype=np.uint8)
    src = np.array([[0, 0], [W, 0], [0, H], [W, H]], np.float32)
    dst = src + MARGIN + rng.uniform(-14, 14, (4, 2)).astype(np.float32)
    return cv2.warpPerspective(frame, cv2.getPerspectiveTransform(src, dst), (W + 2 * MARGIN, H + 2 * MARGIN), flags=cv2.INTER_LINEAR,
                               borderMode=cv2.BORDER_CONSTANT, borderValue=(0, 0, 0))


def extract(mode_val, rgb):
    """the reference CLI's extraction: (status, deskewed frame or None)"""
    m = ORA.mode(mode_val)
    an, W, H = 30, m.image_size_x, m.image_size_y
    dst = np.array([[an, an], [W - an, an], [an, H - an], [W - an, H - an]], np.float32)
    anchors, _ = SO.scan(rgb)
    if anchors is None or len(anchors) < 4:
        return 0, None
    xy = SO.corners(anchors)
    status = 1 if SO.is_granular_scale(xy, W, H) else 2
    frame = cv2.warpPerspective(rgb, cv2.getPerspectiveTransform(np.array(xy, np.float32).reshape(4, 2), dst), (W, H), flags=cv2.INTER_LINEAR)
    return status, frame


def picture_cells(mode_val, rgb, sharpen="no", cc=0):
    """(status, value bits per cell or None, distance per cell or None) of one picture, colour correction 0 or 1 (the oracle restates
    no other per cell); sharpen 'no' / 'all' / 'needed'"""
    status, frame = extract(mode_val, rgb)
    if frame is None:
        return status, None, None
    m = ORA.mode(mode_val)
    sh = {"no": False, "all": True, "needed": status == 2}[sharpen]
    ORA.set_ccm(None)
    _, cells = ORA.decode_raw(m, frame, sharpen=sh, want_cells=True, color_correction=cc)
    ORA.set_ccm(None)
    values = (cells["symbol"].astype(np.int32) | (cells["color"].astype(np.int32) << m.symbol_bits)).astype(np.uint8)
    return status, values, cells["distance"].astype(np.uint8)


def fitted_cells(mode_val, pictures, sharpen="no"):
    """per picture (status, value bits or None, distances or None, the oracle's CC 2 record (good bytes, chunks, mask) or None) under
    colour correction 2, as the reference CLI decodes a batch: one decoder in batch order, FAILURE pictures skipped, each fit (or the
    matrix carried from an earlier picture when a picture has none) kept for the next picture.  cbo_decode_fountain_cc's CC 2 route
    installs the matrix the colour pass uses (its symbol pass, the symbol blocks' RS, the header, CimbReader::init_ccm); the cells
    are then cbo_decode_raw's with that matrix installed: its symbols and distances do not depend on the matrix, and its colour pass
    is the one the CC 2 route runs after the fit."""
    m = ORA.mode(mode_val)
    out = []
    ORA.set_ccm(None)
    try:
        for rgb in pictures:
            status, frame = extract(mode_val, rgb)
            if frame is None:
                out.append((status, None, None, None))
                continue
            sh = {"no": False, "all": True, "needed": status == 2}[sharpen]
            good, chunks, mask = ORA.decode_fountain(m, frame, sharpen=sh, color_correction=2)
            _, cells = ORA.decode_raw(m, frame, sharpen=sh, want_cells=True, color_correction=0)
            values = (cells["symbol"].astype(np.int32) | (cells["color"].astype(np.int32) << m.symbol_bits)).astype(np.uint8)
            out.append((status, values, cells["distance"].astype(np.uint8), (good, chunks.copy(), int(mask))))
    finally:
        ORA.set_ccm(None)
    return out


def vote(values, dists):
    """the rule per cell over k pictures (k x cells arrays, batch order): most pictures, then smallest distance, then earliest"""
    k, cells = values.shape
    dists = dists.astype(np.int32)
    best = values[0].copy()
    best_count = np.zeros(cells, np.int32)
    best_dist = np.full(cells, 256, np.int32)
    for i in range(k):
        seen = np.zeros(cells, bool)
        for j in range(i):
            seen |= values[j] == values[i]
        same = values == values[i]
        count = same.sum(axis=0)
        dist = np.where(same, dists, 256).min(axis=0)
        take = ~seen & ((count > best_count) | ((count == best_count) & (dist < best_dist)))
        best = np.where(take, values[i], best)
        best_count = np.where(take, count, best_count)
        best_dist = np.where(take, dist, best_dist)
    return best


def cells_record(mode_val, values):
    """the record, chunk mask and per-block ok flags of a frame whose final cells are `values` (the oracle's decode of the clean frame
    its renderer draws from them)"""
    m = ORA.mode(mode_val)
    frame = ORA.render_frame(m, np.ascontiguousarray(values, np.uint8))
    ORA.set_ccm(None)
    _, cells = ORA.decode_raw(m, frame, want_cells=True)
    back = (cells["symbol"].astype(np.int32) | (cells["color"].astype(np.int32) << m.symbol_bits)).astype(np.uint8)
    assert np.array_equal(back, values), "the rendered frame does not decode back to its cells"
    _, ok = ORA.decode(m, frame)
    good, chunks, mask = ORA.decode_fountain(m, frame)
    return good, chunks.copy(), int(mask), ok


def group_expectation(mode_val, per_picture, members):
    """(record, mask, used) of one group: per_picture[i] = picture_cells(...) of picture i, members its pictures in batch order"""
    part = [i for i in members if per_picture[i][0] in (1, 2)]
    if not part:
        return None, 0, 0
    v = vote(np.stack([per_picture[i][1] for i in part]), np.stack([per_picture[i][2] for i in part]))
    good, chunks, mask, _ = cells_record(mode_val, v)
    return (good, chunks), mask, len(part)


def clean_picture(mode_val, pad=40):
    """the mode's base frame as a camera picture that extracts to exactly that frame: on a black border, with its four anchor squares
    moved one pixel right and down (the extractor maps the anchors' integer centres, one pixel above and left of where the encoder
    draws them, to 30 and size - 30), so the deskew is a whole-pixel translation of the cells.  K1 decodes such a frame without flags"""
    f = base_frame(mode_val)
    H, W = f.shape[:2]
    p = cv2.copyMakeBorder(f, pad, pad, pad, pad, cv2.BORDER_CONSTANT, value=(0, 0, 0))
    c = 62
    for y0 in (0, H - c):
        for x0 in (0, W - c):
            sq = p[pad + y0:pad + y0 + c, pad + x0:pad + x0 + c].copy()
            p[pad + y0:pad + y0 + c, pad + x0:pad + x0 + c] = 0
            p[pad + y0 + 1:pad + y0 + c + 1, pad + x0 + 1:pad + x0 + c + 1] = sq
    return p
