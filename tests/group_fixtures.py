"""Fixtures and the CPU expectation of the grouped camera call (cb200_scan_extract_decode_chunks_grouped_dev).

The rule of include/cb200.h, restated in numpy: pictures i and j match when both have extract status 1 or 2 and at least half of the
cells have equal symbol bits; in batch order each such picture joins the earliest earlier leader it matches whose group has fewer
than 16 pictures, else it leads; a group is a leader with at least one other picture, numbered in its leaders' order.

Distinct frames: combine_fixtures.capture draws every capture of a mode from one base frame, so the frames here are the oracle's
renderings of a payload seeded per frame, with an encoder frame's anchors pasted into its corners (the path combine_fixtures.base_frame
takes for modes 67, 66 and 8), and their captures the same noise tiles and perspective warp as combine_fixtures.capture."""
import ctypes as C

import cv2
import numpy as np

from combine_fixtures import MARGIN, NOISE, ORA
from oracle_lib import _ptr, load_sample

MAX_GROUP = 16


def agree_matrix(values, symbol_bits):
    """agree(i, j) for every pair: values is a list of per-picture cell bytes (None for a picture without cells)"""
    n = len(values)
    out = np.zeros((n, n), np.int64)
    mask = (1 << symbol_bits) - 1
    for i in range(n):
        for j in range(n):
            if values[i] is not None and values[j] is not None:
                out[i, j] = int(((values[i] & mask) == (values[j] & mask)).sum())
    return out


def match_matrix(values, statuses, symbol_bits, cells):
    """match(i, j) for every pair"""
    elig = np.array([s in (1, 2) for s in statuses], bool)
    return elig[:, None] & elig[None, :] & (2 * agree_matrix(values, symbol_bits) >= cells)


def assign(match, eligible):
    """the assignment of the rule over a boolean match matrix (only j < i is read): (group_of, count)"""
    n = len(eligible)
    lead = [-1] * n
    size = {}
    leaders = []
    for i in range(n):
        if not eligible[i]:
            continue
        for j in leaders:
            if size[j] < MAX_GROUP and match[i][j]:
                lead[i] = j
                size[j] += 1
                break
        else:
            lead[i] = i
            size[i] = 1
            leaders.append(i)
    number = {}
    for j in leaders:
        if size[j] >= 2:
            number[j] = len(number)
    return [number.get(lead[i], -1) if lead[i] >= 0 else -1 for i in range(n)], len(number)


def rule_groups(mode_val, per_picture):
    """(group_of, count) of pictures given as (status, values, ...) tuples (combine_fixtures.picture_cells / fitted_cells)"""
    m = ORA.mode(mode_val)
    statuses = [p[0] for p in per_picture]
    match = match_matrix([p[1] for p in per_picture], statuses, m.symbol_bits, m.total_cells)
    return assign(match, [s in (1, 2) for s in statuses])


def seeded_frame(mode_val, seed):
    """the oracle's rendering of a payload seeded by `seed`, with the anchor squares of an encoder frame in its corners"""
    m = ORA.mode(mode_val)
    nbytes = (ORA.capacity(m) // m.ecc_block_size) * (m.ecc_block_size - m.ecc_bytes)
    payload = np.random.default_rng([mode_val, seed]).integers(0, 256, nbytes, dtype=np.uint8)
    f = ORA.render_frame(m, ORA.payload_to_cells(m, payload)).copy()
    tr, c = load_sample("b/tr_0.png"), 62
    H, W = f.shape[:2]
    for ys, ts in ((slice(0, c), slice(0, c)), (slice(H - c, H), slice(1024 - c, 1024))):
        for xs, us in ((slice(0, c), slice(0, c)), (slice(W - c, W), slice(1024 - c, 1024))):
            f[ys, xs] = tr[ts, us]
    return f


def capture_of(mode_val, frame, seed, rate=NOISE):
    """one synthetic capture of `frame`: noise tiles on `rate` of the cells away from the anchors, a perspective warp of up to 14 px
    per corner onto a canvas 70 px larger on each side"""
    m = ORA.mode(mode_val)
    rng = np.random.default_rng(seed)
    frame = frame.copy()
    H, W = frame.shape[:2]
    xs, ys = np.zeros(m.total_cells, np.int32), np.zeros(m.total_cells, np.int32)
    ORA.lib.cbo_cell_positions(C.byref(m), 0, _ptr(xs, C.c_int), _ptr(ys, C.c_int))
    far = np.ones(m.total_cells, bool)
    for cx, cy in ((0, 0), (W, 0), (0, H), (W, H)):
        far &= np.hypot(xs + 4 - cx, ys + 4 - cy) > 150
    for i in rng.choice(np.flatnonzero(far), int(round(rate * m.total_cells)), replace=False):
        frame[ys[i]:ys[i] + 8, xs[i]:xs[i] + 8] = rng.integers(0, 256, (8, 8, 3), dtype=np.uint8)
    src = np.array([[0, 0], [W, 0], [0, H], [W, H]], np.float32)
    dst = src + MARGIN + rng.uniform(-14, 14, (4, 2)).astype(np.float32)
    return cv2.warpPerspective(frame, cv2.getPerspectiveTransform(src, dst), (W + 2 * MARGIN, H + 2 * MARGIN), flags=cv2.INTER_LINEAR,
                               borderMode=cv2.BORDER_CONSTANT, borderValue=(0, 0, 0))


def frame_captures(mode_val, counts, seed):
    """captures of len(counts) distinct seeded frames, counts[f] of frame f: (pictures, frame of each picture), frames in order"""
    pics, frame_of = [], []
    for f, k in enumerate(counts):
        frame = seeded_frame(mode_val, 1000 * seed + f)
        for s in range(k):
            pics.append(capture_of(mode_val, frame, [seed, f, s]))
            frame_of.append(f)
    return pics, frame_of
