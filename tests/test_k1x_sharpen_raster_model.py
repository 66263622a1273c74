"""Lane-level model of K1x's fast sharpen raster (k1x_flood.cu k_flood_raster_fast<true>): the full-frame needs_sharpen
preprocessing with OpenCV's borders -- filter2D BORDER_REFLECT_101, adaptiveThreshold(7) BORDER_REPLICATE
(CimbReader.cpp:17-46) -- as a row-streaming schedule of one CTA per 64-row band, restated with numpy registers operation for
operation and compared with the oracle over the WHOLE frame (every border case).  The CUDA code transcribes `band()`."""
import numpy as np
import pytest

import oracle_lib as ol
from cpu_support import NT, U, prmt, vmaxu2, vminu2

BAND = 64


def gray_row(rgb, y, nthr):
    row = rgb[y].astype(np.uint32)
    g = (19596 * row[:, 0] + 38470 * row[:, 1] + 7470 * row[:, 2] + 32768) >> 16
    gt = np.zeros((NT, 8), np.uint32)
    gt[:nthr] = g.reshape(nthr, 8)
    gt[nthr:] = gt[nthr - 1]                       # inactive threads shadow the last one
    P = np.stack([gt[:, j] | (gt[:, j + 4] << 16) for j in range(4)]).astype(U)
    E = (gt[:, 0] | (gt[:, 1] << 8) | (gt[:, 6] << 16) | (gt[:, 7] << 24)).astype(U)
    return P, E


def band(rgb, y0, y1):
    """threshold bytes (bit i of byte t = pixel 8t+i) of rows y0..y1-1"""
    H, W = rgb.shape[:2]
    nthr = W // 8
    t = np.arange(NT)
    first, last = (t == 0), (t >= nthr - 1)
    tl, tr = np.maximum(t - 1, 0), np.minimum(t + 1, NT - 1)
    clamp = lambda v: min(max(v, 0), H - 1)
    refl = lambda v: -v if v < 0 else (2 * H - 2 - v if v >= H else v)
    out = {}
    G = [None, None, None]; HL = [None, None, None]     # gray rows u, c, d (packed) and the (lE, rE) of each
    rows_have = (None, None, None)
    Qr = [np.zeros((4, NT), U) for _ in range(4)]       # the last four sharpened rows (ring by sr & 3)
    hr = [np.zeros((4, NT), U) for _ in range(7)]       # the last seven horizontal sums (ring by (sr - first) % 7)
    nV = np.full((4, NT), 0x7FE77FE7, U)

    def load(y):
        P, E = gray_row(rgb, y, nthr)
        # exchange: ex[t] = E; barrier; replicate is NOT what the sharpen wants at the frame edge: REFLECT_101 -> g(-1) = g(1), g(W) = g(W-2)
        lE = np.where(first, prmt(E, E, 0x1111), E[tl])        # byte 3 used (left g7): own g1
        rE = np.where(last, prmt(E, E, 0x2222), E[tr])         # byte 0 used (right g0): own g6
        return P, (lE, rE)

    sr0 = y0 - 3
    for sr in range(y0 - 3, y1 + 3):
        s = clamp(sr)
        want = (refl(s - 1), s, refl(s + 1))
        if rows_have[1] == want[0] and rows_have[2] == want[1]:          # the common case: one new row
            G = [G[1], G[2], None]; HL = [HL[1], HL[2], None]
            G[2], HL[2] = load(want[2])
        elif rows_have == want:
            pass                                                          # a clamped S row repeats (frame top / bottom)
        else:
            for i in range(3):
                G[i], HL[i] = load(want[i])
        rows_have = want
        Pu, Pc, Pd = G
        lE, rE = HL[1]
        Q = np.zeros((4, NT), U)
        for j in range(4):
            Pl = prmt(lE, Pc[3], 0x5453) if j == 0 else Pc[j - 1]
            Pr = prmt(Pc[0], rE, 0x3432) if j == 3 else Pc[j + 1]
            nbr = (Pu[j] + Pd[j] + Pl + Pr).astype(U)
            T = (U(9) * Pc[j] + (U(0x08000800) - U(2) * nbr)).astype(U)
            tc = (vminu2(vmaxu2(T, np.full(NT, 0x08000800, U)), np.full(NT, 0x09FE09FE, U)) - U(0x08000800)).astype(U)
            Q[j] = ((tc + ((tc >> U(1)) & U(0x00010001))) >> U(1)) & U(0x00FF00FF)
        FL = prmt(prmt(Q[0], Q[1], 0x0040), Q[2], 0x0410)                # (s0, s1, s2, .)
        FH = prmt(prmt(Q[1], Q[2], 0x0062), Q[3], 0x0610)                # (s5, s6, s7, .)
        # exchange 2; BORDER_REPLICATE for the box sum: S(-k) = s0, S(W-1+k) = s7
        lF = np.where(first, prmt(FL, FL, 0x0000), FH[tl])
        rF = np.where(last, prmt(FH, FH, 0x2222), FL[tr])
        Qm3 = prmt(lF, Q[1], 0x5450); Qm2 = prmt(lF, Q[2], 0x5451); Qm1 = prmt(lF, Q[3], 0x5452)
        Q4 = prmt(Q[0], rF, 0x3432); Q5 = prmt(Q[1], rF, 0x3532); Q6 = prmt(Q[2], rF, 0x3632)
        h = np.zeros((4, NT), U)
        h[0] = Qm3 + Qm2 + Qm1 + Q[0] + Q[1] + Q[2] + Q[3]
        h[1] = h[0] - Qm3 + Q4
        h[2] = h[1] - Qm2 + Q5
        h[3] = h[2] - Qm1 + Q6
        k = (sr - sr0) % 7
        tj = np.zeros((4, NT), U)
        Qr[sr & 3] = Q
        for j in range(4):
            nV[j] = (nV[j] + hr[k][j] - h[j]).astype(U)
            tj[j] = (U(49) * Qr[(sr - 3) & 3][j] + nV[j]).astype(U)       # centre row sr - 3
        hr[k] = h
        y = sr - 3
        if y >= y0:
            byte = ((tj[0] >> U(15)) & U(0x00010001)) | ((tj[1] >> U(14)) & U(0x00020002)) | \
                   ((tj[2] >> U(13)) & U(0x00040004)) | ((tj[3] >> U(12)) & U(0x00080008))
            byte = (byte | (byte >> U(12))) & U(0xFF)
            out[y] = byte.astype(np.uint8)[:nthr]
    return out


def _whole_frame(rgb):
    H, W = rgb.shape[:2]
    got = np.zeros((H, W), np.uint8)
    for y0 in range(0, H, BAND):
        rows = band(rgb, y0, min(y0 + BAND, H))
        for y, b in rows.items():
            got[y] = np.unpackbits(b, bitorder="little")
    return got


@pytest.mark.parametrize("sample", ["b/ex2434.jpg", "b/tr_0.png"])
def test_fast_sharpen_raster_schedule_matches_oracle(sample):
    o = ol.Oracle()
    rgb = ol.load_sample(sample)
    H, W = rgb.shape[:2]
    want = np.unpackbits(o.preprocess(rgb, sharpen=True)).reshape(H, W)
    assert np.array_equal(_whole_frame(rgb), want)


def test_fast_sharpen_raster_schedule_noise_other_geometry():
    o = ol.Oracle()
    rng = np.random.default_rng(6)
    rgb = rng.integers(0, 256, (637, 736, 3), dtype=np.uint8)           # mode Bu: 92 active threads, last band of 61 rows
    rgb[:, ::3] //= 4
    want = np.unpackbits(o.preprocess(rgb, sharpen=True)).reshape(637, 736)
    assert np.array_equal(_whole_frame(rgb), want)
