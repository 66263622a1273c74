"""Lane-level model of K1's sharpen schedule (k1_decode.cu, template SH) against the oracle's preprocessing.

The kernel cannot run here (no GPU), so the packed 2x16-bit arithmetic, the row lags of the two-barrier stage schedule and
the halo exchange are restated with numpy "registers" (one uint32 per thread) operation for operation, and the raster rows
the symbol stage would read are compared with cbo_preprocess(needs_sharpen=1) -- which is pinned to cv2's
filter2D + adaptiveThreshold(7) (reference: src/lib/cimb_translator/CimbReader.cpp:17-46).  The CUDA code is a transcription
of `stage()` below; variable names are the kernel's.
"""
import numpy as np
import pytest

import oracle_lib as ol
from cpu_support import NT, U, prmt, vmaxu2, vminu2


def umulhi(a, b):
    return ((a.astype(np.uint64) * np.uint64(b)) >> np.uint64(32)).astype(U)


class K1SharpenModel:
    """One CTA walking one whole frame (bands == 1)."""

    def __init__(self, rgb, cell_offset, cells_y):
        self.rgb = rgb
        self.H, self.W = rgb.shape[:2]
        self.cell_offset, self.cells_y = cell_offset, cells_y
        self.nthr_px = self.W // 8
        t = np.arange(NT)
        self.tl = np.where(t == 0, 0, t - 1)
        self.tr = np.where(t + 1 < self.nthr_px, t + 1, t)
        self.raster = np.zeros((2, 10, NT), np.uint8)        # byte t of a raster row = pixels 8t..8t+7, bit i = pixel 8t+i
        z = lambda *s: np.zeros(s + (NT,), U)
        self.Pprev = z(2, 4); self.Qprev = z(3, 4); self.hprev = z(7, 4)
        self.nV = np.full((4, NT), 0x7FE77FE7, U)            # per half: 0x8000 - 25
        self.prevE = z()                                      # halo word of the previous stage's last row

    def gray_rows(self, a0):
        """phase A: P[r][j] = g[j] | g[j+4] << 16 and the halo word E_r = (g0, g1, g6, g7) of the nine staged rows."""
        P = np.zeros((9, 4, NT), U); E = np.zeros((9, NT), U)
        for r in range(9):
            row = self.rgb[a0 + r].astype(np.uint32)                                      # [W][3]
            g = (19596 * row[:, 0] + 38470 * row[:, 1] + 7470 * row[:, 2] + 32768) >> 16   # == cvtColor(RGB2GRAY)
            gt = np.zeros((NT, 8), np.uint32)
            gt[: self.nthr_px] = g.reshape(self.nthr_px, 8)
            for j in range(4):
                P[r, j] = gt[:, j] | (gt[:, j + 4] << 16)
            E[r] = gt[:, 0] | (gt[:, 1] << 8) | (gt[:, 6] << 16) | (gt[:, 7] << 24)
        return P, E

    def stage(self, it, k):
        buf = it & 1
        a0 = self.cell_offset + 9 * k + 4                    # first raw row of the stage (the plain kernel: + 2)
        P, E = self.gray_rows(a0)
        halo = E.copy()                                       # s.halo[r][t] = E[r]
        # ---------------- barrier 1 (raw rows dead, next TMA issued)
        # ---- sharpen: S row i (absolute row a0 - 1 + i), i = 0..8
        Q = np.zeros((9, 4, NT), U)
        FL = np.zeros((9, NT), U); FH = np.zeros((9, NT), U)
        for i in range(9):
            Pc = self.Pprev[1] if i == 0 else P[i - 1]
            Pu = self.Pprev[0] if i == 0 else (self.Pprev[1] if i == 1 else P[i - 2])
            Pd = P[i]
            Ec = self.prevE if i == 0 else halo[i - 1]
            lE, rE = Ec[self.tl], Ec[self.tr]
            for j in range(4):
                Pl = prmt(lE, Pc[3], 0x5453) if j == 0 else Pc[j - 1]        # (gL7, g3)
                Pr = prmt(Pc[0], rE, 0x3432) if j == 3 else Pc[j + 1]        # (g4, gR0)
                nbr = (Pu[j] + Pd[j] + Pl + Pr).astype(U)
                T = (U(9) * Pc[j] + (U(0x08000800) - U(2) * nbr)).astype(U)   # twice + 2048 per half
                tc = (vminu2(vmaxu2(T, np.full(NT, 0x08000800, U)), np.full(NT, 0x09FE09FE, U)) - U(0x08000800)).astype(U)
                x = (tc >> U(1)) & U(0x00010001)
                Q[i, j] = ((tc + x) >> U(1)) & U(0x00FF00FF)
            FL[i] = prmt(prmt(Q[i, 0], Q[i, 1], 0x0040), Q[i, 2], 0x0410)     # bytes (s0, s1, s2, s0)
            FH[i] = prmt(prmt(Q[i, 1], Q[i, 2], 0x0062), Q[i, 3], 0x0610)     # bytes (s5, s6, s7, s5)
        # ---------------- barrier 2
        rows = []
        hs = np.zeros((9, 4, NT), U)
        for i in range(9):
            lF, rF = FH[i][self.tl], FL[i][self.tr]
            Qm3 = prmt(lF, Q[i, 1], 0x5450); Qm2 = prmt(lF, Q[i, 2], 0x5451); Qm1 = prmt(lF, Q[i, 3], 0x5452)
            Q4 = prmt(Q[i, 0], rF, 0x3432); Q5 = prmt(Q[i, 1], rF, 0x3532); Q6 = prmt(Q[i, 2], rF, 0x3632)
            h = np.zeros((4, NT), U)
            h[0] = Qm3 + Qm2 + Qm1 + Q[i, 0] + Q[i, 1] + Q[i, 2] + Q[i, 3]
            h[1] = h[0] - Qm3 + Q4
            h[2] = h[1] - Qm2 + Q5
            h[3] = h[2] - Qm1 + Q6
            tj = np.zeros((4, NT), U)
            for j in range(4):
                hold = self.hprev[i][j] if i < 7 else hs[i - 7][j]
                self.nV[j] = (self.nV[j] + hold - h[j]).astype(U)
                Qc = self.Qprev[i][j] if i < 3 else Q[i - 3][j]
                tj[j] = (U(49) * Qc + self.nV[j]).astype(U)
            hs[i] = h
            dx = prmt(tj[0], tj[1], 0x7531) & U(0x80808080)
            dy = prmt(tj[2], tj[3], 0x7531) & U(0x80808080)
            byte = (umulhi(dx, 0x02200440) + umulhi(dy, 0x08801100)) & U(0xFF)
            rows.append(byte.astype(np.uint8))
        self.raster[buf][0] = self.raster[buf ^ 1][9]
        for i in range(9):
            self.raster[buf][i + 1] = rows[i]
        for i in range(7):
            self.hprev[i] = hs[2 + i]
        for i in range(3):
            self.Qprev[i] = Q[6 + i]
        self.Pprev[0] = P[7]; self.Pprev[1] = P[8]
        self.prevE = halo[8]
        return self.raster[buf]


def _run(rgb, cell_offset, cells_y, want):
    m = K1SharpenModel(rgb, cell_offset, cells_y)
    H, W = rgb.shape[:2]
    checked = 0
    for it, k in enumerate(range(-1, cells_y)):
        rast = m.stage(it, k)
        if k < 0:
            continue
        y = cell_offset + 9 * k
        # window rows y-1 .. y+8 of cell row k; columns the cell windows of this geometry can touch
        got = np.unpackbits(rast[:, : W // 8], axis=1, bitorder="little")
        x_lo, x_hi = cell_offset - 1, W - cell_offset + 1
        assert np.array_equal(got[:, x_lo:x_hi], want[y - 1 : y + 9, x_lo:x_hi]), f"cell row {k}"
        checked += 10
    return checked


@pytest.mark.parametrize("sample", ["b/ex2434.jpg", "b/tr_0.png"])
def test_k1_sharpen_schedule_matches_oracle(sample):
    o = ol.Oracle()
    rgb = ol.load_sample(sample)
    H, W = rgb.shape[:2]
    want = np.unpackbits(o.preprocess(rgb, sharpen=True)).reshape(H, W)
    assert _run(rgb, 8, 112, want) == 1120


def test_k1_sharpen_schedule_random_noise_small_geometry():
    # mode Bu's geometry (736 x 637, offset 9, 69 cell rows) on noise: every rounding / clamping case of the sharpen filter occurs
    o = ol.Oracle()
    rng = np.random.default_rng(5)
    rgb = rng.integers(0, 256, (637, 736, 3), dtype=np.uint8)
    rgb[:, ::3] //= 4                                          # dark columns: negative and saturating filter outputs
    want = np.unpackbits(o.preprocess(rgb, sharpen=True)).reshape(637, 736)
    assert _run(rgb, 9, 69, want) == 690


def test_thread_symbol_search_model_matches_oracle():
    """k1_decode.cu thread_symbol_search (the per-thread P5/P6 search of the sharpen variant): key = dist<<8 | order<<4 | tile
    minimised over drift ids in the order 4,5,7,3,1(,8,0,2,6) and tiles 0..15 == fuzzy_ahash + get_best_symbol of the oracle."""
    import ctypes as C
    o = ol.Oracle()
    o.lib.cbo_tile_hashes.restype = C.POINTER(C.c_uint64)
    T = o.lib.cbo_tile_hashes()
    tiles_L = [int(f"{int(T[i]):064b}"[::-1], 2) for i in range(16)]      # bit (8r+c) = pixel (r, c)
    order = [4, 5, 7, 3, 1, 8, 0, 2, 6]
    rng = np.random.default_rng(11)
    hashes = (C.c_uint64 * 9)()
    doff, ddist = C.c_uint(0), C.c_uint(0)
    for trial in range(1500):
        rows = [int(rng.integers(0, 1024)) for _ in range(10)]             # MSB-first: bit 9 = window column 0
        if trial % 2 == 0:                                                 # a tile with a few flipped bits at a random drift
            t = int(T[int(rng.integers(0, 16))]) ^ (1 << int(rng.integers(0, 64))) ^ (1 << int(rng.integers(0, 64)))
            dx, dy = int(rng.integers(0, 3)), int(rng.integers(0, 3))
            for r in range(8):
                byte = (t >> (8 * (7 - r))) & 0xFF
                rows[dy + r] = (rows[dy + r] & ~(0xFF << (2 - dx))) | (byte << (2 - dx))
        all_ = trial % 3 == 0
        win = [int(f"{v:010b}"[::-1], 2) for v in rows]                    # kernel layout: bit i = window column i
        best = 0xFFFFFFFF
        for q in range(9 if all_ else 5):
            r0, c0 = (0x200201211 >> (4 * q)) & 3, (0x020210121 >> (4 * q)) & 3
            assert (r0, c0) == (order[q] // 3, order[q] % 3)
            L = 0
            for r in range(8):
                L |= ((win[r0 + r] >> c0) & 0xFF) << (8 * r)
            for tile in range(16):
                best = min(best, (bin(L ^ tiles_L[tile]).count("1") << 8) | (q << 4) | tile)
        buf = np.zeros(24, np.uint8)
        for r in range(10):
            v = rows[r] << 6
            buf[2 * r], buf[2 * r + 1] = v >> 8, v & 0xFF
        o.lib.cbo_fuzzy_ahash(ol._ptr(buf), 16, 0, 0, int(all_), hashes)
        s = o.lib.cbo_best_symbol(hashes, int(all_), 16, 0xFE if all_ else 4, C.byref(doff), C.byref(ddist))
        assert (best & 15, order[(best >> 4) & 15], best >> 8) == (s, doff.value, ddist.value), trial
