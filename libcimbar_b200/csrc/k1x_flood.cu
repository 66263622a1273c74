// k1x_flood.cu -- K1x: the exact flood-walk decode for frames the drift-0 pass (K1) cannot prove exact, sm_90a.
//
// Restates the reference's serial semantics on the device (reference file:line relative to /root/reference/):
//   P1  preprocessSymbolGrid (+ sharpen)      src/lib/cimb_translator/CimbReader.cpp:17-46 (full frame, OpenCV borders)
//   P3  FloodDecodePositions                  src/lib/cimb_translator/FloodDecodePositions.cpp:17-134
//       std::priority_queue tie-breaking      libstdc++ bits/stl_heap.h (__push_heap / __adjust_heap), restated exactly:
//                                             equal priorities pop in the order that sift-up/sift-down produces
//   AdjacentCellFinder                        src/lib/cimb_translator/AdjacentCellFinder.cpp:54-105
//   P4  CimbReader::read, CellDrift           src/lib/cimb_translator/CimbReader.cpp:139-162, CellDrift.cpp:23-43
//   P5/P6 fuzzy_ahash + get_best_symbol       src/lib/image_hash/ahash_result.h:70-106, CimbDecoder.cpp:101-132
//   P8/P9 colour at the drift-adjusted cell   src/lib/cimb_translator/Cell.h:30-62, CimbDecoder.cpp:168-217
//
// Four kernels per batch; clean batches cost four empty launches:
//   k_flood_list    compacts the frames K1 flagged into a work list (one CTA, order-preserving)
//   k_flood_raster_fast  threshold raster of every listed frame: one CTA per 64-row band, 8 px per thread, K1's packed-16
//                   SIMD arithmetic (IDP.2A gray, separable 5x5 box sum, one IMAD per pixel pair) with OpenCV's replicate
//                   borders, rolling vertical sums in registers; output in 16x16-pixel TILES (32 B = one sector each) so that
//                   a 10x10 window of the walk touches at most four sectors.  k_flood_raster_fast_sharpen is the same for
//                   needs_sharpen (3x3 sharpen with reflected borders + block 7 with replicated ones, rows streamed through
//                   registers, two barriers per row).  A batch that mixes sharpened and plain frames launches both over the
//                   same work list; each skips the items whose frame is of the other kind (one byte per frame).
//   k_flood_walk    the serial 12 400-step walk, ONE WARP PER FRAME, up to 32 frames per SM in flight (the walk is a chain
//                   of dependent heap and window accesses, so throughput comes from walking many frames at once):
//                   binary heap in shared memory (+ global spill); the sift-down of a pop resolves FIVE heap levels per
//                   memory round trip (31 lanes load the child pairs of a 5-level subtree, one ballot, every lane checks
//                   its ancestors' bits); the drift/cooldown a cell inherits travels inside the 32-bit heap entry, so the
//                   only per-cell state is one priority byte in L2 and a bitmap in shared memory
//                   (batches of at most one wave of big-heap walks keep the WHOLE heap in shared memory: 8 191 entries,
//                   six walks per SM -- with few walks in flight nothing hides the L2 round trips of spilled levels)
//   k_flood_colour  colours at the recorded drift-adjusted positions, one thread per cell
#include "cb200_common.cuh"
#include "k1x_flood.cuh"
#include "ccm.cuh"

namespace cb200 {

constexpr int kFloodMaxEntries = 16384;  // listed frames whose raster/result are resident at once (one chunk, 181 KB each)

__constant__ float cx_adjust[256];
__constant__ unsigned long long cx_tiles_L[16];
__constant__ uint4 cx_tiles_slot[16];            // (L_lo, L_hi, symbol, 0) at the tile's perfect-hash slot ((L_lo * hash_mul) >> 28)

// ---------------------------------------------------------------------------------------------- work list
// order-preserving compaction of the frames that need the exact walk; also writes the per-frame flags.  present: NULL, or one byte
// per frame, 0 for a frame nobody reads (a detect receivers plan's slot that no mode of the geometry decodes): never listed
__global__ void __launch_bounds__(1024)
k_flood_list(const uint32_t* __restrict__ dirty, int n_frames, int no_fallback, int force_all, uint8_t* __restrict__ frame_flags,
             uint32_t* __restrict__ list, uint32_t* __restrict__ counters, int n_counters, const uint8_t* __restrict__ present)
{
    __shared__ uint32_t warp_off[32];
    __shared__ uint32_t base_s, total_s;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) base_s = 0;
    for (int i = 1 + tid; i < n_counters; i += 1024) counters[i] = 0;     // per-chunk work counters of k_flood_walk
    __syncthreads();
    for (int start = 0; start < n_frames; start += 1024) {
        const int f = start + tid;
        const bool need = f < n_frames && (force_all || (dirty[f] & kFrameDirtyK1)) && (!present || present[f]);
        const bool take = need && !no_fallback;
        if (f < n_frames) frame_flags[f] = need ? (no_fallback ? 0x2 : 0x1) : 0;   // CB200_FRAME_INEXACT / CB200_FRAME_FALLBACK
        const uint32_t b = __ballot_sync(0xffffffffu, take);
        const uint32_t prefix = __popc(b & ((1u << lane) - 1u));
        if (lane == 0) warp_off[warp] = __popc(b);
        __syncthreads();
        if (warp == 0) {
            uint32_t v = warp_off[lane], incl = v;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { uint32_t t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
            warp_off[lane] = incl - v;
            if (lane == 31) total_s = incl;
        }
        __syncthreads();
        if (take) list[base_s + warp_off[warp] + prefix] = (uint32_t)f;
        __syncthreads();
        if (tid == 0) base_s += total_s;
        __syncthreads();
    }
    if (tid == 0) counters[0] = base_s;
}

__device__ __forceinline__ int chunk_count(const uint32_t* counters, int base, int cap)
{
    int c = (int)counters[0] - base;
    return c < 0 ? 0 : (c > cap ? cap : c);
}

// ---------------------------------------------------------------------------------------------- preprocessing (P1)
__device__ __forceinline__ int reflect101(int p, int n) { if (p < 0) p = -p; if (p >= n) p = 2 * n - 2 - p; return p; }
__device__ __forceinline__ int clampi(int p, int lo, int hi) { return p < lo ? lo : (p > hi ? hi : p); }

// ---------------------------------------------------------------------------------------------- tiled raster
// 1 bit per pixel in tiles of 16 x 16 pixels: tile (ty, tx) is 16 consecutive uint16 (32 bytes, one DRAM/L2 sector), word r
// of a tile holds row 16 ty + r, bit b of it is pixel 16 tx + b.  A 16-row band of the frame is one contiguous run of 2 W bytes.
__host__ __device__ __forceinline__ size_t raster_words16(int W, int H) { return (size_t)(W >> 4) * (size_t)((H + 15) >> 4) * 16u + 64u; }
__device__ __forceinline__ uint32_t raster_tile_index(int tiles_x, int x, int y)
{
    return ((uint32_t)(y >> 4) * (uint32_t)tiles_x + (uint32_t)(x >> 4)) * 16u + (uint32_t)(y & 15);
}

// ---------------------------------------------------------------------------------------------- fast raster (no sharpen)
// One CTA of 128 threads per (listed frame, band of kFastBand rows).  Thread t owns pixels 8t .. 8t+7 of every row and
// streams down the band: per input row it converts 8 pixels to gray with K1's IDP.2A form, exchanges two halo pixels with
// its neighbours through shared memory (one barrier per row, double buffered; BORDER_REPLICATE at the frame edges by
// clamping), forms the horizontal 5-sums in packed 2x16-bit lanes, keeps the last five of them and the last three gray rows
// in registers, and emits one byte of threshold bits for the row two above.  16 rows of bytes are staged in shared memory
// and written out as whole 16x16 tiles (16 bytes per thread, coalesced).  Arithmetic is K1's, so the bits are OpenCV's:
//   gray = (9798 R + 19235 G + 3735 B + 2^14) >> 15,  bit = 25 gray > boxsum + 12  <=>  gray > round(boxsum / 25).
constexpr int kFastThreads = 128;
constexpr int kFastBand = 64;

__device__ __forceinline__ void gray8_packed(const uint2 q0, const uint2 q1, const uint2 q2, uint32_t P[4], uint32_t& E)
{
    const uint32_t cRG = 19596u | (38470u << 16), cB0 = 7470u, c0R = 19596u << 16, cGB = 38470u | (7470u << 16);
    uint32_t n0, n1, n2, n3, n4, n5, n6, n7;       // (19596 R + 38470 G + 7470 B + 2^15) : gray is byte 2
    n0 = __dp2a_lo(cRG, q0.x, 32768u); n0 = __dp2a_hi(cB0, q0.x, n0);
    n1 = __dp2a_hi(c0R, q0.x, 32768u); n1 = __dp2a_lo(cGB, q0.y, n1);
    n2 = __dp2a_hi(cRG, q0.y, 32768u); n2 = __dp2a_lo(cB0, q1.x, n2);
    n3 = __dp2a_lo(c0R, q1.x, 32768u); n3 = __dp2a_hi(cGB, q1.x, n3);
    n4 = __dp2a_lo(cRG, q1.y, 32768u); n4 = __dp2a_hi(cB0, q1.y, n4);
    n5 = __dp2a_hi(c0R, q1.y, 32768u); n5 = __dp2a_lo(cGB, q2.x, n5);
    n6 = __dp2a_hi(cRG, q2.x, 32768u); n6 = __dp2a_lo(cB0, q2.y, n6);
    n7 = __dp2a_lo(c0R, q2.y, 32768u); n7 = __dp2a_hi(cGB, q2.y, n7);
    P[0] = __byte_perm(n0, n4, 0x7632); P[1] = __byte_perm(n1, n5, 0x7632);     // P[j] = g[j] | g[j+4] << 16
    P[2] = __byte_perm(n2, n6, 0x7632); P[3] = __byte_perm(n3, n7, 0x7632);
    E = __byte_perm(__byte_perm(n0, n1, 0x0062), __byte_perm(n6, n7, 0x6200), 0x7610);   // bytes (g0, g1, g6, g7)
}

__global__ void __launch_bounds__(kFastThreads)
k_flood_raster_fast(const Mode m, const uint8_t* __restrict__ rgb, const uint32_t* __restrict__ list, const uint32_t* __restrict__ counters,
                    int base, int cap, const uint8_t* __restrict__ sharpen_of, uint16_t* __restrict__ ws_raster)
{
    __shared__ uint32_t ex[2][kFastThreads];                       // halo words E of the row in flight (double buffered)
    __shared__ __align__(16) uint8_t outb[2][16][kFastThreads];    // threshold bytes of the 16-row group being collected
    const int W = m.width, H = m.height;
    const int nthr = W >> 3;                                      // active threads (W / 8 <= 128)
    const int nb = (H + kFastBand - 1) / kFastBand;
    const int cnt = chunk_count(counters, base, cap);
    const int t = threadIdx.x;
    const bool act = t < nthr;
    const int tc = act ? t : nthr - 1;                            // inactive threads shadow the last one (loads stay in bounds)
    const size_t row_bytes = (size_t)W * 3;
    const uint32_t kBias = 0x7FF37FF3u;                           // per half: 0x8000 - 13

    for (int item = blockIdx.x; item < cnt * nb; item += gridDim.x) {
        const int e = item / nb, band = item - e * nb;
        const uint32_t f = list[base + e];
        if (sharpen_of && sharpen_of[f]) continue;                // a sharpened frame of a mixed batch: the other raster's
        const uint8_t* frame = rgb + (size_t)f * row_bytes * (size_t)H;
        uint16_t* raster = ws_raster + (size_t)e * raster_words16(W, H);
        const int y0 = band * kFastBand, y1 = (y0 + kFastBand < H) ? y0 + kFastBand : H;
        // input rows y0-2 .. y1+1 (clamped to the frame = BORDER_REPLICATE); the output row lags the input row by two
        uint32_t hr[5][4], Pr[3][4], nV[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            nV[j] = kBias;
#pragma unroll
            for (int i = 0; i < 5; ++i) hr[i][j] = 0;
#pragma unroll
            for (int i = 0; i < 3; ++i) Pr[i][j] = 0;
        }
        auto load_row = [&](int rr, uint2& a, uint2& b, uint2& c) {
            const int yy = rr < 0 ? 0 : (rr > H - 1 ? H - 1 : rr);
            const uint2* rp = reinterpret_cast<const uint2*>(frame + (size_t)yy * row_bytes) + 3 * tc;
            a = __ldg(rp); b = __ldg(rp + 1); c = __ldg(rp + 2);
        };
        uint2 qa, qb, qc;
        load_row(y0 - 2, qa, qb, qc);
        __syncthreads();                                           // the previous item's last flush has been read
        for (int rbase = y0 - 2; rbase < y1 + 2; rbase += 15) {
#pragma unroll
            for (int u = 0; u < 15; ++u) {
                const int rr = rbase + u;
                if (rr >= y1 + 2) break;
                uint32_t (&P)[4] = Pr[u % 3];
                uint32_t E;
                gray8_packed(qa, qb, qc, P, E);
                if (rr + 1 < y1 + 2) load_row(rr + 1, qa, qb, qc);   // next row's pixels fly during this row's arithmetic
                const int par = rr & 1;
                ex[par][t] = E;
                __syncthreads();
                // replicate at the frame's left / right edge: (g-2, g-1) = (g0, g0), (g8, g9) = (g7, g7)
                const uint32_t lE = (t == 0) ? __byte_perm(E, 0, 0x0000) : ex[par][t - 1];          // bytes 2,3 used: g6,g7 of the left
                const uint32_t rE = (t >= nthr - 1) ? __byte_perm(E, 0, 0x3333) : ex[par][t + 1];   // bytes 0,1 used: g0,g1 of the right
                const uint32_t Pm2 = __byte_perm(lE, P[2], 0x5452), Pm1 = __byte_perm(lE, P[3], 0x5453);
                const uint32_t P4 = __byte_perm(P[0], rE, 0x3432), P5 = __byte_perm(P[1], rE, 0x3532);
                uint32_t h[4];
                h[0] = Pm2 + Pm1 + P[0] + P[1] + P[2];
                h[1] = h[0] - Pm2 + P[3];
                h[2] = h[1] - Pm1 + P4;
                h[3] = h[2] - P[0] + P5;
                uint32_t tj[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    nV[j] = nV[j] + hr[u % 5][j] - h[j];              // drops row rr-5, adds row rr: window rr-4 .. rr
                    hr[u % 5][j] = h[j];
                    tj[j] = 25u * Pr[(u + 1) % 3][j] + nV[j];         // centre row rr-2; bit15 / bit31 = (25 g > boxsum + 12)
                }
                const int y = rr - 2;
                if (y >= y0) {
                    uint32_t byte = ((tj[0] >> 15) & 0x00010001u) | ((tj[1] >> 14) & 0x00020002u) |
                                    ((tj[2] >> 13) & 0x00040004u) | ((tj[3] >> 12) & 0x00080008u);
                    byte = (byte | (byte >> 12)) & 0xFFu;
                    outb[(y >> 4) & 1][y & 15][t] = (uint8_t)byte;
                    if ((y & 15) == 15 || y == y1 - 1) {
                        __syncthreads();
                        // 16 rows x nthr bytes -> (nthr / 2) tiles of 32 bytes, contiguous in the tiled raster: thread t writes
                        // rows 8 (t & 1) .. +7 of tile t >> 1 as one 16-byte store
                        if (act) {
                            const uint16_t* ob = reinterpret_cast<const uint16_t*>(&outb[(y >> 4) & 1][0][0]);
                            const int tile = t >> 1, r0 = 8 * (t & 1);
                            uint32_t w[4];
#pragma unroll
                            for (int k = 0; k < 4; ++k)
                                w[k] = (uint32_t)ob[(r0 + 2 * k) * (kFastThreads / 2) + tile] | ((uint32_t)ob[(r0 + 2 * k + 1) * (kFastThreads / 2) + tile] << 16);
                            uint16_t* dst = raster + raster_tile_index(W >> 4, 16 * tile, (y & ~15) + r0);
                            *reinterpret_cast<uint4*>(dst) = make_uint4(w[0], w[1], w[2], w[3]);
                        }
                    }
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------- fast raster, sharpen variant
// needs_sharpen preprocessing of the WHOLE frame with OpenCV's borders (CimbReader.cpp:17-46): gray -> filter2D with
// [0 -1 0; -1 4.5 -1; 0 -1 0] (BORDER_REFLECT_101, cvRound, saturate) -> adaptiveThreshold(MEAN_C, block 7, C = 0, BORDER_REPLICATE).
// Same decomposition as k_flood_raster_fast (one CTA of 128 threads per 64-row band, 8 px per thread, rows streamed, tiled
// output), with K1's packed sharpen arithmetic (k1_decode.cu, template SH): per sharpened row sr the thread holds the gray rows
// above / at / below it (reflected at the frame's top and bottom; one new row per step except where a clamped row repeats),
// exchanges the gray halo (reflected at the left / right edge), forms its eight sharpened pixels, exchanges their halo
// (replicated at the edges), keeps seven rows of horizontal 7-sums and four sharpened rows, and emits the threshold byte of
// row sr - 3: 49 s > boxsum + 24.  Two barriers per row.  A numpy model of exactly this schedule is checked against the
// oracle over whole frames, borders included, in tests/test_k1x_sharpen_raster_model.py.
__global__ void __launch_bounds__(kFastThreads)
k_flood_raster_fast_sharpen(const Mode m, const uint8_t* __restrict__ rgb, const uint32_t* __restrict__ list, const uint32_t* __restrict__ counters,
                            int base, int cap, const uint8_t* __restrict__ sharpen_of, uint16_t* __restrict__ ws_raster)
{
    __shared__ uint32_t ex[2][kFastThreads];                       // gray halo words E (double buffered by load parity)
    __shared__ uint32_t sx[2][2][kFastThreads];                    // sharpened halo words (s0,s1,s2) / (s5,s6,s7) (by row parity)
    __shared__ __align__(16) uint8_t outb[2][16][kFastThreads];
    const int W = m.width, H = m.height;
    const int nthr = W >> 3;
    const int nb = (H + kFastBand - 1) / kFastBand;
    const int cnt = chunk_count(counters, base, cap);
    const int t = threadIdx.x;
    const bool act = t < nthr;
    const int tc = act ? t : nthr - 1;                            // inactive threads shadow the last one
    const bool firstT = t == 0, lastT = t >= nthr - 1;
    const int tl = t > 0 ? t - 1 : 0, tr = t < kFastThreads - 1 ? t + 1 : t;
    const size_t row_bytes = (size_t)W * 3;
    const uint32_t kBias = 0x7FE77FE7u;                           // per half: 0x8000 - 25

    for (int item = blockIdx.x; item < cnt * nb; item += gridDim.x) {
        const int e = item / nb, band = item - e * nb;
        const uint32_t f = list[base + e];
        if (sharpen_of && !sharpen_of[f]) continue;               // a plain frame of a mixed batch: the other raster's
        const uint8_t* frame = rgb + (size_t)f * row_bytes * (size_t)H;
        uint16_t* raster = ws_raster + (size_t)e * raster_words16(W, H);
        const int y0 = band * kFastBand, y1 = (y0 + kFastBand < H) ? y0 + kFastBand : H;
        uint32_t Gu[4], Gc[4], Gd[4], lEc = 0, rEc = 0, lEd = 0, rEd = 0;      // gray rows above / at / below the sharpened row
        uint32_t Qr[4][4], hr[7][4], nV[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            nV[j] = kBias; Gu[j] = Gc[j] = Gd[j] = 0;
#pragma unroll
            for (int i = 0; i < 7; ++i) hr[i][j] = 0;
#pragma unroll
            for (int i = 0; i < 4; ++i) Qr[i][j] = 0;
        }
        int have_u = -9, have_c = -9, have_d = -9;
        unsigned ld = 0;
        uint2 pa = make_uint2(0, 0), pb = pa, pc = pa;             // a row requested one step ahead
        int pf_row = -9;
        auto fetch = [&](int y, uint2& a, uint2& b, uint2& c) {
            const uint2* rp = reinterpret_cast<const uint2*>(frame + (size_t)y * row_bytes) + 3 * tc;
            a = __ldg(rp); b = __ldg(rp + 1); c = __ldg(rp + 2);
        };
        auto load = [&](int y, uint32_t (&P)[4], uint32_t& lE, uint32_t& rE) {
            uint2 a, b, c;
            if (y == pf_row) { a = pa; b = pb; c = pc; } else fetch(y, a, b, c);
            uint32_t E;
            gray8_packed(a, b, c, P, E);
            const unsigned par = ld & 1u; ++ld;
            ex[par][t] = E;
            __syncthreads();
            // filter2D's BORDER_REFLECT_101 at the frame's left / right edge: g(-1) = g(1), g(W) = g(W-2)
            lE = firstT ? __byte_perm(E, 0, 0x1111) : ex[par][tl];      // byte 3 is used: the left neighbour's g7
            rE = lastT ? __byte_perm(E, 0, 0x2222) : ex[par][tr];       // byte 0 is used: the right neighbour's g0
        };
        __syncthreads();                                           // the previous item's last flush has been read
        const int sr0 = y0 - 3;
        for (int srb = sr0; srb < y1 + 3; srb += 7) {
#pragma unroll
            for (int u = 0; u < 7; ++u) {
                const int sr = srb + u;
                if (sr >= y1 + 3) break;
                const int s = clampi(sr, 0, H - 1);                // adaptiveThreshold's BORDER_REPLICATE: the sharpened row repeats
                const int wu = reflect101(s - 1, H), wd = reflect101(s + 1, H);
                if (have_c == wu && have_d == s) {                 // one row further down: the common case
#pragma unroll
                    for (int j = 0; j < 4; ++j) { Gu[j] = Gc[j]; Gc[j] = Gd[j]; }
                    lEc = lEd; rEc = rEd;
                    load(wd, Gd, lEd, rEd);
                } else if (!(have_u == wu && have_c == s && have_d == wd)) {
                    uint32_t dl, dr;
                    load(wu, Gu, dl, dr); load(s, Gc, lEc, rEc); load(wd, Gd, lEd, rEd);
                }
                have_u = wu; have_c = s; have_d = wd;
                {   // the row the next step will want, requested now
                    const int ns = clampi(sr + 1, 0, H - 1);
                    pf_row = reflect101(ns + 1, H);
                    fetch(pf_row, pa, pb, pc);
                }
                // ---- sharpen (k1_decode.cu, SH): twice = 9 c - 2 (up + down + left + right); s = clamp(round-half-even(twice / 2), 0, 255)
                uint32_t Q[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const uint32_t Pl = (j == 0) ? __byte_perm(lEc, Gc[3], 0x5453) : Gc[j > 0 ? j - 1 : 0];
                    const uint32_t Pr = (j == 3) ? __byte_perm(Gc[0], rEc, 0x3432) : Gc[j < 3 ? j + 1 : 3];
                    const uint32_t nbr = Gu[j] + Gd[j] + Pl + Pr;
                    const uint32_t T = 9u * Gc[j] + (0x08000800u - 2u * nbr);
                    const uint32_t tcl = __vminu2(__vmaxu2(T, 0x08000800u), 0x09FE09FEu) - 0x08000800u;
                    Q[j] = ((tcl + ((tcl >> 1) & 0x00010001u)) >> 1) & 0x00FF00FFu;
                }
                const uint32_t FL = __byte_perm(__byte_perm(Q[0], Q[1], 0x0040), Q[2], 0x0410);     // (s0, s1, s2, .)
                const uint32_t FH = __byte_perm(__byte_perm(Q[1], Q[2], 0x0062), Q[3], 0x0610);     // (s5, s6, s7, .)
                const unsigned par2 = (unsigned)(sr - sr0) & 1u;
                sx[par2][0][t] = FL; sx[par2][1][t] = FH;
                __syncthreads();
                // the box sum replicates at the left / right edge: S(-k) = s0, S(W-1+k) = s7
                const uint32_t lF = firstT ? __byte_perm(FL, 0, 0x0000) : sx[par2][1][tl];
                const uint32_t rF = lastT ? __byte_perm(FH, 0, 0x2222) : sx[par2][0][tr];
                const uint32_t Qm3 = __byte_perm(lF, Q[1], 0x5450), Qm2 = __byte_perm(lF, Q[2], 0x5451), Qm1 = __byte_perm(lF, Q[3], 0x5452);
                const uint32_t Q4 = __byte_perm(Q[0], rF, 0x3432), Q5 = __byte_perm(Q[1], rF, 0x3532), Q6 = __byte_perm(Q[2], rF, 0x3632);
                uint32_t h[4];
                h[0] = Qm3 + Qm2 + Qm1 + Q[0] + Q[1] + Q[2] + Q[3];
                h[1] = h[0] - Qm3 + Q4;
                h[2] = h[1] - Qm2 + Q5;
                h[3] = h[2] - Qm1 + Q6;
                uint32_t tj[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    nV[j] = nV[j] + hr[u][j] - h[j];                // drops row sr-7, adds row sr: window sr-6 .. sr
                    hr[u][j] = h[j];
                    Qr[0][j] = Qr[1][j]; Qr[1][j] = Qr[2][j]; Qr[2][j] = Qr[3][j]; Qr[3][j] = Q[j];
                    tj[j] = 49u * Qr[0][j] + nV[j];                  // centre row sr-3; bit15 / bit31 = (49 s > boxsum + 24)
                }
                const int y = sr - 3;
                if (y >= y0) {
                    uint32_t byte = ((tj[0] >> 15) & 0x00010001u) | ((tj[1] >> 14) & 0x00020002u) |
                                    ((tj[2] >> 13) & 0x00040004u) | ((tj[3] >> 12) & 0x00080008u);
                    byte = (byte | (byte >> 12)) & 0xFFu;
                    outb[(y >> 4) & 1][y & 15][t] = (uint8_t)byte;
                    if ((y & 15) == 15 || y == y1 - 1) {
                        __syncthreads();
                        if (act) {
                            const uint16_t* ob = reinterpret_cast<const uint16_t*>(&outb[(y >> 4) & 1][0][0]);
                            const int tile = t >> 1, r0 = 8 * (t & 1);
                            uint32_t w[4];
#pragma unroll
                            for (int k = 0; k < 4; ++k)
                                w[k] = (uint32_t)ob[(r0 + 2 * k) * (kFastThreads / 2) + tile] | ((uint32_t)ob[(r0 + 2 * k + 1) * (kFastThreads / 2) + tile] << 16);
                            uint16_t* dst = raster + raster_tile_index(W >> 4, 16 * tile, (y & ~15) + r0);
                            *reinterpret_cast<uint4*>(dst) = make_uint4(w[0], w[1], w[2], w[3]);
                        }
                    }
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------- heap (warp-uniform)
// 32-bit entries: prio(7) << 25 | cooldown code(3) << 22 | (dy + 8)(4) << 18 | (dx + 8)(4) << 14 | cell index(14).
// std::priority_queue<decode_prio, vector, PrioCompare> with comp(a, b) = a.prio > b.prio: only the priority is compared,
// so the pop order of equal priorities is whatever libstdc++'s sift-up / sift-down produce; both are restated literally.
// Element i lives at shared word i + 1 (so the children 2h+1, 2h+2 are one aligned 64-bit load) while i < hs, else in
// the global spill area at word i - hs (hs is odd, so a pair never straddles the two).  Shared memory is addressed through
// 32-bit shared-window addresses.
// Every lane of the walking warp executes push and pop with the same arguments and keeps the same `n`.  Where the address and
// the value are the same in every lane ("uniform" accesses) EVERY lane stores: the redundant stores merge into one, no branch
// is needed, and each lane later reads back what it wrote itself, so no warp barrier is needed either.  Only the sift-down
// spreads different nodes over the lanes; its results are published with one barrier.
__device__ __forceinline__ uint32_t lds32(uint32_t a) { uint32_t v; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
__device__ __forceinline__ uint2 lds64(uint32_t a) { uint2 v; asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(a)); return v; }
__device__ __forceinline__ void sts32(uint32_t a, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;" :: "r"(a), "r"(v) : "memory"); }
__device__ __forceinline__ void sts64(uint32_t a, uint32_t x, uint32_t y) { asm volatile("st.shared.v2.u32 [%0], {%1, %2};" :: "r"(a), "r"(x), "r"(y) : "memory"); }

struct Heap {
    uint32_t sm;          // shared-window byte address of word 0 (element i at sm + 4 i + 4)
    uint32_t path;        // shared-window byte address of the pop's path scratch: kPathSlots x (node, moved value)
    uint32_t* spill; int n; int hs;
    // element load / store, shared or spill chosen by predicate (no branch)
    __device__ __forceinline__ uint32_t get(int i) const
    {
        uint32_t v;
        asm volatile("{ .reg .pred p; setp.lt.s32 p, %3, %4;\n"
                     "  @p ld.shared.u32 %0, [%1];\n"
                     "  @!p ld.global.cg.u32 %0, [%2]; }"
                     : "=r"(v) : "r"(sm + 4u * (uint32_t)i + 4u), "l"(spill + (i - hs)), "r"(i), "r"(hs));
        return v;
    }
    __device__ __forceinline__ void set(int i, uint32_t v) const
    {
        asm volatile("{ .reg .pred p; setp.lt.s32 p, %3, %4;\n"
                     "  @p st.shared.u32 [%0], %2;\n"
                     "  @!p st.global.cg.u32 [%1], %2; }"
                     :: "r"(sm + 4u * (uint32_t)i + 4u), "l"(spill + (i - hs)), "r"(v), "r"(i), "r"(hs) : "memory");
    }
    __device__ __forceinline__ void set_if(int i, uint32_t v, bool doit) const
    {
        const int in_sm = doit && i < hs, in_gl = doit && i >= hs;
        asm volatile("{ .reg .pred p, q; setp.ne.s32 p, %3, 0; setp.ne.s32 q, %4, 0;\n"
                     "  @p st.shared.u32 [%0], %2;\n"
                     "  @q st.global.cg.u32 [%1], %2; }"
                     :: "r"(sm + 4u * (uint32_t)i + 4u), "l"(spill + (i - hs)), "r"(v), "r"(in_sm), "r"(in_gl) : "memory");
    }
};
__device__ __forceinline__ uint32_t hprio(uint32_t e) { return e >> 25; }

// std::push_heap (__push_heap): append, sift up while parent.prio > prio (strict).  Uniform: every lane does all of it.
// parent0 = the value of the first parent when the caller has already fetched it (parent0_of = its element index), else any.
__device__ __forceinline__ void heap_push(Heap& h, uint32_t e, uint32_t parent0, int parent0_of)
{
    int hole = h.n++;
    const uint32_t prio = hprio(e);
    while (hole > 0) {
        const int parent = (hole - 1) >> 1;
        const uint32_t pe = parent == parent0_of ? parent0 : h.get(parent);
        if (hprio(pe) <= prio) break;
        h.set(hole, pe);
        hole = parent;
        parent0_of = -1;                                       // (the fetched value is only good for the first step)
    }
    h.set(hole, e);
}

// per-lane constants of the five-level subtree a sift-down round works on: lane i < 31 stands for the node at depth d,
// position j of the subtree (heap order: i = 2^d - 1 + j), i.e. node = (hole + 1) * 2^d + j - 1; anc_mask has the bits of its
// ancestors' lanes, anc_want the value each of those bits must have ("ancestor prefers its left child") for the descent to
// pass through this node.  Lane 31 stands for no node (its index is always beyond the heap).
struct SubtreeLane { int pow2d, jm1; bool last; uint32_t anc_mask, anc_want; };
__device__ __forceinline__ SubtreeLane subtree_lane(int lane)
{
    SubtreeLane s;
    const int d = 31 - __clz(lane + 1);
    s.pow2d = 1 << d; s.jm1 = lane - s.pow2d; s.last = d == 4;
    s.anc_mask = 0; s.anc_want = 0;
    for (int i = lane; i > 0;) {
        const int p = (i - 1) >> 1;
        s.anc_mask |= 1u << p;
        if (i & 1) s.anc_want |= 1u << p;            // odd index = left child
        i = p;
    }
    if (lane == 31) { s.pow2d = 0; s.jm1 = 0x3FFFFFFF; s.last = false; s.anc_mask = 0; s.anc_want = 0; }
    return s;
}

// the literal form, one level per step (only reached by heaps of more than 65 535 entries, or when a test asks for it).
// Uniform: returns the new element count.
__device__ __noinline__ int heap_pop_serial(Heap h)
{
    const uint32_t value = h.get(h.n - 1);
    const int len = --h.n;
    if (len == 0) return len;
    int hole = 0, second = 0;
    while (second < ((len - 1) >> 1)) {
        second = 2 * (second + 1);
        uint32_t a = h.get(second);
        const uint32_t b = h.get(second - 1);
        if (hprio(a) > hprio(b)) { second--; a = b; }
        h.set(hole, a);
        hole = second;
    }
    if ((len & 1) == 0 && second == ((len - 2) >> 1)) {
        second = 2 * (second + 1);
        h.set(hole, h.get(second - 1));
        hole = second - 1;
    }
    const uint32_t vp = hprio(value);
    while (hole > 0) {
        const int parent = (hole - 1) >> 1;
        const uint32_t pe = h.get(parent);
        if (hprio(pe) <= vp) break;
        h.set(hole, pe);
        hole = parent;
    }
    h.set(hole, value);
    return len;
}

// std::pop_heap + pop_back (__adjust_heap with the hole at the root, then __push_heap of the last element):
//   while (second < (len - 1) / 2) { second = 2 (second + 1); if (v[second].prio > v[second - 1].prio) second--; v[hole] = v[second]; hole = second; }
//   if (len even && second == (len - 2) / 2) { second = 2 (second + 1); v[hole] = v[second - 1]; hole = second - 1; }
//   sift `value` (the former last element) up from the hole: while (parent.prio > value.prio) { v[hole] = v[parent]; hole = parent; }
// The descent path h_0 = 0, h_1, ..., h_L does not depend on `value`, only on which child each node prefers.  One round
// handles the 31 nodes of the five-level subtree under the current hole: lane i loads the two children of its node, the
// preferences are collected with one ballot, and every lane decides from its ancestors' bits whether the descent passes
// through its node -- a dozen levels cost three memory round trips instead of a dozen.  Nothing of the heap is stored during
// the descent: the lane of path level k writes (h_k, m_k = old v[h_(k+1)], the value that WOULD move up into h_k) to a small
// scratch.  The sift-up walks the same path backwards and undoes those moves while prio(m_k) > prio(value); so with
// s = 1 + max { k : prio(m_k) <= prio(value) } the net effect is v[h_k] = m_k for k < s, v[h_s] = value, everything below
// untouched: lane k stores level k -- s + 1 stores, no reads.
constexpr int kPopRounds = 3;          // 15 levels: heaps of up to 65 535 entries (seven times the largest seen); beyond: heap_pop_serial
constexpr int kPathSlots = 20;
__device__ __forceinline__ void heap_pop(Heap& h, const SubtreeLane& sl, int lane, int serial_above)
{
    if (h.n > serial_above) { h.n = heap_pop_serial(h); __syncwarp(); return; }
    const uint32_t value = h.get(h.n - 1);                     // (often in L2: in flight during the rounds, used after them)
    const int len = --h.n;
    if (len == 0) return;
    const int lim = (len - 1) >> 1;
    int hole = 0;
#pragma unroll
    for (int r = 0; r < kPopRounds; ++r) {
        if (hole < lim) {                                      // warp-uniform
            const int node = (hole + 1) * sl.pow2d + sl.jm1;
            const bool has2 = node < lim;                      // both children inside the heap: the descent continues below it
            const int ce = 2 * node + 2;                       // its right child's element index
            uint2 c = make_uint2(0u, 0u);
            {
                const int in_sm = has2 && ce < h.hs, in_gl = has2 && ce >= h.hs;
                asm volatile("{ .reg .pred p, q; setp.ne.s32 p, %4, 0; setp.ne.s32 q, %5, 0;\n"
                             "  @p ld.shared.v2.u32 {%0, %1}, [%2];\n"
                             "  @q ld.global.cg.v2.u32 {%0, %1}, [%3]; }"
                             : "+r"(c.x), "+r"(c.y) : "r"(h.sm + 4u * (uint32_t)ce), "l"(h.spill + (ce - 1 - h.hs)), "r"(in_sm), "r"(in_gl));
            }
            const bool left = hprio(c.y) > hprio(c.x);         // right child strictly worse -> the left child moves up
            const uint32_t pref = __ballot_sync(0xffffffffu, has2 && left);
            // the descent reaches this node iff its parent has two children ((node - 1) / 2 < lim <=> node <= 2 lim) and every
            // ancestor points towards it
            const bool reached = node <= 2 * lim && (((pref ^ sl.anc_want) & sl.anc_mask) == 0u);
            if (reached && has2) {                             // path level of this node = floor(log2(node + 1))
                const int lvl = 31 - __clz(node + 1);
                sts64(h.path + 8u * (uint32_t)lvl, (uint32_t)node, left ? c.x : c.y);
            }
            // the round ends at the first reached node without two children, or below the subtree's last level: exactly one lane
            const int nxt = has2 ? ce - (left ? 1 : 0) : node;
            hole = (int)__reduce_or_sync(0xffffffffu, (reached && (!has2 || sl.last)) ? (uint32_t)nxt : 0u);
        }
    }
    int last_level = 31 - __clz(hole + 1);                     // level of the hole the descent ends in
    // a last node with only a left child: one more level of the path (uniform)
    if ((len & 1) == 0 && hole == ((len - 2) >> 1)) {
        const uint32_t m_lone = h.get(2 * hole + 1);
        sts64(h.path + 8u * (uint32_t)last_level, (uint32_t)hole, m_lone);
        hole = 2 * hole + 1;
        ++last_level;
    }
    __syncwarp();
    // ---- lane k owns path level k: s = 1 + deepest level whose moved value does not have to go back down
    uint2 pm = make_uint2((uint32_t)hole, 0u);
    if (lane < last_level) pm = lds64(h.path + 8u * (uint32_t)lane);
    const uint32_t vp = hprio(value);
    const uint32_t keep = __ballot_sync(0xffffffffu, lane < last_level && hprio(pm.y) <= vp);
    const int s = 32 - __clz(keep);                            // = 1 + highest set bit, 0 if none (always <= last_level)
    h.set_if((int)pm.x, lane == s ? value : pm.y, lane <= s);
    __syncwarp();
}
// cooldown values (CellDrift::calculate_cooldown, CellDrift.cpp:34-43): 4, 0xFF, 0xFE (initial), or an odd drift id 1/3/5/7
__device__ __forceinline__ uint32_t cd_code(uint32_t cd) { return cd == 4u ? 0u : cd == 0xFFu ? 1u : cd == 0xFEu ? 2u : 3u + (cd >> 1); }
__device__ __forceinline__ uint32_t cd_value(uint32_t code) { return __byte_perm(0x01FEFF04u, 0x00070503u, code) & 0xFFu; }   // byte `code` of 04 FF FE 01 03 05 07
constexpr uint32_t kSeedCode = 7u;     // entry pushed by reset(): its cell's inherit record is NOT in the entry
__device__ __forceinline__ uint32_t make_entry(uint32_t idx, int dx, int dy, uint32_t code, uint32_t prio)
{
    return (prio << 25) | (code << 22) | ((uint32_t)(dy + 8) << 18) | ((uint32_t)(dx + 8) << 14) | idx;
}

// top-left pixel of linear cell ci (CellPositions::compute_linear, CellPositions.cpp:5-50), branch-free
// (everything comes from kernel parameters = constant-bank operands: no registers are tied up)
__device__ __forceinline__ void cell_pixel(const Mode& m, float rcp_narrow, float rcp_wide, int ci, int& px, int& py)
{
    const int top_mid = m.top_cells + m.mid_cells;
    const bool mid = ci >= m.top_cells && ci < top_mid, bot = ci >= top_mid;
    const int q = ci - (mid ? m.top_cells : (bot ? top_mid : 0));
    const int width = mid ? m.cells_x : m.cells_x - 2 * m.corner;
    const int kk = __float2int_rz(((float)q + 0.5f) * (mid ? rcp_wide : rcp_narrow));     // exact floor for q < 2^14
    const int c = q - kk * width;
    px = m.cell_offset + kSpacing * (c + (mid ? 0 : m.corner));
    py = m.cell_offset + kSpacing * (kk + (mid ? m.corner : (bot ? m.cells_y - m.corner : 0)));
}

// ---------------------------------------------------------------------------------------------- the walk
// Shared memory of one walking warp: heap[hs + 1] words, the _remaining bitmap (1 bit per cell), the pop's path scratch.
// One byte per cell lives in a per-slot global array (L2 resident, read by the 12 candidate lanes in parallel):
//   0 = decoded (FloodDecodePositions::_remaining false), else best_prio + 1 (0xFF for the initial 0xFE).
// Why the inherit record (drift, best_prio, cooldown; FloodDecodePositions.h:17) can ride in the heap entry: update()
// only rewrites it when the new error is strictly lower (FloodDecodePositions.cpp:75), and pushes an entry with that
// error, so of all entries of a cell the one that pops first is always the latest, and it carries the record as it stands.
// The exception are the eight entries reset() seeds with priority 0/1 while the record says (0,0,0xFE,0xFE): when such an
// entry pops, the record is the latest update still sitting in the heap (found by a warp-wide scan), else the initial one.
// Memory latency is taken off the chain by running one cell ahead: as soon as a pop has settled, the NEW heap top names the
// cell of the next iteration (unless a push with a lower priority overtakes it, which the next iteration checks), so its
// window rows and its neighbour-table row are requested right away and arrive while the current cell is scored and pushed.
__global__ void __launch_bounds__(32, 32)
k_flood_walk(const Mode m, const uint32_t* __restrict__ list, const uint32_t* __restrict__ counters, int base, int cap, uint32_t* next_counter,
             int heap_smem, const uint16_t* __restrict__ ws_raster, uint32_t* __restrict__ ws_result, uint32_t* ws_spill, size_t spill_cap,
             uint8_t* ws_prio, const uint16_t* __restrict__ cinfo, CellTrace* __restrict__ trace, int serial_above,
             float rcp_narrow, float rcp_wide)
{
    extern __shared__ __align__(16) uint8_t walk_smem[];
    // [heap: heap_smem + 1 words][_remaining bitmap: kMaxCells / 32 words][path scratch of the pop: kPathSlots x 2 words]
    const uint32_t sm_base = (uint32_t)__cvta_generic_to_shared(walk_smem);
    const uint32_t rem_base = sm_base + 4u * (uint32_t)(heap_smem + 1);
    uint8_t* prio = ws_prio + (size_t)blockIdx.x * kMaxCells;
    const int lane = threadIdx.x;
    const int W = m.width, ncells = m.num_cells, tiles_x = W >> 4;
    const size_t rwords = raster_words16(W, m.height);
    const int cnt = chunk_count(counters, base, cap);
    const unsigned long long tileL = cx_tiles_L[lane & 15];
    const int narrow = m.cells_x - 2 * m.corner;
    const SubtreeLane sl = subtree_lane(lane);
    Heap heap; heap.sm = sm_base; heap.path = rem_base + 4u * (uint32_t)(kMaxCells / 32);
    heap.spill = ws_spill + (size_t)blockIdx.x * spill_cap; heap.n = 0; heap.hs = heap_smem;

    while (true) {
        uint32_t k = 0;
        if (lane == 0) k = atomicAdd(next_counter, 1u);
        k = __shfl_sync(0xffffffffu, k, 0);
        if (k >= (uint32_t)cnt) break;
        const uint32_t f = list[base + k];
        const uint16_t* raster = ws_raster + (size_t)k * rwords;
        uint32_t* result = ws_result + (size_t)k * ncells;

        // ---- FloodDecodePositions::reset (FloodDecodePositions.cpp:17-42)
        for (int i = lane; i < kMaxCells / 16; i += 32) __stcg(reinterpret_cast<uint4*>(prio) + i, make_uint4(~0u, ~0u, ~0u, ~0u));
        for (int i = lane; i < (ncells + 31) / 32; i += 32) sts32(rem_base + 4u * (uint32_t)i, 0xFFFFFFFFu);
        __syncwarp();
        heap.n = 0;
        {
            const int last = ncells - 1, bmb = m.top_cells;
            heap_push(heap, make_entry(0, 0, 0, kSeedCode, 0), 0u, -1); heap_push(heap, make_entry((uint32_t)(narrow - 1), 0, 0, kSeedCode, 0), 0u, -1);
            heap_push(heap, make_entry((uint32_t)last, 0, 0, kSeedCode, 0), 0u, -1); heap_push(heap, make_entry((uint32_t)(last - (narrow - 1)), 0, 0, kSeedCode, 0), 0u, -1);
            heap_push(heap, make_entry((uint32_t)bmb, 0, 0, kSeedCode, 1), 0u, -1); heap_push(heap, make_entry((uint32_t)(bmb + m.cells_x - 1), 0, 0, kSeedCode, 1), 0u, -1);
            heap_push(heap, make_entry((uint32_t)(last - bmb), 0, 0, kSeedCode, 1), 0u, -1);
            heap_push(heap, make_entry((uint32_t)(last - (bmb + m.cells_x - 1)), 0, 0, kSeedCode, 1), 0u, -1);
        }

        // what was requested ahead for the entry `ahead_e`: window words of this lane's row, neighbour-table entry
        uint32_t ahead_e = 0xFFFFFFFFu, ahead_ra = 0, ahead_rb = 0, ahead_cv = 0;
        int ahead_x = 0, ahead_y = 0;
        int count = 0;
        while (count < ncells) {
            // ---- FloodDecodePositions::next (FloodDecodePositions.cpp:49-67): the entry about to pop is the heap's first element
            if (heap.n == 0) break;                          // heap exhausted (cannot happen on a connected grid)
            const uint32_t e = lds32(sm_base + 4u);
            const int ci = (int)(e & 0x3FFFu);
            const uint32_t rem_bit = 1u << (ci & 31);
            const uint32_t rem_addr = rem_base + 4u * (uint32_t)(ci >> 5);
            const uint32_t rem_word = lds32(rem_addr);
            if (!(rem_word & rem_bit)) {                     // stale entry of a cell that is already decoded: skipped
                __syncwarp();                                // every lane has read the top before the pop rewrites it
                heap_pop(heap, sl, lane, serial_above);
                continue;
            }
            ++count;
            uint32_t code = (e >> 22) & 7u, prev_err = e >> 25;
            int ddx = (int)((e >> 14) & 15u) - 8, ddy = (int)((e >> 18) & 15u) - 8;
            if (code == kSeedCode) {                         // (scanned before the pop: the seed entry itself is excluded either way)
                uint32_t latest = 0xFFFFFFFFu;
                for (int i = lane; i < heap.n; i += 32) {
                    const uint32_t t = heap.get(i);
                    if ((t & 0x3FFFu) == (uint32_t)ci && ((t >> 22) & 7u) != kSeedCode && t < latest) latest = t;
                }
                latest = __reduce_min_sync(0xffffffffu, latest);
                if (latest != 0xFFFFFFFFu) {
                    code = (latest >> 22) & 7u; prev_err = latest >> 25;
                    ddx = (int)((latest >> 14) & 15u) - 8; ddy = (int)((latest >> 18) & 15u) - 8;
                } else { code = 2u; prev_err = 0xFEu; ddx = 0; ddy = 0; }
            }
            const uint32_t cooldown = cd_value(code);
            // ---- neighbour-table row (lanes 0-3 right / left / bottom / top, 4-11 the horizon chains, see flood_build_cinfo) and the
            // 10x10 window at (x-1, y-1) (lane r < 10: row r from at most two tiles): taken from the look-ahead when it was for this
            // very entry (a seed entry's drift is not in the entry: never looked ahead), else requested now.  The rasters are read
            // once per window and are far bigger than the L2: streaming loads, so that they do not evict the heaps and priority bytes.
            uint32_t ra, rb, cv;
            int x, y;                                             // CimbReader.cpp:146-148: position + drift
            if (e == ahead_e) { ra = ahead_ra; rb = ahead_rb; cv = ahead_cv; x = ahead_x; y = ahead_y; }
            else {
                int px, py;
                cell_pixel(m, rcp_narrow, rcp_wide, ci, px, py);
                x = px + ddx; y = py + ddy;
                ra = 0; rb = 0;
                cv = lane < 12 ? (uint32_t)__ldg(&cinfo[ci * 16 + lane]) : 0xFFFFu;
                if (lane < 10) {
                    const uint32_t ti = raster_tile_index(tiles_x, x - 1, y - 1 + lane);
                    ra = __ldcs(raster + ti); rb = __ldcs(raster + ti + 16);
                }
            }
            // every lane has read the heap top / bitmap before they are rewritten, and the priority bytes the last iteration's
            // pushes marked (stored by other lanes) are ordered before the loads below
            __syncwarp();
            const uint32_t rshift = (uint32_t)(x - 1) & 15u;
            // the candidates' priority bytes: requested now, needed after the scoring
            uint32_t pv = 0;
            if (cv != 0xFFFFu) pv = __ldcg(prio + cv);
            heap_pop(heap, sl, lane, serial_above);
            sts32(rem_addr, rem_word & ~rem_bit);
            __stcg(prio + ci, (uint8_t)0);
            // ---- look ahead: the new top is (most probably) the next cell
            const uint32_t parent_of = (uint32_t)((heap.n - 1) >> 1);                 // parent of the slot the first push will take
            const uint32_t parent_val = heap.n > 0 ? heap.get((int)parent_of) : 0u;
            ahead_e = 0xFFFFFFFFu;
            if (heap.n > 0) {
                const uint32_t ne = lds32(sm_base + 4u);
                if (((ne >> 22) & 7u) != kSeedCode) {
                    ahead_e = ne;
                    const int nci = (int)(ne & 0x3FFFu);
                    int npx, npy;
                    cell_pixel(m, rcp_narrow, rcp_wide, nci, npx, npy);
                    const int nx = npx + (int)((ne >> 14) & 15u) - 8, ny = npy + (int)((ne >> 18) & 15u) - 8;
                    ahead_x = nx; ahead_y = ny;
                    ahead_cv = lane < 12 ? (uint32_t)__ldg(&cinfo[nci * 16 + lane]) : 0xFFFFu;
                    ahead_ra = 0; ahead_rb = 0;
                    if (lane < 10) {
                        const uint32_t ti = raster_tile_index(tiles_x, nx - 1, ny - 1 + lane);
                        ahead_ra = __ldcs(raster + ti); ahead_rb = __ldcs(raster + ti + 16);
                    }
                }
            }
            const uint32_t myrow = ((ra | (rb << 16)) >> rshift) & 0x3FFu;     // bit i = window col i
            // ---- fast path: the centre hash (drift id 4 = rows 1..8, cols 1..8) is a dictionary tile.  The reference's search
            // starts with id 4 and returns at once on distance 0 (CimbDecoder.cpp:101-132), whatever the cooldown.
            uint32_t dist, sym, ncd;
            int id, ndx, ndy, rx, ry;
            bool exact;
            {
                const uint32_t b = (myrow >> 1) & 0xFFu;
                const uint32_t plo = (lane >= 1 && lane <= 4) ? b << (8 * (lane - 1)) : 0u;
                const uint32_t phi = (lane >= 5 && lane <= 8) ? b << (8 * (lane - 5)) : 0u;
                const uint32_t clo = __reduce_or_sync(0xffffffffu, plo), chi = __reduce_or_sync(0xffffffffu, phi);
                const uint4 te = cx_tiles_slot[(clo * m.hash_mul) >> 28];          // uniform index: one constant-bank read
                exact = te.x == clo && te.y == chi;
                sym = te.z;
            }
            if (exact) {                                     // warp-uniform
                dist = 0; id = 4; ncd = 4; ndx = ddx; ndy = ddy; rx = x; ry = y;
            } else {
                uint32_t win[10];
#pragma unroll
                for (int r = 0; r < 10; ++r) win[r] = __shfl_sync(0xffffffffu, myrow, r);
                // ---- candidates (id order 4,5,7,3,1,8,0,2,6; tiles 0..15), key = dist<<8 | order<<4 | tile
                // lane q < 9 extracts the hash at drift id order[q]: the window's 8-bit columns c0..c0+7 of all ten rows form one
                // 80-bit string, the hash at row offset r0 is bits [8 r0, 8 r0 + 64) of it (ahash_result::extract, ahash_result.h:70-106)
                uint32_t hlo, hhi;
                {
                    const int qq = lane < 9 ? lane : 0;
                    const int r0 = (int)((0x200201211ULL >> (4 * qq)) & 3u), c0 = (int)((0x020210121ULL >> (4 * qq)) & 3u);   // id / 3, id % 3
                    uint32_t b[10];
#pragma unroll
                    for (int r = 0; r < 10; ++r) b[r] = (win[r] >> c0) & 0xFFu;
                    const uint32_t w0 = b[0] | (b[1] << 8) | (b[2] << 16) | (b[3] << 24);
                    const uint32_t w1 = b[4] | (b[5] << 8) | (b[6] << 16) | (b[7] << 24);
                    const uint32_t w2 = b[8] | (b[9] << 8);
                    hlo = __funnelshift_r(w0, w1, 8 * r0); hhi = __funnelshift_r(w1, w2, 8 * r0);
                }
                // every lane scores its tile (lane & 15) against the hashes q = 2 it + (lane >> 4)
                const bool all = (cooldown == 0xFEu);                 // CimbDecoder.cpp:144
                const int nq = all ? 9 : 5;
                const uint32_t tile_lo = (uint32_t)tileL, tile_hi = (uint32_t)(tileL >> 32);
                uint32_t best_key = 0xFFFFFFFFu;
#pragma unroll
                for (int it = 0; it < 5; ++it) {
                    if (it >= 3 && !all) break;                       // warp-uniform
                    const int q = 2 * it + (lane >> 4);
                    const uint32_t lo = __shfl_sync(0xffffffffu, hlo, q & 15), hi = __shfl_sync(0xffffffffu, hhi, q & 15);
                    const int qid = (int)((0x620813754ULL >> (4 * q)) & 0xF);         // packed order table, nibble q
                    const bool valid = q < nq && !((uint32_t)qid == cooldown && qid != 4);   // CimbDecoder.cpp:116
                    const uint32_t d = (uint32_t)(__popc(lo ^ tile_lo) + __popc(hi ^ tile_hi));
                    const uint32_t key = valid ? ((d << 8) | ((uint32_t)q << 4) | (uint32_t)(lane & 15)) : 0xFFFFFFFFu;
                    best_key = key < best_key ? key : best_key;
                }
                best_key = __reduce_min_sync(0xffffffffu, best_key);
                // every lane derives the (warp-uniform) decision from the reduced key
                dist = best_key >> 8; sym = best_key & 0xFu;
                id = (int)((0x620813754ULL >> (4 * ((best_key >> 4) & 0xFu))) & 0xF);
                const int bx = id % 3 - 1, by = id / 3 - 1;                       // CellDrift::driftPairs, CellDrift.h:13-15
                ndx = clampi(ddx + bx, -7, 7); ndy = clampi(ddy + by, -7, 7);     // CellDrift.cpp:23-31
                rx = x + bx; ry = y + by;
                // CellDrift::calculate_cooldown, CellDrift.cpp:34-43
                if (id == 4) ncd = 4; else if ((id & 1) == 0) ncd = 0xFF; else if (((cooldown ^ (uint32_t)id) & 0xFFu) == 6) ncd = 0xFF; else ncd = (uint32_t)id;
            }
            __stcs(result + ci, ((uint32_t)rx & 0x7FFu) | (((uint32_t)ry & 0x7FFu) << 11) | (sym << 22));     // (uniform: every lane, one store)
            if (trace && lane == 0) {
                CellTrace tr;
                tr.order = (uint16_t)(count - 1); tr.x = (int16_t)rx; tr.y = (int16_t)ry;
                tr.drift_offset = (uint8_t)id; tr.distance = (uint8_t)dist;
                trace[(size_t)f * ncells + ci] = tr;
            }
            // ---- FloodDecodePositions::update (FloodDecodePositions.cpp:86-129) with update_adjacents (:69-83):
            // lanes 0..11 test one candidate each (still remaining and stored priority > err  <=>  byte >= err + 2); the new
            // priority is recorded and the survivors are pushed in the reference's order (adjacents, horizon, vert).
            const bool horizon = prev_err < 3u && dist < 3u && cooldown == 4u && ncd == 4u;
            const bool push = cv != 0xFFFFu && (lane < 4 || horizon) && pv >= dist + 2u;
            if (push) __stcg(prio + cv, (uint8_t)(dist + 1u));
            uint32_t todo = __ballot_sync(0xffffffffu, push);
            const uint32_t entry = make_entry(0, ndx, ndy, cd_code(ncd), dist);
            int first_parent = (int)parent_of;
            while (todo) {
                const int l = __ffs(todo) - 1;
                todo &= todo - 1;
                const uint32_t c = __shfl_sync(0xffffffffu, cv, l);
                heap_push(heap, entry | c, parent_val, first_parent);
                first_parent = -1;
            }
        }
        __syncwarp();
    }
}


// ---------------------------------------------------------------------------------------------- colour (P8/P9)
__device__ uint32_t flood_best_color(const float* adjust_tab, const Mode& m, uint32_t ri, uint32_t gi, uint32_t bi)
{   // CimbDecoder.cpp:168-200, float32 op for op (see k1_decode.cu best_color)
    float r = (float)ri, g = (float)gi, b = (float)bi;
    float mx = fmaxf(fmaxf(r, g), fmaxf(b, 1.0f));
    float mn = fminf(fminf(r, g), fminf(b, 48.0f));
    if (mn >= mx) mn = 0.0f;
    float adjust = adjust_tab[(int)(mx - mn)];
    int c[3];
    float in[3] = {r, g, b};
    for (int k = 0; k < 3; ++k) {
        float v = __fmul_rn(__fsub_rn(in[k], mn), adjust);
        if (v > __fsub_rn(245.0f, mn)) v = 255.0f;
        if (v < 0.0f) v = 0.0f;
        c[k] = (int)__float2uint_rz(v);
    }
    int a0 = c[0] - c[1], a1 = c[1] - c[2], a2 = c[2] - c[0];
    uint32_t best = 0, best_d = 0x7fffffffu;
    int num_colors = 1 << m.color_bits;
    for (int i = 0; i < num_colors; ++i) {
        int pr = m.palette[i][0], pg = m.palette[i][1], pb = m.palette[i][2];
        int d0 = a0 - (pr - pg), d1 = a1 - (pg - pb), d2 = a2 - (pb - pr);
        uint32_t d = (uint32_t)(d0 * d0 + d1 * d1 + d2 * d2);
        if (d < best_d) { best_d = d; best = (uint32_t)i; }
    }
    return best;
}

// colours at the drift-adjusted positions (CimbReader::read_color, CimbReader.cpp:133-137); one thread per cell
__global__ void __launch_bounds__(256)
k_flood_colour(const Mode m, const uint8_t* __restrict__ rgb, const uint32_t* __restrict__ list, const uint32_t* __restrict__ counters,
               int base, int cap, const uint32_t* __restrict__ ws_result, uint8_t* __restrict__ cellvals, const CcmArg cc)
{
    __shared__ float adjust[256];
    adjust[threadIdx.x] = cx_adjust[threadIdx.x];
    __syncthreads();
    const int W = m.width, ncells = m.num_cells;
    const size_t frame_bytes = (size_t)W * m.height * 3;
    const int cnt = chunk_count(counters, base, cap);
    const int num_colors = 1 << m.color_bits;
    const size_t total = (size_t)cnt * ncells;
    for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (size_t)gridDim.x * 256) {
        const int e = (int)(i / (size_t)ncells), ci = (int)(i - (size_t)e * ncells);
        const uint32_t f = list[base + e];
        const uint8_t* frame = rgb + (size_t)f * frame_bytes;
        const uint32_t rec = ws_result[i];
        const int x = (int)(rec & 0x7FFu), y = (int)((rec >> 11) & 0x7FFu);
        const uint32_t sym = (rec >> 22) & 0xFu;
        uint32_t col = 0;
        if (num_colors > 1) {
            uint32_t R = 0, G = 0, B = 0;
            for (int r = 1; r <= 6; ++r) {
                const uint8_t* p = frame + ((size_t)(y + r) * W + (size_t)(x + 1)) * 3;
                for (int c = 0; c < 6; ++c) { R += p[3 * c]; G += p[3 * c + 1]; B += p[3 * c + 2]; }
            }
            if (cc.means) cc.means[(size_t)f * ncells + ci] = (R / 36u) | ((G / 36u) << 8) | ((B / 36u) << 16);
            else if (cc.active && (!cc.per_frame_active || cc.per_frame_active[f])) {
                float mat[9];
#pragma unroll
                for (int q = 0; q < 9; ++q) mat[q] = cc.per_frame ? cc.per_frame[(size_t)f * 9 + q] : cc.m[q];
                col = best_color_ccm<0>(mat, m, R / 36u, G / 36u, B / 36u);
            } else col = flood_best_color(adjust, m, R / 36u, G / 36u, B / 36u);
        }
        cellvals[(size_t)f * ncells + ci] = (uint8_t)(sym | (col << m.symbol_bits));
    }
}

// ---------------------------------------------------------------------------------------------- host side
cudaError_t flood_init_tables(const float* adjust256, const unsigned long long* tiles_L16, uint32_t hash_mul)
{
    cudaError_t e = cudaMemcpyToSymbol(cx_adjust, adjust256, sizeof(float) * 256);
    if (e != cudaSuccess) return e;
    uint4 slots[16];
    for (int t = 0; t < 16; ++t) {
        const uint32_t lo = (uint32_t)tiles_L16[t], hi = (uint32_t)(tiles_L16[t] >> 32);
        slots[(lo * hash_mul) >> 28] = make_uint4(lo, hi, (uint32_t)t, 0u);
    }
    if ((e = cudaMemcpyToSymbol(cx_tiles_slot, slots, sizeof(slots))) != cudaSuccess) return e;
    return cudaMemcpyToSymbol(cx_tiles_L, tiles_L16, sizeof(unsigned long long) * 16);
}

// per cell 16 x u16: the 12 cells FloodDecodePositions::update may touch, in the reference's push order -- 0..3 the direct
// neighbours (right, left, bottom, top; update_adjacents), 4,5 right+1 / right+2, 6,7 left+1 / left+2 (horizontal horizon,
// only when BOTH right and left exist, FloodDecodePositions.cpp:102), 8,9 top+1 / top+2, 10,11 bottom+1 / bottom+2 (vertical,
// only when both top and bottom exist, :116); 0xFFFF = none.  Built from AdjacentCellFinder::find for every cell (adj_host).
static void flood_build_cinfo(const Mode& m, const uint16_t* adj, std::vector<uint16_t>& out)
{
    auto nb = [&](int cell, int dir) -> int { if (cell < 0) return -1; unsigned v = adj[(size_t)cell * 4 + dir]; return v == 0xFFFFu ? -1 : (int)v; };
    out.assign((size_t)m.num_cells * 16, 0xFFFFu);
    for (int i = 0; i < m.num_cells; ++i) {
        uint16_t* o = &out[(size_t)i * 16];
        for (int d = 0; d < 4; ++d) { int c = nb(i, d); if (c >= 0) o[d] = (uint16_t)c; }
        const int right = nb(i, 0), left = nb(i, 1), bottom = nb(i, 2), top = nb(i, 3);
        auto chain = [&](int first_from, int dir, int slot) {
            int a = nb(first_from, dir), b = nb(a, dir);
            if (a >= 0) o[slot] = (uint16_t)a;
            if (b >= 0) o[slot + 1] = (uint16_t)b;
        };
        if (right >= 0 && left >= 0) { chain(right, 0, 4); chain(left, 1, 6); }
        if (top >= 0 && bottom >= 0) { chain(top, 3, 8); chain(bottom, 2, 10); }
        int k, cc, rbase, ncols, x0;                       // slots 12, 13: the cell's top-left pixel
        cell_row_col(m, i, k, cc);
        cell_row_geom(m, k, rbase, ncols, x0);
        o[12] = (uint16_t)(x0 + kSpacing * cc);
        o[13] = (uint16_t)(m.cell_offset + kSpacing * k);
    }
}

cudaError_t flood_workspace_create(const Mode& m, int sm_count, const uint16_t* adj_host, FloodWorkspace* ws)
{
    ws->sm_count = sm_count;
    // shared-memory heap entries per walking warp (must be odd): 1023 = the ten top levels; deeper levels go to the
    // per-slot spill area in L2.  Shared memory per walk decides how many walks an SM holds (at most 32 blocks).
    ws->heap_smem = 1023;
    ws->walk_smem = (size_t)(ws->heap_smem + 1) * 4 + (size_t)(kMaxCells / 32) * 4 + (size_t)kPathSlots * 8;
    // few frames (the one-frame-per-call shape of the mirrors and the facade, small camera batches): nothing hides the L2 round
    // trips of the spilled heap levels then (a photograph's heap grows to ~4 500 entries, 19 500 pushes), so each walk gets the
    // whole heap in shared memory -- 8 191 entries, 34 KB, six walks per SM -- and the spill area is only the overflow
    ws->heap_smem_few = 8191;
    ws->walk_smem_few = (size_t)(ws->heap_smem_few + 1) * 4 + (size_t)(kMaxCells / 32) * 4 + (size_t)kPathSlots * 8;
    ws->few_frames = sm_count * (int)((227u * 1024u) / (ws->walk_smem_few + 1024));
    int per_sm = (int)((227u * 1024u) / (ws->walk_smem + 1024));
    if (per_sm > 32) per_sm = 32;
    if (per_sm < 1) per_sm = 1;
    ws->slots = sm_count * per_sm;
    ws->max_entries = kFloodMaxEntries;
    if (const char* s = getenv("CB200_K1X_MAX_ENTRIES")) { int v = atoi(s); if (v >= 1 && v <= kFloodMaxEntries) ws->max_entries = v; }   // tests: force several chunks
    ws->serial_above = 65536;                        // heaps beyond three five-level rounds pop one level at a time
    if (const char* s = getenv("CB200_K1X_SERIAL_ABOVE")) ws->serial_above = atoi(s);      // tests: 0 forces the literal pop
    ws->spill_cap = 16 + 12 * (size_t)m.num_cells;   // every decoded cell pushes at most 12 entries (4 + 8 horizon)
    cudaError_t e;
    if ((e = cudaFuncSetAttribute(k_flood_walk, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  (int)(ws->walk_smem > ws->walk_smem_few ? ws->walk_smem : ws->walk_smem_few))) != cudaSuccess) return e;
    if ((e = ws->spill.ensure(ws->spill_cap * (size_t)ws->slots)) != cudaSuccess) return e;
    if ((e = ws->prio.ensure((size_t)kMaxCells * (size_t)ws->slots)) != cudaSuccess) return e;
    std::vector<uint16_t> cinfo;
    flood_build_cinfo(m, adj_host, cinfo);
    if ((e = ws->cinfo.ensure(cinfo.size())) != cudaSuccess) return e;
    if ((e = cudaMemcpy(ws->cinfo, cinfo.data(), cinfo.size() * sizeof(uint16_t), cudaMemcpyHostToDevice)) != cudaSuccess) return e;
    return cudaSuccess;
}

bool flood_workspace_fits(const FloodWorkspace& ws, int n_frames)
{
    const int want = n_frames < ws.max_entries ? n_frames : ws.max_entries;
    return ws.list.capacity() >= (size_t)n_frames && ws.counters.capacity() >= 2 + ws.list.capacity() && want <= ws.entry_cap;
}

// grows the per-batch buffers (cudaFree synchronises, so no kernel still reads the old ones)
cudaError_t flood_workspace_ensure(const Mode& m, FloodWorkspace& ws, int n_frames)
{
    cudaError_t e;
    const size_t rw = raster_words16(m.width, m.height);
    size_t list_cap = ws.list.capacity() ? ws.list.capacity() : 256;
    while (list_cap < (size_t)n_frames) list_cap *= 2;
    if ((e = ws.list.ensure(list_cap)) != cudaSuccess) return e;
    if ((e = ws.counters.ensure(2 + list_cap)) != cudaSuccess) return e;   // 1 + one per chunk (>= 1 frame each)
    const int want = n_frames < ws.max_entries ? n_frames : ws.max_entries;
    if (want > ws.entry_cap) {
        int cap = (want + 1023) / 1024 * 1024;          // in steps of 1024 frames (185 MB)
        if (want <= 64) cap = 64; else if (want <= 256) cap = 256;
        if (cap > ws.max_entries) cap = ws.max_entries;
        ws.entry_cap = 0;
        if ((e = ws.raster.ensure(rw * (size_t)cap)) != cudaSuccess) return e;
        if ((e = cudaMemset(ws.raster, 0, rw * (size_t)cap * sizeof(uint16_t))) != cudaSuccess) return e;
        if ((e = ws.result.ensure((size_t)m.num_cells * (size_t)cap)) != cudaSuccess) return e;
        ws.entry_cap = cap;
    }
    return cudaSuccess;
}

cudaError_t flood_launch(const Mode& m, FloodWorkspace& ws, const uint8_t* d_rgb, int n_frames, bool no_fallback,
                         bool force_all, bool sharpen, const uint8_t* d_sharpen_of, uint8_t* d_cellvals, const uint32_t* d_dirty,
                         uint8_t* d_flags, CellTrace* d_trace, const CcmArg& cc, cudaStream_t st, uint32_t* keep, const uint8_t* d_present)
{
    if (n_frames <= 0) return cudaSuccess;
    cudaError_t e = flood_workspace_ensure(m, ws, n_frames);
    if (e != cudaSuccess) return e;
    const int nchunks = (n_frames + ws.entry_cap - 1) / ws.entry_cap;
    k_flood_list<<<1, 1024, 0, st>>>(d_dirty, n_frames, no_fallback ? 1 : 0, force_all ? 1 : 0, d_flags, ws.list, ws.counters, 1 + nchunks,
                                     d_present); count_launch();
    if (no_fallback) return cudaGetLastError();
    for (int c = 0; c < nchunks; ++c) {
        const int base = c * ws.entry_cap;
        const int cap = n_frames - base < ws.entry_cap ? n_frames - base : ws.entry_cap;
        const long long items = (long long)cap * ((m.height + kFastBand - 1) / kFastBand);
        const int rgrid = (int)(items < (long long)ws.sm_count * 8 ? items : (long long)ws.sm_count * 8);
        // a mixed batch runs both rasters over the chunk, each skipping the other kind's items
        if (d_sharpen_of || !sharpen) { k_flood_raster_fast<<<rgrid, kFastThreads, 0, st>>>(m, d_rgb, ws.list, ws.counters, base, cap, d_sharpen_of, ws.raster); count_launch(); }
        if (d_sharpen_of || sharpen) { k_flood_raster_fast_sharpen<<<rgrid, kFastThreads, 0, st>>>(m, d_rgb, ws.list, ws.counters, base, cap, d_sharpen_of, ws.raster); count_launch(); }
        int wgrid = cap < ws.slots ? cap : ws.slots;
        const bool few = cap <= ws.few_frames;              // at most one wave of big-heap walks: latency over occupancy
        uint32_t* result = keep ? keep + (size_t)base * m.num_cells : ws.result.get();
        k_flood_walk<<<wgrid, 32, few ? ws.walk_smem_few : ws.walk_smem, st>>>(m, ws.list, ws.counters, base, cap, ws.counters + 1 + c,
                                                      few ? ws.heap_smem_few : ws.heap_smem, ws.raster, result,
                                                      ws.spill, ws.spill_cap, ws.prio, ws.cinfo, d_trace, ws.serial_above,
                                                      1.0f / (float)(m.cells_x - 2 * m.corner), 1.0f / (float)m.cells_x); count_launch();
        long long cthreads = (long long)cap * m.num_cells;
        long long cblocks = (cthreads + 255) / 256;
        int cgrid = (int)(cblocks < (long long)ws.sm_count * 8 ? cblocks : (long long)ws.sm_count * 8);
        k_flood_colour<<<cgrid, 256, 0, st>>>(m, d_rgb, ws.list, ws.counters, base, cap, result, d_cellvals, cc); count_launch();
    }
    return cudaGetLastError();
}

// the colours of another context's walk (flood_launch with `keep`), in its chunks: the work list and its counters are `walked`'s
cudaError_t flood_colour_launch(const Mode& m, const FloodWorkspace& walked, const uint8_t* d_rgb, int n_frames, const uint32_t* kept,
                                uint8_t* d_cellvals, const CcmArg& cc, cudaStream_t st)
{
    if (n_frames <= 0) return cudaSuccess;
    const int nchunks = (n_frames + walked.entry_cap - 1) / walked.entry_cap;
    for (int c = 0; c < nchunks; ++c) {
        const int base = c * walked.entry_cap;
        const int cap = n_frames - base < walked.entry_cap ? n_frames - base : walked.entry_cap;
        long long cthreads = (long long)cap * m.num_cells;
        long long cblocks = (cthreads + 255) / 256;
        int cgrid = (int)(cblocks < (long long)walked.sm_count * 8 ? cblocks : (long long)walked.sm_count * 8);
        k_flood_colour<<<cgrid, 256, 0, st>>>(m, d_rgb, walked.list, walked.counters, base, cap, kept + (size_t)base * m.num_cells, d_cellvals, cc);
        count_launch();
    }
    return cudaGetLastError();
}

}  // namespace cb200
