// k1_decode.cu -- K1: fused preprocess + average-hash + colour kernel for clean (drift-0) frames, sm_90a.
//
// Replaces, for one RGB8 frame resident in HBM (reference file:line relative to /root/reference/):
//   P1  preprocessSymbolGrid            src/lib/cimb_translator/CimbReader.cpp:30-46  (cvtColor + adaptiveThreshold(5, C=0))
//   P5  fuzzy_ahash<8>(bitmatrix)       src/lib/image_hash/average_hash.h:63-75, ahash_result.h:70-106
//   P6  CimbDecoder::get_best_symbol    src/lib/cimb_translator/CimbDecoder.cpp:101-132
//   P8  Cell::mean_rgb_continuous       src/lib/cimb_translator/Cell.h:30-62 (inner 6x6, CimbDecoder.cpp:202-209)
//   P9  CimbDecoder::get_best_color     src/lib/cimb_translator/CimbDecoder.cpp:168-200
// for every cell at drift (0,0).  The reference walks cells serially in heap order and lets drift propagate
// (FloodDecodePositions.cpp:49-134); that walk provably degenerates to this embarrassingly parallel pass when the
// centre hash wins for every cell (SURVEY.md appendix A.8).  A cell where it does not sets bit 7 of its result
// byte and the frame's dirty flag; such frames are re-done by the exact flood-walk kernel (k1x_flood.cu).
//
// Data flow per CTA (128 threads, thread 0 doubles as the TMA producer; 4 CTAs/SM):
//   HBM --cp.async.bulk (TMA, one copy of 9 full-width rows = 27 KB per stage, one mbarrier per stage)--> smem
//   phase A: 8 px/thread: gray = (19596R+38470G+7470B+32768)>>16 via 2x IDP.2A per px, packed 2x16 bit
//   phase B: separable 5x5 box sum in packed-16 SIMD (5 IADD3 + 4 PRMT per 8 px), rolling vertical sum in
//            registers, threshold 25*g > sum+12 as ONE IMAD per pixel pair, 1-bit raster row -> smem
//   phase C: one thread per cell: 8x8 hash by funnel shifts from the raster, perfect-hash exact match against
//            the 16-tile dictionary (full 5/9-way popcount search only when inexact), 6x6 RGB mean via IDP.4A
//            from the staged raw rows, colour classification, one result byte per cell -> HBM
// Every HBM byte of the frame is read exactly once (plus 4 warm-up rows per band).
#include "cb200_common.cuh"
#include "k1_decode.cuh"
#include "ccm.cuh"

namespace cb200 {

constexpr int kK1Threads = 128;            // 128 threads x 8 px = one full 1024-px row
constexpr int kK1CtasPerSm = 4;            // resident CTAs per SM without sharpen: caps the registers at 128 (5 -> 96)
constexpr int kStageRows = 9;              // raw rows per cell row (stage)
constexpr int kMaxW = 1024;
constexpr int kRastPitch = 144;            // bytes per raster row: 1024 bits + funnel-shift overread pad
constexpr int kRastWords = kRastPitch / 4;

struct __align__(128) K1Smem {
    uint8_t ring[kStageRows * kMaxW * 3];     // the raw RGB rows of ONE stage, filled by TMA (row r at r * row_bytes)
    uint32_t halo[2][kStageRows][kK1Threads]; // per row and thread: gray of px 0,1,6,7 of its eight (what the neighbours' box sums need)
    uint32_t raster[2][10][kRastWords];       // 1-bit threshold rows of the current / previous stage
    uint4 tiles_by_slot[16];                  // (L_lo, L_hi, symbol, 0), indexed by the perfect hash
    uint2 tiles_by_sym[16];                   // (L_lo, L_hi), indexed by symbol (tie-break order of the full search)
    float adjust[256];                        // copy of c_adjust: indexed per lane, so not read through the constant cache
    unsigned long long full_bar[2];
    float ccm[12];                            // CCM variant only: the current frame's 3x3 colour correction matrix
};

__constant__ float c_adjust[256];             // (float)(255.0 / (double)d), d = max-min (CimbDecoder.cpp:185)
__constant__ unsigned long long c_tiles_L[16]; // tile dictionary, bit (8r+c) = pixel(r,c)  (bit-reversed reference hash)

// ---------------------------------------------------------------------------------------------- PTX helpers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned long long* bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(unsigned long long* bar, uint32_t parity)
{
    uint32_t ok;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.b32 %0, 1, 0, p;\n"
        "}\n" : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, uint32_t parity)
{
    while (!mbar_try_wait(bar, parity)) {}
}
// TMA 1-D bulk copy global -> shared, completion signalled on an mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void tma_bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, unsigned long long* bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void consumer_sync() { __syncthreads(); }

// ---------------------------------------------------------------------------------------------- colour
// P9 get_best_color with integer inputs (no CCM): float32 arithmetic restated op for op (CimbDecoder.cpp:27-36, :168-200)
template <int NC>
__device__ __forceinline__ uint32_t best_color(const float* adjust_tab, const Mode& m, uint32_t ri, uint32_t gi, uint32_t bi)
{
    // max/min with the floors 1 and 48 on integers (exact: the inputs are integer means); if (min >= max) min = 0
    uint32_t mxi = max(max(ri, gi), max(bi, 1u));
    uint32_t mni = min(min(ri, gi), min(bi, 48u));
    if (mni >= mxi) mni = 0;
    const float adjust = adjust_tab[mxi - mni];
    const float mn = (float)mni;
    const float hi_thr = __fsub_rn(245.0f, mn);
    // fix_single_color: c -= down; c *= adjustUp; if (c > 245 - down) c = 255; (c < 0 cannot happen: down <= c); (uchar)c
    float fr = __fmul_rn((float)(ri - mni), adjust), fg = __fmul_rn((float)(gi - mni), adjust), fb = __fmul_rn((float)(bi - mni), adjust);
    int cr = (fr > hi_thr) ? 255 : (int)__float2uint_rz(fr);
    int cg = (fg > hi_thr) ? 255 : (int)__float2uint_rz(fg);
    int cb = (fb > hi_thr) ? 255 : (int)__float2uint_rz(fb);
    const int a0 = cr - cg, a1 = cg - cb;
    // color_diff = sum_j (a_j - p_ij)^2 = |a|^2 + |p_i|^2 - 2 a.p_i, and a2 = -a0 - a1: the first term is common, so the
    // strict-'<' argmin over i of pal_c[i] - (a0 pal_u[i] + a1 pal_w[i]) is the reference's argmin (same ties)
    uint32_t best = 0;
    int best_d = 0x7fffffff;
#pragma unroll
    for (int i = 0; i < NC; ++i) {
        const int d = m.pal_c[i] - (a0 * m.pal_u[i] + a1 * m.pal_w[i]);
        if (d < best_d) { best_d = d; best = (uint32_t)i; }
    }
    return best;
}

// sum of R,G,B over 6 consecutive pixels starting at pixel x of one staged raw row (P8, one row of the 6x6)
__device__ __forceinline__ void rgb_row6(const uint8_t* row, int x, uint32_t& R, uint32_t& G, uint32_t& B)
{
    uint32_t bo = 3u * (uint32_t)x;
    const uint32_t* w = reinterpret_cast<const uint32_t*>(row) + (bo >> 2);
    uint32_t sh = (bo & 3u) * 8u;
    uint32_t w0 = w[0], w1 = w[1], w2 = w[2], w3 = w[3], w4 = w[4], w5 = w[5];
    // realign so that a0 starts at the first pixel's R byte
    uint32_t a0 = __funnelshift_r(w0, w1, sh), a1 = __funnelshift_r(w1, w2, sh), a2 = __funnelshift_r(w2, w3, sh);
    uint32_t a3 = __funnelshift_r(w3, w4, sh), a4 = __funnelshift_r(w4, w5, sh);
    // a0 = R0 G0 B0 R1 | a1 = G1 B1 R2 G2 | a2 = B2 R3 G3 B3 | a3 = R4 G4 B4 R5 | a4 = G5 B5 x x
    R = __dp4a(a0, 0x01000001u, R); R = __dp4a(a1, 0x00010000u, R); R = __dp4a(a2, 0x00000100u, R); R = __dp4a(a3, 0x01000001u, R);
    G = __dp4a(a0, 0x00000100u, G); G = __dp4a(a1, 0x01000001u, G); G = __dp4a(a2, 0x00010000u, G); G = __dp4a(a3, 0x00000100u, G);
    G = __dp4a(a4, 0x00000001u, G);
    B = __dp4a(a0, 0x00010000u, B); B = __dp4a(a1, 0x00000100u, B); B = __dp4a(a2, 0x01000001u, B); B = __dp4a(a3, 0x00010000u, B);
    B = __dp4a(a4, 0x00000100u, B);
}

// ---------------------------------------------------------------------------------------------- symbols
// 32 raster bits starting at pixel `o` of window row `r`
__device__ __forceinline__ uint32_t raster_bits(const K1Smem& s, uint32_t rbuf, int r, uint32_t o)
{
    uint32_t idx = o >> 5;
    return __funnelshift_r(s.raster[rbuf][r][idx], s.raster[rbuf][r][idx + 1], o & 31u);
}

// full P5+P6 search at drift 0 for ONE cell, done by the whole warp: FAST = ids {4,5,7,3,1}, ALL adds {8,0,2,6}
// (ahash_result.h:26), tiles 0..15; the reference keeps the first minimum in that iteration order (strict '<'; its early
// return on distance 0 cannot change the result), which is the minimum of key = dist<<8 | order<<4 | tile.
// o = pixel x of window column 0.  Every lane returns the same key.
__device__ __forceinline__ uint32_t warp_symbol_search(const K1Smem& s, uint32_t rbuf, uint32_t o, bool all, int lane)
{
    // lanes 0..9 fetch the ten 10-bit window rows, every lane gets all of them
    const uint32_t myrow = raster_bits(s, rbuf, lane < 10 ? lane : 0, o) & 0x3FFu;
    uint32_t win[10];
#pragma unroll
    for (int r = 0; r < 10; ++r) win[r] = __shfl_sync(0xffffffffu, myrow, r);
    // lane q < 9 extracts the hash at drift id order[q]: columns c0..c0+7 of the ten rows form an 80-bit string, the hash
    // at row offset r0 is bits [8 r0, 8 r0 + 64) of it (ahash_result::extract, ahash_result.h:70-106)
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
    const uint2 tl = s.tiles_by_sym[lane & 15];
    const int nq = all ? 9 : 5;
    uint32_t best_key = 0xFFFFFFFFu;
#pragma unroll
    for (int it = 0; it < 5; ++it) {
        if (it >= 3 && !all) break;                       // warp-uniform
        const int q = 2 * it + (lane >> 4);
        const uint32_t lo = __shfl_sync(0xffffffffu, hlo, q & 15), hi = __shfl_sync(0xffffffffu, hhi, q & 15);
        const uint32_t d = (uint32_t)(__popc(lo ^ tl.x) + __popc(hi ^ tl.y));
        const uint32_t key = q < nq ? ((d << 8) | ((uint32_t)q << 4) | (uint32_t)(lane & 15)) : 0xFFFFFFFFu;
        best_key = key < best_key ? key : best_key;
    }
    return __reduce_min_sync(0xffffffffu, best_key);
}

// the same search done by ONE thread for its own cell (used by the sharpen variant, where most cells are inexact): identical
// keys, so identical results.  o = pixel x of window column 0.
__device__ __forceinline__ uint32_t thread_symbol_search(const K1Smem& s, uint32_t rbuf, uint32_t o, bool all)
{
    uint32_t win[10];
#pragma unroll
    for (int r = 0; r < 10; ++r) win[r] = raster_bits(s, rbuf, r, o) & 0x3FFu;
    uint32_t best_key = 0xFFFFFFFFu;
#pragma unroll
    for (int q = 0; q < 9; ++q) {
        if (q >= 5 && !all) break;
        const int r0 = (int)((0x200201211ULL >> (4 * q)) & 3u), c0 = (int)((0x020210121ULL >> (4 * q)) & 3u);   // id / 3, id % 3
        uint32_t b[8];
#pragma unroll
        for (int r = 0; r < 8; ++r) b[r] = (win[r0 + r] >> c0) & 0xFFu;
        const uint32_t lo = b[0] | (b[1] << 8) | (b[2] << 16) | (b[3] << 24);
        const uint32_t hi = b[4] | (b[5] << 8) | (b[6] << 16) | (b[7] << 24);
#pragma unroll 4
        for (int tile = 0; tile < 16; ++tile) {
            const uint2 tl = s.tiles_by_sym[tile];
            const uint32_t d = (uint32_t)(__popc(lo ^ tl.x) + __popc(hi ^ tl.y));
            const uint32_t key = (d << 8) | ((uint32_t)q << 4) | (uint32_t)tile;
            best_key = key < best_key ? key : best_key;
        }
    }
    return best_key;
}

// ---------------------------------------------------------------------------------------------- the kernel
// 128 threads (8 px each), 4 CTAs/SM.  On an H100 it reads frames at 0.90 of the 3.35 TB/s data-sheet HBM3 bandwidth.  Shared
// memory per CTA is 41 KB -- the raw rows of exactly one stage (every raw byte is consumed before the stage barrier, so the next
// stage lands in the same place while the box sums and the symbols run) plus a 9 KB exchange array for the box-filter halo
// words -- which would admit five CTAs per SM; five CTAs would need 96 registers, and the scheduler needs 128 to keep a stage's
// loads in flight, so the cap is 128.
// One barrier per stage.  Iteration for stage `it` (cell row k, raw rows [y_k+2, y_k+10]):
//   wait full[it&1]
//   A(k):   gray of the thread's 8 px in each of the 9 rows -> packed pairs in registers; one halo word E_r per row
//           (bytes g0,g1,g6,g7) goes to a small double-buffered exchange array
//   col(k): 6x6 RGB means of cell row k straight from the staged raw rows (drift 0: positions are static), and the
//           first row of cell row k+1's window (its other rows come with the next stage)
//   ---- __syncthreads ----   nobody reads the raw rows any more: thread 0 issues the TMA of stage it+1 into the same
//                             27 KB, it lands while B and S run
//   B(k):   box sums, threshold -> raster[it&1]
//   S(k-1): symbols of cell row k-1 from raster[(it-1)&1] (complete since this barrier) + col(k-1) -> result bytes
// CCM: the colour classifier runs the reference's float path with a 3x3 colour correction matrix (ccm.cuh) instead of the
// integer restatement; the matrix of the frame is staged in shared memory when a CTA starts on it.
// CM = 0: integer classifier; 1: CCM classifier; 2: no decision, the cell's mean colour is stored for the fitted-CCM pass
// SH: needs_sharpen preprocessing (CimbReader.cpp:17-40): gray -> filter2D [0 -1 0; -1 4.5 -1; 0 -1 0] -> adaptiveThreshold
// with block 7.  The stage then starts two rows further down (raw rows [y_k+4, y_k+12]), has a second barrier (the
// sharpened rows' halo pixels come from the neighbours, whose sharpened values need THEIR neighbours' gray first) and keeps
// seven rows of horizontal sums; three CTAs per SM at up to 168 registers.  Schedule per stage:
//   A(k), col(k)  ---- barrier 1 (TMA of the next stage) ----  sharpen: S rows a0-1 .. a0+7 from gray rows a0-2 .. a0+8
//   (two carried), their halo words (s0,s1,s2 | s5,s6,s7) -> smem  ---- barrier 2 ----  7x7 box sums, threshold rows
//   a0-4 .. a0+4 = y_k .. y_k+8, S(k-1).  Frame borders are never reached: the cell windows stay 3 pixels inside.
// A lane-level numpy model of exactly this schedule is checked against the oracle in tests/test_k1_sharpen_model.py.
// frame_list: NULL = the n_frames frames of the batch; else the batch indices of the n_frames frames this launch decodes (one
// kind of a batch that mixes sharpened and plain frames).  Every output stays batch-indexed.
// DC: the list's length is only known on the device (a selection built there, k_select in api.cu): n_frames, bands and the
// list's first entry come from sched[0..2] instead, and the launch is the persistent grid whatever the count.
template <int NC, bool G1024, int CM, bool SH, bool DC>
__global__ void __launch_bounds__(kK1Threads, SH ? 3 : kK1CtasPerSm)
k1_decode_kernel(const Mode mm, const uint8_t* __restrict__ rgb, const uint32_t* __restrict__ frame_list, int n_frames, int bands,
                 uint8_t* __restrict__ cellvals, uint32_t* __restrict__ dirty_flags, const CcmArg cc, const int* __restrict__ sched)
{
    if constexpr (DC) { n_frames = __ldg(sched); bands = __ldg(sched + 1); frame_list += __ldg(sched + 2); }
    // G1024: the 1024x1024 / 112x112-cell geometry of modes B, 4C and 8C as compile-time constants (GridConf.h:121-141);
    // the other modes (Bm 1024x720, Bu 736x637) take every dimension from the Mode struct
    struct Geo {
        const Mode& q;
        __device__ __forceinline__ int width() const { return G1024 ? 1024 : q.width; }
        __device__ __forceinline__ int height() const { return G1024 ? 1024 : q.height; }
        __device__ __forceinline__ int cells_x() const { return G1024 ? 112 : q.cells_x; }
        __device__ __forceinline__ int cells_y() const { return G1024 ? 112 : q.cells_y; }
        __device__ __forceinline__ int corner() const { return G1024 ? 6 : q.corner; }
        __device__ __forceinline__ int cell_offset() const { return G1024 ? 8 : q.cell_offset; }
        __device__ __forceinline__ int num_cells() const { return G1024 ? 12400 : q.num_cells; }
        __device__ __forceinline__ int top_cells() const { return G1024 ? 600 : q.top_cells; }
        __device__ __forceinline__ int mid_cells() const { return G1024 ? 11200 : q.mid_cells; }
        __device__ __forceinline__ int symbol_bits() const { return G1024 ? 4 : q.symbol_bits; }
        __device__ __forceinline__ void row_geom(int k, int& base, int& ncols, int& x0) const
        {
            const int narrow = cells_x() - 2 * corner();
            if (k < corner()) { base = k * narrow; ncols = narrow; x0 = cell_offset() + kSpacing * corner(); }
            else if (k < cells_y() - corner()) { base = top_cells() + (k - corner()) * cells_x(); ncols = cells_x(); x0 = cell_offset(); }
            else { base = top_cells() + mid_cells() + (k - (cells_y() - corner())) * narrow; ncols = narrow; x0 = cell_offset() + kSpacing * corner(); }
        }
    };
    const Geo m{mm};
    extern __shared__ __align__(128) uint8_t smem_raw[];
    K1Smem& s = *reinterpret_cast<K1Smem*>(smem_raw);
    const int tid = threadIdx.x;
    const int W = m.width();
    const uint32_t row_bytes = (uint32_t)W * 3u;
    const uint32_t stage_bytes = row_bytes * kStageRows;
    const size_t frame_bytes = (size_t)row_bytes * (size_t)m.height();
    const int n_units = n_frames * bands;

    if (tid == 0) {
        mbar_init(&s.full_bar[0], 1); mbar_init(&s.full_bar[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    if (tid < 16) {
        unsigned long long L = c_tiles_L[tid];
        uint32_t lo = (uint32_t)L, hi = (uint32_t)(L >> 32);
        s.tiles_by_sym[tid] = make_uint2(lo, hi);
        s.tiles_by_slot[(lo * mm.hash_mul) >> 28] = make_uint4(lo, hi, (uint32_t)tid, 0u);
    }
    for (int i = tid; i < 256; i += kK1Threads) s.adjust[i] = c_adjust[i];
    __syncthreads();

    const int t = tid;                          // owns pixels 8t .. 8t+7 of every row, and cell t of every cell row
    const int nthr_px = W / 8;
    const bool px_active = t < nthr_px;
    const int tl = (t == 0) ? 0 : t - 1, tr = (t + 1 < nthr_px) ? t + 1 : t;   // halo sources (frame borders are never used)
    const uint32_t cRG = 19596u | (38470u << 16), cB0 = 7470u, c0R = 19596u << 16, cGB = 38470u | (7470u << 16);
    const uint32_t kBias = SH ? 0x7FE77FE7u : 0x7FF37FF3u;   // per half: 0x8000 - 13 (block 5), 0x8000 - 25 (block 7)
    constexpr int kBox = SH ? 7 : 5;            // adaptiveThreshold block size
    constexpr int kFirstRow = SH ? 4 : 2;       // first raw row of a stage relative to the cell row's y
    uint32_t* const sh_hi = reinterpret_cast<uint32_t*>(smem_raw + sizeof(K1Smem));   // SH only: [kStageRows][kK1Threads], (s5,s6,s7) halo words
    const int narrow = m.cells_x() - 2 * m.corner(), last_cell = m.num_cells() - 1, first_mid = m.top_cells();

    // ---- stage stream of this CTA: (unit u, cell row k = k0-1 .. k1-1).  Thread 0 is the TMA producer.
    struct Cursor { int u, k, kend; const uint8_t* src; bool valid; };
    auto cursor_unit = [&](Cursor& c) {          // position at the first (virtual) stage of unit c.u
        c.valid = c.u < n_units;
        if (!c.valid) return;
        const int e = c.u / bands, b = c.u - e * bands;
        const int f = frame_list ? (int)frame_list[e] : e;
        c.k = (m.cells_y() * b) / bands - 1;
        c.kend = (m.cells_y() * (b + 1)) / bands;
        c.src = rgb + (size_t)f * frame_bytes + (size_t)(m.cell_offset() + kSpacing * c.k + kFirstRow) * row_bytes;
    };
    auto cursor_next = [&](Cursor& c) {
        if (++c.k < c.kend) { c.src += stage_bytes; return; }   // consecutive stages are contiguous in the frame
        c.u += gridDim.x;
        cursor_unit(c);
    };
    // the nine source rows of a stage are contiguous in the frame: one bulk copy into the (single-stage) ring
    auto issue_stage = [&](const Cursor& c, uint32_t i) {
        unsigned long long* bar = &s.full_bar[i & 1u];
        mbar_expect_tx(bar, stage_bytes);
        tma_bulk_g2s(s.ring, c.src, stage_bytes, bar);
    };
    Cursor nxt;                                   // next stage to load into shared memory (thread 0's)
    nxt.u = blockIdx.x; nxt.valid = false;
    if (tid == 0) {
        cursor_unit(nxt);
        if (nxt.valid) { issue_stage(nxt, 0u); cursor_next(nxt); }
    }

    // symbol stage for one cell row from a finished raster (P5/P6 at drift 0) + the colour decided earlier.
    // Exact dictionary hits are resolved per thread through the perfect hash; the rare inexact cells (threshold edge
    // artefacts, ~1 % of a clean frame) are searched one at a time by the whole warp.
    auto symbol_stage = [&](int k, uint32_t rbuf, uint32_t col, uint8_t* out, bool& any_dirty) {
        int base, ncols, x0;
        m.row_geom(k, base, ncols, x0);
        const bool active = t < ncols;
        const uint32_t (*rast)[kRastWords] = s.raster[rbuf];
        const uint32_t o = (uint32_t)(x0 + kSpacing * t);     // window col 1 == pixel x
        const int cell = base + t;
        uint32_t sym = 0, dirty = 0;
        bool exact = true;
        if (active) {
            uint32_t fr[8];
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                const uint32_t idx = o >> 5, sh = o & 31u;
                fr[q] = __funnelshift_r(rast[1 + q][idx], rast[1 + q][idx + 1], sh);      // byte 0 = hash row q
            }
            const uint32_t lo = __byte_perm(__byte_perm(fr[0], fr[1], 0x0040), __byte_perm(fr[2], fr[3], 0x0040), 0x5410);
            const uint32_t hi = __byte_perm(__byte_perm(fr[4], fr[5], 0x0040), __byte_perm(fr[6], fr[7], 0x0040), 0x5410);
            uint4 te = s.tiles_by_slot[(lo * mm.hash_mul) >> 28];
            exact = (te.x == lo) & (te.y == hi);
            sym = te.z;
        }
        uint32_t need = __ballot_sync(0xffffffffu, !exact);
        const int lane = tid & 31;
        if constexpr (SH) {
            // a sharpened raster rarely reproduces a dictionary tile bit for bit (five cells in six of a clean frame are
            // inexact), so the one-cell-at-a-time warp search would dominate: with more than two inexact cells in the warp
            // every thread searches its own cell instead (same keys, same minimum)
            if (__popc(need) > 2) {
                if (!exact) {
                    const bool seed = (cell == 0) | (cell == narrow - 1) | (cell == last_cell) | (cell == last_cell - (narrow - 1)) |
                                      (cell == first_mid) | (cell == first_mid + m.cells_x() - 1) | (cell == last_cell - first_mid) |
                                      (cell == last_cell - (first_mid + m.cells_x() - 1));
                    const uint32_t key = thread_symbol_search(s, rbuf, o - 1u, seed);
                    sym = key & 15u;
                    if (((key >> 4) & 15u) != 0u) { dirty = kCellDirty; any_dirty = true; }
                }
                need = 0;
            }
        }
        while (need) {
            const int leader = __ffs(need) - 1;
            need &= need - 1;
            const uint32_t lo_ = __shfl_sync(0xffffffffu, o, leader);
            const int lcell = __shfl_sync(0xffffffffu, cell, leader);
            const bool seed = (lcell == 0) | (lcell == narrow - 1) | (lcell == last_cell) | (lcell == last_cell - (narrow - 1)) |
                              (lcell == first_mid) | (lcell == first_mid + m.cells_x() - 1) | (lcell == last_cell - first_mid) |
                              (lcell == last_cell - (first_mid + m.cells_x() - 1));
            const uint32_t key = warp_symbol_search(s, rbuf, lo_ - 1u, seed, lane);
            if (lane == leader) {
                sym = key & 15u;
                if (((key >> 4) & 15u) != 0u) { dirty = kCellDirty; any_dirty = true; }   // order index 0 == centre hash (id 4)
            }
        }
        if (active) out[cell] = (uint8_t)(sym | (col << m.symbol_bits()) | dirty);
    };

    uint32_t it = 0;
    for (int u = blockIdx.x; u < n_units; u += gridDim.x) {
        const int e = u / bands, b = u - e * bands;
        const int f = frame_list ? (int)frame_list[e] : e;
        int k0 = (m.cells_y() * b) / bands, k1 = (m.cells_y() * (b + 1)) / bands;
        uint8_t* out = cellvals + (size_t)f * (size_t)m.num_cells();
        if (CM == 1) {  // nobody reads s.ccm between the last colour pass of the previous unit and this barrier
            if (tid < 9) s.ccm[tid] = cc.per_frame ? cc.per_frame[(size_t)f * 9 + tid] : cc.m[tid];
            __syncthreads();
        }

        uint32_t hprev[kBox][4], Pprev[2][4], nV[4];
        uint32_t Qprev[3][4], prevL = 0, prevR = 0;    // SH: the last three sharpened rows, the halo words of the last gray row
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            nV[j] = kBias;
#pragma unroll
            for (int i = 0; i < kBox; ++i) hprev[i][j] = 0;
            Pprev[0][j] = Pprev[1][j] = 0;
            Qprev[0][j] = Qprev[1][j] = Qprev[2][j] = 0;
        }
        uint32_t carryR = 0, carryG = 0, carryB = 0;   // colour sums of row y+1 of the upcoming cell row
        uint32_t col_prev = 0;                         // colour of this thread's cell in the row whose symbols are pending
        bool any_dirty = false;

        for (int k = k0 - 1; k < k1; ++k, ++it) {
            const uint32_t buf = it & 1u, ph = (it >> 1) & 1u;
            uint8_t* const ub[3] = {s.ring, s.ring + 3u * row_bytes, s.ring + 6u * row_bytes};   // stage rows 0-2, 3-5, 6-8
            mbar_wait(&s.full_bar[buf], ph);

            // ---------------- A(k): gray, packed pairs P[r][j] = (g[j], g[j+4]); halo word E_r = (g0,g1,g6,g7)
            uint32_t P[kStageRows][4];
            {   // (threads beyond the row width of the narrower modes compute on in-bounds garbage; their stores are masked)
                uint32_t E[kStageRows];
#pragma unroll
                for (int r = 0; r < kStageRows; ++r) {
                    const uint2* rp = reinterpret_cast<const uint2*>(ub[r / 3] + (uint32_t)(r % 3) * row_bytes) + 3 * t;
                    uint2 q0 = rp[0], q1 = rp[1], q2 = rp[2];
                    uint32_t n0, n1, n2, n3, n4, n5, n6, n7;
                    n0 = __dp2a_lo(cRG, q0.x, 32768u); n0 = __dp2a_hi(cB0, q0.x, n0);
                    n1 = __dp2a_hi(c0R, q0.x, 32768u); n1 = __dp2a_lo(cGB, q0.y, n1);
                    n2 = __dp2a_hi(cRG, q0.y, 32768u); n2 = __dp2a_lo(cB0, q1.x, n2);
                    n3 = __dp2a_lo(c0R, q1.x, 32768u); n3 = __dp2a_hi(cGB, q1.x, n3);
                    n4 = __dp2a_lo(cRG, q1.y, 32768u); n4 = __dp2a_hi(cB0, q1.y, n4);
                    n5 = __dp2a_hi(c0R, q1.y, 32768u); n5 = __dp2a_lo(cGB, q2.x, n5);
                    n6 = __dp2a_hi(cRG, q2.x, 32768u); n6 = __dp2a_lo(cB0, q2.y, n6);
                    n7 = __dp2a_lo(c0R, q2.y, 32768u); n7 = __dp2a_hi(cGB, q2.y, n7);
                    P[r][0] = __byte_perm(n0, n4, 0x7632); P[r][1] = __byte_perm(n1, n5, 0x7632);
                    P[r][2] = __byte_perm(n2, n6, 0x7632); P[r][3] = __byte_perm(n3, n7, 0x7632);
                    // gray is byte 2 of each numerator
                    E[r] = __byte_perm(__byte_perm(n0, n1, 0x0062), __byte_perm(n6, n7, 0x6200), 0x7610);
                }
                // E_0..E_8 go to the halo buffer of this stage (double buffered: a warp may start A(k+1) while another is still in B(k))
#pragma unroll
                for (int r = 0; r < kStageRows; ++r) s.halo[SH ? 0u : buf][r][t] = E[r];   // (SH: single buffer, two barriers per stage)
            }

            // ---------------- col(k): inner 6x6 = rows y+1..y+6 (row y+1 carried from the previous stage), px x+1..x+6
            uint32_t col = 0;
            {
                int base, ncols, x0;
                if (k >= k0) {
                    m.row_geom(k, base, ncols, x0);
                    if (t < ncols && NC > 1) {
                        const int x = x0 + kSpacing * t + 1;
                        uint32_t R = carryR, G = carryG, B = carryB;
                        rgb_row6(ub[0], x, R, G, B);
                        rgb_row6(ub[0] + row_bytes, x, R, G, B);
                        rgb_row6(ub[0] + 2u * row_bytes, x, R, G, B);
                        if (!SH) {                     // SH: rows y+1..y+3 were carried, rows y+4..y+6 are stage rows 0..2
                            rgb_row6(ub[1], x, R, G, B);
                            rgb_row6(ub[1] + row_bytes, x, R, G, B);
                        }
                        if (CM == 2) cc.means[(size_t)f * (size_t)m.num_cells() + (size_t)(base + t)] = (R / 36u) | ((G / 36u) << 8) | ((B / 36u) << 16);
                        else col = CM == 1 ? best_color_ccm<NC>(s.ccm, mm, R / 36u, G / 36u, B / 36u) : best_color<NC>(s.adjust, mm, R / 36u, G / 36u, B / 36u);
                    }
                }
                carryR = carryG = carryB = 0;          // colour carry for cell row k+1: its row y'+1 = last row of this stage
                if (k + 1 < k1) {
                    m.row_geom(k + 1, base, ncols, x0);
                    if (t < ncols) {
                        if (SH) {                      // its rows y'+1..y'+3 = stage rows 6..8
                            rgb_row6(ub[2], x0 + kSpacing * t + 1, carryR, carryG, carryB);
                            rgb_row6(ub[2] + row_bytes, x0 + kSpacing * t + 1, carryR, carryG, carryB);
                        }
                        rgb_row6(ub[2] + 2u * row_bytes, x0 + kSpacing * t + 1, carryR, carryG, carryB);
                    }
                }
            }
            __syncthreads();
            // the raw rows are dead now (gray is in registers, the colour sums are taken): the next stage may overwrite them
            if (tid == 0 && nxt.valid) { issue_stage(nxt, it + 1u); cursor_next(nxt); }

            // ---------------- B(k): 5x5 box sum, threshold, raster rows 1..9 (row 0 = row 9 of the previous stage)
            if constexpr (!SH) {
                uint8_t* rast8 = reinterpret_cast<uint8_t*>(&s.raster[buf][0][0]);
                const uint8_t* prev8 = reinterpret_cast<const uint8_t*>(&s.raster[buf ^ 1u][0][0]);
                if (px_active) rast8[t] = prev8[9 * kRastPitch + t];
                uint32_t h[kStageRows][4];
#pragma unroll
                for (int r = 0; r < kStageRows; ++r) {
                    const uint32_t lE = s.halo[buf][r][tl], rE = s.halo[buf][r][tr];
                    uint32_t Pm2 = __byte_perm(lE, P[r][2], 0x5452), Pm1 = __byte_perm(lE, P[r][3], 0x5453);
                    uint32_t P4 = __byte_perm(P[r][0], rE, 0x3432), P5 = __byte_perm(P[r][1], rE, 0x3532);
                    h[r][0] = Pm2 + Pm1 + P[r][0] + P[r][1] + P[r][2];
                    h[r][1] = h[r][0] - Pm2 + P[r][3];
                    h[r][2] = h[r][1] - Pm1 + P4;
                    h[r][3] = h[r][2] - P[r][0] + P5;
                    uint32_t tj[4];
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        uint32_t hold = (r < 5) ? hprev[r][j] : h[r - 5][j];
                        nV[j] = nV[j] + hold - h[r][j];
                        uint32_t Pc = (r < 2) ? Pprev[r][j] : P[r - 2][j];
                        tj[j] = 25u * Pc + nV[j];             // bit15 / bit31 = (25 g > boxsum + 12)
                    }
                    // the eight decisions are bit 7 of bytes 1 and 3 of tj[0..3]: px 0,4 | 1,5 | 2,6 | 3,7.  Two byte permutes put
                    // them into two words (px 0,4,1,5 and px 2,6,3,7 at bits 7,15,23,31); the high half of a 32x32 product with a
                    // constant that has one bit per source (bit 32 + k - s for source bit s -> result bit k) moves all four to
                    // their places at once -- every partial product lands on its own bit, so nothing carries, and the strays
                    // fall outside bits 32..39.  Only the low byte of the sum is stored.
                    const uint32_t dx = __byte_perm(tj[0], tj[1], 0x7531) & 0x80808080u;
                    const uint32_t dy = __byte_perm(tj[2], tj[3], 0x7531) & 0x80808080u;
                    const uint32_t byte = __umulhi(dx, 0x02200440u) + __umulhi(dy, 0x08801100u);
                    if (px_active) rast8[(r + 1) * kRastPitch + t] = (uint8_t)byte;
                }
#pragma unroll
                for (int j = 0; j < 4; ++j) {
#pragma unroll
                    for (int i = 0; i < 5; ++i) hprev[i][j] = h[4 + i][j];
                    Pprev[0][j] = P[7][j]; Pprev[1][j] = P[8][j];
                }
            } else {
                // ---------------- sharpen: S row i = absolute row a0-1+i, Q[i][j] = (s[j], s[j+4]) like P.  Per half:
                // twice = 9 c - 2 (up + down + left + right) = 2 x the float result; cvRound (half to even) and saturate_cast:
                // tc = clamp(twice, 0, 510), s = (tc + ((tc >> 1) & 1)) >> 1
                uint32_t Q[kStageRows][4];
#pragma unroll
                for (int i = 0; i < kStageRows; ++i) {
                    const uint32_t* Pc = (i == 0) ? Pprev[1] : P[i > 0 ? i - 1 : 0];
                    const uint32_t* Pu = (i == 0) ? Pprev[0] : ((i == 1) ? Pprev[1] : P[i > 1 ? i - 2 : 0]);
                    const uint32_t* Pd = P[i];
                    const uint32_t lE = (i == 0) ? prevL : s.halo[0][i > 0 ? i - 1 : 0][tl];
                    const uint32_t rE = (i == 0) ? prevR : s.halo[0][i > 0 ? i - 1 : 0][tr];
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const uint32_t Pl = (j == 0) ? __byte_perm(lE, Pc[3], 0x5453) : Pc[j > 0 ? j - 1 : 0];   // (gL7, g3)
                        const uint32_t Pr = (j == 3) ? __byte_perm(Pc[0], rE, 0x3432) : Pc[j < 3 ? j + 1 : 3];   // (g4, gR0)
                        const uint32_t nbr = Pu[j] + Pd[j] + Pl + Pr;
                        const uint32_t T = 9u * Pc[j] + (0x08000800u - 2u * nbr);                  // twice + 2048 per half
                        const uint32_t tc = __vminu2(__vmaxu2(T, 0x08000800u), 0x09FE09FEu) - 0x08000800u;
                        Q[i][j] = ((tc + ((tc >> 1) & 0x00010001u)) >> 1) & 0x00FF00FFu;
                    }
                    s.halo[1][i][t] = __byte_perm(__byte_perm(Q[i][0], Q[i][1], 0x0040), Q[i][2], 0x0410);   // bytes (s0, s1, s2, .)
                    sh_hi[i * kK1Threads + t] = __byte_perm(__byte_perm(Q[i][1], Q[i][2], 0x0062), Q[i][3], 0x0610);   // (s5, s6, s7, .)
                }
                prevL = s.halo[0][kStageRows - 1][tl]; prevR = s.halo[0][kStageRows - 1][tr];
                __syncthreads();
                // ---------------- B(k): 7x7 box sum of the sharpened rows, threshold 49 s > sum + 24, raster rows 1..9
                uint8_t* rast8 = reinterpret_cast<uint8_t*>(&s.raster[buf][0][0]);
                const uint8_t* prev8 = reinterpret_cast<const uint8_t*>(&s.raster[buf ^ 1u][0][0]);
                if (px_active) rast8[t] = prev8[9 * kRastPitch + t];
                uint32_t h[kStageRows][4];
#pragma unroll
                for (int i = 0; i < kStageRows; ++i) {
                    const uint32_t lF = sh_hi[i * kK1Threads + tl], rF = s.halo[1][i][tr];
                    const uint32_t Qm3 = __byte_perm(lF, Q[i][1], 0x5450), Qm2 = __byte_perm(lF, Q[i][2], 0x5451), Qm1 = __byte_perm(lF, Q[i][3], 0x5452);
                    const uint32_t Q4 = __byte_perm(Q[i][0], rF, 0x3432), Q5 = __byte_perm(Q[i][1], rF, 0x3532), Q6 = __byte_perm(Q[i][2], rF, 0x3632);
                    h[i][0] = Qm3 + Qm2 + Qm1 + Q[i][0] + Q[i][1] + Q[i][2] + Q[i][3];
                    h[i][1] = h[i][0] - Qm3 + Q4;
                    h[i][2] = h[i][1] - Qm2 + Q5;
                    h[i][3] = h[i][2] - Qm1 + Q6;
                    uint32_t tj[4];
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const uint32_t hold = (i < 7) ? hprev[i < 7 ? i : 0][j] : h[i >= 7 ? i - 7 : 0][j];
                        nV[j] = nV[j] + hold - h[i][j];
                        const uint32_t Qc = (i < 3) ? Qprev[i < 3 ? i : 0][j] : Q[i >= 3 ? i - 3 : 0][j];
                        tj[j] = 49u * Qc + nV[j];             // bit15 / bit31 = (49 s > boxsum + 24)
                    }
                    const uint32_t dx = __byte_perm(tj[0], tj[1], 0x7531) & 0x80808080u;
                    const uint32_t dy = __byte_perm(tj[2], tj[3], 0x7531) & 0x80808080u;
                    const uint32_t byte = __umulhi(dx, 0x02200440u) + __umulhi(dy, 0x08801100u);
                    if (px_active) rast8[(i + 1) * kRastPitch + t] = (uint8_t)byte;
                }
#pragma unroll
                for (int j = 0; j < 4; ++j) {
#pragma unroll
                    for (int i = 0; i < 7; ++i) hprev[i < kBox ? i : 0][j] = h[2 + i][j];
#pragma unroll
                    for (int i = 0; i < 3; ++i) Qprev[i][j] = Q[6 + i][j];
                    Pprev[0][j] = P[7][j]; Pprev[1][j] = P[8][j];
                }
            }

            // ---------------- S(k-1): its raster was finished by every thread before the barrier above
            if (k - 1 >= k0) symbol_stage(k - 1, buf ^ 1u, col_prev, out, any_dirty);
            col_prev = col;
        }
        // the last cell row of the unit still needs its symbols: one more barrier to see its complete raster
        __syncthreads();
        symbol_stage(k1 - 1, (it - 1u) & 1u, col_prev, out, any_dirty);
        if (any_dirty) atomicOr(&dirty_flags[f], (uint32_t)kFrameDirtyK1);
    }
}

// ---------------------------------------------------------------------------------------------- single-cell API
// CimbDecoder::decode_symbol(bitmatrix) for a batch of pre-thresholded 10x10 windows (rows MSB-first, bit 9 = col 0)
__global__ void k_decode_symbols(const uint16_t* __restrict__ windows, const uint8_t* __restrict__ cooldown, int n,
                                 uint8_t* __restrict__ symbol, uint8_t* __restrict__ drift_offset, uint8_t* __restrict__ distance)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t rows[10];
    for (int r = 0; r < 10; ++r) rows[r] = windows[(size_t)i * 10 + r] & 0x3FFu;
    uint32_t cd = cooldown ? cooldown[i] : 0xFFu;
    const int order[9] = {4, 5, 7, 3, 1, 8, 0, 2, 6};
    int nids = (cd == 0xFEu) ? 9 : 5;                          // CimbDecoder.cpp:144
    uint32_t best = 1000, best_sym = 0, best_id = 0;
    for (int q = 0; q < nids; ++q) {
        int id = order[q];
        if ((uint32_t)id == cd && id != 4) continue;           // CimbDecoder.cpp:116
        int r0 = id / 3, c0 = id % 3;
        unsigned long long H = 0;
        for (int k = 0; k < 8; ++k) H = (H << 8) | ((rows[r0 + k] >> (2 - c0)) & 0xFFu);
        unsigned long long L = __brevll(H);
        for (int t = 0; t < 16; ++t) {
            uint32_t d = __popcll(L ^ c_tiles_L[t]);
            if (d < best) { best = d; best_sym = (uint32_t)t; best_id = (uint32_t)id; }
        }
    }
    symbol[i] = (uint8_t)best_sym; drift_offset[i] = (uint8_t)best_id; distance[i] = (uint8_t)best;
}

__global__ void k_best_colors(const Mode m, const uint8_t* __restrict__ rgb, int n, uint8_t* __restrict__ color, const CcmArg cc)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (cc.active) { color[i] = (uint8_t)best_color_ccm<0>(cc.m, m, rgb[3 * i], rgb[3 * i + 1], rgb[3 * i + 2]); return; }
    color[i] = (uint8_t)((m.color_bits == 3) ? best_color<8>(c_adjust, m, rgb[3 * i], rgb[3 * i + 1], rgb[3 * i + 2])
                                              : best_color<4>(c_adjust, m, rgb[3 * i], rgb[3 * i + 1], rgb[3 * i + 2]));
}

cudaError_t k1_symbols_launch(const uint16_t* d_windows, const uint8_t* d_cooldown, int n, uint8_t* d_sym, uint8_t* d_off, uint8_t* d_dist, cudaStream_t st)
{
    k_decode_symbols<<<(n + 127) / 128, 128, 0, st>>>(d_windows, d_cooldown, n, d_sym, d_off, d_dist); count_launch();
    return cudaGetLastError();
}
cudaError_t k1_colors_launch(const Mode& m, const uint8_t* d_rgb, int n, uint8_t* d_color, const CcmArg& cc, cudaStream_t st)
{
    k_best_colors<<<(n + 127) / 128, 128, 0, st>>>(m, d_rgb, n, d_color, cc); count_launch();
    return cudaGetLastError();
}

constexpr size_t kSharpenExtraSmem = sizeof(uint32_t) * kStageRows * kK1Threads;   // the second halo word of the sharpened rows
size_t k1_smem_bytes(bool sharpen) { return sizeof(K1Smem) + (sharpen ? kSharpenExtraSmem : 0); }
int k1_ctas_per_sm(bool sharpen) { return sharpen ? 3 : kK1CtasPerSm; }

cudaError_t k1_init_tables(const float* adjust256, const unsigned long long* tiles_L16)
{
    cudaError_t e = cudaMemcpyToSymbol(c_adjust, adjust256, sizeof(float) * 256);
    if (e != cudaSuccess) return e;
    e = cudaMemcpyToSymbol(c_tiles_L, tiles_L16, sizeof(unsigned long long) * 16);
    if (e != cudaSuccess) return e;
    const int smem_max = (int)(sizeof(K1Smem) + kSharpenExtraSmem);
#define CB200_K1_ATTR3(NC, G, C, S, D) \
    if ((e = cudaFuncSetAttribute(k1_decode_kernel<NC, G, C, S, D>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_max)) != cudaSuccess) return e;
#define CB200_K1_ATTR2(NC, G, C, S) CB200_K1_ATTR3(NC, G, C, S, false) CB200_K1_ATTR3(NC, G, C, S, true)
#define CB200_K1_ATTR(NC, G, C) CB200_K1_ATTR2(NC, G, C, false) CB200_K1_ATTR2(NC, G, C, true)
    CB200_K1_ATTR(4, true, 0) CB200_K1_ATTR(4, false, 0) CB200_K1_ATTR(8, true, 0) CB200_K1_ATTR(8, false, 0)
    CB200_K1_ATTR(4, true, 1) CB200_K1_ATTR(4, false, 1) CB200_K1_ATTR(8, true, 1) CB200_K1_ATTR(8, false, 1)
    CB200_K1_ATTR(4, true, 2) CB200_K1_ATTR(4, false, 2) CB200_K1_ATTR(8, true, 2) CB200_K1_ATTR(8, false, 2)
#undef CB200_K1_ATTR
#undef CB200_K1_ATTR2
#undef CB200_K1_ATTR3
    return cudaSuccess;
}

cudaError_t k1_launch(const Mode& m, const uint8_t* d_rgb, const uint32_t* d_list, int n_frames, int bands, int grid, bool sharpen,
                      uint8_t* d_cellvals, uint32_t* d_dirty, const CcmArg& cc, cudaStream_t stream, const int* d_sched)
{
    const size_t smem = k1_smem_bytes(sharpen);
    const bool g1024 = m.width == 1024 && m.height == 1024 && m.cells_x == 112 && m.cells_y == 112 && m.corner == 6 &&
                       m.cell_offset == 8 && m.symbol_bits == 4;
    const int cm = cc.means ? 2 : (cc.active ? 1 : 0);
#define CB200_K1_GO2(NC, G, C, S, D) k1_decode_kernel<NC, G, C, S, D><<<grid, kK1Threads, smem, stream>>>(m, d_rgb, d_list, n_frames, bands, d_cellvals, d_dirty, cc, d_sched)
#define CB200_K1_GO(NC, G, C, S) do { if (d_sched) CB200_K1_GO2(NC, G, C, S, true); else CB200_K1_GO2(NC, G, C, S, false); } while (0)
#define CB200_K1_SH(NC, G, C) do { if (sharpen) CB200_K1_GO(NC, G, C, true); else CB200_K1_GO(NC, G, C, false); } while (0)
#define CB200_K1_CM(NC, G) do { if (cm == 2) CB200_K1_SH(NC, G, 2); else if (cm == 1) CB200_K1_SH(NC, G, 1); else CB200_K1_SH(NC, G, 0); } while (0)
    if (m.color_bits == 3) { if (g1024) CB200_K1_CM(8, true); else CB200_K1_CM(8, false); }
    else { if (g1024) CB200_K1_CM(4, true); else CB200_K1_CM(4, false); }
#undef CB200_K1_CM
#undef CB200_K1_SH
#undef CB200_K1_GO
#undef CB200_K1_GO2
    count_launch();
    return cudaGetLastError();
}

}  // namespace cb200
