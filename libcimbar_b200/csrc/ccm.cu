// ccm.cu -- color_correction == 1: one von Kries adaptation matrix per frame from the anchors' white (see ccm.cuh)
#include "ccm.cuh"
#include <cstring>

namespace cb200 {

__device__ __forceinline__ void matx33_mul_rn(const float* a, const float* b, float* out)
{
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) out[3 * i + j] = dot3_rn(a[3 * i], a[3 * i + 1], a[3 * i + 2], b[j], b[3 + j], b[6 + j]);
}

// cv::Matx<float,3,3>::inv(): closed-form 3x3 (opencv2/core/operations.hpp): determinant in float, d = 1 / d, cofactors * d
__device__ __forceinline__ bool matx33_inv_rn(const float* a, float* b)
{
    auto mm = [](float x, float y, float z, float w) { return __fsub_rn(__fmul_rn(x, y), __fmul_rn(z, w)); };   // x*y - z*w
    float d = __fadd_rn(__fsub_rn(__fmul_rn(a[0], mm(a[4], a[8], a[7], a[5])), __fmul_rn(a[1], mm(a[3], a[8], a[6], a[5]))),
                        __fmul_rn(a[2], mm(a[3], a[7], a[6], a[4])));
    if (d == 0.0f) return false;
    d = __fdiv_rn(1.0f, d);
    b[0] = __fmul_rn(mm(a[4], a[8], a[5], a[7]), d); b[1] = __fmul_rn(mm(a[2], a[7], a[1], a[8]), d); b[2] = __fmul_rn(mm(a[1], a[5], a[2], a[4]), d);
    b[3] = __fmul_rn(mm(a[5], a[6], a[3], a[8]), d); b[4] = __fmul_rn(mm(a[0], a[8], a[2], a[6]), d); b[5] = __fmul_rn(mm(a[2], a[3], a[0], a[5]), d);
    b[6] = __fmul_rn(mm(a[3], a[7], a[4], a[6]), d); b[7] = __fmul_rn(mm(a[1], a[6], a[0], a[7]), d); b[8] = __fmul_rn(mm(a[0], a[4], a[1], a[3]), d);
    return true;
}

// one thread per frame: calculateWhite (dark layout: anchors top-left, bottom-left, top-right; 4x4 means; floor 1) and
// get_adaptation_matrix<von_kries>(white, (255,255,255)) = T.inv() * diag((T*desired) / (T*white)) * T
__global__ void k_ccm_simple(const Mode m, const uint8_t* __restrict__ rgb, int n_frames, float* __restrict__ ccm)
{
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n_frames) return;
    const int W = m.width, H = m.height;
    const uint8_t* frame = rgb + (size_t)f * W * H * 3;
    const int tl = 30 - 2, right = W - 30 - 2, bottom = H - 30 - 2;       // Config::anchor_size() == 30, padding 0
    const int ax[3] = {tl, tl, right}, ay[3] = {tl, bottom, tl};
    float white[3] = {1.0f, 1.0f, 1.0f};
    for (int a = 0; a < 3; ++a) {
        uint32_t sum[3] = {0, 0, 0};
        for (int y = 0; y < 4; ++y)
            for (int x = 0; x < 4; ++x) {
                const uint8_t* p = frame + ((size_t)(ay[a] + y) * W + (ax[a] + x)) * 3;
                sum[0] += p[0]; sum[1] += p[1]; sum[2] += p[2];
            }
        for (int c = 0; c < 3; ++c) { const float v = (float)((double)sum[c] / 16.0); if (v > white[c]) white[c] = v; }   // cv::mean is double
    }
    const float T[9] = {0.4002400f, 0.7076000f, -0.0808100f, -0.2263000f, 1.1653200f, 0.0457000f, 0.0000000f, 0.0000000f, 0.9182200f};
    float d[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, ti[9], tmp[9], out[9];
    for (int i = 0; i < 3; ++i) {
        const float m1 = dot3_rn(T[3 * i], T[3 * i + 1], T[3 * i + 2], white[0], white[1], white[2]);
        const float m2 = dot3_rn(T[3 * i], T[3 * i + 1], T[3 * i + 2], 255.0f, 255.0f, 255.0f);
        d[4 * i] = __fdiv_rn(m2, m1);
    }
    if (!matx33_inv_rn(T, ti)) for (int i = 0; i < 9; ++i) ti[i] = 0.0f;
    matx33_mul_rn(ti, d, tmp);
    matx33_mul_rn(tmp, T, out);
    for (int i = 0; i < 9; ++i) ccm[(size_t)f * 9 + i] = out[i];
}

cudaError_t ccm_simple_launch(const Mode& m, const uint8_t* d_rgb, int n_frames, float* d_ccm, cudaStream_t st)
{
    k_ccm_simple<<<(n_frames + 63) / 64, 64, 0, st>>>(m, d_rgb, n_frames, d_ccm); count_launch();
    return cudaGetLastError();
}

}  // namespace cb200

// ================================================================================================ color_correction == 2
// CimbReader::init_ccm (src/lib/cimb_translator/CimbReader.cpp:169-267) with color_correction::get_moore_penrose_lsm
// (chromatic_adaptation/color_correction.h:26-39) and OpenCV's float Jacobi SVD restated operation by operation
// (oracle/cimbar_oracle.c: cbo_moore_penrose_lsm has the derivation).  All arithmetic goes through the _rn intrinsics so
// that nvcc cannot contract multiply-adds (the reference's x86-64 code has no FMAs).
namespace cb200 {
namespace {

__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double ddiv(double a, double b) { return __ddiv_rn(a, b); }
__device__ __forceinline__ float fmul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float fadd(float a, float b) { return __fadd_rn(a, b); }
// std::hypot for finite, unscaled arguments: x^2 + y^2 in double-double, square root with one Newton correction (the result
// is the correctly rounded one except in astronomically rare half-way cases, like glibc's)
__device__ double hypot_acc(double x, double y)
{
    x = fabs(x); y = fabs(y);
    if (x < y) { const double t = x; x = y; y = t; }
    if (y == 0.0) return x;
    const double xx = dmul(x, x), exx = __fma_rn(x, x, -xx);
    const double yy = dmul(y, y), eyy = __fma_rn(y, y, -yy);
    const double sum = dadd(xx, yy);
    const double bv = dsub(sum, xx), err = dadd(dadd(dsub(xx, dsub(sum, bv)), dsub(yy, bv)), dadd(exx, eyy));   // two-sum + low parts
    double h = __dsqrt_rn(sum);
    const double r = dadd(__fma_rn(-h, h, sum), err);           // (x^2 + y^2) - h^2
    return dadd(h, ddiv(r, dmul(2.0, h)));
}

constexpr int kMaxRows = 9;       // 8 colours + white
constexpr int kAStep = 12;

__device__ void jacobi_svd_f32(float* At, float* Wout, float* Vt, int m, int n)
{
    double W[3];
    const float eps = 2.384185791015625e-07f;         // FLT_EPSILON * 2
    for (int i = 0; i < n; ++i) {
        double sd = 0;
        for (int k = 0; k < m; ++k) { const double t = At[i * kAStep + k]; sd = dadd(sd, dmul(t, t)); }
        W[i] = sd;
        for (int k = 0; k < n; ++k) Vt[i * n + k] = 0;
        Vt[i * n + i] = 1;
    }
    const int max_iter = m > 30 ? m : 30;
    for (int iter = 0; iter < max_iter; ++iter) {
        bool changed = false;
        for (int i = 0; i < n - 1; ++i)
            for (int j = i + 1; j < n; ++j) {
                float *Ai = At + i * kAStep, *Aj = At + j * kAStep;
                double a = W[i], p = 0, b = W[j];
                for (int k = 0; k < m; ++k) p = dadd(p, dmul((double)Ai[k], (double)Aj[k]));
                if (fabs(p) <= dmul((double)eps, __dsqrt_rn(dmul(a, b)))) continue;
                p = dmul(p, 2.0);
                const double beta = dsub(a, b), gamma = hypot_acc(p, beta);
                float c, sn;
                if (beta < 0) {
                    const double delta = dmul(dsub(gamma, beta), 0.5);
                    sn = __double2float_rn(__dsqrt_rn(ddiv(delta, gamma)));
                    c = __double2float_rn(ddiv(p, dmul(dmul(gamma, (double)sn), 2.0)));
                } else {
                    c = __double2float_rn(__dsqrt_rn(ddiv(dadd(gamma, beta), dmul(gamma, 2.0))));
                    sn = __double2float_rn(ddiv(p, dmul(dmul(gamma, (double)c), 2.0)));
                }
                a = b = 0;
                for (int k = 0; k < m; ++k) {
                    const float t0 = fadd(fmul(c, Ai[k]), fmul(sn, Aj[k]));
                    const float t1 = fadd(fmul(-sn, Ai[k]), fmul(c, Aj[k]));
                    Ai[k] = t0; Aj[k] = t1;
                    a = dadd(a, dmul((double)t0, (double)t0)); b = dadd(b, dmul((double)t1, (double)t1));
                }
                W[i] = a; W[j] = b;
                changed = true;
                float *Vi = Vt + i * n, *Vj = Vt + j * n;
                for (int k = 0; k < n; ++k) {
                    const float t0 = fadd(fmul(c, Vi[k]), fmul(sn, Vj[k]));
                    const float t1 = fadd(fmul(-sn, Vi[k]), fmul(c, Vj[k]));
                    Vi[k] = t0; Vj[k] = t1;
                }
            }
        if (!changed) break;
    }
    for (int i = 0; i < n; ++i) {
        double sd = 0;
        for (int k = 0; k < m; ++k) { const double t = At[i * kAStep + k]; sd = dadd(sd, dmul(t, t)); }
        W[i] = __dsqrt_rn(sd);
    }
    for (int i = 0; i < n - 1; ++i) {
        int j = i;
        for (int k = i + 1; k < n; ++k) if (W[j] < W[k]) j = k;
        if (i != j) {
            const double tw = W[i]; W[i] = W[j]; W[j] = tw;
            for (int k = 0; k < m; ++k) { const float t = At[i * kAStep + k]; At[i * kAStep + k] = At[j * kAStep + k]; At[j * kAStep + k] = t; }
            for (int k = 0; k < n; ++k) { const float t = Vt[i * n + k]; Vt[i * n + k] = Vt[j * n + k]; Vt[j * n + k] = t; }
        }
    }
    for (int i = 0; i < n; ++i) Wout[i] = __double2float_rn(W[i]);
    for (int i = 0; i < n; ++i) {
        const double sd = W[i];
        const float s = __double2float_rn(sd > 1.17549435e-38 ? ddiv(1.0, sd) : 0.0);
        for (int k = 0; k < m; ++k) At[i * kAStep + k] = fmul(At[i * kAStep + k], s);
    }
}

__device__ bool moore_penrose_lsm(const float* actual, const float* desired, int rows, float* out)
{
    const int N = rows;
    float At[3 * kAStep], Vt[9], W[3];
    for (int r = 0; r < 3; ++r) for (int k = 0; k < N; ++k) At[r * kAStep + k] = actual[k * 3 + r];
    jacobi_svd_f32(At, W, Vt, N, 3);
    float z[kMaxRows * 3];
    for (int i = 0; i < N * 3; ++i) z[i] = 0;
    double threshold = 0;
    for (int i = 0; i < 3; ++i) threshold = dadd(threshold, (double)W[i]);
    threshold = dmul(threshold, (double)2.384185791015625e-07f);
    for (int i = 0; i < 3; ++i) {
        double wi = W[i];
        if (fabs(wi) <= threshold) continue;
        wi = ddiv(1.0, wi);
        double buffer[3];
        for (int j = 0; j < 3; ++j) buffer[j] = dmul((double)Vt[i * 3 + j], wi);
        for (int r = 0; r < N; ++r) {
            const double sv = At[i * kAStep + r];
            for (int j = 0; j < 3; ++j) z[r * 3 + j] = __double2float_rn(dadd((double)z[r * 3 + j], dmul(sv, buffer[j])));
        }
    }
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            double acc = 0;
            for (int k = 0; k < N; ++k) acc = dadd(acc, dmul((double)desired[k * 3 + i], (double)z[k * 3 + j]));
            out[i * 3 + j] = __double2float_rn(acc);
        }
    return true;
}

__device__ __forceinline__ uint32_t md_file_size(const uint8_t* md)
{   // FountainMetadata::file_size, FountainMetadata.h:74-82
    return (uint32_t)md[3] | ((uint32_t)md[2] << 8) | ((uint32_t)md[1] << 16) | (((uint32_t)md[0] & 0x80u) << 17);
}
__device__ __forceinline__ void md_increment(uint8_t* md, uint32_t radioactive)
{   // FountainMetadata::increment_block_id, FountainMetadata.h:66-72
    uint32_t next = (((uint32_t)md[4] << 8) | md[5]) + 1u;
    if (next == radioactive) next += 1u;
    md[4] = (uint8_t)((next >> 8) & 0xFFu); md[5] = (uint8_t)(next & 0xFFu);
}

struct FitSmem {
    uint32_t cnt[8], sr[8], sg[8], sb[8], first[8];
    uint8_t hdr[8];
    uint32_t radioactive;
    int has;
};

// one warp per frame
__global__ void __launch_bounds__(128)
k_ccm_fit(const Mode m, const uint8_t* __restrict__ rgb, const uint8_t* __restrict__ data, const uint8_t* __restrict__ ok,
          const uint16_t* __restrict__ idx, int n_frames, float* __restrict__ fit, uint8_t* __restrict__ valid, const GivenHeader given)
{
    __shared__ FitSmem sm[4];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const int f = blockIdx.x * 4 + wib;
    if (f >= n_frames) return;
    FitSmem& s = sm[wib];
    const int W = m.width, H = m.height;
    const uint8_t* frame = rgb + (size_t)f * W * H * 3;
    if (lane < 8) { s.cnt[lane] = s.sr[lane] = s.sg[lane] = s.sb[lane] = 0; s.first[lane] = 0xFFFFFFFFu; }
    if (lane == 0 && given.use) {
        // CimbReader::init_ccm called by a host that kept the header itself (CimbReader::update_metadata on the host side)
        for (int k = 0; k < 6; ++k) s.hdr[k] = given.hdr[k];
        s.radioactive = given.radioactive;
        s.has = (given.hdr[0] | given.hdr[1] | given.hdr[2] | given.hdr[3]) != 0;
    } else if (lane == 0) {
        // what the symbol stream's chunk events leave in CimbReader::_fountainColorHeader (aligned_stream.h:39-116 with five
        // whole RS blocks per chunk: a chunk whose last block is bad raises no event and passes its bad flag on; otherwise the
        // event is a flush of the chunk when all its blocks are good and no flag was pending, else the "bad chunk" callback)
        const int nbs = m.nblocks_sym, bpc = m.blocks_per_chunk, msg = m.msg_len;
        const uint8_t* okf = ok + (size_t)f * m.nblocks;
        const uint8_t* df = data + (size_t)f * m.nblocks * msg;
        uint8_t hdr[6] = {0, 0, 0, 0, 0, 0};
        uint32_t radioactive = 0;
        bool carry = false;
        for (int q = 0; q * bpc + bpc <= nbs; ++q) {
            bool all = true;
            for (int k = 0; k < bpc; ++k) all = all && okf[q * bpc + k] != 0;
            const bool last_ok = okf[q * bpc + bpc - 1] != 0;
            if (!last_ok) { carry = true; continue; }
            const bool good = all && !carry;
            carry = false;
            const bool id_zero = (hdr[0] | hdr[1] | hdr[2] | hdr[3]) == 0;
            if (!good && id_zero) continue;                                   // update_metadata(nullptr, 0) without a header
            if (id_zero) for (int k = 0; k < 6; ++k) hdr[k] = df[(size_t)q * bpc * msg + k];
            if (radioactive == 0) { const uint32_t fs = md_file_size(hdr); radioactive = (fs % (uint32_t)m.chunk_size == 0) ? 0xFFFFFFFFu : fs / (uint32_t)m.chunk_size; }
            md_increment(hdr, radioactive);
        }
        for (int k = 0; k < 6; ++k) s.hdr[k] = hdr[k];
        s.radioactive = radioactive;
        s.has = (hdr[0] | hdr[1] | hdr[2] | hdr[3]) != 0;
    }
    __syncwarp();
    if (!s.has || m.color_bits == 0) { if (lane == 0) valid[f] = 0; return; }

    // ---- the colours the header predicts at the head of each colour-stream chunk vs the observed cell means
    const int color_bits = m.color_bits;
    const uint32_t end = (uint32_t)m.cap_col * 8u / (uint32_t)color_bits;
    const uint32_t interval = (uint32_t)m.cap_all * 8u / (uint32_t)m.chunks_per_frame / (uint32_t)color_bits;
    const uint32_t header_len = 48u / (uint32_t)color_bits;
    const uint32_t nchunks = (end + interval - 1) / interval;
    for (uint32_t sidx = lane; sidx < nchunks * header_len; sidx += 32) {
        const uint32_t c = sidx / header_len, i = sidx - c * header_len;
        uint8_t hdr[6];
        for (int k = 0; k < 6; ++k) hdr[k] = s.hdr[k];
        for (uint32_t k = 0; k < c; ++k) md_increment(hdr, s.radioactive);
        uint32_t expected = 0;
        for (int k = 0; k < color_bits; ++k) { const uint32_t bit = i * color_bits + k; expected = (expected << 1) | ((hdr[bit >> 3] >> (7 - (bit & 7))) & 1u); }
        const int cell = idx[c * interval + i];
        int k, col, base, ncols, x0;
        cell_row_col(m, cell, k, col);
        cell_row_geom(m, k, base, ncols, x0);
        const int x = x0 + kSpacing * col, y = m.cell_offset + kSpacing * k;
        uint32_t R = 0, G = 0, B = 0;
        for (int r = 1; r <= 6; ++r) {
            const uint8_t* p = frame + ((size_t)(y + r) * W + (size_t)(x + 1)) * 3;
            for (int cc = 0; cc < 6; ++cc) { R += p[3 * cc]; G += p[3 * cc + 1]; B += p[3 * cc + 2]; }
        }
        atomicAdd(&s.cnt[expected], 1u); atomicAdd(&s.sr[expected], R / 36u); atomicAdd(&s.sg[expected], G / 36u); atomicAdd(&s.sb[expected], B / 36u);
        atomicMin(&s.first[expected], sidx);
    }
    __syncwarp();
    if (lane != 0) return;
    // rows in the iteration order of libstdc++'s unordered_map<uint16_t, ...>: reverse order of first appearance
    float actual[kMaxRows * 3], desired[kMaxRows * 3];
    int rows = 0;
    const int nc = 1 << color_bits;
    uint32_t done = 0;
    for (int r = 0; r < nc; ++r) {
        int best = -1; uint32_t bf = 0;
        for (int c = 0; c < nc; ++c) if (!((done >> c) & 1u) && s.cnt[c] && (best < 0 || s.first[c] > bf)) { best = c; bf = s.first[c]; }
        if (best < 0) break;
        done |= 1u << best;
        actual[rows * 3] = (float)(s.sr[best] / s.cnt[best]); actual[rows * 3 + 1] = (float)(s.sg[best] / s.cnt[best]); actual[rows * 3 + 2] = (float)(s.sb[best] / s.cnt[best]);
        desired[rows * 3] = (float)m.palette[best][0]; desired[rows * 3 + 1] = (float)m.palette[best][1]; desired[rows * 3 + 2] = (float)m.palette[best][2];
        ++rows;
    }
    if (rows < 4) { valid[f] = 0; return; }
    {   // calculateWhite (dark), CimbReader.cpp:55-72
        const int tl = 30 - 2, right = W - 30 - 2, bottom = H - 30 - 2;
        const int ax[3] = {tl, tl, right}, ay[3] = {tl, bottom, tl};
        float white[3] = {1.0f, 1.0f, 1.0f};
        for (int a = 0; a < 3; ++a) {
            uint32_t sum[3] = {0, 0, 0};
            for (int y = 0; y < 4; ++y)
                for (int x = 0; x < 4; ++x) {
                    const uint8_t* p = frame + ((size_t)(ay[a] + y) * W + (ax[a] + x)) * 3;
                    sum[0] += p[0]; sum[1] += p[1]; sum[2] += p[2];
                }
            for (int c = 0; c < 3; ++c) { const float v = (float)((double)sum[c] / 16.0); if (v > white[c]) white[c] = v; }
        }
        actual[rows * 3] = white[0]; actual[rows * 3 + 1] = white[1]; actual[rows * 3 + 2] = white[2];
        desired[rows * 3] = desired[rows * 3 + 1] = desired[rows * 3 + 2] = 255.0f;
        ++rows;
    }
    float out[9];
    moore_penrose_lsm(actual, desired, rows, out);
    for (int i = 0; i < 9; ++i) fit[(size_t)f * 9 + i] = out[i];
    valid[f] = 1;
}

// the decoder's CCM is whatever the last successful fit left (thread-local state, CimbDecoder.cpp:69-85): frame f uses its own
// fit if it has one, else the matrix of frame f-1 (frame 0: the context's).  The context's matrix is initial.m / initial.active,
// or, with initial.per_frame set, 9 floats and an activity byte in device memory (an earlier batch still in flight left it there)
__global__ void __launch_bounds__(1024)
k_ccm_carry(int n_frames, const float* __restrict__ fit, const uint8_t* __restrict__ valid, const CcmArg initial,
            float* __restrict__ used, uint8_t* __restrict__ used_active)
{
    float im[9];
    for (int i = 0; i < 9; ++i) im[i] = initial.per_frame ? initial.per_frame[i] : initial.m[i];
    const bool iactive = initial.per_frame ? initial.per_frame_active[0] != 0 : initial.active != 0;
    // "index of the last frame <= f with a fit" is a running maximum: every thread scans a contiguous segment, the segment
    // results are combined by a block-wide inclusive max scan, then every thread replays its segment with the right start
    __shared__ int seg_last[1024];
    const int t = threadIdx.x;
    const int seg = (n_frames + 1023) / 1024, f0 = t * seg, f1 = min(f0 + seg, n_frames);
    int last = -1;
    for (int f = f0; f < f1; ++f) if (valid[f]) last = f;
    seg_last[t] = last;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {
        const int v = t >= o ? seg_last[t - o] : -1;
        __syncthreads();
        if (v > seg_last[t]) seg_last[t] = v;
        __syncthreads();
    }
    int cur = t > 0 ? seg_last[t - 1] : -1;
    for (int f = f0; f < f1; ++f) {
        if (valid[f]) cur = f;
        for (int i = 0; i < 9; ++i) used[(size_t)f * 9 + i] = cur >= 0 ? fit[(size_t)cur * 9 + i] : im[i];
        used_active[f] = (cur >= 0 || iactive) ? 1 : 0;
    }
}

// CimbDecoder::get_best_color for every cell from the mean colours the first pass stored.  blockIdx.y walks the frames (the
// frame's matrix sits in shared memory), blockIdx.x the cells.
__global__ void __launch_bounds__(256)
k_ccm_apply(const Mode m, const uint32_t* __restrict__ means, int n_frames, const float* __restrict__ used,
            const uint8_t* __restrict__ used_active, uint8_t* __restrict__ cellvals)
{
    __shared__ float mat[9];
    const int ci = blockIdx.x * 256 + threadIdx.x;
    const uint32_t color_mask = ((1u << m.color_bits) - 1u) << m.symbol_bits;
    for (int f = blockIdx.y; f < n_frames; f += gridDim.y) {
        __syncthreads();                                   // the previous frame's readers of mat[] are done
        const bool active = used_active[f] != 0;
        if (active && threadIdx.x < 9) mat[threadIdx.x] = used[(size_t)f * 9 + threadIdx.x];
        __syncthreads();
        if (ci >= m.num_cells) continue;
        const size_t i = (size_t)f * m.num_cells + ci;
        const uint32_t v = means[i], ri = v & 0xFFu, gi = (v >> 8) & 0xFFu, bi = (v >> 16) & 0xFFu;
        uint32_t col;
        if (active) col = best_color_ccm<0>(mat, m, ri, gi, bi);
        else {
            // integer inputs: max/min with the floors, scale through the table, same decision as the float code (k1_decode.cu)
            uint32_t mxi = max(max(ri, gi), max(bi, 1u)), mni = min(min(ri, gi), min(bi, 48u));
            if (mni >= mxi) mni = 0;
            // (float)(255.0 / (double)d) == the single-precision quotient (see best_color_ccm)
            const float adj = __fdiv_rn(255.0f, (float)(mxi - mni)), mn = (float)mni, hi_thr = __fsub_rn(245.0f, mn);
            const float fr = __fmul_rn((float)(ri - mni), adj), fg = __fmul_rn((float)(gi - mni), adj), fb = __fmul_rn((float)(bi - mni), adj);
            const int cr = (fr > hi_thr) ? 255 : (int)__float2uint_rz(fr), cg = (fg > hi_thr) ? 255 : (int)__float2uint_rz(fg),
                      cb = (fb > hi_thr) ? 255 : (int)__float2uint_rz(fb);
            const int a0 = cr - cg, a1 = cg - cb;
            int best_d = 0x7fffffff; col = 0;
            for (int c = 0; c < (1 << m.color_bits); ++c) {
                const int d = m.pal_c[c] - (a0 * m.pal_u[c] + a1 * m.pal_w[c]);
                if (d < best_d) { best_d = d; col = (uint32_t)c; }
            }
        }
        cellvals[i] = (uint8_t)((cellvals[i] & ~color_mask) | (col << m.symbol_bits));
    }
}

}  // namespace

cudaError_t ccm_fit_launch(const Mode& m, const uint8_t* d_rgb, const uint8_t* d_data, const uint8_t* d_ok, const uint16_t* d_idx,
                           int n_frames, float* d_fit, uint8_t* d_valid, cudaStream_t st, const GivenHeader* given)
{
    GivenHeader g;
    memset(&g, 0, sizeof(g));
    if (given) g = *given;
    k_ccm_fit<<<(n_frames + 3) / 4, 128, 0, st>>>(m, d_rgb, d_data, d_ok, d_idx, n_frames, d_fit, d_valid, g); count_launch();
    return cudaGetLastError();
}
cudaError_t ccm_carry_launch(int n_frames, const float* d_fit, const uint8_t* d_valid, const CcmArg& initial, float* d_used,
                             uint8_t* d_used_active, cudaStream_t st)
{
    k_ccm_carry<<<1, 1024, 0, st>>>(n_frames, d_fit, d_valid, initial, d_used, d_used_active); count_launch();
    return cudaGetLastError();
}
cudaError_t ccm_apply_launch(const Mode& m, const uint32_t* d_means, int n_frames, const float* d_used, const uint8_t* d_used_active,
                             uint8_t* d_cellvals, cudaStream_t st)
{
    dim3 grid((unsigned)((m.num_cells + 255) / 256), (unsigned)(n_frames < 2048 ? n_frames : 2048));
    k_ccm_apply<<<grid, 256, 0, st>>>(m, d_means, n_frames, d_used, d_used_active, d_cellvals); count_launch();
    return cudaGetLastError();
}

}  // namespace cb200
