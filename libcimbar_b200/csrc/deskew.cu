// deskew.cu -- the extractor's deskew in front of the decode path (SURVEY.md 8f-2), sm_90a.
//
// Replaces (reference file:line relative to /root/reference/):
//   Deskewer::deskew        src/lib/extractor/Deskewer.h:25-40: cv::getPerspectiveTransform(corners, outputPoints) +
//                           cv::warpPerspective(img, output, transform, size, cv::INTER_LINEAR) to the mode's image size
//   (Extractor::extract     src/lib/extractor/Extractor.h:30-46 calls it with the four anchor centres Scanner found: scan.cu, or
//                           corners the caller supplies)
// OpenCV is a third-party dependency of the reference; its arithmetic is restated here and pinned against cv2 itself
// (tests/test_deskew.py): getPerspectiveTransform and cv::invert(3x3) in extract_core.cuh, warpPerspective(INTER_LINEAR,
// BORDER_CONSTANT 0) =
//   per destination pixel, in double:  W = 32 / (M6 x + M7 y + M8);  X = cvRound((M0 x + M1 y + M2) W), Y likewise,
//   evaluated block-wise exactly as OpenCV does (X0 = M0 bx + M1 y + M2 for the 64-pixel block origin bx, then + M0 x1);
//   source pixel (X >> 5, Y >> 5) with 5-bit fractions ax, ay and the fixed-point bilinear weights
//   (32-ax)(32-ay), ax(32-ay), (32-ax)ay, ax ay (x 32 = OpenCV's 15-bit table, which is exact for these fractions),
//   result (sum + 512) >> 10, taps outside the source count as 0.
// The output frames land in device memory in the layout cb200_decode_*_dev take: a camera frame goes H2D once and never
// returns to the host before its chunks do.
#include "ctx.cuh"
#include "extract_core.cuh"

#include <cfloat>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

namespace cb200 {

struct DeskewState {
    DevBuf<uint8_t> d_table;       // n x 9 inverse maps (destination -> source) in double, then n PicDesc (the sources)
    DevBuf<uint8_t> d_src;         // staging for the host-pointer entry point
    DevBuf<uint8_t> d_dst;         // deskewed frames of the host-pointer entry points
};

void deskew_destroy(DeskewState* d) { delete d; }

// one thread = four consecutive destination pixels (12 bytes = three aligned words); blockIdx.y = frame (grid-strided), so the
// index arithmetic is 32-bit.  Frame f reads its source picture (base, size) from desc[f]; the pictures may differ in size, the
// frames do not.  No branch sits between the address arithmetic and the loads, so the loads of a thread's four pixels
// are all in flight together, and the two horizontal taps of a source row -- six consecutive bytes -- are fetched as aligned 32-bit
// words and realigned by funnel shifts: a source that lies rotated in the photograph makes every lane hit its own sector, and the
// kernel is then bound by L1 sector look-ups (ncu: 27 sectors per request), so fewer, wider requests are what counts.
// A tap outside the source gets weight 0 (== BORDER_CONSTANT 0); its bytes come from a clamped, valid address.
__device__ __forceinline__ void load_row_pair(const uint8_t* __restrict__ p, const uint8_t* __restrict__ end, uint32_t& lo, uint32_t& hi)
{   // bytes p[0..5] -> lo = p[0..3], hi = p[4..5] (upper half unspecified); `end` = one past the last readable byte
    const uintptr_t addr = reinterpret_cast<uintptr_t>(p);
    const uint32_t a = (uint32_t)(addr & 3u);
    const uint8_t* base = p - a;
    if (base + 12 <= end) {
        const uint32_t* w = reinterpret_cast<const uint32_t*>(base);
        const uint32_t w0 = __ldg(w), w1 = __ldg(w + 1);
        const uint32_t w2 = (a == 3u) ? __ldg(w + 2) : 0u;           // six bytes from offset 3 reach into the third word
        lo = __funnelshift_r(w0, w1, 8u * a);
        hi = __funnelshift_r(w1, w2, 8u * a);
    } else {                                                        // the last few bytes of the buffer: byte loads
        lo = (uint32_t)__ldg(p) | ((uint32_t)__ldg(p + 1) << 8) | ((uint32_t)__ldg(p + 2) << 16) | ((uint32_t)__ldg(p + 3) << 24);
        hi = (uint32_t)__ldg(p + 4) | ((uint32_t)__ldg(p + 5) << 8);
    }
}

__global__ void __launch_bounds__(256)
k_deskew(const uint8_t* __restrict__ src, size_t src_bytes, const double* __restrict__ minv, const PicDesc* __restrict__ desc, int n,
         int dst_w, int dst_h, int bw0, uint8_t* __restrict__ dst)
{
    const int quads = dst_w >> 2;
    const int per_frame = dst_h * quads;
    const int i = (int)(blockIdx.x * blockDim.x + threadIdx.x);
    if (i >= per_frame) return;
    const int y = i / quads, q = i - y * quads;
    const int x = 4 * q, bx = (x / bw0) * bw0;
    const uint8_t* const end = src + src_bytes;
    for (int f = (int)blockIdx.y; f < n; f += (int)gridDim.y) {
        const double* M = minv + (size_t)f * 9;
        const uint8_t* s = src + __ldg(&desc[f].src);
        const int src_w = __ldg(&desc[f].w), src_h = __ldg(&desc[f].h);
        const double M0 = __ldg(M), M1 = __ldg(M + 1), M2 = __ldg(M + 2), M3 = __ldg(M + 3), M4 = __ldg(M + 4), M5 = __ldg(M + 5),
                     M6 = __ldg(M + 6), M7 = __ldg(M + 7), M8 = __ldg(M + 8);
        // no FMA contraction: OpenCV's x86-64 code rounds after every multiply and add
        const double X0 = __dadd_rn(__dadd_rn(__dmul_rn(M0, (double)bx), __dmul_rn(M1, (double)y)), M2);
        const double Y0 = __dadd_rn(__dadd_rn(__dmul_rn(M3, (double)bx), __dmul_rn(M4, (double)y)), M5);
        const double W0 = __dadd_rn(__dadd_rn(__dmul_rn(M6, (double)bx), __dmul_rn(M7, (double)y)), M8);
        uint32_t wgt[4][4];
        uint32_t off[4][2];                      // byte offsets of the two row pairs inside the source picture (< 4 GB)
        bool left[4], right[4];                  // the pair was clamped: tap x1 is the pair's first pixel / tap x0 its second
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const double x1 = (double)(x + u - bx);
            double W = __dadd_rn(W0, __dmul_rn(M6, x1));
            W = W != 0. ? __ddiv_rn(32.0, W) : 0.;
            double fX = __dmul_rn(__dadd_rn(X0, __dmul_rn(M0, x1)), W), fY = __dmul_rn(__dadd_rn(Y0, __dmul_rn(M3, x1)), W);
            fX = fmax(-2147483648.0, fmin(2147483647.0, fX)); fY = fmax(-2147483648.0, fmin(2147483647.0, fY));
            const int X = __double2int_rn(fX), Y = __double2int_rn(fY);        // cvRound: to nearest, ties to even
            int sx = X >> 5, sy = Y >> 5;
            sx = sx < -32768 ? -32768 : (sx > 32767 ? 32767 : sx); sy = sy < -32768 ? -32768 : (sy > 32767 ? 32767 : sy);   // saturate_cast<short>
            const uint32_t ax = (uint32_t)(X & 31), ay = (uint32_t)(Y & 31);
            const bool x0in = sx >= 0 && sx < src_w, x1in = sx + 1 >= 0 && sx + 1 < src_w;
            const bool y0in = sy >= 0 && sy < src_h, y1in = sy + 1 >= 0 && sy + 1 < src_h;
            wgt[u][0] = (x0in && y0in) ? (32u - ax) * (32u - ay) : 0u;
            wgt[u][1] = (x1in && y0in) ? ax * (32u - ay) : 0u;
            wgt[u][2] = (x0in && y1in) ? (32u - ax) * ay : 0u;
            wgt[u][3] = (x1in && y1in) ? ax * ay : 0u;
            // the pair of source pixels (c, c + 1) that holds whichever of the taps sx, sx + 1 are inside the row
            const int c = sx < 0 ? 0 : (sx > src_w - 2 ? src_w - 2 : sx);
            left[u] = sx < c; right[u] = sx > c;
            const int cy0 = sy < 0 ? 0 : (sy >= src_h ? src_h - 1 : sy), cy1 = sy + 1 < 0 ? 0 : (sy + 1 >= src_h ? src_h - 1 : sy + 1);
            off[u][0] = 3u * ((uint32_t)cy0 * (uint32_t)src_w + (uint32_t)c);
            off[u][1] = 3u * ((uint32_t)cy1 * (uint32_t)src_w + (uint32_t)c);
        }
        uint32_t lo[4][2], hi[4][2];
#pragma unroll
        for (int u = 0; u < 4; ++u) { load_row_pair(s + off[u][0], end, lo[u][0], hi[u][0]); load_row_pair(s + off[u][1], end, lo[u][1], hi[u][1]); }
        uint32_t px[4][3];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) {
                uint32_t acc = 512u;
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    const uint32_t pa = (lo[u][r] >> (8 * ch)) & 0xFFu;                                   // pixel c
                    const uint32_t pb = ch == 0 ? lo[u][r] >> 24 : (hi[u][r] >> (8 * (ch - 1))) & 0xFFu;  // pixel c + 1
                    const uint32_t v0 = right[u] ? pb : pa, v1 = left[u] ? pa : pb;                      // taps sx, sx + 1
                    acc += wgt[u][2 * r] * v0 + wgt[u][2 * r + 1] * v1;
                }
                px[u][ch] = acc >> 10;
            }
        }
        uint32_t* out = reinterpret_cast<uint32_t*>(dst + ((size_t)f * dst_h + y) * (size_t)dst_w * 3 + (size_t)x * 3);
        out[0] = px[0][0] | (px[0][1] << 8) | (px[0][2] << 16) | (px[1][0] << 24);
        out[1] = px[1][1] | (px[1][2] << 8) | (px[2][0] << 16) | (px[2][1] << 24);
        out[2] = px[2][2] | (px[3][0] << 8) | (px[3][1] << 16) | (px[3][2] << 24);
    }
}

static DeskewState* dstate(cb200_ctx* c)
{
    if (!c->deskew) c->deskew = new DeskewState();
    return c->deskew;
}

// the host-pointer entry points: n source pictures of w x h into the staging buffer
static int stage_sources(cb200_ctx* c, const uint8_t* src, int w, int h, int n)
{
    DeskewState* d = dstate(c);
    const size_t sb = (size_t)n * w * h * 3;
    CK(d->d_src.ensure(sb), "cudaMalloc deskew source");
    CK(cudaMemcpyAsync(d->d_src, src, sb, cudaMemcpyHostToDevice, c->stream), "H2D camera frames");
    return CB200_OK;
}

// room for n deskewed frames in the output buffer
static int ensure_frames(cb200_ctx* c, int n)
{
    return grow(c, dstate(c)->d_dst, (size_t)n * c->mode.width * c->mode.height * 3, "deskew output");
}

}  // namespace cb200

int cb200::deskew_reserve(cb200_ctx* c, int n) { return ensure_frames(c, n); }

int cb200::deskew_frames(cb200_ctx* c, int n, uint8_t** frames)
{
    int rc = ensure_frames(c, n); if (rc) return rc;
    *frames = c->deskew->d_dst;
    return CB200_OK;
}

namespace cb200 {

// warpPerspective of n source pictures of sizes wh (n x (w, h), host) packed in d_src, one frame each
static int deskew_run(cb200_ctx* c, const uint8_t* d_src, const int32_t* wh, int n, const double* m9, uint8_t* d_dst)
{
    size_t src_bytes = 0;
    for (int f = 0; f < n; ++f) {
        if (wh[2 * f] < 2 || wh[2 * f + 1] < 2) return fail(CB200_ERR_ARG, "bad arguments");
        const size_t b = (size_t)wh[2 * f] * (size_t)wh[2 * f + 1] * 3;
        if (b >= ((size_t)1 << 32)) return fail(CB200_ERR_ARG, "source picture " + std::to_string(f) + " of 4 GB or more");
        src_bytes += b;
    }
    if (n == 0) return CB200_OK;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    DeskewState* d = dstate(c);
    const size_t table_bytes = (sizeof(double) * 9 + sizeof(PicDesc)) * (size_t)n;
    CK(d->d_table.ensure(table_bytes), "cudaMalloc transforms");
    // warpPerspective inverts the transform it is given (no WARP_INVERSE_MAP): cv::invert, DECOMP_LU; a singular matrix maps
    // everything to (0, 0) there (invert leaves zeros) -- reported here instead
    int slot;
    uint8_t* table;
    int rc = stage_take(c, table_bytes, &slot, &table); if (rc) return rc;
    double* inv = reinterpret_cast<double*>(table);
    PicDesc* desc = reinterpret_cast<PicDesc*>(inv + 9 * (size_t)n);
    size_t off = 0;
    for (int f = 0; f < n; ++f) {
        if (!extract::invert3(m9 + (size_t)f * 9, inv + (size_t)f * 9)) return fail(CB200_ERR_ARG, "singular perspective transform");
        desc[f] = PicDesc{off, 0, wh[2 * f], wh[2 * f + 1], 0, 0};
        off += (size_t)wh[2 * f] * (size_t)wh[2 * f + 1] * 3;
    }
    rc = stage_send(c, slot, d->d_table, table_bytes, "H2D transforms"); if (rc) return rc;
    const double* d_inv = reinterpret_cast<const double*>(d->d_table.get());
    return deskew_launch(c, d_src, src_bytes, d_inv, reinterpret_cast<const PicDesc*>(d_inv + 9 * (size_t)n), n, d_dst);
}

}  // namespace cb200

int cb200::deskew_launch(cb200_ctx* c, const uint8_t* d_src, size_t src_bytes, const double* d_minv, const PicDesc* d_desc, int n, uint8_t* d_dst)
{
    const Mode& m = c->mode;
    // OpenCV's block geometry (WarpPerspectiveInvoker): bh0 = min(16, H); bw0 = min(1024 / bh0, W)
    const int bh0 = m.height < 16 ? m.height : 16;
    int bw0 = 1024 / bh0; if (bw0 > m.width) bw0 = m.width;
    const int per_frame = m.height * (m.width / 4);
    const dim3 grid((unsigned)((per_frame + 255) / 256), (unsigned)(n < 32768 ? n : 32768));
    k_deskew<<<grid, 256, 0, c->stream>>>(d_src, src_bytes, d_minv, d_desc, n, m.width, m.height, bw0, d_dst);
    count_launch();
    CK(cudaGetLastError(), "deskew launch");
    return CB200_OK;
}

namespace cb200 {

}  // namespace cb200

using namespace cb200;

extern "C" {

int cb200_perspective_transform(const float* src_xy, const float* dst_xy, double* m9_out)
{
    if (!src_xy || !dst_xy || !m9_out) return fail(CB200_ERR_ARG, "null argument");
    if (!extract::perspective_transform(src_xy, dst_xy, m9_out)) return fail(CB200_ERR_ARG, "degenerate corner quadrilateral");
    return CB200_OK;
}

int cb200_deskew_dev(cb200_ctx* c, const uint8_t* d_src, int src_w, int src_h, int n, const double* m9, uint8_t* d_dst)
{
    if (!c || !d_src || !m9 || !d_dst || n < 0 || src_w < 2 || src_h < 2) return fail(CB200_ERR_ARG, "bad arguments");
    if ((size_t)src_w * (size_t)src_h * 3 >= ((size_t)1 << 32)) return fail(CB200_ERR_ARG, "source picture of 4 GB or more");
    int rc = check_frozen_deskew(c, n); if (rc) return rc;
    return deskew_run(c, d_src, uniform_sizes(src_w, src_h, n).data(), n, m9, d_dst);
}

int cb200_deskew(cb200_ctx* c, const uint8_t* src, int src_w, int src_h, int n, const double* m9, uint8_t* dst)
{
    if (!c || !src || !dst || n < 0 || n > c->max_frames) return fail(CB200_ERR_ARG, "bad arguments");
    if (n == 0) return CB200_OK;
    int rc = check_frozen_deskew(c, n); if (rc) return rc;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    rc = stage_sources(c, src, src_w, src_h, n); if (rc) return rc;
    rc = ensure_frames(c, n); if (rc) return rc;
    const DeskewState* d = c->deskew;
    rc = cb200_deskew_dev(c, d->d_src, src_w, src_h, n, m9, d->d_dst); if (rc) return rc;
    CK(cudaMemcpyAsync(dst, d->d_dst, (size_t)n * c->mode.width * c->mode.height * 3, cudaMemcpyDeviceToHost, c->stream), "D2H frames");
    CK(cudaStreamSynchronize(c->stream), "sync");
    return CB200_OK;
}

}  // extern "C"

// both sharpen flags together are a contradiction (CB200_FLAG_SHARPEN_IF_NEEDED is the CLI's --preprocess -1, SHARPEN its 1)
int cb200::check_camera_flags(uint32_t flags)
{
    if ((flags & CB200_FLAG_SHARPEN) && (flags & CB200_FLAG_SHARPEN_IF_NEEDED))
        return fail(CB200_ERR_ARG, "CB200_FLAG_SHARPEN and CB200_FLAG_SHARPEN_IF_NEEDED are exclusive");
    return CB200_OK;
}

// the pictures are already in device memory (the scan entry points stage them once for scan + deskew)
int cb200::extract_decode_to_host(cb200_ctx* c, const uint8_t* d_src, const int32_t* wh, int n, const float* corners, uint32_t flags,
                                  const uint8_t* sharpen, uint8_t* chunks_out, uint32_t* chunk_count, uint32_t* chunk_mask, uint8_t* frame_flags)
{
    if (!c || !d_src || !corners || !chunks_out || !chunk_count || n < 0 || n > c->max_frames) return fail(CB200_ERR_ARG, "bad arguments");
    if (n == 0) return CB200_OK;
    int rc = check_frozen_deskew(c, n); if (rc) return rc;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    const Mode& m = c->mode;
    float outp[8];
    extract::output_points(m.width, m.height, outp);
    std::vector<double> m9((size_t)n * 9);
    for (int f = 0; f < n; ++f) {
        rc = cb200_perspective_transform(corners + (size_t)f * 8, outp, m9.data() + (size_t)f * 9); if (rc) return rc;
    }
    rc = ensure_frames(c, n); if (rc) return rc;
    rc = deskew_run(c, d_src, wh, n, m9.data(), c->deskew->d_dst); if (rc) return rc;
    // the deskewed frames never leave the device: straight into the decode
    return decode_fountain_to_host(c, c->deskew->d_dst, n, flags, sharpen, chunks_out, chunk_count, chunk_mask, frame_flags);
}

// Extractor::extract (Extractor.h:30-46): NEEDS_SHARPEN unless every side of the corner quadrilateral spans more than the frame in x
// or in y (Corners::is_granular_scale, Corners.h:57-75)
std::vector<uint8_t> cb200::sharpen_from_corners(const cb200_ctx* c, const float* corners, int n)
{
    std::vector<uint8_t> sharpen((size_t)n);
    for (int i = 0; i < n; ++i) sharpen[(size_t)i] = extract::is_granular_scale(corners + 8 * (size_t)i, c->mode.width, c->mode.height) ? 0 : 1;
    return sharpen;
}

extern "C" {

int cb200_extract_decode_fountain_dev(cb200_ctx* c, const uint8_t* d_src, int src_w, int src_h, int n, const float* corners, uint32_t flags,
                                      uint8_t* chunks_out, uint32_t* chunk_count, uint32_t* chunk_mask, uint8_t* frame_flags)
{
    int rc = check_camera_flags(flags); if (rc) return rc;
    const std::vector<int32_t> wh = uniform_sizes(src_w, src_h, n);
    if (!(flags & CB200_FLAG_SHARPEN_IF_NEEDED) || !c || !corners || n < 0 || n > c->max_frames)
        return extract_decode_to_host(c, d_src, wh.data(), n, corners, flags, nullptr, chunks_out, chunk_count, chunk_mask, frame_flags);
    return extract_decode_to_host(c, d_src, wh.data(), n, corners, flags & ~CB200_FLAG_SHARPEN_IF_NEEDED, sharpen_from_corners(c, corners, n).data(),
                                  chunks_out, chunk_count, chunk_mask, frame_flags);
}

int cb200_extract_decode_fountain_ragged_dev(cb200_ctx* c, const uint8_t* d_src, const int32_t* wh, int n, const float* corners, uint32_t flags,
                                             uint8_t* chunks_out, uint32_t* chunk_count, uint32_t* chunk_mask, uint8_t* frame_flags)
{
    int rc = check_camera_flags(flags); if (rc) return rc;
    if (n < 0) return fail(CB200_ERR_ARG, "n < 0");
    if (!wh) return fail(CB200_ERR_ARG, "null wh");
    if (!d_src) return fail(CB200_ERR_ARG, "null pictures");
    rc = check_picture_sizes(wh, n); if (rc) return rc;
    if (!c) return fail(CB200_ERR_ARG, "null context");
    if (!corners || !chunks_out || !chunk_count) return fail(CB200_ERR_ARG, !corners ? "null corners" : "null output");
    if (n > c->max_frames) return fail(CB200_ERR_ARG, "n = " + std::to_string(n) + " > max_frames = " + std::to_string(c->max_frames));
    if (!(flags & CB200_FLAG_SHARPEN_IF_NEEDED))
        return extract_decode_to_host(c, d_src, wh, n, corners, flags, nullptr, chunks_out, chunk_count, chunk_mask, frame_flags);
    return extract_decode_to_host(c, d_src, wh, n, corners, flags & ~CB200_FLAG_SHARPEN_IF_NEEDED, sharpen_from_corners(c, corners, n).data(),
                                  chunks_out, chunk_count, chunk_mask, frame_flags);
}

int cb200_extract_decode_fountain(cb200_ctx* c, const uint8_t* src, int src_w, int src_h, int n, const float* corners, uint32_t flags,
                                  uint8_t* chunks_out, uint32_t* chunk_count, uint32_t* chunk_mask, uint8_t* frame_flags)
{
    int rc = check_camera_flags(flags); if (rc) return rc;
    if (!c || !src || !corners || !chunks_out || !chunk_count || n < 0 || n > c->max_frames) return fail(CB200_ERR_ARG, "bad arguments");
    if (n == 0) return CB200_OK;
    rc = check_frozen_deskew(c, n); if (rc) return rc;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    rc = stage_sources(c, src, src_w, src_h, n); if (rc) return rc;
    return cb200_extract_decode_fountain_dev(c, c->deskew->d_src, src_w, src_h, n, corners, flags, chunks_out, chunk_count, chunk_mask, frame_flags);
}

}  // extern "C"
