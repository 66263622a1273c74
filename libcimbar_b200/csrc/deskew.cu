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
#include "layout_core.cuh"

#include <cfloat>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

namespace cb200 {

struct DeskewState {
    DevBuf<uint8_t> d_table;       // n x 9 inverse maps (destination -> source) in double, then n PicDesc (the sources)
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
// The taps are fetched per the picture's layout (layout_core.cuh): the six bytes of a packed 3-byte pair or the eight of a 4-byte
// pair as above, two bytes from each plane of a planar picture, and reordered into the packed RGB pair the blend below reads; the
// frames are packed RGB whatever the pictures' layout.  Word loads stop short of the end of the picture (of each plane).  Without
// kLayouts every picture is packed RGB (row pitch 3 w) and the layout is not read: the packed batches' code, in fewer registers.
template <bool kLayouts>
__global__ void __launch_bounds__(256)
k_deskew(const double* __restrict__ minv, const PicDesc* __restrict__ desc, int n, int dst_w, int dst_h, int bw0, uint8_t* __restrict__ dst)
{
    const int quads = dst_w >> 2;
    const int per_frame = dst_h * quads;
    const int i = (int)(blockIdx.x * blockDim.x + threadIdx.x);
    if (i >= per_frame) return;
    const int y = i / quads, q = i - y * quads;
    const int x = 4 * q, bx = (x / bw0) * bw0;
    for (int f = (int)blockIdx.y; f < n; f += (int)gridDim.y) {
        const double* M = minv + (size_t)f * 9;
        const uint8_t* s = reinterpret_cast<const uint8_t*>(__ldg(&desc[f].src));
        const int src_w = __ldg(&desc[f].w), src_h = __ldg(&desc[f].h), lay = kLayouts ? __ldg(&desc[f].layout) : CB200_LAYOUT_RGB;
        const uint32_t pitch = kLayouts ? (uint32_t)__ldg(&desc[f].pitch) : 3u * (uint32_t)src_w, cpp = (uint32_t)layout::channels(lay);
        const uint64_t plane = kLayouts ? __ldg(&desc[f].plane) : 0;
        const uint8_t* const end = s + (size_t)(src_h - 1) * pitch + (size_t)src_w * cpp;
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
            off[u][0] = (uint32_t)cy0 * pitch + cpp * (uint32_t)c;
            off[u][1] = (uint32_t)cy1 * pitch + cpp * (uint32_t)c;
        }
        uint32_t lo[4][2], hi[4][2];
        if (lay == CB200_LAYOUT_RGB_PLANAR) {
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                layout::planar_pair(s + off[u][0], plane, end, lo[u][0], hi[u][0]);
                layout::planar_pair(s + off[u][1], plane, end, lo[u][1], hi[u][1]);
            }
        } else {
            const uint32_t nb = 2u * cpp;
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                layout::load_bytes(s + off[u][0], end, nb, lo[u][0], hi[u][0]);
                layout::load_bytes(s + off[u][1], end, nb, lo[u][1], hi[u][1]);
            }
            if (lay != CB200_LAYOUT_RGB) {
#pragma unroll
                for (int u = 0; u < 4; ++u) { layout::pair_rgb(lay, lo[u][0], hi[u][0]); layout::pair_rgb(lay, lo[u][1], hi[u][1]); }
            }
        }
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

// room for n deskewed frames in the output buffer
static int ensure_frames(cb200_ctx* c, int n)
{
    return grow(c, dstate(c)->d_dst, (size_t)n * c->mode.width * c->mode.height * 3, "deskew output");
}

// the batch of the uniform deskew and corner calls: n pictures of w x h packed from d (in host memory when `host`).  The deskew
// reads any picture of 2 x 2 or more: the scan's size rule is not theirs
static int deskew_batch(const uint8_t* d, int w, int h, int n, bool host, CameraBatch& b)
{
    if (n < 0) return fail(CB200_ERR_ARG, "n < 0");
    if (!d) return fail(CB200_ERR_ARG, "null pictures");
    if (n > 0 && (w < 2 || h < 2))
        return fail(CB200_ERR_ARG, "pictures of " + std::to_string(w) + " x " + std::to_string(h) + ": the deskew needs 2 x 2 or more");
    b.wh = uniform_sizes(w, h, n);
    b.pack(d);
    b.host = host;
    return CB200_OK;
}

// warpPerspective of the pictures of a device batch with the transforms m9 (n x 9, host), one frame each into d_dst
static int deskew_run(cb200_ctx* c, const CameraBatch& b, const double* m9, uint8_t* d_dst)
{
    const int n = b.n();
    DeskewState* d = dstate(c);
    const size_t table_bytes = (sizeof(double) * 9 + sizeof(PicDesc)) * (size_t)n;
    CK(d->d_table.ensure(table_bytes), "cudaMalloc transforms");
    // warpPerspective inverts the transform it is given (no WARP_INVERSE_MAP): cv::invert, DECOMP_LU; a singular matrix maps
    // everything to (0, 0) there (invert leaves zeros) -- reported here instead
    int slot;
    uint8_t* table;
    int rc = c->upload.take(table_bytes, &slot, &table); if (rc) return rc;
    double* inv = reinterpret_cast<double*>(table);
    PicDesc* desc = reinterpret_cast<PicDesc*>(inv + 9 * (size_t)n);
    for (int f = 0; f < n; ++f) {
        if (!extract::invert3(m9 + (size_t)f * 9, inv + (size_t)f * 9)) return fail(CB200_ERR_ARG, "singular perspective transform");
        const cb200_picture& p = b.pics[(size_t)f];
        const uint64_t plane = p.layout == CB200_LAYOUT_RGB_PLANAR ? (uint64_t)p.plane_pitch : 0;     // ignored in the other layouts
        desc[f] = PicDesc{reinterpret_cast<uint64_t>(p.data), 0, p.w, p.h, 0, 0, (uint64_t)p.row_pitch, plane, p.layout};
    }
    rc = c->upload.send(c->stream, slot, d->d_table, table_bytes); if (rc) return rc;
    const double* d_inv = reinterpret_cast<const double*>(d->d_table.get());
    return deskew_launch(c, b, d_inv, reinterpret_cast<const PicDesc*>(d_inv + 9 * (size_t)n), d_dst);
}

// Extractor::extract (Extractor.h:30-46): NEEDS_SHARPEN unless every side of the corner quadrilateral spans more than the frame in x
// or in y (Corners::is_granular_scale, Corners.h:57-75)
static std::vector<uint8_t> sharpen_from_corners(const cb200_ctx* c, const float* corners, int n)
{
    std::vector<uint8_t> sharpen((size_t)n);
    for (int i = 0; i < n; ++i) sharpen[(size_t)i] = extract::is_granular_scale(corners + 8 * (size_t)i, c->mode.width, c->mode.height) ? 0 : 1;
    return sharpen;
}

// the corner calls: the batch checked and staged, deskewed on the caller's corners and decoded, the results copied out.  With
// CB200_FLAG_SHARPEN_IF_NEEDED the corners decide which frames are sharpened
template <class Build>
static int extract_decode(cb200_ctx* c, Build&& build, const float* corners, uint32_t flags, uint8_t* chunks_out, uint32_t* chunk_count,
                          uint32_t* chunk_mask, uint8_t* frame_flags)
{
    CameraBatch b;
    int rc = check_camera_call(c, flags, build, b, !corners ? "null corners" : chunks_out && chunk_count ? nullptr : "null output");
    if (rc) return rc;
    const int n = b.n();
    if (n == 0) return CB200_OK;
    rc = check_frozen_deskew(c, n); if (rc) return rc;
    const Mode& m = c->mode;
    float outp[8];
    extract::output_points(m.width, m.height, outp);
    std::vector<double> m9((size_t)n * 9);
    for (int f = 0; f < n; ++f) {
        rc = cb200_perspective_transform(corners + (size_t)f * 8, outp, m9.data() + (size_t)f * 9); if (rc) return rc;
    }
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    rc = stage_batch(c, b); if (rc) return rc;
    rc = ensure_frames(c, n); if (rc) return rc;
    rc = deskew_run(c, b, m9.data(), c->deskew->d_dst); if (rc) return rc;
    // the deskewed frames never leave the device: straight into the decode
    const bool if_needed = (flags & CB200_FLAG_SHARPEN_IF_NEEDED) != 0;
    const std::vector<uint8_t> sharpen = if_needed ? sharpen_from_corners(c, corners, n) : std::vector<uint8_t>();
    return decode_fountain_to_host(c, c->deskew->d_dst, n, flags & ~CB200_FLAG_SHARPEN_IF_NEEDED, if_needed ? sharpen.data() : nullptr,
                                   chunks_out, chunk_count, chunk_mask, frame_flags);
}

}  // namespace cb200

int cb200::deskew_reserve(cb200_ctx* c, int n) { return ensure_frames(c, n); }

int cb200::deskew_frames(cb200_ctx* c, int n, uint8_t** frames)
{
    int rc = ensure_frames(c, n); if (rc) return rc;
    *frames = c->deskew->d_dst;
    return CB200_OK;
}

int cb200::deskew_launch(cb200_ctx* c, const CameraBatch& b, const double* d_minv, const PicDesc* d_desc, uint8_t* d_dst)
{
    const Mode& m = c->mode;
    const int n = b.n();
    // OpenCV's block geometry (WarpPerspectiveInvoker): bh0 = min(16, H); bw0 = min(1024 / bh0, W)
    const int bh0 = m.height < 16 ? m.height : 16;
    int bw0 = 1024 / bh0; if (bw0 > m.width) bw0 = m.width;
    const int per_frame = m.height * (m.width / 4);
    const dim3 grid((unsigned)((per_frame + 255) / 256), (unsigned)(n < 32768 ? n : 32768));
    if (!b.packed) k_deskew<true><<<grid, 256, 0, c->stream>>>(d_minv, d_desc, n, m.width, m.height, bw0, d_dst);
    else k_deskew<false><<<grid, 256, 0, c->stream>>>(d_minv, d_desc, n, m.width, m.height, bw0, d_dst);
    count_launch();
    CK(cudaGetLastError(), "deskew launch");
    return CB200_OK;
}

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
    CameraBatch b;
    int rc = deskew_batch(d_src, src_w, src_h, n, false, b);
    if (rc || (rc = check_spans(b))) return rc;
    if (!c || !m9 || !d_dst) return fail(CB200_ERR_ARG, !c ? "null context" : "null argument");
    rc = check_frozen_deskew(c, n); if (rc) return rc;
    if (n == 0) return CB200_OK;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    return deskew_run(c, b, m9, d_dst);
}

int cb200_deskew_pictures_dev(cb200_ctx* c, const cb200_picture* pics, int n, const double* m9, uint8_t* d_dst)
{
    CameraBatch b;
    int rc = picture_batch(pics, n, b);
    if (rc || (rc = check_spans(b))) return rc;
    if (!c || !m9 || !d_dst) return fail(CB200_ERR_ARG, !c ? "null context" : "null argument");
    rc = check_frozen_deskew(c, n); if (rc) return rc;
    if (n == 0) return CB200_OK;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    return deskew_run(c, b, m9, d_dst);
}

int cb200_deskew(cb200_ctx* c, const uint8_t* src, int src_w, int src_h, int n, const double* m9, uint8_t* dst)
{
    CameraBatch b;
    int rc = deskew_batch(src, src_w, src_h, n, true, b);
    if (rc || (rc = check_spans(b))) return rc;
    if (!c || !dst) return fail(CB200_ERR_ARG, !c ? "null context" : "null output");
    if (n > c->max_frames) return fail(CB200_ERR_ARG, "n = " + std::to_string(n) + " > max_frames = " + std::to_string(c->max_frames));
    if (n == 0) return CB200_OK;
    if (!m9) return fail(CB200_ERR_ARG, "null argument");
    rc = check_frozen_deskew(c, n); if (rc) return rc;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    rc = stage_batch(c, b); if (rc) return rc;
    rc = ensure_frames(c, n); if (rc) return rc;
    rc = deskew_run(c, b, m9, c->deskew->d_dst); if (rc) return rc;
    CK(cudaMemcpyAsync(dst, c->deskew->d_dst, (size_t)n * c->mode.width * c->mode.height * 3, cudaMemcpyDeviceToHost, c->stream), "D2H frames");
    CK(cudaStreamSynchronize(c->stream), "sync");
    return CB200_OK;
}

int cb200_extract_decode_fountain_dev(cb200_ctx* c, const uint8_t* d_src, int src_w, int src_h, int n, const float* corners, uint32_t flags,
                                      uint8_t* chunks_out, uint32_t* chunk_count, uint32_t* chunk_mask, uint8_t* frame_flags)
{
    auto build = [&](CameraBatch& b) { return deskew_batch(d_src, src_w, src_h, n, false, b); };
    return extract_decode(c, build, corners, flags, chunks_out, chunk_count, chunk_mask, frame_flags);
}

int cb200_extract_decode_fountain_ragged_dev(cb200_ctx* c, const uint8_t* d_src, const int32_t* wh, int n, const float* corners, uint32_t flags,
                                             uint8_t* chunks_out, uint32_t* chunk_count, uint32_t* chunk_mask, uint8_t* frame_flags)
{
    auto build = [&](CameraBatch& b) { return packed_batch(d_src, wh, n, b); };
    return extract_decode(c, build, corners, flags, chunks_out, chunk_count, chunk_mask, frame_flags);
}

int cb200_extract_decode_fountain(cb200_ctx* c, const uint8_t* src, int src_w, int src_h, int n, const float* corners, uint32_t flags,
                                  uint8_t* chunks_out, uint32_t* chunk_count, uint32_t* chunk_mask, uint8_t* frame_flags)
{
    auto build = [&](CameraBatch& b) { return deskew_batch(src, src_w, src_h, n, true, b); };
    return extract_decode(c, build, corners, flags, chunks_out, chunk_count, chunk_mask, frame_flags);
}

}  // extern "C"
