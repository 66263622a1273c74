// scan.cu -- the extractor's anchor scan on the device (SURVEY.md 8f-2: the step in front of the deskew), sm_90a.
//
// Replaces, for a batch of camera pictures resident in HBM (reference file:line relative to /root/reference/src/lib/extractor/):
//   Scanner::Scanner / preprocess_image(fast)   Scanner.h:146-174   cvtColor(RGB2GRAY) + GaussianBlur(unit x unit, sigma 0) + Otsu
//   Scanner::scan                               Scanner.cpp:182-199 scan_primary (t1 rows -> t2 column -> t3 diagonal -> t4 confirm,
//                                                                   filter_candidates, sort_top_to_bottom) + add_bottom_right_corner
//   Extractor::extract                          Extractor.h:30-46   scan -> Corners -> Deskewer (deskew.cu) -> NEEDS_SHARPEN test
// Four kernels:
//   k_scan_blur4<R>  gray + separable fixed-point Gaussian (OpenCV's 8-bit path: coefficients / 256 from its small-kernel
//                    table, BORDER_REFLECT_101, (sum + 2^15) >> 16) in 128 x 32 tiles staged in shared memory, plus the
//                    picture's 256-bin histogram (shared-memory atomics, one global atomic per bin and tile)
//   k_scan_otsu      getThreshVal_Otsu_8u in double precision, one thread per picture (no FMA contraction)
//   k_scan_anchors   one CTA per picture runs scan_core.cuh's scan_picture: the rows of a t1 pass and the confirmation chains
//                    of its hits are spread over the threads, the order-dependent tail (on_t1_scan's shadow test, libstdc++'s
//                    std::sort, the bottom-right window) runs on thread 0
//   k_extract        one thread per picture runs extract_core.cuh's extract_picture on the scan's results in place: status,
//                    corners, getPerspectiveTransform, its inverse (k_deskew's map) and the sharpen byte -- the camera calls
//                    never bring the anchors to the host
// The pixel work (gray/blur/histogram) moves 3 bytes in and 1 out per pixel (bound by
// instruction issue, not by HBM); the scan itself touches ~60 rows and a few hundred short lines of the blurred picture.
#include "ctx.cuh"
#include "scan_core.cuh"
#include "extract_core.cuh"
#include "layout_core.cuh"
#include "receivers_core.cuh"
#include "combine_core.cuh"
#include "k2_rs.cuh"

#include <algorithm>
#include <string>
#include <vector>

namespace cb200 {

using namespace scan;

struct ScanScratch {                 // per-context scratch of the scan entry points
    DevBuf<uint8_t> d_pics;                                 // host pictures of any call, staged (stage_batch)
    DevBuf<uint8_t> d_blur;                                 // blurred gray, n x h x w
    DevBuf<unsigned> d_hist; DevBuf<int> d_thr;
    DevBuf<Anchor> d_rowbuf; DevBuf<int> d_rowcnt; DevBuf<Anchor> d_pts; DevBuf<Anchor> d_res; DevBuf<int> d_nres;
    int ws_pics = 0, ws_rows_cap = 0;
    DevBuf<int4> d_anchors; DevBuf<int> d_count; DevBuf<unsigned> d_cutoff; DevBuf<int> d_status;
    PinnedBuf<int4> h_anchors; PinnedBuf<int> h_count;      // results: [n][4] anchors, then count / cutoff / status per picture
    DevBuf<uint8_t> d_table;                                // n PicDesc, then the pictures grouped by blur radius (n int)
    // the camera calls: per picture the inverse map k_deskew reads, the forward map (cb200_camera_transforms), the status of the
    // synchronous entry points; camera_n = the pictures of the last camera call
    DevBuf<double> d_minv, d_fwd; DevBuf<int32_t> d_ext_status;
    int camera_n = 0;
};

void scan_destroy(ScanScratch* s) { delete s; }

// ---------------------------------------------------------------------------------------------- gray + blur + histogram
template <int R> struct BlurK;
template <> struct BlurK<1> { __device__ static constexpr unsigned c(int i) { return i == 1 ? 128u : 64u; } };
template <> struct BlurK<2> { __device__ static constexpr unsigned c(int i) { return i == 2 ? 96u : ((i == 1 || i == 3) ? 64u : 16u); } };
template <> struct BlurK<3> { __device__ static constexpr unsigned c(int i) { return i == 3 ? 72u : ((i == 2 || i == 4) ? 56u : ((i == 1 || i == 5) ? 28u : 8u)); } };
template <> struct BlurK<4> {
    __device__ static constexpr unsigned c(int i) { return i == 4 ? 60u : ((i == 3 || i == 5) ? 51u : ((i == 2 || i == 6) ? 30u : ((i == 1 || i == 7) ? 13u : 4u))); }
};

__device__ __forceinline__ int reflect101_clamped(int p, int n)
{   // BORDER_REFLECT_101 for the positions a filter tap can reach (|overshoot| < n); far-outside tile padding is clamped (unused)
    if (p < 0) p = -p;
    if (p >= n) p = 2 * n - 2 - p;
    return p < 0 ? 0 : (p >= n ? n - 1 : p);
}

constexpr int kBlurTW = 128, kBlurTH = 32, kBlurThreads = 256;

// The pixel work is bound by instruction issue, not by HBM, so every thread takes four consecutive pixels: the twelve RGB bytes come
// as three aligned words and are converted with K1's IDP.2A form (8 instructions per four pixels), the horizontal taps are IDP.4A dot
// products of realigned gray words with the packed coefficients, the vertical pass reads four 16-bit sums per 64-bit load, and a warp
// owns a tile row (no divisions).
// The word path needs 4-byte aligned rows: a picture width that is a multiple of four, aligned source and blurred bases and an
// aligned row (and plane) pitch (decided per picture by the host: in a packed batch a picture that follows one of odd area starts
// unaligned); otherwise, and in tiles that cross the right edge, pixels are fetched one by one.  The gray comes from the picture's
// layout (layout_core.cuh): the IDP.2A form with the coefficients in the channel order for 3-byte pixels, one word per 4-byte
// pixel, one word per plane for planar pictures.
template <int R> struct BlurKW {     // the 2R+1 coefficients as bytes of up to three words (IDP.4A operands)
    __device__ static constexpr uint32_t w(int i)
    {
        return (4 * i + 0 <= 2 * R ? BlurK<R>::c(4 * i + 0) : 0u) | ((4 * i + 1 <= 2 * R ? BlurK<R>::c(4 * i + 1) : 0u) << 8) |
               ((4 * i + 2 <= 2 * R ? BlurK<R>::c(4 * i + 2) : 0u) << 16) | ((4 * i + 3 <= 2 * R ? BlurK<R>::c(4 * i + 3) : 0u) << 24);
    }
};

// One launch per radius over the flattened tiles of that radius' pictures: order[0 .. npics) lists them (batch indices into the
// descriptor table, in batch order), their tiles are numbered consecutively from desc[order[k]].tile0, row-major inside a picture.
// A CTA finds its picture by division when all listed pictures have one size (uniform_tiles tiles each), else by binary search.
// kLayouts: the pictures' layouts and pitches come from the table; without it every picture is packed RGB (row pitch 3 w), the
// code the packed batches have always run (fewer registers)
// The tile body, shared by k_scan_blur4 (tile t = its block) and k_scan_blur4_list (a grid-stride loop over the listed tiles).  Every
// shared array a tile writes is read only before its last barrier, so the next tile of the same CTA may start at once
static_assert(kBlurTW == layout::kBlurTileW && kBlurTH == layout::kBlurTileH, "the plan's tile counts are the blur's");
template <int R, bool kLayouts>
__device__ __forceinline__ void blur_tile(uint8_t* __restrict__ out, const PicDesc* __restrict__ desc, const int* __restrict__ order, int npics,
                                          int uniform_tiles, unsigned* __restrict__ hist, const int t)
{
    constexpr int GH = kBlurTH + 2 * R, GP = kBlurTW + 8, NW = (2 * R + 1 + 3) / 4;      // gray pitch: interior at byte 4
    __shared__ __align__(16) uint8_t g[GH][GP];
    __shared__ __align__(16) uint16_t hs[GH][kBlurTW];
    __shared__ unsigned lh[256];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    int k;
    if (uniform_tiles) {
        k = t / uniform_tiles;
    } else {
        int lo = 0, hi = npics - 1;
        while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (__ldg(&desc[__ldg(order + mid)].tile0) <= t) lo = mid; else hi = mid - 1; }
        k = lo;
    }
    const int pic = __ldg(order + k);
    const PicDesc* d = desc + pic;
    const int w = __ldg(&d->w), h = __ldg(&d->h), words_ok = __ldg(&d->words);
    const int tiles_x = (w + kBlurTW - 1) / kBlurTW, tl = t - __ldg(&d->tile0), tyi = tl / tiles_x;
    const int tx0 = (tl - tyi * tiles_x) * kBlurTW, ty0 = tyi * kBlurTH;
    const uint8_t* src = reinterpret_cast<const uint8_t*>(__ldg(&d->src));
    const size_t pitch = kLayouts ? __ldg(&d->pitch) : 3 * (size_t)w;
    const uint64_t plane = kLayouts ? __ldg(&d->plane) : 0;
    const int lay = kLayouts ? __ldg(&d->layout) : CB200_LAYOUT_RGB;
    const layout::Fetch fx = layout::fetch_of(lay, plane);
    lh[tid] = 0;
    // ---- gray of the tile and its halo
    const int x = tx0 + 4 * lane;
    for (int r = warp; r < GH; r += kBlurThreads / 32) {
        const int y = reflect101_clamped(ty0 - R + r, h);
        const uint8_t* row = src + (size_t)y * pitch;
        uint32_t g4;
        if (words_ok && x + 3 < w) {
            g4 = layout::gray4_words(row, x, plane, lay);
        } else {
            g4 = 0;
#pragma unroll
            for (int k = 0; k < 4; ++k) g4 |= layout::gray_px(row, reflect101_clamped(x + k, w), fx) << (8 * k);
        }
        *reinterpret_cast<uint32_t*>(&g[r][4 + 4 * lane]) = g4;
        if (lane < 2 * R) {                               // halo columns: R to the left of the tile, R to the right
            const int xx = lane < R ? tx0 - R + lane : tx0 + kBlurTW + (lane - R);
            g[r][lane < R ? 4 - R + lane : 4 + kBlurTW + (lane - R)] = (uint8_t)layout::gray_px(row, reflect101_clamped(xx, w), fx);
        }
    }
    __syncthreads();
    // ---- horizontal pass: output j of the thread is pixel 4 lane + j = gray byte 8 + 4 lane + j - 4; its taps start at byte 4 + j - R of the
    // 16-byte window (wA, wB, wC, 0) that begins at byte 4 lane of the row
    for (int r = warp; r < GH; r += kBlurThreads / 32) {
        const uint32_t* gw = reinterpret_cast<const uint32_t*>(&g[r][4 * lane]);
        const uint32_t W4[5] = {gw[0], gw[1], gw[2], 0u, 0u};
        uint32_t sums[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int t = 4 + j - R, wi = t >> 2, sh = 8 * (t & 3);
            uint32_t acc = 0;
#pragma unroll
            for (int k = 0; k < NW; ++k) {
                const uint32_t d = sh ? __funnelshift_r(W4[wi + k], W4[wi + k + 1 < 5 ? wi + k + 1 : 4], sh) : W4[wi + k];
                acc = __dp4a(d, BlurKW<R>::w(k), acc);
            }
            sums[j] = acc;                                // <= 255 * 256
        }
        *reinterpret_cast<uint2*>(&hs[r][4 * lane]) = make_uint2(sums[0] | (sums[1] << 16), sums[2] | (sums[3] << 16));
    }
    __syncthreads();
    // ---- vertical pass, histogram, store
    uint8_t* dst = out + __ldg(&d->blur);
    for (int r = warp; r < kBlurTH; r += kBlurThreads / 32) {
        const int y = ty0 + r;
        if (y >= h) break;
        uint32_t a0 = 32768u, a1 = 32768u, a2 = 32768u, a3 = 32768u;
#pragma unroll
        for (int k = 0; k < 2 * R + 1; ++k) {
            const uint2 v = *reinterpret_cast<const uint2*>(&hs[r + k][4 * lane]);
            const uint32_t c = BlurK<R>::c(k);
            a0 += c * (v.x & 0xFFFFu); a1 += c * (v.x >> 16); a2 += c * (v.y & 0xFFFFu); a3 += c * (v.y >> 16);
        }
        const uint32_t v0 = a0 >> 16, v1 = a1 >> 16, v2 = a2 >> 16, v3 = a3 >> 16;
        uint8_t* o = dst + (size_t)y * w + x;
        if (x + 3 < w) {
            if (words_ok) *reinterpret_cast<uint32_t*>(o) = v0 | (v1 << 8) | (v2 << 16) | (v3 << 24);
            else { o[0] = (uint8_t)v0; o[1] = (uint8_t)v1; o[2] = (uint8_t)v2; o[3] = (uint8_t)v3; }
            atomicAdd(&lh[v0], 1u); atomicAdd(&lh[v1], 1u); atomicAdd(&lh[v2], 1u); atomicAdd(&lh[v3], 1u);
        } else {
            if (x < w) { o[0] = (uint8_t)v0; atomicAdd(&lh[v0], 1u); }
            if (x + 1 < w) { o[1] = (uint8_t)v1; atomicAdd(&lh[v1], 1u); }
            if (x + 2 < w) { o[2] = (uint8_t)v2; atomicAdd(&lh[v2], 1u); }
        }
    }
    __syncthreads();
    if (lh[tid]) atomicAdd(&hist[(size_t)pic * 256 + tid], lh[tid]);
}

template <int R, bool kLayouts>
__global__ void __launch_bounds__(kBlurThreads)
k_scan_blur4(uint8_t* __restrict__ out, const PicDesc* __restrict__ desc, const int* __restrict__ order, int npics, int uniform_tiles,
             unsigned* __restrict__ hist)
{
    blur_tile<R, kLayouts>(out, desc, order, npics, uniform_tiles, hist, (int)blockIdx.x);
}

// k_scan_blur4 over a plan's device table (k_plan_pictures): radius group `group` lists counts[group] pictures in order, with
// counts[3 + group] tiles between them, both written at this launch -- persistent CTAs walk the tiles, none idle while tiles remain
template <int R>
__global__ void __launch_bounds__(kBlurThreads)
k_scan_blur4_list(uint8_t* __restrict__ out, const PicDesc* __restrict__ desc, const int* __restrict__ order, const int* __restrict__ counts,
                  int group, unsigned* __restrict__ hist)
{
    const int npics = counts[group], tiles = counts[3 + group];
    for (int t = (int)blockIdx.x; t < tiles; t += (int)gridDim.x) blur_tile<R, true>(out, desc, order, npics, 0, hist, t);
}

// k_scan_blur4_list's grid: as many CTAs as the GPU holds at once (more would wait for a whole CTA's share of the tiles), at most one
// per tile of the largest batch
template <int R>
static int blur_list_grid(const cb200_ctx* c, int64_t most, unsigned* grid)
{
    int per_sm = 0;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_scan_blur4_list<R>, kBlurThreads, 0), "blur occupancy");
    *grid = (unsigned)std::max<int64_t>(1, std::min<int64_t>(most, (int64_t)per_sm * c->sm_count));
    return CB200_OK;
}

// ---------------------------------------------------------------------------------------------- Otsu
// cv::threshold(THRESH_OTSU) -> getThreshVal_Otsu_8u (modules/imgproc/src/thresh.cpp), double precision, operation for operation
__global__ void k_scan_otsu(const unsigned* __restrict__ hist, const PicDesc* __restrict__ desc, int n, int* __restrict__ thr)
{
    const int pic = blockIdx.x * blockDim.x + threadIdx.x;
    if (pic >= n) return;
    const unsigned* hh = hist + (size_t)pic * 256;
    const double npx = (double)((long long)desc[pic].w * desc[pic].h);
    const double scale = ddiv(1., npx);
    double mu = 0;
    for (int i = 0; i < 256; ++i) mu = dadd(mu, dmul((double)i, (double)hh[i]));
    mu = dmul(mu, scale);
    double mu1 = 0, q1 = 0, max_sigma = 0;
    int max_val = 0;
    const double eps = 1.1920928955078125e-07;        // FLT_EPSILON
    for (int i = 0; i < 256; ++i) {
        const double p_i = dmul((double)hh[i], scale);
        mu1 = dmul(mu1, q1);
        q1 = dadd(q1, p_i);
        const double q2 = dsub(1., q1);
        const double lo = q1 < q2 ? q1 : q2, hi = q1 > q2 ? q1 : q2;
        if (lo < eps || hi > dsub(1., eps)) continue;
        mu1 = ddiv(dadd(mu1, dmul((double)i, p_i)), q1);
        const double mu2 = ddiv(dsub(mu, dmul(q1, mu1)), q2);
        const double d = dsub(mu1, mu2);
        const double sigma = dmul(dmul(dmul(q1, q2), d), d);
        if (sigma > max_sigma) { max_sigma = sigma; max_val = i; }
    }
    thr[pic] = max_val;
}

// ---------------------------------------------------------------------------------------------- the scan
constexpr int kScanThreads = 256;

__global__ void __launch_bounds__(kScanThreads)
k_scan_anchors(const uint8_t* __restrict__ blurred, const PicDesc* __restrict__ desc, const int* __restrict__ thr, int rows_cap,
               Anchor* rowbuf, int* rowcnt, Anchor* pts, Anchor* res, int* nres,
               int4* __restrict__ anchors_out, int* __restrict__ count_out, unsigned* __restrict__ cutoff_out, int* __restrict__ status_out)
{
    __shared__ PicShared sh;
    const int pic = blockIdx.x;
    Anchor* out = reinterpret_cast<Anchor*>(anchors_out + (size_t)pic * 4);
    if (threadIdx.x < 4) out[threadIdx.x] = mk(0, 0, 0, 0);
    __syncthreads();
    Img im;
    im.px = blurred + desc[pic].blur; im.w = desc[pic].w; im.h = desc[pic].h; im.thr = thr[pic];
    PicWs ws;
    ws.rowbuf = rowbuf + (size_t)pic * rows_cap * kRowCap; ws.rowcnt = rowcnt + (size_t)pic * rows_cap;
    ws.pts = pts + (size_t)pic * kPtsCap; ws.res = res + (size_t)pic * kPtsCap * kResCap; ws.nres = nres + (size_t)pic * kPtsCap;
    ws.rows_cap = rows_cap;
    Exec ex;
    ex.tid = threadIdx.x; ex.nthreads = kScanThreads;
    const int count = scan_picture(ex, im, ws, sh, out, cutoff_out + pic, status_out + pic);
    if (threadIdx.x == 0) count_out[pic] = count;
}

static ScanScratch* sstate(cb200_ctx* c)
{
    if (!c->scan) c->scan = new ScanScratch();
    return c->scan;
}

static int scan_blur_radius(int w, int h) { return layout::blur_radius(w, h); }

int check_picture_sizes(const int32_t* wh, int n)
{
    for (int i = 0; i < n; ++i) {
        const int w = wh[2 * i], h = wh[2 * i + 1];
        if ((w < h ? w : h) < 60)
            return fail(CB200_ERR_ARG, "picture " + std::to_string(i) + " is " + std::to_string(w) + " x " + std::to_string(h) +
                                           ": smaller than 60 pixels on its short side (Scanner's row step would be 0)");
        if (scan_blur_radius(w, h) > 4)
            return fail(CB200_ERR_ARG, "picture " + std::to_string(i) + " is " + std::to_string(w) + " x " + std::to_string(h) +
                                           ": pictures with a short side of 4500 pixels or more need a Gaussian kernel beyond 9 taps, which is not restated");
    }
    return CB200_OK;
}

std::vector<int32_t> uniform_sizes(int w, int h, int n)
{
    std::vector<int32_t> wh(2 * (size_t)(n > 0 ? n : 0));
    for (int i = 0; i < n; ++i) { wh[2 * (size_t)i] = w; wh[2 * (size_t)i + 1] = h; }
    return wh;
}

void CameraBatch::pack(const uint8_t* d)
{
    pics.resize((size_t)n());
    size_t off = 0;
    for (int i = 0; i < n(); ++i) {
        const int w = wh[2 * (size_t)i], h = wh[2 * (size_t)i + 1];
        pics[(size_t)i] = cb200_picture{d ? d + off : nullptr, w, h, 3 * (int64_t)w, 0, CB200_LAYOUT_RGB};
        off += 3 * (size_t)w * (size_t)h;
    }
    packed = true;
}

// the checks every builder of a packed or host batch starts with; b.wh = the sizes
static int sized_batch(const void* pictures, const int32_t* wh, int n, CameraBatch& b)
{
    if (n < 0) return fail(CB200_ERR_ARG, "n < 0");
    if (!wh) return fail(CB200_ERR_ARG, "null wh");
    if (!pictures) return fail(CB200_ERR_ARG, "null pictures");
    int rc = check_picture_sizes(wh, n); if (rc) return rc;
    b.wh.assign(wh, wh + 2 * (size_t)n);
    return CB200_OK;
}

int packed_batch(const uint8_t* d, const int32_t* wh, int n, CameraBatch& b)
{
    int rc = sized_batch(d, wh, n, b); if (rc) return rc;
    b.pack(d);
    return CB200_OK;
}

int uniform_batch(const uint8_t* d, int w, int h, int n, CameraBatch& b)
{
    if (n < 0) return fail(CB200_ERR_ARG, "n < 0");
    if (!d) return fail(CB200_ERR_ARG, "null pictures");
    b.wh = uniform_sizes(w, h, n);
    int rc = check_picture_sizes(b.wh.data(), n); if (rc) return rc;
    b.pack(d);
    return CB200_OK;
}

int host_batch(const uint8_t* const* pictures, const int32_t* wh, int n, CameraBatch& b)
{
    int rc = sized_batch(pictures, wh, n, b); if (rc) return rc;
    b.pack(nullptr);
    for (int i = 0; i < n; ++i) {
        if (!pictures[i]) return fail(CB200_ERR_ARG, "picture " + std::to_string(i) + " is a null pointer");
        b.pics[(size_t)i].data = pictures[i];
    }
    b.host = true;
    return CB200_OK;
}

int picture_batch(const cb200_picture* pics, int n, CameraBatch& b)
{
    if (n < 0) return fail(CB200_ERR_ARG, "n < 0");
    if (!pics) return fail(CB200_ERR_ARG, "null pictures");
    b.wh.assign(2 * (size_t)n, 0);
    for (int i = 0; i < n; ++i) {
        const cb200_picture& p = pics[i];
        const std::string name = "picture " + std::to_string(i);
        if (!p.data) return fail(CB200_ERR_ARG, name + " has a null data pointer");
        if (!layout::known(p.layout)) return fail(CB200_ERR_ARG, name + " has an unknown layout " + std::to_string(p.layout));
        if (p.row_pitch < 0 || p.plane_pitch < 0)
            return fail(CB200_ERR_ARG, name + " has a negative " + (p.row_pitch < 0 ? "row" : "plane") + " pitch");
        b.wh[2 * (size_t)i] = p.w; b.wh[2 * (size_t)i + 1] = p.h;
    }
    int rc = check_picture_sizes(b.wh.data(), n); if (rc) return rc;
    b.packed = true;
    for (int i = 0; i < n; ++i) {
        const cb200_picture& p = pics[i];
        const int64_t row = (int64_t)p.w * layout::channels(p.layout);
        if (p.row_pitch < row)
            return fail(CB200_ERR_ARG, "picture " + std::to_string(i) + " has a row pitch of " + std::to_string(p.row_pitch) +
                                           " bytes, below w x channels = " + std::to_string(row));
        if (p.layout == CB200_LAYOUT_RGB_PLANAR && p.plane_pitch < (int64_t)p.h * p.row_pitch)
            return fail(CB200_ERR_ARG, "picture " + std::to_string(i) + " has overlapping planes: a plane pitch of " + std::to_string(p.plane_pitch) +
                                           " bytes, below h x row pitch = " + std::to_string((int64_t)p.h * p.row_pitch));
        b.packed = b.packed && p.layout == CB200_LAYOUT_RGB && p.row_pitch == row;
    }
    b.pics.assign(pics, pics + n);
    return CB200_OK;
}

int device_batch(const cb200_picture* d_pics, int n, const cb200_picture_bounds* bounds, CameraBatch& b)
{
    if (n < 0) return fail(CB200_ERR_ARG, "n < 0");
    if (!d_pics) return fail(CB200_ERR_ARG, "null d_pics");
    if (reinterpret_cast<uintptr_t>(d_pics) % 8) return fail(CB200_ERR_ARG, "d_pics is not 8-byte aligned");
    if (!bounds) return fail(CB200_ERR_ARG, "null bounds");
    const cb200_picture_bounds bd = *bounds;
    const std::string is = " (bounds " + std::to_string(bd.min_short) + ", " + std::to_string(bd.max_short) + ", " + std::to_string(bd.max_long) + ")";
    if (bd.min_short < 60) return fail(CB200_ERR_ARG, "min_short < 60: the scan's row step would be 0" + is);
    if (bd.max_short > 4499) return fail(CB200_ERR_ARG, "max_short > 4499: a short side of 4500 or more needs a Gaussian beyond 9 taps" + is);
    if (bd.min_short > bd.max_short) return fail(CB200_ERR_ARG, "min_short > max_short" + is);
    if (bd.max_long < bd.max_short) return fail(CB200_ERR_ARG, "max_long < max_short" + is);
    // the largest picture in either orientation: its blur tiles over n slots, and the scan rows of the smallest short side
    const int64_t tiles = std::max(layout::blur_tiles(bd.max_long, bd.max_short), layout::blur_tiles(bd.max_short, bd.max_long));
    if (tiles * n > 0x7FFFFFFFll) return fail(CB200_ERR_ARG, "n x the blur tiles of a max_long x max_short picture exceed 2^31 - 1" + is);
    const int64_t skip = bd.min_short / 60, rows = 2 * ((bd.max_long + skip - 1) / skip) + 4;
    if (rows > 0x7FFFFFFFll) return fail(CB200_ERR_ARG, "the scan rows of a max_long picture exceed 2^31 - 1" + is);
    b.pics.clear(); b.wh.clear();
    b.d_pics = d_pics; b.dev_n = n; b.bounds = bd;
    b.packed = false; b.host = false;
    return CB200_OK;
}

int check_spans(const CameraBatch& b)
{
    const int64_t lim = (int64_t)1 << 32;
    for (int i = 0; i < (int)b.pics.size(); ++i) {      // (a device batch: none on the host, each launch checks its own)
        const cb200_picture& p = b.pics[(size_t)i];
        const bool planar = p.layout == CB200_LAYOUT_RGB_PLANAR;
        if (p.row_pitch >= lim || (planar && p.plane_pitch >= lim) ||
            (planar ? 2 * p.plane_pitch : 0) + (int64_t)(p.h - 1) * p.row_pitch + (int64_t)p.w * layout::channels(p.layout) >= lim)
            return fail(CB200_ERR_ARG, "picture " + std::to_string(i) + " spans 4 GB or more");
    }
    return CB200_OK;
}

int stage_batch(cb200_ctx* c, CameraBatch& b)
{
    if (!b.host) return CB200_OK;
    ScanScratch* s = sstate(c);
    size_t bytes = 0;
    for (int i = 0; i < b.n(); ++i) bytes += 3 * (size_t)b.pics[(size_t)i].w * (size_t)b.pics[(size_t)i].h;
    CK(s->d_pics.ensure(bytes), "cudaMalloc picture staging");
    size_t off = 0;
    for (int i = 0; i < b.n();) {
        const uint8_t* src = b.pics[(size_t)i].data;
        size_t run = 0;
        do run += 3 * (size_t)b.pics[(size_t)i].w * (size_t)b.pics[(size_t)i].h;
        while (++i < b.n() && b.pics[(size_t)i].data == src + run);
        CK(cudaMemcpyAsync(s->d_pics + off, src, run, cudaMemcpyHostToDevice, c->stream), "H2D pictures");
        off += run;
    }
    b.pack(s->d_pics);
    b.host = false;
    return CB200_OK;
}

// rows of a scan pass for one picture: the primary pass scans h / skip rows, the bottom-right window at most 2 h / skip (half the step)
static int scan_rows(int w, int h)
{
    const int skip = (w < h ? w : h) / 60;
    return 2 * ((h + skip - 1) / skip) + 4;
}

// a device batch: each slot's blurred picture at a fixed offset, slot x this many bytes (a multiple of 4)
static size_t plan_slot_bytes(const cb200_picture_bounds& bd) { return ((size_t)bd.max_long * (size_t)bd.max_short + 3) & ~(size_t)3; }

// the scan's buffers for n pictures of npx pixels in all, whose scans take at most rows_cap rows
static int scan_reserve_for(cb200_ctx* c, int n, size_t npx, int rows_cap)
{
    ScanScratch* s = sstate(c);
    int rc;
    if ((rc = grow(c, s->d_blur, npx, "blurred pictures")) || (rc = grow(c, s->d_hist, 256 * (size_t)n, "histograms")) ||
        (rc = grow(c, s->d_thr, (size_t)n, "thresholds")) || (rc = grow(c, s->d_anchors, 4 * (size_t)n, "anchors")) ||
        (rc = grow(c, s->d_count, (size_t)n, "counts")) || (rc = grow(c, s->d_cutoff, (size_t)n, "cutoffs")) ||
        (rc = grow(c, s->d_status, (size_t)n, "status")))
        return rc;
    // the per-picture scan lists: k_scan_anchors strides them by the largest row count seen so far (raised once they fit)
    const size_t np = (size_t)(n > s->ws_pics ? n : s->ws_pics), rows = (size_t)(rows_cap > s->ws_rows_cap ? rows_cap : s->ws_rows_cap);
    if ((rc = grow(c, s->d_rowbuf, np * rows * kRowCap, "scan rows")) || (rc = grow(c, s->d_rowcnt, np * rows, "scan row counts")) ||
        (rc = grow(c, s->d_pts, np * kPtsCap, "scan points")) || (rc = grow(c, s->d_res, np * kPtsCap * kResCap, "scan results")) ||
        (rc = grow(c, s->d_nres, np * kPtsCap, "scan result counts")))
        return rc;
    s->ws_pics = (int)np; s->ws_rows_cap = (int)rows;
    return CB200_OK;
}

int scan_reserve(cb200_ctx* c, const int32_t* wh, int n)
{
    size_t npx = 0;
    int rows_cap = 0;
    for (int i = 0; i < n; ++i) {
        npx += (size_t)wh[2 * i] * (size_t)wh[2 * i + 1];
        const int rc = scan_rows(wh[2 * i], wh[2 * i + 1]);
        if (rc > rows_cap) rows_cap = rc;
    }
    return scan_reserve_for(c, n, npx, rows_cap);
}

// a device batch: every accepted picture's scan takes at most the rows of a min_short x max_long one (device_batch checked that
// they fit an int)
int scan_reserve(cb200_ctx* c, const CameraBatch& b)
{
    if (!b.d_pics) return scan_reserve(c, b.wh.data(), b.n());
    const cb200_picture_bounds& bd = b.bounds;
    return scan_reserve_for(c, b.n(), (size_t)b.n() * plan_slot_bytes(bd), scan_rows(bd.min_short, bd.max_long));
}

// the launch geometry of the blur: per radius its pictures, their first entry in the order list, their tiles, one size or not
struct BlurGroups {
    int count[5] = {}, group0[5] = {};
    long long tiles[5] = {};
    bool same[5] = {true, true, true, true, true};
};

// the descriptor table (batch order), then the pictures grouped by blur radius (batch order inside a group) into `table`; the tiles
// of one radius are numbered across its pictures.  The word path depends on where the pictures and the scan's blurred buffer are
static int pic_table(const ScanScratch* s, const CameraBatch& b, uint8_t* table, BlurGroups& g)
{
    const int n = b.n();
    const int32_t* wh = b.wh.data();
    const cb200_picture* pics = b.pics.data();
    PicDesc* desc = reinterpret_cast<PicDesc*>(table);
    int* order = reinterpret_cast<int*>(desc + n);
    int first[5] = {};
    for (int i = 0; i < n; ++i) {
        const int R = scan_blur_radius(wh[2 * i], wh[2 * i + 1]);
        if (!g.count[R]) first[R] = i;
        else g.same[R] = g.same[R] && wh[2 * i] == wh[2 * first[R]] && wh[2 * i + 1] == wh[2 * first[R] + 1];
        ++g.count[R];
    }
    size_t off = 0;
    int next[5] = {};
    for (int R = 1, at = 0; R <= 4; ++R) { next[R] = at; at += g.count[R]; }
    for (int R = 1; R <= 4; ++R) g.group0[R] = next[R];
    for (int i = 0; i < n; ++i) {
        const int w = wh[2 * i], h = wh[2 * i + 1], R = scan_blur_radius(w, h);
        const cb200_picture& p = pics[i];
        const bool planar = p.layout == CB200_LAYOUT_RGB_PLANAR;
        PicDesc& d = desc[i];
        d.src = reinterpret_cast<uint64_t>(p.data); d.blur = off; d.w = w; d.h = h;
        d.pitch = (uint64_t)p.row_pitch; d.plane = planar ? (uint64_t)p.plane_pitch : 0; d.layout = p.layout;
        d.words = (w % 4 == 0) && (d.src % 4 == 0) && (d.pitch % 4 == 0) && (d.plane % 4 == 0) &&
                  (reinterpret_cast<uintptr_t>(s->d_blur + d.blur) % 4 == 0);
        d.tile0 = (int)g.tiles[R];
        g.tiles[R] += (long long)((w + kBlurTW - 1) / kBlurTW) * ((h + kBlurTH - 1) / kBlurTH);
        if (g.tiles[R] > 0x7FFFFFFFll) return fail(CB200_ERR_ARG, "more than 2^31 blur tiles in one batch");
        order[next[R]++] = i;
        off += (size_t)w * (size_t)h;
    }
    return CB200_OK;
}

PlanTable::PlanTable(const CameraBatch& b)
{
    const size_t n = (size_t)b.n();
    order = sizeof(PicDesc) * n;
    groups = order + sizeof(int) * 3 * n;
    of = groups + sizeof(int) * 6;
    refused = of + sizeof(int32_t) * n;
    standin = (refused + n + 15) & ~(size_t)15;
    bytes = standin + 3 * (size_t)b.bounds.min_short + 16;
}

// A plan's picture table from the descriptors and the map of this launch (layout::plan_slot per slot; in a detect plan, the
// candidates too: a slot with no candidate mode below n_modes is empty, receivers::plan_modes), in one CTA whatever n: chunks
// of kPlanThreads slots, each numbered by a block scan of six sums (per radius group: slots, tiles) on top of the chunks before it.
// So each group's list is in slot order and its tiles are numbered consecutively in that order, as pic_table numbers them
constexpr int kPlanThreads = 1024;
__global__ void __launch_bounds__(kPlanThreads)
k_plan_pictures(int n, const cb200_picture* __restrict__ pics, const int32_t* __restrict__ receiver_of, int receivers,
                const uint32_t* __restrict__ cand, int n_modes, cb200_picture_bounds bounds, uint64_t standin, uint64_t blur_base, uint64_t slot_bytes, PicDesc* __restrict__ desc, int* __restrict__ order,
                int* __restrict__ counts, int32_t* __restrict__ of, uint8_t* __restrict__ refused)
{
    __shared__ int wsum[kPlanThreads / 32][6];
    __shared__ int carry[6];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid < 6) carry[tid] = 0;
    __syncthreads();
    for (int base = 0; base < n; base += kPlanThreads) {
        const int i = base + tid;
        layout::PlanSlot ps = {-1, 0, false};
        PicDesc d;
        int32_t r = -1;
        if (i < n) {
            r = receiver_of[i];
            const bool empty = receivers::plan_modes(cand ? cand[i] : ~0u, r, receivers, n_modes) == 0;
            ps = layout::plan_slot(pics, empty, bounds, standin, blur_base, slot_bytes, i, d);
        }
        int v[6];
#pragma unroll
        for (int k = 0; k < 3; ++k) { v[k] = ps.group == k; v[3 + k] = ps.group == k ? ps.tiles : 0; }
#pragma unroll
        for (int k = 0; k < 6; ++k)
            for (int o = 1; o < 32; o <<= 1) { const int u = __shfl_up_sync(~0u, v[k], o); if (lane >= o) v[k] += u; }
        if (lane == 31)
            for (int k = 0; k < 6; ++k) wsum[warp][k] = v[k];
        __syncthreads();
        if (warp == 0)
            for (int k = 0; k < 6; ++k) {
                int x = wsum[lane][k];
                for (int o = 1; o < 32; o <<= 1) { const int u = __shfl_up_sync(~0u, x, o); if (lane >= o) x += u; }
                wsum[lane][k] = x;
            }
        __syncthreads();
        if (i < n) {
            int at = 0, tile0 = 0;
#pragma unroll
            for (int k = 0; k < 3; ++k)
                if (ps.group == k) {
                    at = carry[k] + (warp ? wsum[warp - 1][k] : 0) + v[k] - 1;
                    tile0 = carry[3 + k] + (warp ? wsum[warp - 1][3 + k] : 0) + v[3 + k] - ps.tiles;
                }
            d.tile0 = tile0;
            desc[i] = d;
            order[(size_t)ps.group * n + at] = i;
            of[i] = ps.refused ? -1 : r;
            refused[i] = ps.refused;
        }
        __syncthreads();
        if (tid < 6) carry[tid] += wsum[kPlanThreads / 32 - 1][tid];
        __syncthreads();
    }
    if (tid < 6) counts[tid] = carry[tid];
}

int plan_pictures_launch(cb200_ctx* c, const CameraBatch& b, const int32_t* d_receiver_of, int receivers, uint8_t* d_table,
                         const uint32_t* d_cand, int n_modes)
{
    const PlanTable t(b);
    const ScanScratch* s = sstate(c);
    k_plan_pictures<<<1, kPlanThreads, 0, c->stream>>>(b.n(), b.d_pics, d_receiver_of, receivers, d_cand, n_modes, b.bounds, reinterpret_cast<uint64_t>(d_table + t.standin),
                                                      reinterpret_cast<uint64_t>(s->d_blur.get()), plan_slot_bytes(b.bounds),
                                                      reinterpret_cast<PicDesc*>(d_table), reinterpret_cast<int*>(d_table + t.order),
                                                      reinterpret_cast<int*>(d_table + t.groups), reinterpret_cast<int32_t*>(d_table + t.of),
                                                      d_table + t.refused);
    count_launch();
    CK(cudaGetLastError(), "plan pictures launch");
    return CB200_OK;
}

int camera_pictures(cb200_ctx* c) { return sstate(c)->camera_n; }
void set_camera_pictures(cb200_ctx* c, int n) { sstate(c)->camera_n = n; }

int pic_table(cb200_ctx* c, const CameraBatch& b, std::vector<uint8_t>& table)
{
    table.assign((sizeof(PicDesc) + sizeof(int)) * (size_t)b.n(), 0);
    BlurGroups g;
    return pic_table(sstate(c), b, table.data(), g);
}

// blurred pictures + thresholds + anchors for a device batch, in the state's device arrays; enqueued only.  The picture table
// (PicDesc, in s->d_table) is this call's one upload -- unless d_table holds it already (a camera plan's): then *d_desc = d_table
// and nothing is uploaded.  A receivers call's map travels behind the table, in the same slot, and so do a detect receivers call's
// lists (`tail`, 8-byte aligned on the device at *d_tail)
int camera_scan(cb200_ctx* c, const CameraBatch& b, const PicDesc* d_table, const PicDesc** d_desc_out, Receivers* recv,
                const std::vector<uint8_t>* tail, const uint8_t** d_tail)
{
    ScanScratch* s = sstate(c);
    cudaStream_t st = c->stream;
    const int n = b.n();
    int err = scan_reserve(c, b); if (err) return err;
    const size_t table_bytes = (sizeof(PicDesc) + sizeof(int)) * (size_t)n;
    BlurGroups g;
    const PicDesc* d_desc = d_table;
    if (b.d_pics) {
        // a plan over device descriptors: k_plan_pictures writes d_table at each launch, the host knows no sizes
    } else if (d_table) {
        std::vector<uint8_t> table(table_bytes);
        err = pic_table(s, b, table.data(), g); if (err) return err;
    } else {
        const size_t map_bytes = recv ? recv->bytes() : 0, tail_at = (table_bytes + map_bytes + 7) & ~(size_t)7;
        const size_t bytes = tail ? tail_at + tail->size() : table_bytes + map_bytes;
        CK(s->d_table.ensure(bytes), "cudaMalloc picture table");
        int slot;
        uint8_t* h_table;
        err = c->upload.take(bytes, &slot, &h_table); if (err) return err;
        err = pic_table(s, b, h_table, g); if (err) return err;
        if (recv) memcpy(h_table + table_bytes, recv->map.data(), map_bytes);
        if (tail) memcpy(h_table + tail_at, tail->data(), tail->size());
        err = c->upload.send(st, slot, s->d_table, bytes); if (err) return err;
        d_desc = reinterpret_cast<const PicDesc*>(s->d_table.get());
        if (recv) recv->map_on_device(reinterpret_cast<const int32_t*>(s->d_table + table_bytes), n);
        if (tail) *d_tail = s->d_table + tail_at;
    }
    if (d_desc_out) *d_desc_out = d_desc;
    const int* count = g.count;
    const int* group0 = g.group0;
    const long long* tiles = g.tiles;
    const bool* same = g.same;
    const bool layouts = !b.packed;
    const int* d_order = reinterpret_cast<const int*>(d_desc + n);
    CK(cudaMemsetAsync(s->d_hist, 0, sizeof(unsigned) * 256 * (size_t)n, st), "memset histograms");
    // cb200_set_timing: one event set per scan -- [blur + histogram (all radii), Otsu, anchors] through cb200_get_timing
    begin_timed_call(c);
    mark(c);
    if (b.d_pics) {
        // one launch per radius group the bounds reach (short sides min_short .. max_short), persistent CTAs over the listed tiles
        const PlanTable t(b);
        const uint8_t* tb = reinterpret_cast<const uint8_t*>(d_table);
        const int* d_ord = reinterpret_cast<const int*>(tb + t.order);
        const int* d_counts = reinterpret_cast<const int*>(tb + t.groups);
        const cb200_picture_bounds& bd = b.bounds;
        const int64_t most = (int64_t)n * std::max(layout::blur_tiles(bd.max_long, bd.max_short), layout::blur_tiles(bd.max_short, bd.max_long));
        const int g0 = layout::radius_group(layout::blur_radius(bd.min_short, bd.min_short));
        const int g1 = layout::radius_group(layout::blur_radius(bd.max_short, bd.max_short));
        for (int gi = g0; gi <= g1; ++gi) {
            const int* ord = d_ord + (size_t)gi * n;
            unsigned grid = 0;
            switch (gi) {
            case 0: if ((err = blur_list_grid<1>(c, most, &grid))) return err;
                    k_scan_blur4_list<1><<<grid, kBlurThreads, 0, st>>>(s->d_blur, d_desc, ord, d_counts, gi, s->d_hist); break;
            case 1: if ((err = blur_list_grid<2>(c, most, &grid))) return err;
                    k_scan_blur4_list<2><<<grid, kBlurThreads, 0, st>>>(s->d_blur, d_desc, ord, d_counts, gi, s->d_hist); break;
            default: if ((err = blur_list_grid<4>(c, most, &grid))) return err;
                     k_scan_blur4_list<4><<<grid, kBlurThreads, 0, st>>>(s->d_blur, d_desc, ord, d_counts, gi, s->d_hist); break;
            }
            count_launch();
        }
    }
    for (int R = 1; R <= 4 && !b.d_pics; ++R) {
        if (!count[R]) continue;
        const int uniform = same[R] ? (int)(tiles[R] / count[R]) : 0;
        const unsigned grid = (unsigned)tiles[R];
        const int* ord = d_order + group0[R];
        switch (R) {
        case 1: if (layouts) k_scan_blur4<1, true><<<grid, kBlurThreads, 0, st>>>(s->d_blur, d_desc, ord, count[R], uniform, s->d_hist);
                 else k_scan_blur4<1, false><<<grid, kBlurThreads, 0, st>>>(s->d_blur, d_desc, ord, count[R], uniform, s->d_hist); break;
        case 2: if (layouts) k_scan_blur4<2, true><<<grid, kBlurThreads, 0, st>>>(s->d_blur, d_desc, ord, count[R], uniform, s->d_hist);
                 else k_scan_blur4<2, false><<<grid, kBlurThreads, 0, st>>>(s->d_blur, d_desc, ord, count[R], uniform, s->d_hist); break;
        case 3: if (layouts) k_scan_blur4<3, true><<<grid, kBlurThreads, 0, st>>>(s->d_blur, d_desc, ord, count[R], uniform, s->d_hist);
                 else k_scan_blur4<3, false><<<grid, kBlurThreads, 0, st>>>(s->d_blur, d_desc, ord, count[R], uniform, s->d_hist); break;
        default: if (layouts) k_scan_blur4<4, true><<<grid, kBlurThreads, 0, st>>>(s->d_blur, d_desc, ord, count[R], uniform, s->d_hist);
                 else k_scan_blur4<4, false><<<grid, kBlurThreads, 0, st>>>(s->d_blur, d_desc, ord, count[R], uniform, s->d_hist); break;
        }
        count_launch();
    }
    mark(c);
    k_scan_otsu<<<(n + 63) / 64, 64, 0, st>>>(s->d_hist, d_desc, n, s->d_thr); count_launch();
    mark(c);
    k_scan_anchors<<<n, kScanThreads, 0, st>>>(s->d_blur, d_desc, s->d_thr, s->ws_rows_cap, s->d_rowbuf, s->d_rowcnt, s->d_pts, s->d_res, s->d_nres,
                                               s->d_anchors, s->d_count, s->d_cutoff, s->d_status); count_launch();
    mark(c);
    CK(cudaGetLastError(), "scan launch");
    return CB200_OK;
}

// camera_scan, then its results into the pinned host arrays of the state
static int scan_run(cb200_ctx* c, const CameraBatch& b)
{
    const int n = b.n();
    int rc = camera_scan(c, b, nullptr, nullptr); if (rc) return rc;
    ScanScratch* s = c->scan;
    cudaStream_t st = c->stream;
    CK(s->h_anchors.ensure(4 * (size_t)n), "cudaMallocHost anchors");
    CK(s->h_count.ensure(3 * (size_t)n), "cudaMallocHost counts");
    CK(cudaMemcpyAsync(s->h_anchors, s->d_anchors, sizeof(int4) * 4 * (size_t)n, cudaMemcpyDeviceToHost, st), "D2H anchors");
    CK(cudaMemcpyAsync(s->h_count, s->d_count, sizeof(int) * (size_t)n, cudaMemcpyDeviceToHost, st), "D2H counts");
    CK(cudaMemcpyAsync(s->h_count + n, s->d_cutoff, sizeof(unsigned) * (size_t)n, cudaMemcpyDeviceToHost, st), "D2H cutoffs");
    CK(cudaMemcpyAsync(s->h_count + 2 * (size_t)n, s->d_status, sizeof(int) * (size_t)n, cudaMemcpyDeviceToHost, st), "D2H status");
    CK(cudaStreamSynchronize(st), "sync (scan)");
    return CB200_OK;
}

static int scan_results(cb200_ctx* c, int n, int32_t* anchors, int32_t* count, uint32_t* cutoff)
{
    const ScanScratch* s = c->scan;
    for (int i = 0; i < n; ++i) {
        const bool overflow = (s->h_count[2 * (size_t)n + i] & kScanOverflow) != 0;
        count[i] = overflow ? -1 : s->h_count[i];
        if (cutoff) cutoff[i] = (uint32_t)s->h_count[(size_t)n + i];
    }
    if (anchors) memcpy(anchors, s->h_anchors, sizeof(int32_t) * 16 * (size_t)n);
    return CB200_OK;
}

// Extractor::extract (Extractor.h:30-46) of every picture of a scan, on the device: one thread per picture.  slots: NULL, or picture
// i of a sub-batch is the scan's picture slots[i] (a detect receivers call's geometry).  words: NULL, or a receiver flags table
// (Receivers::d_words) with the batch's map `of` and refused bytes: a slot whose receiver's word is invalid leaves the map (receiver
// -1) as refused, and every other slot's sharpen byte follows its receiver's word (an empty slot is not sharpened).  The receiver is
// the picture's (pic_of, indexed as the scan's pictures and checked against [0, receivers)), so every mode of a detect call's geometry
// takes the same sharpen bytes, whichever of them decodes the picture
struct ExtractWords { const uint32_t* words; const int32_t* pic_of; int receivers; int32_t* of; uint8_t* refused; };
__global__ void k_extract(const int4* __restrict__ anchors, const int* __restrict__ count, const int* __restrict__ scan_status, int n,
                          int width, int height, int32_t* __restrict__ status, double* __restrict__ minv, double* __restrict__ fwd,
                          uint8_t* __restrict__ sharpen, const int32_t* __restrict__ slots, const ExtractWords xw)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int s = slots ? slots[i] : i;
    const int st = extract::extract_picture(reinterpret_cast<const Anchor*>(anchors + 4 * (size_t)s), count[s], (scan_status[s] & kScanOverflow) != 0,
                                            width, height, fwd + 9 * (size_t)i, minv + 9 * (size_t)i);
    status[i] = st;
    if (xw.words) {
        const int32_t r = xw.pic_of[s];
        const bool in = (uint32_t)r < (uint32_t)xw.receivers;          // !receivers::empty_slot(r, xw.receivers)
        const uint32_t w = in ? xw.words[r] : 0u;
        const bool bad = in && receivers::word_refused(w);
        if (bad) { xw.of[i] = -1; xw.refused[i] = 1; }
        sharpen[i] = in && !bad && receivers::word_sharpens(w, st);
    } else if (sharpen) {
        sharpen[i] = st == 2;                      // CB200_FLAG_SHARPEN_IF_NEEDED: the CLI sharpens exactly the NEEDS_SHARPEN pictures
    }
}

// a picture that failed extraction yields no chunks.  of: NULL, or the receivers map, where an empty slot (receiver -1) yields no
// chunks either and its status, which k_extract wrote before, becomes CB200_EXTRACT_EMPTY -- CB200_EXTRACT_REFUSED where refused
// (NULL, or a plan over device descriptors: k_plan_pictures refused the slot's descriptor) is set
__global__ void k_mask_failed(int32_t* __restrict__ status, int n, uint32_t* __restrict__ mask, const int32_t* __restrict__ of,
                              const uint8_t* __restrict__ refused)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (of && of[i] < 0) status[i] = refused && refused[i] ? CB200_EXTRACT_REFUSED : CB200_EXTRACT_EMPTY;
    if (status[i] <= 0) mask[i] = 0;
}

// a receivers call with a flags table: the record (record_bytes) of every refused picture zeroed, one CTA per picture
__global__ void k_zero_refused(const int32_t* __restrict__ status, uint8_t* __restrict__ records, int record_bytes)
{
    if (status[blockIdx.x] != CB200_EXTRACT_REFUSED) return;
    uint8_t* r = records + (size_t)blockIdx.x * record_bytes;
    for (int k = threadIdx.x; k < record_bytes; k += blockDim.x) r[k] = 0;
}

int camera_reserve_for(cb200_ctx* c, const int32_t* wh, int n, bool scans, bool walks)
{
    ScanScratch* s = sstate(c);
    int rc;
    if ((rc = grow(c, s->d_minv, 9 * (size_t)n, "inverse maps")) || (rc = grow(c, s->d_fwd, 9 * (size_t)n, "transforms")) ||
        (rc = grow(c, c->d_sel, (size_t)c->max_frames * 5, "selection")) || (walks && (rc = deskew_reserve(c, n))) ||
        (scans && (rc = scan_reserve(c, wh, n))))
        return rc;
    return walks ? flood_reserve(c, n) : CB200_OK;
}

int camera_reserve(cb200_ctx* c, const int32_t* wh, int n) { return camera_reserve_for(c, wh, n, true, true); }

int camera_reserve(cb200_ctx* c, const CameraBatch& b)
{
    if (!b.d_pics) return camera_reserve(c, b.wh.data(), b.n());
    const int rc = camera_reserve_for(c, nullptr, b.n(), false, true);
    return rc ? rc : scan_reserve(c, b);
}

int camera_after_scan(cb200_ctx* c, const cb200_ctx* scanned, const CameraBatch& b, const PicDesc* d_desc, uint32_t flags, uint8_t* frames,
                      bool deskew, uint8_t* d_chunks, uint32_t* d_mask, uint8_t* d_frame_flags, int32_t* d_status, Receivers* recv,
                      const int32_t* d_slots, CellTrace* d_trace)
{
    const Mode& m = c->mode;
    const int n = b.n();
    ScanScratch* s = sstate(c);
    const ScanScratch* s0 = scanned->scan;
    // a flags table's slots are refused and their sharpen bytes written by k_extract, which may rewrite the map in place (the map is
    // this call's upload, or the plan's own)
    const uint32_t* words = recv ? recv->d_words : nullptr;
    const bool if_needed = (flags & CB200_FLAG_SHARPEN_IF_NEEDED) != 0 || words;
    uint8_t* d_sharp = if_needed ? c->d_sel + 4 * (size_t)n : nullptr;
    ExtractWords xw = {};
    if (words) xw = {words, recv->d_pic_of ? recv->d_pic_of : recv->d_map, recv->receivers, const_cast<int32_t*>(recv->d_map),
                     const_cast<uint8_t*>(recv->d_refused)};
    k_extract<<<(n + 127) / 128, 128, 0, c->stream>>>(s0->d_anchors, s0->d_count, s0->d_status, n, m.width, m.height, d_status, s->d_minv, s->d_fwd, d_sharp,
                                                      d_slots, xw);
    count_launch();
    CK(cudaGetLastError(), "extract launch");
    s->camera_n = n;
    int rc;
    if (deskew) { rc = deskew_launch(c, b, s->d_minv, d_desc, frames); if (rc) return rc; }
    rc = decode_chunks(c, frames, n, flags & ~CB200_FLAG_SHARPEN_IF_NEEDED, nullptr, d_chunks, d_mask, d_frame_flags, d_sharp, true, recv,
                       d_trace);
    if (rc) return rc;
    k_mask_failed<<<(n + 127) / 128, 128, 0, c->stream>>>(d_status, n, d_mask, recv ? recv->d_map : nullptr, recv ? recv->d_refused : nullptr);
    count_launch();
    CK(cudaGetLastError(), "mask launch");
    if (words) {
        k_zero_refused<<<n, 256, 0, c->stream>>>(d_status, d_chunks, m.data_bytes);
        count_launch();
        CK(cudaGetLastError(), "zero refused launch");
    }
    return CB200_OK;
}

// Extractor::extract + Decoder::decode_fountain for a device batch, enqueued on the context's stream without a host round trip:
// scan, k_extract, deskew with the scan's picture table, decode (with CB200_FLAG_SHARPEN_IF_NEEDED the frame lists are built on
// the device), masks of failed pictures cleared
int camera_enqueue(cb200_ctx* c, const CameraBatch& b, uint32_t flags, uint8_t* d_chunks, uint32_t* d_mask, uint8_t* d_frame_flags,
                   int32_t* d_status, const PicDesc* d_table, Receivers* recv)
{
    int rc = camera_reserve(c, b); if (rc) return rc;
    uint8_t* frames;
    rc = deskew_frames(c, b.n(), &frames); if (rc) return rc;
    const PicDesc* d_desc;
    rc = camera_scan(c, b, d_table, &d_desc, recv); if (rc) return rc;
    return camera_after_scan(c, c, b, d_desc, flags, frames, true, d_chunks, d_mask, d_frame_flags, d_status, recv);
}

int check_receiver_flags(const uint32_t* d_receiver_flags, uint32_t flags)
{
    if (!d_receiver_flags) return fail(CB200_ERR_ARG, "null d_receiver_flags");
    if (reinterpret_cast<uintptr_t>(d_receiver_flags) % 4) return fail(CB200_ERR_ARG, "d_receiver_flags is not 4-byte aligned");
    if (flags & receivers::kWordBits)
        return fail(CB200_ERR_ARG, "flags hold a per-receiver bit (SHARPEN, SHARPEN_IF_NEEDED, CC_SIMPLE, CC_FIT): those come from "
                                   "d_receiver_flags");
    return CB200_OK;
}

int check_camera_flags(uint32_t flags)
{
    // both sharpen flags together are a contradiction (CB200_FLAG_SHARPEN_IF_NEEDED is the CLI's --preprocess -1, SHARPEN its 1)
    if ((flags & CB200_FLAG_SHARPEN) && (flags & CB200_FLAG_SHARPEN_IF_NEEDED))
        return fail(CB200_ERR_ARG, "CB200_FLAG_SHARPEN and CB200_FLAG_SHARPEN_IF_NEEDED are exclusive");
    if ((flags & CB200_FLAG_CC_FIT) && (flags & CB200_FLAG_CC_SIMPLE)) return fail(CB200_ERR_ARG, "CC_SIMPLE and CC_FIT are exclusive");
    return CB200_OK;
}

// the synchronous camera entry points: the batch checked and staged, the enqueue-only path into the context's buffers, one copy
// back, one synchronise
template <class Build>
static int scan_extract_decode(cb200_ctx* c, Build&& build, uint32_t flags, uint8_t* chunks_out, uint32_t* chunk_count, uint32_t* chunk_mask,
                               uint8_t* frame_flags, int32_t* extract_status)
{
    CameraBatch b;
    int rc = check_camera_call(c, flags, build, b, chunks_out && chunk_count && extract_status ? nullptr : "null output"); if (rc) return rc;
    const int n = b.n();
    if (n == 0) return empty_stripe(c, flags, true);
    rc = check_frozen_camera(c, b.wh.data(), n); if (rc) return rc;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    rc = stage_batch(c, b); if (rc) return rc;
    ScanScratch* s = sstate(c);
    CK(s->d_ext_status.ensure((size_t)n), "cudaMalloc extract status");
    rc = camera_enqueue(c, b, flags, c->d_data, c->d_mask, nullptr, s->d_ext_status); if (rc) return rc;
    return fetch_fountain(c, n, s->d_ext_status, chunks_out, chunk_count, chunk_mask, frame_flags, extract_status);
}

// the receiver arguments of cb200_scan_extract_decode_chunks_receivers_dev (and the flags table of its _flags_ form, else NULL)
struct ReceiverArgs { const int32_t* of; int n, count; cb200_receiver_state* d_states; const uint32_t* d_words; };

// the enqueue-only camera entry points on device pictures.  A receivers call (ra) checks its receivers first; it is never chained,
// so with no pictures it does nothing
template <class Build>
static int scan_extract_decode_dev(cb200_ctx* c, Build&& build, uint32_t flags, uint8_t* d_chunks, uint32_t* d_chunk_mask, uint8_t* d_frame_flags,
                                   int32_t* d_extract_status, const ReceiverArgs* ra = nullptr)
{
    CameraBatch b;
    int rc = ra ? check_receivers(c, ra->of, ra->n, ra->count, ra->d_states) : CB200_OK; if (rc) return rc;
    rc = check_camera_call(c, flags, build, b, d_chunks && d_chunk_mask && d_extract_status ? nullptr : "null output"); if (rc) return rc;
    if (b.n() == 0) return empty_stripe(c, flags, true);
    rc = check_frozen_camera(c, b.wh.data(), b.n()); if (rc) return rc;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    if (!ra) return camera_enqueue(c, b, flags, d_chunks, d_chunk_mask, d_frame_flags, d_extract_status);
    Receivers r(ra->of, b.n(), ra->count, ra->d_states);
    if ((r.d_words = ra->d_words)) { r.refused_bytes(b.n()); r.receivers = ra->count; }
    return camera_enqueue(c, b, flags, d_chunks, d_chunk_mask, d_frame_flags, d_extract_status, nullptr, &r);
}

// ---- the combined call (cb200_scan_extract_decode_chunks_combined_dev): per-cell vote over groups of pictures of one frame
int check_groups(uint32_t flags, const CameraGroups& g, int n)
{
    if (g.found) {
        if (flags & CB200_FLAG_NO_FALLBACK) return fail(CB200_ERR_ARG, "CB200_FLAG_NO_FALLBACK: the vote needs every picture's walk");
        return g.outputs ? CB200_OK : fail(CB200_ERR_ARG, "null group output");
    }
    if (g.m > 0 && (flags & CB200_FLAG_NO_FALLBACK))
        return fail(CB200_ERR_ARG, "CB200_FLAG_NO_FALLBACK with m > 0: the vote needs every picture's walk");
    if (g.m < 0) return fail(CB200_ERR_ARG, "m = " + std::to_string(g.m) + " < 0");
    if (!g.of) return g.m > 0 ? fail(CB200_ERR_ARG, "null group_of with m > 0") : CB200_OK;
    int at = 0;
    switch (combine::group_error(g.of, n, g.m, &at)) {
    case 1: return fail(CB200_ERR_ARG, "picture " + std::to_string(at) + ": group " + std::to_string(g.of[at]) + " outside [-1, " +
                                       std::to_string(g.m) + ")");
    case 2: return fail(CB200_ERR_ARG, "picture " + std::to_string(at) + ": group " + std::to_string(g.of[at]) + " has more than " +
                                       std::to_string(combine::kMaxGroup) + " pictures");
    default: break;
    }
    if (g.m > 0 && !g.outputs) return fail(CB200_ERR_ARG, "null group output");
    return CB200_OK;
}

// the combined and grouped calls' own buffers: the groups' cells and the pictures' traces, and with `pairs` (the grouped calls) the
// match rows and the group table with the assignment's scratch (`receivers`: the grouped receivers call's, 2 n ints more).  With
// live plans grow() makes no CUDA call and refuses what would grow, so the calls run this before any CUDA call then
static int combine_reserve(cb200_ctx* c, int n, int m, bool pairs, bool receivers = false)
{
    const size_t cells = (size_t)c->mode.num_cells;
    int rc;
    if ((rc = grow(c, c->d_combined, (size_t)m * cells, "combined cells")) || (rc = grow(c, c->d_traces, (size_t)n * cells, "cell traces")))
        return rc;
    if (pairs && ((rc = grow(c, c->d_pairs, (size_t)n * (((size_t)n + 31) / 32), "match rows")) ||
                  (rc = grow(c, c->d_groups, (size_t)m + 1 + (receivers ? 5 : 3) * (size_t)n, "group table"))))
        return rc;
    return CB200_OK;
}

// combine::vote per (group, cell), one thread each, over the CSR group table (offsets[0 .. m], members): the participating pictures'
// value bits from their final cell bytes and their walk distances from the trace, into the groups' contiguous cell frames; the cell-0
// thread of a group writes its participant count
__global__ void k_combine(int m, int cells, const int32_t* __restrict__ offsets, const int32_t* __restrict__ members,
                          const int32_t* __restrict__ status, const uint8_t* __restrict__ cellvals, const CellTrace* __restrict__ trace,
                          uint8_t* __restrict__ out, int32_t* __restrict__ used)
{
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)m * cells) return;
    const int g = (int)(t / cells), cell = (int)(t - (long long)g * cells);
    uint8_t v[combine::kMaxGroup], d[combine::kMaxGroup];
    int k = 0;
    for (int j = offsets[g], end = offsets[g + 1]; j < end; ++j) {
        const int p = members[j];
        if (!combine::takes_part(status[p])) continue;
        const size_t at = (size_t)p * cells + cell;
        v[k] = cellvals[at] & combine::kValueBits;
        d[k] = trace[at].distance;
        ++k;
    }
    out[t] = k ? combine::vote(v, d, k) : 0;
    if (cell == 0) used[g] = k;
}

// every group of a call without pictures: zeroed records, mask 0, no pictures
static int combine_empty(cb200_ctx* c, int m, uint8_t* d_group_chunks, uint32_t* d_group_mask, int32_t* d_group_used)
{
    CK(cudaMemsetAsync(d_group_chunks, 0, (size_t)m * c->mode.data_bytes, c->stream), "memset group records");
    CK(cudaMemsetAsync(d_group_mask, 0, sizeof(uint32_t) * (size_t)m, c->stream), "memset group masks");
    CK(cudaMemsetAsync(d_group_used, 0, sizeof(int32_t) * (size_t)m, c->stream), "memset group counts");
    return CB200_OK;
}

// camera_enqueue with the walk's traces kept and `tail` (or nothing) behind the picture table, at *d_tail on the device.  recv: a
// grouped receivers call's receivers, whose map goes up between the table and the tail
static int combine_pictures(cb200_ctx* c, const CameraBatch& b, int m, bool pairs, const std::vector<uint8_t>* tail, const uint8_t** d_tail,
                            uint32_t flags, uint8_t* d_chunks, uint32_t* d_chunk_mask, uint8_t* d_frame_flags, int32_t* d_extract_status,
                            Receivers* recv = nullptr)
{
    const int n = b.n();
    int rc;
    if ((rc = combine_reserve(c, n, m, pairs, recv != nullptr)) || (rc = camera_reserve(c, b))) return rc;
    uint8_t* frames;
    if ((rc = deskew_frames(c, n, &frames))) return rc;
    const PicDesc* d_desc;
    if ((rc = camera_scan(c, b, nullptr, &d_desc, recv, tail, d_tail))) return rc;
    return camera_after_scan(c, c, b, d_desc, flags, frames, true, d_chunks, d_chunk_mask, d_frame_flags, d_extract_status, recv, nullptr,
                             c->d_traces);
}

// the vote and the decode of the m groups of the table at d_table (offsets[0 .. m], then the members): the route of a call without
// colour correction (k2_rs_fused_launch: the frame-pair kernel where it applies), the chunk masks, and mask 0 for a group without
// pictures (k_mask_failed on the counts).  The members' cells and traces: the context's (d_cellvals, d_traces), or a history's
// staging region (members are then its positions).  Four launches
static int combine_groups(cb200_ctx* c, int m, const int32_t* d_table, uint32_t flags, const int32_t* d_extract_status, uint8_t* d_group_chunks,
                          uint32_t* d_group_mask, int32_t* d_group_used, const uint8_t* d_cellvals = nullptr,
                          const CellTrace* d_traces = nullptr)
{
    const Mode& md = c->mode;
    const long long threads = (long long)m * md.num_cells;
    k_combine<<<(unsigned)((threads + 255) / 256), 256, 0, c->stream>>>(m, md.num_cells, d_table, d_table + m + 1, d_extract_status,
                                                                       d_cellvals ? d_cellvals : c->d_cellvals.get(),
                                                                       d_traces ? d_traces : c->d_traces.get(), c->d_combined, d_group_used);
    count_launch();
    CK(cudaGetLastError(), "combine launch");
    const uint16_t* idx = (flags & CB200_FLAG_NO_INTERLEAVE) ? c->d_idx_ident.get() : c->d_idx.get();
    CK(k2_rs_fused_launch(md, c->d_combined, idx, m, d_group_chunks, c->d_ok, c->d_rho, c->sm_count, c->stream), "rs launch (groups)");
    CK(k2_mask_launch(md, c->d_ok, m, d_group_mask, c->stream), "mask launch (groups)");
    k_mask_failed<<<(m + 127) / 128, 128, 0, c->stream>>>(d_group_used, m, d_group_mask, nullptr, nullptr);
    count_launch();
    CK(cudaGetLastError(), "group mask launch");
    return CB200_OK;
}

// the combined call with groups: the group table travels behind the picture table (one upload).  Four launches more than the
// pictures call
static int combine_enqueue(cb200_ctx* c, const CameraBatch& b, const int32_t* group_of, int m, uint32_t flags, uint8_t* d_chunks,
                           uint32_t* d_chunk_mask, uint8_t* d_frame_flags, int32_t* d_extract_status, uint8_t* d_group_chunks,
                           uint32_t* d_group_mask, int32_t* d_group_used)
{
    const int n = b.n();
    std::vector<int32_t> table((size_t)m + 1 + (size_t)n);
    combine::group_table(group_of, n, m, table.data(), table.data() + m + 1);
    table.resize((size_t)m + 1 + (size_t)table[(size_t)m]);
    std::vector<uint8_t> tail(table.size() * sizeof(int32_t));
    memcpy(tail.data(), table.data(), tail.size());
    const uint8_t* d_tail;
    int rc = combine_pictures(c, b, m, false, &tail, &d_tail, flags, d_chunks, d_chunk_mask, d_frame_flags, d_extract_status);
    if (rc) return rc;
    return combine_groups(c, m, reinterpret_cast<const int32_t*>(d_tail), flags, d_extract_status, d_group_chunks, d_group_mask, d_group_used);
}

// ---- the grouped call (cb200_scan_extract_decode_chunks_grouped_dev): the groups found on the device from the pictures' cells
// the grouped call after the argument checks, n >= 2: the pictures call with traces, find_groups (group.cu) into d_group_of,
// d_group_count and the table in c->d_groups (n / 2 slots), then combine_groups over the slots.  Six launches more than the pictures
// call, and no wait of its own
static int grouped_enqueue(cb200_ctx* c, const CameraBatch& b, uint32_t flags, uint8_t* d_chunks, uint32_t* d_chunk_mask, uint8_t* d_frame_flags,
                           int32_t* d_extract_status, int32_t* d_group_of, int32_t* d_group_count, uint8_t* d_group_chunks,
                           uint32_t* d_group_mask, int32_t* d_group_used)
{
    const int n = b.n(), slots = n / 2;
    int rc = combine_pictures(c, b, slots, true, nullptr, nullptr, flags, d_chunks, d_chunk_mask, d_frame_flags, d_extract_status);
    if (rc) return rc;
    if ((rc = find_groups(c, n, d_extract_status, d_group_of, d_group_count))) return rc;
    return combine_groups(c, slots, c->d_groups, flags, d_extract_status, d_group_chunks, d_group_mask, d_group_used);
}

// ---- the grouped history call (cb200_scan_extract_decode_chunks_grouped_history_dev): the grouped call over a batch that follows a
// history's pictures.  Its own buffers on the context: n voted frames and traces, and the pairing and assignment over N = H + n
// positions.  With live plans grow() refuses before any CUDA call
static int history_reserve_ctx(cb200_ctx* c, int N, int n)
{
    int rc;
    if ((rc = combine_reserve(c, n, n, false)) || (rc = grow(c, c->d_pairs, (size_t)N * (((size_t)N + 31) / 32), "match rows")) ||
        (rc = grow(c, c->d_groups, (size_t)(N / 2) + 1 + 3 * (size_t)N, "group table")))
        return rc;
    return CB200_OK;
}

// after the argument checks, n >= 1: the pictures call with traces; history_groups (the batch staged behind the history, the
// pairing, the assignment and the groups with a batch member); the vote and decode of n slots from the staging region; history_settle
// (the new history).  Nine launches more than the pictures call (three more than the grouped call), three device copies, no wait
static int grouped_history_enqueue(cb200_ctx* c, cb200_group_history* h, const CameraBatch& b, uint32_t flags, uint8_t* d_chunks,
                                   uint32_t* d_chunk_mask, uint8_t* d_frame_flags, int32_t* d_extract_status, int32_t* d_group_of,
                                   int32_t* d_group_count, uint8_t* d_group_chunks, uint32_t* d_group_mask, int32_t* d_group_used)
{
    const int n = b.n();
    int rc;
    if ((rc = history_reserve_ctx(c, history_positions(h) + n, n)) || (rc = history_reserve(c, h, n))) return rc;
    if ((rc = combine_pictures(c, b, n, false, nullptr, nullptr, flags, d_chunks, d_chunk_mask, d_frame_flags, d_extract_status))) return rc;
    HistoryStage st;
    if ((rc = history_groups(c, h, n, d_extract_status, d_group_of, d_group_count, &st))) return rc;
    if ((rc = combine_groups(c, n, st.table, flags, st.status, d_group_chunks, d_group_mask, d_group_used, st.cells, st.traces))) return rc;
    return history_settle(c, h, n, d_chunk_mask, d_group_count, d_group_mask);
}

// ---- the grouped receivers call (cb200_scan_extract_decode_chunks_grouped_receivers_dev): the grouped call's rule within each
// receiver.  After the argument checks, n >= 2: the receivers call with traces, whose one upload carries the picture table, the map
// and the host lists of find_groups (combine::pair_tiles' tile pairs, then combine::segment_starts); find_groups with those lists;
// combine_groups over the n / 2 slots.  Six launches more than the receivers call, and no wait of its own
static int grouped_receivers_enqueue(cb200_ctx* c, const CameraBatch& b, uint32_t flags, Receivers& r, uint8_t* d_chunks,
                                     uint32_t* d_chunk_mask, uint8_t* d_frame_flags, int32_t* d_extract_status, int32_t* d_group_of,
                                     int32_t* d_group_count, uint8_t* d_group_chunks, uint32_t* d_group_mask, int32_t* d_group_used,
                                     int32_t* d_group_receiver)
{
    const int n = b.n(), slots = n / 2;
    const int32_t* order = r.map.data() + n;
    std::vector<int32_t> tiles, starts;
    combine::pair_tiles(r.map.data(), order, n, combine::kPairTile, tiles);
    combine::segment_starts(r.map.data(), order, n, starts);
    std::vector<uint8_t> tail(sizeof(int32_t) * (tiles.size() + starts.size()));
    memcpy(tail.data(), tiles.data(), sizeof(int32_t) * tiles.size());
    memcpy(tail.data() + sizeof(int32_t) * tiles.size(), starts.data(), sizeof(int32_t) * starts.size());
    const uint8_t* d_tail;
    int rc = combine_pictures(c, b, slots, true, &tail, &d_tail, flags, d_chunks, d_chunk_mask, d_frame_flags, d_extract_status, &r);
    if (rc) return rc;
    const int ntiles = (int)(tiles.size() / 2);
    const GroupLists lists = {r.d_map, reinterpret_cast<const int2*>(d_tail), ntiles, reinterpret_cast<const int32_t*>(d_tail) + 2 * (size_t)ntiles,
                              (int)starts.size() - 1, d_group_receiver};
    if ((rc = find_groups(c, n, d_extract_status, d_group_of, d_group_count, &lists))) return rc;
    return combine_groups(c, slots, c->d_groups, flags, d_extract_status, d_group_chunks, d_group_mask, d_group_used);
}

// the scan entry points: the batch, the context and the count output checked, the batch staged and scanned, the results copied out
static int scan_call(cb200_ctx* c, int built, CameraBatch& b, int32_t* anchors, int32_t* count, uint32_t* cutoff)
{
    if (built) return built;
    if (!c || !count) return fail(CB200_ERR_ARG, !c ? "null context" : "null count");
    const int n = b.n();
    if (n == 0) return CB200_OK;
    int rc = check_frozen_scan(c, b.wh.data(), n); if (rc) return rc;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    rc = stage_batch(c, b); if (rc) return rc;
    rc = scan_run(c, b); if (rc) return rc;
    return scan_results(c, n, anchors, count, cutoff);
}

}  // namespace cb200

using namespace cb200;

extern "C" {

int cb200_scan_dev(cb200_ctx* c, const uint8_t* d_pictures, int w, int h, int n, int32_t* anchors, int32_t* count, uint32_t* cutoff)
{
    CameraBatch b;
    const int rc = uniform_batch(d_pictures, w, h, n, b);
    return scan_call(c, rc, b, anchors, count, cutoff);
}

int cb200_scan(cb200_ctx* c, const uint8_t* pictures, int w, int h, int n, int32_t* anchors, int32_t* count, uint32_t* cutoff)
{
    CameraBatch b;
    const int rc = uniform_batch(pictures, w, h, n, b);
    b.host = true;
    return scan_call(c, rc, b, anchors, count, cutoff);
}

int cb200_scan_ragged_dev(cb200_ctx* c, const uint8_t* d_pictures, const int32_t* wh, int n, int32_t* anchors, int32_t* count, uint32_t* cutoff)
{
    CameraBatch b;
    const int rc = packed_batch(d_pictures, wh, n, b);
    return scan_call(c, rc, b, anchors, count, cutoff);
}

int cb200_scan_ragged(cb200_ctx* c, const uint8_t* const* pictures, const int32_t* wh, int n, int32_t* anchors, int32_t* count, uint32_t* cutoff)
{
    CameraBatch b;
    const int rc = host_batch(pictures, wh, n, b);
    return scan_call(c, rc, b, anchors, count, cutoff);
}

// the first npx blurred bytes and n thresholds of the last scan
static int read_blurred(cb200_ctx* c, uint8_t* blurred_out, int32_t* thresholds_out, size_t npx, int n)
{
    if (!c || !c->scan || n < 0 || npx > c->scan->d_blur.capacity() || (size_t)n > c->scan->d_thr.capacity())
        return fail(CB200_ERR_ARG, "no scan of that size to read back");
    if (n == 0) return CB200_OK;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    if (blurred_out) CK(cudaMemcpyAsync(blurred_out, c->scan->d_blur, npx, cudaMemcpyDeviceToHost, c->stream), "D2H blurred");
    if (thresholds_out) CK(cudaMemcpyAsync(thresholds_out, c->scan->d_thr, sizeof(int) * (size_t)n, cudaMemcpyDeviceToHost, c->stream), "D2H thresholds");
    CK(cudaStreamSynchronize(c->stream), "sync");
    return CB200_OK;
}

int cb200_scan_blurred(cb200_ctx* c, uint8_t* blurred_out, int32_t* thresholds_out, int w, int h, int n)
{
    return read_blurred(c, blurred_out, thresholds_out, (size_t)w * h * (size_t)(n < 0 ? 0 : n), n);
}

int cb200_scan_blurred_ragged(cb200_ctx* c, uint8_t* blurred_out, int32_t* thresholds_out, const int32_t* wh, int n)
{
    if (n < 0 || !wh) return fail(CB200_ERR_ARG, n < 0 ? "n < 0" : "null wh");
    size_t npx = 0;
    for (int i = 0; i < n; ++i) npx += (size_t)wh[2 * i] * (size_t)wh[2 * i + 1];
    return read_blurred(c, blurred_out, thresholds_out, npx, n);
}

int cb200_scan_extract_decode_fountain(cb200_ctx* c, const uint8_t* pictures, int w, int h, int n, uint32_t flags,
                                       uint8_t* chunks_out, uint32_t* chunk_count, uint32_t* chunk_mask, uint8_t* frame_flags,
                                       int32_t* extract_status)
{
    auto build = [&](CameraBatch& b) {
        const int rc = uniform_batch(pictures, w, h, n, b);
        b.host = true;
        return rc;
    };
    return scan_extract_decode(c, build, flags, chunks_out, chunk_count, chunk_mask, frame_flags, extract_status);
}

int cb200_scan_extract_decode_fountain_ragged(cb200_ctx* c, const uint8_t* const* pictures, const int32_t* wh, int n, uint32_t flags,
                                              uint8_t* chunks_out, uint32_t* chunk_count, uint32_t* chunk_mask, uint8_t* frame_flags,
                                              int32_t* extract_status)
{
    auto build = [&](CameraBatch& b) { return host_batch(pictures, wh, n, b); };
    return scan_extract_decode(c, build, flags, chunks_out, chunk_count, chunk_mask, frame_flags, extract_status);
}

int cb200_scan_extract_decode_chunks_ragged_dev(cb200_ctx* c, const uint8_t* d_pictures, const int32_t* wh, int n, uint32_t flags,
                                                uint8_t* d_chunks, uint32_t* d_chunk_mask, uint8_t* d_frame_flags, int32_t* d_extract_status)
{
    auto build = [&](CameraBatch& b) { return packed_batch(d_pictures, wh, n, b); };
    return scan_extract_decode_dev(c, build, flags, d_chunks, d_chunk_mask, d_frame_flags, d_extract_status);
}

int cb200_scan_extract_decode_chunks_dev(cb200_ctx* c, const uint8_t* d_pictures, int w, int h, int n, uint32_t flags, uint8_t* d_chunks,
                                         uint32_t* d_chunk_mask, uint8_t* d_frame_flags, int32_t* d_extract_status)
{
    auto build = [&](CameraBatch& b) { return uniform_batch(d_pictures, w, h, n, b); };
    return scan_extract_decode_dev(c, build, flags, d_chunks, d_chunk_mask, d_frame_flags, d_extract_status);
}

int cb200_scan_extract_decode_chunks_pictures_dev(cb200_ctx* c, const cb200_picture* pics, int n, uint32_t flags, uint8_t* d_chunks,
                                                  uint32_t* d_chunk_mask, uint8_t* d_frame_flags, int32_t* d_extract_status)
{
    auto build = [&](CameraBatch& b) { return picture_batch(pics, n, b); };
    return scan_extract_decode_dev(c, build, flags, d_chunks, d_chunk_mask, d_frame_flags, d_extract_status);
}

int cb200_scan_extract_decode_chunks_combined_dev(cb200_ctx* c, const cb200_picture* pics, int n, const int32_t* group_of, int m, uint32_t flags,
                                                  uint8_t* d_chunks, uint32_t* d_chunk_mask, uint8_t* d_frame_flags, int32_t* d_extract_status,
                                                  uint8_t* d_group_chunks, uint32_t* d_group_mask, int32_t* d_group_used)
{
    CameraBatch b;
    auto build = [&](CameraBatch& bb) { return picture_batch(pics, n, bb); };
    const CameraGroups groups = {group_of, m, d_group_chunks && d_group_mask && d_group_used};
    int rc = check_camera_call(c, flags, build, b, d_chunks && d_chunk_mask && d_extract_status ? nullptr : "null output", &groups);
    if (rc) return rc;
    const int nb = b.n();
    if (nb == 0) {
        if ((rc = empty_stripe(c, flags, true)) || m == 0) return rc;
        CK(cudaSetDevice(c->device), "cudaSetDevice");
        return combine_empty(c, m, d_group_chunks, d_group_mask, d_group_used);
    }
    if ((rc = check_frozen_camera(c, b.wh.data(), nb)) || (m > 0 && !c->plans.empty() && (rc = combine_reserve(c, nb, m, false)))) return rc;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    if (m == 0) return camera_enqueue(c, b, flags, d_chunks, d_chunk_mask, d_frame_flags, d_extract_status);
    return combine_enqueue(c, b, group_of, m, flags, d_chunks, d_chunk_mask, d_frame_flags, d_extract_status, d_group_chunks, d_group_mask,
                           d_group_used);
}

int cb200_scan_extract_decode_chunks_grouped_dev(cb200_ctx* c, const cb200_picture* pics, int n, uint32_t flags, uint8_t* d_chunks,
                                                 uint32_t* d_chunk_mask, uint8_t* d_frame_flags, int32_t* d_extract_status, int32_t* d_group_of,
                                                 int32_t* d_group_count, uint8_t* d_group_chunks, uint32_t* d_group_mask, int32_t* d_group_used)
{
    CameraBatch b;
    auto build = [&](CameraBatch& bb) { return picture_batch(pics, n, bb); };
    const CameraGroups groups = {nullptr, 0, d_group_of && d_group_count && d_group_chunks && d_group_mask && d_group_used, true};
    int rc = check_camera_call(c, flags, build, b, d_chunks && d_chunk_mask && d_extract_status ? nullptr : "null output", &groups);
    if (rc) return rc;
    const int nb = b.n();
    if (nb == 0) {
        rc = empty_stripe(c, flags, true);
    } else {
        if ((rc = check_frozen_camera(c, b.wh.data(), nb)) || (nb >= 2 && !c->plans.empty() && (rc = combine_reserve(c, nb, nb / 2, true))))
            return rc;
        CK(cudaSetDevice(c->device), "cudaSetDevice");
        if (nb >= 2)
            return grouped_enqueue(c, b, flags, d_chunks, d_chunk_mask, d_frame_flags, d_extract_status, d_group_of, d_group_count,
                                   d_group_chunks, d_group_mask, d_group_used);
        rc = camera_enqueue(c, b, flags, d_chunks, d_chunk_mask, d_frame_flags, d_extract_status);
    }
    if (rc) return rc;
    // fewer than two pictures form no group
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    CK(cudaMemsetAsync(d_group_of, 0xFF, sizeof(int32_t) * (size_t)nb, c->stream), "memset group_of");
    CK(cudaMemsetAsync(d_group_count, 0, sizeof(int32_t), c->stream), "memset group count");
    return CB200_OK;
}

int cb200_scan_extract_decode_chunks_grouped_history_dev(cb200_ctx* c, cb200_group_history* h, const cb200_picture* pics, int n, uint32_t flags,
                                                         uint8_t* d_chunks, uint32_t* d_chunk_mask, uint8_t* d_frame_flags,
                                                         int32_t* d_extract_status, int32_t* d_group_of, int32_t* d_group_count,
                                                         uint8_t* d_group_chunks, uint32_t* d_group_mask, int32_t* d_group_used)
{
    CameraBatch b;
    auto build = [&](CameraBatch& bb) { return picture_batch(pics, n, bb); };
    const CameraGroups groups = {nullptr, 0, d_group_of && d_group_count && d_group_chunks && d_group_mask && d_group_used, true};
    int rc = check_camera_call(c, flags, build, b, d_chunks && d_chunk_mask && d_extract_status ? nullptr : "null output", &groups);
    if (rc || (rc = history_check(c, h))) return rc;
    const int nb = b.n();
    if (nb == 0) {
        // the history and the group outputs stay as they are; the call is counted
        if ((rc = empty_stripe(c, flags, true))) return rc;
        history_skip(h);
        return CB200_OK;
    }
    if ((rc = check_frozen_camera(c, b.wh.data(), nb)) ||
        (!c->plans.empty() && (rc = history_reserve_ctx(c, history_positions(h) + nb, nb))))
        return rc;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    return grouped_history_enqueue(c, h, b, flags, d_chunks, d_chunk_mask, d_frame_flags, d_extract_status, d_group_of, d_group_count,
                                   d_group_chunks, d_group_mask, d_group_used);
}

int cb200_scan_extract_decode_chunks_receivers_dev(cb200_ctx* c, const cb200_picture* pics, int n, uint32_t flags, const int32_t* receiver_of,
                                                   int n_receivers, cb200_receiver_state* d_states, uint8_t* d_chunks, uint32_t* d_chunk_mask,
                                                   uint8_t* d_frame_flags, int32_t* d_extract_status)
{
    auto build = [&](CameraBatch& b) { return picture_batch(pics, n, b); };
    const ReceiverArgs ra = {receiver_of, n, n_receivers, d_states, nullptr};
    return scan_extract_decode_dev(c, build, flags, d_chunks, d_chunk_mask, d_frame_flags, d_extract_status, &ra);
}

int cb200_scan_extract_decode_chunks_receivers_flags_dev(cb200_ctx* c, const cb200_picture* pics, int n, uint32_t flags,
                                                         const int32_t* receiver_of, int n_receivers, cb200_receiver_state* d_states,
                                                         const uint32_t* d_receiver_flags, uint8_t* d_chunks, uint32_t* d_chunk_mask,
                                                         uint8_t* d_frame_flags, int32_t* d_extract_status)
{
    int rc = check_receiver_flags(d_receiver_flags, flags); if (rc) return rc;
    auto build = [&](CameraBatch& b) { return picture_batch(pics, n, b); };
    const ReceiverArgs ra = {receiver_of, n, n_receivers, d_states, d_receiver_flags};
    return scan_extract_decode_dev(c, build, flags, d_chunks, d_chunk_mask, d_frame_flags, d_extract_status, &ra);
}

// both grouped receivers entry points (ra->d_words: the flags form's table, checked by the caller).  The receivers call's checks,
// then the grouped call's (check_camera_call with the groups: NO_FALLBACK and the six group outputs before the context)
static int grouped_receivers(cb200_ctx* c, const cb200_picture* pics, int n, uint32_t flags, const ReceiverArgs& ra, uint8_t* d_chunks,
                             uint32_t* d_chunk_mask, uint8_t* d_frame_flags, int32_t* d_extract_status, int32_t* d_group_of,
                             int32_t* d_group_count, uint8_t* d_group_chunks, uint32_t* d_group_mask, int32_t* d_group_used,
                             int32_t* d_group_receiver)
{
    CameraBatch b;
    int rc = check_receivers(c, ra.of, ra.n, ra.count, ra.d_states); if (rc) return rc;
    auto build = [&](CameraBatch& bb) { return picture_batch(pics, n, bb); };
    const CameraGroups groups = {nullptr, 0, d_group_of && d_group_count && d_group_chunks && d_group_mask && d_group_used && d_group_receiver,
                                 true};
    rc = check_camera_call(c, flags, build, b, d_chunks && d_chunk_mask && d_extract_status ? nullptr : "null output", &groups);
    if (rc) return rc;
    const int nb = b.n();
    if (nb == 0) {
        rc = empty_stripe(c, flags, true);
    } else {
        if ((rc = check_frozen_camera(c, b.wh.data(), nb)) ||
            (nb >= 2 && !c->plans.empty() && (rc = combine_reserve(c, nb, nb / 2, true, true))))
            return rc;
        CK(cudaSetDevice(c->device), "cudaSetDevice");
        Receivers r(ra.of, nb, ra.count, ra.d_states);
        if ((r.d_words = ra.d_words)) { r.refused_bytes(nb); r.receivers = ra.count; }
        if (nb >= 2)
            return grouped_receivers_enqueue(c, b, flags, r, d_chunks, d_chunk_mask, d_frame_flags, d_extract_status, d_group_of,
                                             d_group_count, d_group_chunks, d_group_mask, d_group_used, d_group_receiver);
        rc = camera_enqueue(c, b, flags, d_chunks, d_chunk_mask, d_frame_flags, d_extract_status, nullptr, &r);
    }
    if (rc) return rc;
    // fewer than two pictures form no group, and there are no slots
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    CK(cudaMemsetAsync(d_group_of, 0xFF, sizeof(int32_t) * (size_t)nb, c->stream), "memset group_of");
    CK(cudaMemsetAsync(d_group_count, 0, sizeof(int32_t), c->stream), "memset group count");
    return CB200_OK;
}

int cb200_scan_extract_decode_chunks_grouped_receivers_dev(cb200_ctx* c, const cb200_picture* pics, int n, uint32_t flags,
                                                           const int32_t* receiver_of, int n_receivers, cb200_receiver_state* d_states,
                                                           uint8_t* d_chunks, uint32_t* d_chunk_mask, uint8_t* d_frame_flags,
                                                           int32_t* d_extract_status, int32_t* d_group_of, int32_t* d_group_count,
                                                           uint8_t* d_group_chunks, uint32_t* d_group_mask, int32_t* d_group_used,
                                                           int32_t* d_group_receiver)
{
    const ReceiverArgs ra = {receiver_of, n, n_receivers, d_states, nullptr};
    return grouped_receivers(c, pics, n, flags, ra, d_chunks, d_chunk_mask, d_frame_flags, d_extract_status, d_group_of, d_group_count,
                             d_group_chunks, d_group_mask, d_group_used, d_group_receiver);
}

int cb200_scan_extract_decode_chunks_grouped_receivers_flags_dev(cb200_ctx* c, const cb200_picture* pics, int n, uint32_t flags,
                                                                 const int32_t* receiver_of, int n_receivers, cb200_receiver_state* d_states,
                                                                 const uint32_t* d_receiver_flags, uint8_t* d_chunks, uint32_t* d_chunk_mask,
                                                                 uint8_t* d_frame_flags, int32_t* d_extract_status, int32_t* d_group_of,
                                                                 int32_t* d_group_count, uint8_t* d_group_chunks, uint32_t* d_group_mask,
                                                                 int32_t* d_group_used, int32_t* d_group_receiver)
{
    int rc = check_receiver_flags(d_receiver_flags, flags); if (rc) return rc;
    const ReceiverArgs ra = {receiver_of, n, n_receivers, d_states, d_receiver_flags};
    return grouped_receivers(c, pics, n, flags, ra, d_chunks, d_chunk_mask, d_frame_flags, d_extract_status, d_group_of, d_group_count,
                             d_group_chunks, d_group_mask, d_group_used, d_group_receiver);
}

int cb200_camera_transforms(cb200_ctx* c, double* m9_out, int n)
{
    if (!c || !m9_out || n < 0) return fail(CB200_ERR_ARG, "bad arguments");
    if (!c->scan || n > c->scan->camera_n)
        return fail(CB200_ERR_ARG, "the last camera call had " + std::to_string(c->scan ? c->scan->camera_n : 0) + " pictures");
    if (n == 0) return CB200_OK;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    CK(cudaMemcpyAsync(m9_out, c->scan->d_fwd, sizeof(double) * 9 * (size_t)n, cudaMemcpyDeviceToHost, c->stream), "D2H transforms");
    CK(cudaStreamSynchronize(c->stream), "sync");
    return CB200_OK;
}

}  // extern "C"
