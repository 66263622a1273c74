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

#include <string>
#include <vector>

namespace cb200 {

using namespace scan;

struct ScanScratch {                 // per-context scratch of the scan entry points
    DevBuf<uint8_t> d_pics;                                 // staging of host pictures
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
// The word path needs 4-byte aligned rows: a picture width that is a multiple of four and aligned source and blurred bases (decided
// per picture by the host: in a packed batch a picture that follows one of odd area starts unaligned); otherwise, and in tiles that
// cross the right edge, pixels are fetched one by one.
template <int R> struct BlurKW {     // the 2R+1 coefficients as bytes of up to three words (IDP.4A operands)
    __device__ static constexpr uint32_t w(int i)
    {
        return (4 * i + 0 <= 2 * R ? BlurK<R>::c(4 * i + 0) : 0u) | ((4 * i + 1 <= 2 * R ? BlurK<R>::c(4 * i + 1) : 0u) << 8) |
               ((4 * i + 2 <= 2 * R ? BlurK<R>::c(4 * i + 2) : 0u) << 16) | ((4 * i + 3 <= 2 * R ? BlurK<R>::c(4 * i + 3) : 0u) << 24);
    }
};

__device__ __forceinline__ uint32_t gray_scalar(const uint8_t* p)
{
    return (9798u * p[0] + 19235u * p[1] + 3735u * p[2] + 16384u) >> 15;
}

// One launch per radius over the flattened tiles of that radius' pictures: order[0 .. npics) lists them (batch indices into the
// descriptor table, in batch order), their tiles are numbered consecutively from desc[order[k]].tile0, row-major inside a picture.
// A CTA finds its picture by division when all listed pictures have one size (uniform_tiles tiles each), else by binary search.
template <int R>
__global__ void __launch_bounds__(kBlurThreads)
k_scan_blur4(const uint8_t* __restrict__ rgb, uint8_t* __restrict__ out, const PicDesc* __restrict__ desc, const int* __restrict__ order,
             int npics, int uniform_tiles, unsigned* __restrict__ hist)
{
    constexpr int GH = kBlurTH + 2 * R, GP = kBlurTW + 8, NW = (2 * R + 1 + 3) / 4;      // gray pitch: interior at byte 4
    __shared__ __align__(16) uint8_t g[GH][GP];
    __shared__ __align__(16) uint16_t hs[GH][kBlurTW];
    __shared__ unsigned lh[256];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int t = (int)blockIdx.x;
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
    const uint8_t* src = rgb + __ldg(&d->src);
    lh[tid] = 0;
    // ---- gray of the tile and its halo
    const int x = tx0 + 4 * lane;
    for (int r = warp; r < GH; r += kBlurThreads / 32) {
        const int y = reflect101_clamped(ty0 - R + r, h);
        const uint8_t* row = src + (size_t)y * (size_t)w * 3;
        uint32_t g4;
        if (words_ok && x + 3 < w) {
            const uint32_t* p = reinterpret_cast<const uint32_t*>(row + 3 * (size_t)x);
            const uint32_t q0 = __ldg(p), q1 = __ldg(p + 1), q2 = __ldg(p + 2);          // R0 G0 B0 R1 | G1 B1 R2 G2 | B2 R3 G3 B3
            const uint32_t cRG = 19596u | (38470u << 16), cB0 = 7470u, c0R = 19596u << 16, cGB = 38470u | (7470u << 16);
            uint32_t n0, n1, n2, n3;                     // (19596 R + 38470 G + 7470 B + 2^15): gray is byte 2 (== (9798 R + 19235 G + 3735 B + 2^14) >> 15)
            n0 = __dp2a_lo(cRG, q0, 32768u); n0 = __dp2a_hi(cB0, q0, n0);
            n1 = __dp2a_hi(c0R, q0, 32768u); n1 = __dp2a_lo(cGB, q1, n1);
            n2 = __dp2a_hi(cRG, q1, 32768u); n2 = __dp2a_lo(cB0, q2, n2);
            n3 = __dp2a_lo(c0R, q2, 32768u); n3 = __dp2a_hi(cGB, q2, n3);
            g4 = __byte_perm(__byte_perm(n0, n1, 0x0062), __byte_perm(n2, n3, 0x6200), 0x7610);
        } else {
            g4 = 0;
#pragma unroll
            for (int k = 0; k < 4; ++k) g4 |= gray_scalar(row + 3 * (size_t)reflect101_clamped(x + k, w)) << (8 * k);
        }
        *reinterpret_cast<uint32_t*>(&g[r][4 + 4 * lane]) = g4;
        if (lane < 2 * R) {                               // halo columns: R to the left of the tile, R to the right
            const int xx = lane < R ? tx0 - R + lane : tx0 + kBlurTW + (lane - R);
            g[r][lane < R ? 4 - R + lane : 4 + kBlurTW + (lane - R)] = (uint8_t)gray_scalar(row + 3 * (size_t)reflect101_clamped(xx, w));
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

static int scan_blur_radius(int w, int h)               // Scanner.h:93-103, :155-157
{
    unsigned v = (unsigned)((w < h ? w : h) * 0.002);
    v--;
    v |= v >> 1; v |= v >> 2; v |= v >> 4; v |= v >> 8; v |= v >> 16;
    unsigned unit = v + 2;
    if (unit < 3u) unit = 3u;
    return (int)(unit / 2);
}

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

// rows of a scan pass for one picture: the primary pass scans h / skip rows, the bottom-right window at most 2 h / skip (half the step)
static int scan_rows(int w, int h)
{
    const int skip = (w < h ? w : h) / 60;
    return 2 * ((h + skip - 1) / skip) + 4;
}

int scan_reserve(cb200_ctx* c, const int32_t* wh, int n)
{
    ScanScratch* s = sstate(c);
    size_t npx = 0;
    int rows_cap = 0;
    for (int i = 0; i < n; ++i) {
        npx += (size_t)wh[2 * i] * (size_t)wh[2 * i + 1];
        const int rc = scan_rows(wh[2 * i], wh[2 * i + 1]);
        if (rc > rows_cap) rows_cap = rc;
    }
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

// the launch geometry of the blur: per radius its pictures, their first entry in the order list, their tiles, one size or not
struct BlurGroups {
    int count[5] = {}, group0[5] = {};
    long long tiles[5] = {};
    bool same[5] = {true, true, true, true, true};
};

// the descriptor table (batch order), then the pictures grouped by blur radius (batch order inside a group) into `table`; the tiles
// of one radius are numbered across its pictures.  The word path depends on where d_pics and the scan's blurred buffer are
static int pic_table(const ScanScratch* s, const uint8_t* d_pics, const int32_t* wh, int n, uint8_t* table, BlurGroups& g)
{
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
        PicDesc& d = desc[i];
        d.src = 3 * off; d.blur = off; d.w = w; d.h = h;
        d.words = (w % 4 == 0) && (reinterpret_cast<uintptr_t>(d_pics + d.src) % 4 == 0) && (reinterpret_cast<uintptr_t>(s->d_blur + d.blur) % 4 == 0);
        d.tile0 = (int)g.tiles[R];
        g.tiles[R] += (long long)((w + kBlurTW - 1) / kBlurTW) * ((h + kBlurTH - 1) / kBlurTH);
        if (g.tiles[R] > 0x7FFFFFFFll) return fail(CB200_ERR_ARG, "more than 2^31 blur tiles in one batch");
        order[next[R]++] = i;
        off += (size_t)w * (size_t)h;
    }
    return CB200_OK;
}

int camera_pictures(cb200_ctx* c) { return sstate(c)->camera_n; }
void set_camera_pictures(cb200_ctx* c, int n) { sstate(c)->camera_n = n; }

int camera_table(cb200_ctx* c, const uint8_t* d_pics, const int32_t* wh, int n, std::vector<uint8_t>& table)
{
    table.assign((sizeof(PicDesc) + sizeof(int)) * (size_t)n, 0);
    BlurGroups g;
    return pic_table(sstate(c), d_pics, wh, n, table.data(), g);
}

// blurred pictures + thresholds + anchors for n pictures of sizes wh (checked by check_picture_sizes) packed in device memory, in
// the state's device arrays; enqueued only.  The picture table (PicDesc, in s->d_table) is this call's one upload -- unless
// d_table holds it already (a camera plan's): then *d_desc = d_table and nothing is uploaded
static int scan_enqueue(cb200_ctx* c, const uint8_t* d_pics, const int32_t* wh, int n, const PicDesc* d_table = nullptr,
                        const PicDesc** d_desc_out = nullptr)
{
    ScanScratch* s = sstate(c);
    cudaStream_t st = c->stream;
    int err = scan_reserve(c, wh, n); if (err) return err;
    const size_t table_bytes = (sizeof(PicDesc) + sizeof(int)) * (size_t)n;
    BlurGroups g;
    const PicDesc* d_desc = d_table;
    if (d_table) {
        std::vector<uint8_t> table(table_bytes);
        err = pic_table(s, d_pics, wh, n, table.data(), g); if (err) return err;
    } else {
        CK(s->d_table.ensure(table_bytes), "cudaMalloc picture table");
        int slot;
        uint8_t* h_table;
        err = stage_take(c, table_bytes, &slot, &h_table); if (err) return err;
        err = pic_table(s, d_pics, wh, n, h_table, g); if (err) return err;
        err = stage_send(c, slot, s->d_table, table_bytes, "H2D picture table"); if (err) return err;
        d_desc = reinterpret_cast<const PicDesc*>(s->d_table.get());
    }
    if (d_desc_out) *d_desc_out = d_desc;
    const int* count = g.count;
    const int* group0 = g.group0;
    const long long* tiles = g.tiles;
    const bool* same = g.same;
    const int* d_order = reinterpret_cast<const int*>(d_desc + n);
    CK(cudaMemsetAsync(s->d_hist, 0, sizeof(unsigned) * 256 * (size_t)n, st), "memset histograms");
    // cb200_set_timing: one event set per scan -- [blur + histogram (all radii), Otsu, anchors] through cb200_get_timing
    begin_timed_call(c);
    mark(c);
    for (int R = 1; R <= 4; ++R) {
        if (!count[R]) continue;
        const int uniform = same[R] ? (int)(tiles[R] / count[R]) : 0;
        const unsigned grid = (unsigned)tiles[R];
        const int* ord = d_order + group0[R];
        switch (R) {
        case 1: k_scan_blur4<1><<<grid, kBlurThreads, 0, st>>>(d_pics, s->d_blur, d_desc, ord, count[R], uniform, s->d_hist); break;
        case 2: k_scan_blur4<2><<<grid, kBlurThreads, 0, st>>>(d_pics, s->d_blur, d_desc, ord, count[R], uniform, s->d_hist); break;
        case 3: k_scan_blur4<3><<<grid, kBlurThreads, 0, st>>>(d_pics, s->d_blur, d_desc, ord, count[R], uniform, s->d_hist); break;
        default: k_scan_blur4<4><<<grid, kBlurThreads, 0, st>>>(d_pics, s->d_blur, d_desc, ord, count[R], uniform, s->d_hist); break;
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

// scan_enqueue, then its results into the pinned host arrays of the state
static int scan_run(cb200_ctx* c, const uint8_t* d_pics, const int32_t* wh, int n)
{
    int rc = scan_enqueue(c, d_pics, wh, n); if (rc) return rc;
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

// the host pictures, packed into the staging buffer with one copy each
static int stage_pictures(cb200_ctx* c, const uint8_t* const* pics, const int32_t* wh, int n, const uint8_t** d_out)
{
    ScanScratch* s = sstate(c);
    size_t bytes = 0;
    for (int i = 0; i < n; ++i) bytes += (size_t)wh[2 * i] * (size_t)wh[2 * i + 1] * 3;
    CK(s->d_pics.ensure(bytes), "cudaMalloc picture staging");
    size_t off = 0;
    for (int i = 0; i < n; ++i) {
        const size_t b = (size_t)wh[2 * i] * (size_t)wh[2 * i + 1] * 3;
        CK(cudaMemcpyAsync(s->d_pics + off, pics[i], b, cudaMemcpyHostToDevice, c->stream), "H2D pictures");
        off += b;
    }
    *d_out = s->d_pics;
    return CB200_OK;
}

// the host pointers of a uniform batch (picture i at pics + i w h 3)
static std::vector<const uint8_t*> uniform_pointers(const uint8_t* pics, int w, int h, int n)
{
    std::vector<const uint8_t*> p((size_t)n);
    for (int i = 0; i < n; ++i) p[(size_t)i] = pics + (size_t)i * w * h * 3;
    return p;
}

// Extractor::extract (Extractor.h:30-46) of every picture of a scan, on the device: one thread per picture
__global__ void k_extract(const int4* __restrict__ anchors, const int* __restrict__ count, const int* __restrict__ scan_status, int n,
                          int width, int height, int32_t* __restrict__ status, double* __restrict__ minv, double* __restrict__ fwd,
                          uint8_t* __restrict__ sharpen)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int st = extract::extract_picture(reinterpret_cast<const Anchor*>(anchors + 4 * (size_t)i), count[i], (scan_status[i] & kScanOverflow) != 0,
                                            width, height, fwd + 9 * (size_t)i, minv + 9 * (size_t)i);
    status[i] = st;
    if (sharpen) sharpen[i] = st == 2;             // CB200_FLAG_SHARPEN_IF_NEEDED: the CLI sharpens exactly the NEEDS_SHARPEN pictures
}

// a picture that failed extraction yields no chunks
__global__ void k_mask_failed(const int32_t* __restrict__ status, int n, uint32_t* __restrict__ mask)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && status[i] <= 0) mask[i] = 0;
}

// Extractor::extract + Decoder::decode_fountain for n pictures of sizes wh packed in device memory, enqueued on the context's stream
// without a host round trip: scan, k_extract, deskew with the scan's picture table, decode (with CB200_FLAG_SHARPEN_IF_NEEDED the
// frame lists are built on the device), masks of failed pictures cleared.  The arguments are checked by the caller
int camera_enqueue(cb200_ctx* c, const uint8_t* d, const int32_t* wh, int n, uint32_t flags, uint8_t* d_chunks, uint32_t* d_mask,
                   uint8_t* d_frame_flags, int32_t* d_status)
{
    return camera_enqueue_table(c, d, wh, n, flags, d_chunks, d_mask, d_frame_flags, d_status, nullptr);
}

int camera_reserve(cb200_ctx* c, const int32_t* wh, int n)
{
    ScanScratch* s = sstate(c);
    int rc;
    if ((rc = grow(c, s->d_minv, 9 * (size_t)n, "inverse maps")) || (rc = grow(c, s->d_fwd, 9 * (size_t)n, "transforms")) ||
        (rc = grow(c, c->d_sel, (size_t)c->max_frames * 5, "selection")) || (rc = deskew_reserve(c, n)) || (rc = scan_reserve(c, wh, n)))
        return rc;
    return flood_reserve(c, n);
}

int camera_enqueue_table(cb200_ctx* c, const uint8_t* d, const int32_t* wh, int n, uint32_t flags, uint8_t* d_chunks, uint32_t* d_mask,
                         uint8_t* d_frame_flags, int32_t* d_status, const PicDesc* d_table)
{
    const Mode& m = c->mode;
    size_t src_bytes = 0;
    for (int i = 0; i < n; ++i) {
        const size_t b = (size_t)wh[2 * i] * (size_t)wh[2 * i + 1] * 3;
        if (b >= ((size_t)1 << 32)) return fail(CB200_ERR_ARG, "source picture " + std::to_string(i) + " of 4 GB or more");   // k_deskew's offsets
        src_bytes += b;
    }
    ScanScratch* s = sstate(c);
    int rc = camera_reserve(c, wh, n); if (rc) return rc;
    uint8_t* frames;
    rc = deskew_frames(c, n, &frames); if (rc) return rc;
    const PicDesc* d_desc;
    rc = scan_enqueue(c, d, wh, n, d_table, &d_desc); if (rc) return rc;
    const bool if_needed = (flags & CB200_FLAG_SHARPEN_IF_NEEDED) != 0;
    uint8_t* d_sharp = if_needed ? c->d_sel + 4 * (size_t)n : nullptr;
    k_extract<<<(n + 127) / 128, 128, 0, c->stream>>>(s->d_anchors, s->d_count, s->d_status, n, m.width, m.height, d_status, s->d_minv, s->d_fwd, d_sharp);
    count_launch();
    CK(cudaGetLastError(), "extract launch");
    s->camera_n = n;
    rc = deskew_launch(c, d, src_bytes, s->d_minv, d_desc, n, frames); if (rc) return rc;
    rc = decode_chunks_enqueue(c, frames, n, flags & ~CB200_FLAG_SHARPEN_IF_NEEDED, d_sharp, d_chunks, d_mask, d_frame_flags); if (rc) return rc;
    k_mask_failed<<<(n + 127) / 128, 128, 0, c->stream>>>(d_status, n, d_mask);
    count_launch();
    CK(cudaGetLastError(), "mask launch");
    return CB200_OK;
}

// the synchronous camera entry points: the enqueue-only path into the context's buffers, one copy back, one synchronise
static int scan_extract_decode(cb200_ctx* c, const uint8_t* d, const int32_t* wh, int n, uint32_t flags, uint8_t* chunks_out,
                               uint32_t* chunk_count, uint32_t* chunk_mask, uint8_t* frame_flags, int32_t* extract_status)
{
    ScanScratch* s = sstate(c);
    CK(s->d_ext_status.ensure((size_t)n), "cudaMalloc extract status");
    int rc = camera_enqueue(c, d, wh, n, flags, c->d_data, c->d_mask, nullptr, s->d_ext_status); if (rc) return rc;
    return fetch_fountain(c, n, s->d_ext_status, chunks_out, chunk_count, chunk_mask, frame_flags, extract_status);
}

// the argument checks of the ragged entry points, all before any CUDA call
static int check_ragged(const int32_t* wh, const void* pictures, int n)
{
    if (n < 0) return fail(CB200_ERR_ARG, "n < 0");
    if (!wh) return fail(CB200_ERR_ARG, "null wh");
    if (!pictures) return fail(CB200_ERR_ARG, "null pictures");
    return check_picture_sizes(wh, n);
}

static int check_host_pictures(const uint8_t* const* pictures, int n)
{
    for (int i = 0; i < n; ++i)
        if (!pictures[i]) return fail(CB200_ERR_ARG, "picture " + std::to_string(i) + " is a null pointer");
    return CB200_OK;
}

int check_camera_dev_flags(uint32_t flags)
{
    int rc = check_camera_flags(flags); if (rc) return rc;
    if ((flags & CB200_FLAG_CC_FIT) && (flags & CB200_FLAG_CC_SIMPLE)) return fail(CB200_ERR_ARG, "CC_SIMPLE and CC_FIT are exclusive");
    return CB200_OK;
}

int check_camera_dev_outputs(cb200_ctx* c, int n, const uint8_t* d_chunks, const uint32_t* d_chunk_mask, const int32_t* d_extract_status)
{
    if (!c) return fail(CB200_ERR_ARG, "null context");
    if (!d_chunks || !d_chunk_mask || !d_extract_status) return fail(CB200_ERR_ARG, "null output");
    if (n > c->max_frames) return fail(CB200_ERR_ARG, "n = " + std::to_string(n) + " > max_frames = " + std::to_string(c->max_frames));
    return CB200_OK;
}

// the argument checks of the enqueue-only camera entry point, all before any CUDA call
static int check_camera_dev(cb200_ctx* c, const uint8_t* d_pictures, const int32_t* wh, int n, uint32_t flags, const uint8_t* d_chunks,
                            const uint32_t* d_chunk_mask, const int32_t* d_extract_status)
{
    int rc = check_camera_dev_flags(flags); if (rc) return rc;
    rc = check_ragged(wh, d_pictures, n); if (rc) return rc;
    rc = check_camera_dev_outputs(c, n, d_chunks, d_chunk_mask, d_extract_status); if (rc) return rc;
    rc = check_chain_call(c, flags); if (rc) return rc;
    return check_frozen_camera(c, wh, n);
}

int camera_empty(cb200_ctx* c, uint32_t flags)
{
    if (!chain_linked(c, flags)) return CB200_OK;
    return decode_chunks_enqueue(c, nullptr, 0, flags & ~CB200_FLAG_SHARPEN_IF_NEEDED, nullptr, nullptr, nullptr, nullptr);
}

}  // namespace cb200

using namespace cb200;

extern "C" {

int cb200_scan_dev(cb200_ctx* c, const uint8_t* d_pictures, int w, int h, int n, int32_t* anchors, int32_t* count, uint32_t* cutoff)
{
    if (!c || !d_pictures || !count || n < 0 || w < 1 || h < 1) return fail(CB200_ERR_ARG, "bad arguments");
    if (n == 0) return CB200_OK;
    const std::vector<int32_t> wh = uniform_sizes(w, h, n);
    int rc = check_picture_sizes(wh.data(), 1); if (rc) return rc;
    rc = check_frozen_scan(c, wh.data(), n); if (rc) return rc;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    rc = scan_run(c, d_pictures, wh.data(), n); if (rc) return rc;
    return scan_results(c, n, anchors, count, cutoff);
}

int cb200_scan(cb200_ctx* c, const uint8_t* pictures, int w, int h, int n, int32_t* anchors, int32_t* count, uint32_t* cutoff)
{
    if (!c || !pictures || !count || n < 0 || w < 1 || h < 1) return fail(CB200_ERR_ARG, "bad arguments");
    if (n == 0) return CB200_OK;
    const std::vector<int32_t> wh = uniform_sizes(w, h, n);
    int rc = check_picture_sizes(wh.data(), 1); if (rc) return rc;
    rc = check_frozen_scan(c, wh.data(), n); if (rc) return rc;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    const uint8_t* d = nullptr;
    rc = stage_pictures(c, uniform_pointers(pictures, w, h, n).data(), wh.data(), n, &d); if (rc) return rc;
    rc = scan_run(c, d, wh.data(), n); if (rc) return rc;
    return scan_results(c, n, anchors, count, cutoff);
}

int cb200_scan_ragged_dev(cb200_ctx* c, const uint8_t* d_pictures, const int32_t* wh, int n, int32_t* anchors, int32_t* count, uint32_t* cutoff)
{
    int rc = check_ragged(wh, d_pictures, n); if (rc) return rc;
    if (!c || !count) return fail(CB200_ERR_ARG, !c ? "null context" : "null count");
    if (n == 0) return CB200_OK;
    rc = check_frozen_scan(c, wh, n); if (rc) return rc;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    rc = scan_run(c, d_pictures, wh, n); if (rc) return rc;
    return scan_results(c, n, anchors, count, cutoff);
}

int cb200_scan_ragged(cb200_ctx* c, const uint8_t* const* pictures, const int32_t* wh, int n, int32_t* anchors, int32_t* count, uint32_t* cutoff)
{
    int rc = check_ragged(wh, pictures, n); if (rc) return rc;
    rc = check_host_pictures(pictures, n); if (rc) return rc;
    if (!c || !count) return fail(CB200_ERR_ARG, !c ? "null context" : "null count");
    if (n == 0) return CB200_OK;
    rc = check_frozen_scan(c, wh, n); if (rc) return rc;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    const uint8_t* d = nullptr;
    rc = stage_pictures(c, pictures, wh, n, &d); if (rc) return rc;
    rc = scan_run(c, d, wh, n); if (rc) return rc;
    return scan_results(c, n, anchors, count, cutoff);
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
    int rc = check_camera_flags(flags); if (rc) return rc;
    if (!c || !pictures || !chunks_out || !chunk_count || !extract_status || n < 0 || n > c->max_frames || w < 2 || h < 2)
        return fail(CB200_ERR_ARG, "bad arguments");
    rc = check_chain_call(c, flags); if (rc) return rc;
    if (n == 0) return camera_empty(c, flags);
    const std::vector<int32_t> wh = uniform_sizes(w, h, n);
    rc = check_picture_sizes(wh.data(), 1); if (rc) return rc;
    rc = check_frozen_camera(c, wh.data(), n); if (rc) return rc;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    const uint8_t* d = nullptr;
    rc = stage_pictures(c, uniform_pointers(pictures, w, h, n).data(), wh.data(), n, &d); if (rc) return rc;
    return scan_extract_decode(c, d, wh.data(), n, flags, chunks_out, chunk_count, chunk_mask, frame_flags, extract_status);
}

int cb200_scan_extract_decode_fountain_ragged(cb200_ctx* c, const uint8_t* const* pictures, const int32_t* wh, int n, uint32_t flags,
                                              uint8_t* chunks_out, uint32_t* chunk_count, uint32_t* chunk_mask, uint8_t* frame_flags,
                                              int32_t* extract_status)
{
    int rc = check_camera_flags(flags); if (rc) return rc;
    rc = check_ragged(wh, pictures, n); if (rc) return rc;
    rc = check_host_pictures(pictures, n); if (rc) return rc;
    if (!c) return fail(CB200_ERR_ARG, "null context");
    if (!chunks_out || !chunk_count || !extract_status) return fail(CB200_ERR_ARG, "null output");
    if (n > c->max_frames) return fail(CB200_ERR_ARG, "n = " + std::to_string(n) + " > max_frames = " + std::to_string(c->max_frames));
    rc = check_chain_call(c, flags); if (rc) return rc;
    if (n == 0) return camera_empty(c, flags);
    rc = check_frozen_camera(c, wh, n); if (rc) return rc;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    const uint8_t* d = nullptr;
    rc = stage_pictures(c, pictures, wh, n, &d); if (rc) return rc;
    return scan_extract_decode(c, d, wh, n, flags, chunks_out, chunk_count, chunk_mask, frame_flags, extract_status);
}

int cb200_scan_extract_decode_chunks_ragged_dev(cb200_ctx* c, const uint8_t* d_pictures, const int32_t* wh, int n, uint32_t flags,
                                                uint8_t* d_chunks, uint32_t* d_chunk_mask, uint8_t* d_frame_flags, int32_t* d_extract_status)
{
    int rc = check_camera_dev(c, d_pictures, wh, n, flags, d_chunks, d_chunk_mask, d_extract_status); if (rc) return rc;
    if (n == 0) return camera_empty(c, flags);
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    return camera_enqueue(c, d_pictures, wh, n, flags, d_chunks, d_chunk_mask, d_frame_flags, d_extract_status);
}

int cb200_scan_extract_decode_chunks_dev(cb200_ctx* c, const uint8_t* d_pictures, int w, int h, int n, uint32_t flags, uint8_t* d_chunks,
                                         uint32_t* d_chunk_mask, uint8_t* d_frame_flags, int32_t* d_extract_status)
{
    if (n < 0) return fail(CB200_ERR_ARG, "n < 0");
    const std::vector<int32_t> wh = uniform_sizes(w, h, n);
    return cb200_scan_extract_decode_chunks_ragged_dev(c, d_pictures, wh.data(), n, flags, d_chunks, d_chunk_mask, d_frame_flags, d_extract_status);
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
