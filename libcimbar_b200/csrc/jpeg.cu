// jpeg.cu -- JPEG photographs decoded on the device, bit-exact to cv2.imread + cvtColor(BGR2RGB), and run through the camera path
// (sm_90a).  Replaces the first step of the reference CLI's decode loop, `cv::imread(file)` + `cvtColor(BGR2RGB)`
// (src/exe/cimbar/cimbar.cpp:132-133, reference-relative), for a batch of files in host memory.
//
// The host parses the markers (jpeg_core.cuh parse: tables, scans, restart intervals, EXIF orientation) and uploads the picture,
// scan, segment and table descriptors together with the compressed files in one copy from a pinned ring of its own (ctx.cuh
// FileUpload, the type the PNG calls use too).  Then,
// enqueued on the context's stream:
//   k_jpeg_init     the per-picture corrupt flag from the parse (a file that ends inside its data)
//   k_jpeg_unstuff  one CTA per segment (restart interval, or whole scan): FF 00 stuffing out by a flag + block-wide prefix sum
//                   compaction, into the unstuffed buffer at the segment's offset
//   k_jpeg_decode   one launch per round r = the r-th scan of every picture (a picture's scans run in file order, pictures side by
//                   side), one CTA of kSegThreads per segment, the scan's Huffman tables in shared memory.  Sequential, DC and
//                   AC-first scans: the self-synchronising parallel decode of jpeg_core.cuh (speculative subsequences, sync rounds
//                   until every start state is its predecessor's end state, prefix sums of blocks and DC differences, write pass).
//                   AC refinement scans: the CTA builds every block's nonzero mask, one thread decodes the segment in order into
//                   per-block correction masks, and the CTA applies them.  Corrupt data set the picture's flag
//   k_jpeg_idct     one thread per 8 x 8 block: dequantise + jpeg_idct_islow into the component's sample plane
//   k_jpeg_rgb      one thread per output pixel: EXIF orientation, fancy upsampling, YCbCr -> RGB, into the packed ragged RGB8
//                   batch (a corrupt picture is written black)
// The coefficient, plane and unstuffed buffers belong to the context and grow as batches need.
#include "ctx.cuh"
#include "jpeg_core.cuh"

#include <string>
#include <vector>

namespace cb200 {

using namespace jpeg;

constexpr int kSegThreads = 512;       // threads per segment in k_jpeg_unstuff / k_jpeg_decode

struct JpegState {
    FileUpload up;                     // the calls' uploads (descriptors + files)
    DevBuf<uint8_t> d_blob;            // the call's upload (descriptors + files)
    DevBuf<uint8_t> d_unstuffed;       // the segments' bytes without FF 00 stuffing, at their offsets in the data section
    DevBuf<uint32_t> d_ulen;           // per segment: its unstuffed bytes
    DevBuf<int16_t> d_coef;            // coefficients of every component plane
    DevBuf<uint8_t> d_planes;          // sample planes
    DevBuf<uint64_t> d_masks;          // AC refinement: 4 masks per block (jpeg_core.cuh decode_refine)
    DevBuf<int> d_bad;                 // per picture: corrupt data
    DevBuf<uint8_t> d_rgb;             // the camera call's decoded pictures
};

void jpeg_destroy(JpegState* j) { delete j; }

static JpegState* jstate(cb200_ctx* c)
{
    if (!c->jpeg) c->jpeg = new JpegState();
    return c->jpeg;
}

__global__ void k_jpeg_init(const Pic* __restrict__ pics, int n, int* __restrict__ bad)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) bad[i] = pics[i].bad;
}

// block-wide exclusive prefix sum of v over kSegThreads threads (scratch: kSegThreads / 32 words); *total gets the sum
__device__ uint32_t block_scan(uint32_t v, uint32_t* scratch, uint32_t* total)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t x = v;
    for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, x, o); if (lane >= o) x += y; }
    if (lane == 31) scratch[warp] = x;
    __syncthreads();
    if (warp == 0) {
        uint32_t w = lane < kSegThreads / 32 ? scratch[lane] : 0;
        for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, w, o); if (lane >= o) w += y; }
        if (lane < kSegThreads / 32) scratch[lane] = w;
    }
    __syncthreads();
    const uint32_t before = (warp ? scratch[warp - 1] : 0) + x - v;
    *total = scratch[kSegThreads / 32 - 1];
    __syncthreads();
    return before;
}

__global__ void __launch_bounds__(kSegThreads) k_jpeg_unstuff(const uint8_t* __restrict__ raw, const Seg* __restrict__ segs,
                                                              uint8_t* __restrict__ u, uint32_t* __restrict__ ulen)
{
    __shared__ uint32_t scratch[kSegThreads / 32];
    const Seg& sg = segs[blockIdx.x];
    uint32_t kept_so_far = 0;
    for (uint64_t i0 = sg.begin; i0 < sg.end; i0 += kSegThreads) {
        const uint64_t i = i0 + threadIdx.x;
        const bool k = i < sg.end && kept(raw, i, sg.begin);
        uint32_t total;
        const uint32_t at = block_scan(k ? 1u : 0u, scratch, &total);
        if (k) u[sg.begin + kept_so_far + at] = raw[i];
        kept_so_far += total;
    }
    if (threadIdx.x == 0) ulen[blockIdx.x] = kept_so_far;
}

// one segment per CTA: the parallel decode of jpeg_core.cuh (decode_segment_sync is its host restatement), or, for an AC refinement
// scan, refine_prep / decode_refine (thread 0) / refine_apply
__global__ void __launch_bounds__(kSegThreads) k_jpeg_decode(const uint8_t* __restrict__ u, const uint32_t* __restrict__ ulens,
                                                             const Pic* __restrict__ pics, const Scan* __restrict__ scans,
                                                             const Seg* __restrict__ segs, const Huff* __restrict__ huffs, uint32_t seg0,
                                                             int16_t* __restrict__ coef, uint64_t* __restrict__ masks, int* __restrict__ bad)
{
    __shared__ Huff tab[8];                                   // DC tables of scan slots 0..3, then AC tables
    __shared__ Unit ends[kSegThreads];
    __shared__ uint32_t scratch[kSegThreads / 32];
    __shared__ int sbad;
    const uint32_t si = seg0 + blockIdx.x;
    const Seg& sg = segs[si];
    const Scan& sc = scans[sg.scan];
    const Pic& P = pics[sc.pic];
    if (threadIdx.x == 0) sbad = bad[sc.pic];                 // read once: another segment's CTA may set it meanwhile
    __syncthreads();
    if (sbad) return;
    const uint8_t* d = u + sg.begin;
    const uint32_t ulen = ulens[si];
    if (sc.kind == kAcRefine) {                               // the blocks' nonzero masks, the decode in order, the masks applied
        const uint32_t nb = segment_blocks(sc, sg);
        for (uint32_t k = threadIdx.x; k < nb; k += kSegThreads) {
            const uint64_t o = block_offset(P, sc, sg, k);
            refine_prep(coef + o, sc.ss, sc.se, masks + 4 * (o / 64));
        }
        __syncthreads();
        if (threadIdx.x == 0 && !decode_refine(d, ulen, P, sc, sg, huffs[sc.ac[0]], masks)) bad[sc.pic] = 1;
        __syncthreads();
        for (uint32_t k = threadIdx.x; k < nb; k += kSegThreads) {
            const uint64_t o = block_offset(P, sc, sg, k);
            refine_apply(coef + o, sc.al, masks + 4 * (o / 64));
        }
        return;
    }
    // the scan's tables into shared memory
    const bool need_dc = sc.kind == kSequential || sc.kind == kDcFirst, need_ac = sc.kind == kSequential || sc.kind == kAcFirst;
    constexpr int kWords = (int)(sizeof(Huff) / 4);
    for (int w = threadIdx.x; w < 8 * kWords; w += kSegThreads) {
        const int t = w / kWords, s = t & 3;
        if (s >= sc.ncomp || (t < 4 ? !need_dc : !need_ac)) continue;
        const Huff* src = huffs + (t < 4 ? sc.dc[s] : sc.ac[s]);
        reinterpret_cast<uint32_t*>(&tab[t])[w % kWords] = reinterpret_cast<const uint32_t*>(src)[w % kWords];
    }
    __syncthreads();
    const Huff* dct[4] = {&tab[0], &tab[1], &tab[2], &tab[3]};
    const Huff* act[4] = {&tab[4], &tab[5], &tab[6], &tab[7]};
    const int t = threadIdx.x;
    const uint32_t S = sub_size(ulen, kSegThreads), stop = sub_end(S, t, kSegThreads, ulen), total = segment_blocks(sc, sg);
    // speculative decode of every subsequence, then the sync rounds
    Unit start = {sub_begin(S, t, ulen), 0};
    Region R;
    run_region(d, ulen, P, sc, sg, dct, act, start, stop, 0, nullptr, nullptr, R);
    ends[t] = R.end;
    __syncthreads();
    for (;;) {
        const Unit in = t ? ends[t - 1] : start;
        __syncthreads();
        bool changed = false;
        if (!same(in, start)) {
            start = in;
            const Unit old = R.end;
            run_region(d, ulen, P, sc, sg, dct, act, start, stop, 0, nullptr, nullptr, R);
            ends[t] = R.end;
            changed = !same(old, R.end);
        }
        if (!__syncthreads_or(changed)) break;
    }
    // first block and DC predictions of every thread, then the write pass
    uint32_t sum;
    const uint32_t g0 = block_scan(R.blocks, scratch, &sum);
    int pred[4] = {0, 0, 0, 0};
    if (sc.kind == kSequential || sc.kind == kDcFirst)
        for (int s = 0; s < sc.ncomp; ++s) pred[s] = (int)block_scan((uint32_t)R.dc[s], scratch, &sum);
    Region W;
    run_region(d, ulen, P, sc, sg, dct, act, start, stop, g0, pred, coef, W);
    if (!region_ok(start, W, g0, total, ulen)) sbad = 1;
    const int tail = __syncthreads_or(W.tail != kNoState);
    if (t == 0 && (sbad || !tail)) bad[sc.pic] = 1;
}

__global__ void k_jpeg_idct(const Pic* __restrict__ pics, const uint16_t* __restrict__ quant, const int16_t* __restrict__ coef,
                            uint8_t* __restrict__ planes)
{
    const Pic& P = pics[blockIdx.y / 3];
    const int c = blockIdx.y % 3;
    if (c >= P.ncomp) return;
    const Comp& C = P.comp[c];
    const int blk = blockIdx.x * blockDim.x + threadIdx.x;
    if (blk >= C.bw * C.bh) return;
    const int by = blk / C.bw, bx = blk - by * C.bw;
    idct_islow(coef + C.coef + (size_t)blk * 64, quant + C.quant, planes + C.plane + (size_t)by * 64 * C.bw + (size_t)bx * 8, (size_t)C.bw * 8);
}

__global__ void k_jpeg_rgb(const Pic* __restrict__ pics, const uint8_t* __restrict__ planes, const int* __restrict__ bad, uint8_t* __restrict__ out)
{
    const Pic& P = pics[blockIdx.y];
    const int px = blockIdx.x * blockDim.x + threadIdx.x;
    if (px >= P.ow * P.oh) return;
    const int oy = px / P.ow, ox = px - oy * P.ow;
    uint8_t rgb[3] = {0, 0, 0};
    if (!bad[blockIdx.y]) pixel_rgb(planes, P, ox, oy, rgb);
    uint8_t* o = out + P.out + 3 * (size_t)px;
    o[0] = rgb[0]; o[1] = rgb[1]; o[2] = rgb[2];
}

// the files' headers, all before any CUDA call: CB200_ERR_ARG naming the picture for a refused file or size
static int parse_files(const uint8_t* const* files, const uint64_t* sizes, int n, std::vector<Parsed>& ps, std::vector<int32_t>& wh)
{
    if (n < 0) return fail(CB200_ERR_ARG, "n < 0");
    if (!files) return fail(CB200_ERR_ARG, "null files");
    if (!sizes) return fail(CB200_ERR_ARG, "null sizes");
    if (3 * (long long)n > 65535) return fail(CB200_ERR_ARG, "more than 21845 pictures in one call");
    ps.resize((size_t)n);
    wh.resize(2 * (size_t)n);
    for (int i = 0; i < n; ++i) {
        if (!files[i]) return fail(CB200_ERR_ARG, "picture " + std::to_string(i) + " is a null pointer");
        const std::string why = parse(files[i], sizes[i], ps[(size_t)i]);
        if (!why.empty()) return fail(CB200_ERR_ARG, "picture " + std::to_string(i) + ": " + why);
        wh[2 * (size_t)i] = ps[(size_t)i].pic.ow;
        wh[2 * (size_t)i + 1] = ps[(size_t)i].pic.oh;
    }
    return check_picture_sizes(wh.data(), n);
}

// the decode of parsed files into d_rgb (the packed ragged RGB8 batch), enqueued on the context's stream.  With cb200_set_timing:
// [0] unstuffing, [1] entropy decode (all rounds), [2] IDCT, [3] upsampling + colour
static int jpeg_enqueue(cb200_ctx* c, const std::vector<Parsed>& ps, const uint8_t* const* files, const uint64_t* sizes, uint8_t* d_rgb)
{
    JpegState* j = jstate(c);
    const int n = (int)ps.size();
    const Layout L = layout(ps, sizes);
    cudaStream_t st = c->stream;
    const size_t nseg = L.round0.back();
    CK(j->d_blob.ensure(L.bytes), "cudaMalloc JPEG upload");
    CK(j->d_unstuffed.ensure(L.bytes - L.data), "cudaMalloc JPEG unstuffed data");
    CK(j->d_ulen.ensure(nseg ? nseg : 1), "cudaMalloc JPEG segment lengths");
    CK(j->d_coef.ensure(L.coef), "cudaMalloc JPEG coefficients");
    CK(j->d_planes.ensure(L.planes), "cudaMalloc JPEG planes");
    CK(j->d_masks.ensure(4 * (L.coef / 64)), "cudaMalloc JPEG refinement masks");
    CK(j->d_bad.ensure((size_t)n), "cudaMalloc JPEG flags");
    int slot, rc;
    uint8_t* h;
    rc = j->up.take(L.bytes, &slot, &h); if (rc) return rc;
    pack(ps, files, sizes, L, h);
    rc = j->up.send(st, slot, j->d_blob, L.bytes); if (rc) return rc;
    const uint8_t* b = j->d_blob;
    const Pic* pics = reinterpret_cast<const Pic*>(b + L.pics);
    const Seg* segs = reinterpret_cast<const Seg*>(b + L.segs);
    CK(cudaMemsetAsync(j->d_coef, 0, sizeof(int16_t) * L.coef, st), "memset JPEG coefficients");
    begin_timed_call(c);
    mark(c);
    k_jpeg_init<<<(n + 127) / 128, 128, 0, st>>>(pics, n, j->d_bad); count_launch();
    if (nseg) { k_jpeg_unstuff<<<(unsigned)nseg, kSegThreads, 0, st>>>(b + L.data, segs, j->d_unstuffed, j->d_ulen); count_launch(); }
    mark(c);
    for (size_t r = 0; r + 1 < L.round0.size(); ++r) {
        const uint32_t s0 = L.round0[r], ns = L.round0[r + 1] - s0;
        if (!ns) continue;
        k_jpeg_decode<<<ns, kSegThreads, 0, st>>>(j->d_unstuffed, j->d_ulen, pics, reinterpret_cast<const Scan*>(b + L.scans), segs,
                                                  reinterpret_cast<const Huff*>(b + L.huffs), s0, j->d_coef, j->d_masks, j->d_bad);
        count_launch();
    }
    mark(c);
    k_jpeg_idct<<<dim3((L.max_blocks + 127) / 128, 3 * n), 128, 0, st>>>(pics, reinterpret_cast<const uint16_t*>(b + L.quant), j->d_coef, j->d_planes);
    count_launch();
    mark(c);
    k_jpeg_rgb<<<dim3((L.max_px + 255) / 256, n), 256, 0, st>>>(pics, j->d_planes, j->d_bad, d_rgb);
    count_launch();
    mark(c);
    CK(cudaGetLastError(), "JPEG launch");
    return CB200_OK;
}

}  // namespace cb200

using namespace cb200;

extern "C" {

int cb200_jpeg_info(const uint8_t* file, uint64_t size, int32_t* w, int32_t* h)
{
    if (!file || !w || !h) return fail(CB200_ERR_ARG, "null argument");
    std::vector<Parsed> ps;
    std::vector<int32_t> wh;
    int rc = parse_files(&file, &size, 1, ps, wh); if (rc) return rc;
    *w = wh[0];
    *h = wh[1];
    return CB200_OK;
}

int cb200_jpeg_decode_dev(cb200_ctx* c, const uint8_t* const* files, const uint64_t* sizes, int n, uint8_t* d_rgb_out, int32_t* d_status)
{
    std::vector<Parsed> ps;
    std::vector<int32_t> wh;
    int rc = parse_files(files, sizes, n, ps, wh); if (rc) return rc;
    if (!c) return fail(CB200_ERR_ARG, "null context");
    if (!d_rgb_out) return fail(CB200_ERR_ARG, "null output");
    if (n == 0) return CB200_OK;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    rc = jpeg_enqueue(c, ps, files, sizes, d_rgb_out); if (rc) return rc;
    if (d_status) {
        CK(cudaMemsetAsync(d_status, 0, sizeof(int32_t) * (size_t)n, c->stream), "memset status");
        return file_status(c, c->jpeg->d_bad, n, d_status, nullptr);
    }
    return CB200_OK;
}

int cb200_jpeg_scan_extract_decode_chunks_dev(cb200_ctx* c, const uint8_t* const* files, const uint64_t* sizes, int n, uint32_t flags,
                                              uint8_t* d_chunks, uint32_t* d_chunk_mask, uint8_t* d_frame_flags, int32_t* d_extract_status)
{
    std::vector<Parsed> ps;
    std::vector<int32_t> wh;
    int rc = parse_files(files, sizes, n, ps, wh); if (rc) return rc;
    rc = check_camera_dev_flags(flags); if (rc) return rc;
    rc = check_camera_dev_outputs(c, n, d_chunks, d_chunk_mask, d_extract_status); if (rc) return rc;
    rc = check_chain_call(c, flags); if (rc) return rc;
    if (n == 0) return camera_empty(c, flags);
    rc = check_frozen_camera(c, wh.data(), n); if (rc) return rc;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    JpegState* j = jstate(c);
    uint64_t rgb = 0;
    for (int i = 0; i < n; ++i) rgb += 3 * (uint64_t)wh[2 * (size_t)i] * (uint64_t)wh[2 * (size_t)i + 1];
    CK(j->d_rgb.ensure(rgb), "cudaMalloc JPEG pictures");
    rc = jpeg_enqueue(c, ps, files, sizes, j->d_rgb); if (rc) return rc;
    rc = camera_enqueue(c, j->d_rgb, wh.data(), n, flags, d_chunks, d_chunk_mask, d_frame_flags, d_extract_status); if (rc) return rc;
    return file_status(c, j->d_bad, n, d_extract_status, d_chunk_mask);
}

}  // extern "C"
