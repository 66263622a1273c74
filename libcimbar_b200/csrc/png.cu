// png.cu -- PNG files decoded on the device, bit-exact to cv2.imread + cvtColor(BGR2RGB), and run through the camera path (sm_90a).
// Replaces the first step of the reference CLI's decode loop, `cv::imread(file)` + `cvtColor(BGR2RGB)`
// (src/exe/cimbar/cimbar.cpp:132-133, reference-relative), for PNG files in host memory: camera pictures saved as PNG, and the
// encoder's extracted frames (the CLI's --no-deskew input).
//
// The host walks the chunks (png_core.cuh parse: IHDR, PLTE, eXIf, the IDAT chunks, the zlib header) and uploads the picture and
// IDAT chunk descriptors, the palettes and each file's IDAT payloads back to back (its zlib stream) in one copy from the file
// calls' pinned ring (ctx.cuh UploadRing).  Then, enqueued on the context's stream:
//   k_png_crc       one warp per IDAT chunk: CRC-32 of 32 pieces, combined (png_core.cuh crc_piece / chunk_crc); a mismatch sets
//                   the picture's corrupt flag
//   k_png_inflate   one warp per file: lane 0 reads block headers and decodes batches of up to 32 tokens from a 64-bit bit buffer;
//                   for each Huffman block the warp fills the 10-bit look-up tables in shared memory; the warp places the batch by a
//                   prefix sum over the token lengths, stores its literals together and copies its matches in order (lanes 32
//                   bytes apart, the periodic form for d < 32).  The 32 KB window is the output itself: the filtered scanlines,
//                   h x (1 + stride) bytes per file in the scanline buffer.  Then the Adler-32 (lanes' sums combined) and libpng's
//                   rules for the stream's end
//   k_png_unfilter  one warp per file, rows in order: None in place, Up across the row, Sub as a per-byte-lane prefix sum (warp
//                   scans), Avg and Paeth as serial chains, one lane per byte of a pixel.  A filter type above 4 sets the flag
//   k_png_rgb       one thread per output pixel: eXIf orientation, sub-byte unpacking, palette, grey replicated, 16 -> 8 bit by
//                   truncation, alpha dropped, into the packed ragged RGB8 batch (a corrupt picture is written black)
// With cb200_set_timing: [0] CRC + inflate, [1] unfilter, [2] expand.
#include "ctx.cuh"
#include "png_core.cuh"

#include <string>
#include <vector>

namespace cb200 {

using namespace png;

struct PngState {
    UploadRing up;                     // the calls' uploads (descriptors + IDAT payloads)
    DevBuf<uint8_t> d_blob;            // the call's upload
    DevBuf<uint8_t> d_raw;             // filtered, then unfiltered, scanlines of every file
    DevBuf<int> d_bad;                 // per picture: corrupt data
    DevBuf<uint8_t> d_rgb;             // the camera call's decoded pictures
};

void png_destroy(PngState* p) { delete p; }

static PngState* pstate(cb200_ctx* c)
{
    if (!c->png) c->png = new PngState();
    return c->png;
}

__global__ void __launch_bounds__(32) k_png_crc(const Chunk* __restrict__ chunks, const uint8_t* __restrict__ data, int* __restrict__ bad)
{
    const Chunk& C = chunks[blockIdx.x];
    uint32_t x = crc_piece(data + C.begin, C.len, threadIdx.x, 32);
    for (int o = 16; o; o >>= 1) x ^= __shfl_xor_sync(0xFFFFFFFFu, x, o);
    if (threadIdx.x == 0 && chunk_crc(x, C.len) != C.crc) bad[C.pic] = 1;
}

enum Cmd { kCmdTables = 0, kCmdStored = 1, kCmdTokens = 2, kCmdEnd = 3, kCmdBad = 4 };

__global__ void __launch_bounds__(32) k_png_inflate(const Pic* __restrict__ pics, const Chunk* __restrict__ chunks,
                                                     const uint8_t* __restrict__ data, uint8_t* __restrict__ raw, int* __restrict__ bad)
{
    __shared__ Huff lit, dist;
    __shared__ uint8_t lens[320];
    __shared__ Tok tok[kBatch];
    __shared__ uint64_t s_p, s_src;
    __shared__ uint32_t s_len;
    __shared__ int s_cmd, s_nt, s_st;
    const Pic& P = pics[blockIdx.x];
    const int lane = threadIdx.x;
    const uint64_t cap = (uint64_t)P.h * (1 + P.stride);
    uint8_t* out = raw + P.raw;
    const uint8_t* z = data + P.z;
    Inflate I;
    if (lane == 0) inflate_init(I, P, chunks + P.chunk0, data);
    for (;;) {
        if (lane == 0) {
            s_p = I.out;
            int cmd = kCmdTokens;
            if (I.block == kNeedHeader) {
                int nlit = 0, ndist = 0;
                if (!block_header(I, lens, &nlit, &ndist, dist) || consumed(I.b) > 8 * I.b.zlen) cmd = kCmdBad;
                else if (I.block == kStored) cmd = kCmdStored;
                else cmd = build(lit, lens, nlit, false) && build(dist, lens + 288, ndist, false) ? kCmdTables : kCmdBad;
            } else if (I.block == kFinished) {
                cmd = kCmdEnd;
            }
            if (cmd == kCmdStored) {
                uint64_t src;
                uint32_t len;
                if (stored_step(I, &src, &len)) { s_src = src; s_len = len; } else cmd = kCmdBad;
            } else if (cmd == kCmdTokens) {
                int nt;
                const int st = decode_batch(I, lit, dist, tok, &nt);
                s_nt = nt;
                s_st = st;
                if (st == kEndOfBlock) I.block = I.last ? kFinished : kNeedHeader;
            }
            s_cmd = cmd;
        }
        __syncwarp();
        const int cmd = s_cmd;
        const uint64_t p = s_p;
        if (cmd == kCmdBad || cmd == kCmdEnd) break;
        if (cmd == kCmdTables) {
            for (uint32_t e = lane; e < (1u << kLookBits); e += 32) { fill_look(lit, e); fill_look(dist, e); }
        } else if (cmd == kCmdStored) {
            const uint64_t src = s_src;
            const uint32_t len = s_len;
            for (uint32_t i = lane; i < len; i += 32)
                if (p + i < cap) out[p + i] = z[src + i];
        } else {
            // the batch: token k at lane k, its first byte by a prefix sum of the lengths
            const int nt = s_nt;
            const uint32_t len = lane < nt ? tok[lane].len : 0, v = lane < nt ? tok[lane].v : 0;
            uint32_t at = len;
            for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, at, o); if (lane >= o) at += y; }
            const uint64_t q = p + at - len;
            if (len == 1 && q < cap) out[q] = (uint8_t)v;
            __syncwarp();
            for (int k = 0; k < nt; ++k) {
                const uint32_t lk = __shfl_sync(0xFFFFFFFFu, len, k), dk = __shfl_sync(0xFFFFFFFFu, v, k);
                const uint64_t qk = __shfl_sync(0xFFFFFFFFu, q, k);
                if (lk > 1) { copy_match(out, qk, lk, dk, cap, lane, 32); __syncwarp(); }
            }
            if (s_st == kBad) { if (lane == 0) s_cmd = kCmdBad; __syncwarp(); break; }
        }
        __syncwarp();
    }
    __syncwarp();
    if (s_cmd == kCmdBad) { if (lane == 0) bad[blockIdx.x] = 1; return; }
    uint32_t a, b;
    adler_piece(out, cap, lane, 32, &a, &b);
    for (int o = 16; o; o >>= 1) {
        a = (a + __shfl_xor_sync(0xFFFFFFFFu, a, o)) % 65521;
        b = (b + __shfl_xor_sync(0xFFFFFFFFu, b, o)) % 65521;
    }
    if (lane == 0 && !stream_end_ok(I, chunks + P.chunk0, P.nchunks, P.z, adler_of(a, b, cap))) bad[blockIdx.x] = 1;
}

__global__ void __launch_bounds__(32) k_png_unfilter(const Pic* __restrict__ pics, uint8_t* __restrict__ raw, int* __restrict__ bad)
{
    const Pic& P = pics[blockIdx.x];
    if (bad[blockIdx.x]) return;
    const int lane = threadIdx.x, bpp = P.bpp;
    const uint32_t stride = P.stride;
    for (int y = 0; y < P.h; ++y) {
        uint8_t* row = raw + P.raw + (uint64_t)y * (1 + stride);
        const int f = row[0];
        uint8_t* cur = row + 1;
        const uint8_t* prev = y ? cur - (1 + stride) : nullptr;
        if (f > 4) { if (lane == 0) bad[blockIdx.x] = 1; return; }
        if (f == 2 && prev) {
            for (uint32_t x = lane; x < stride; x += 32) cur[x] = (uint8_t)(cur[x] + prev[x]);
        } else if (f == 1) {
            // pixel base + lane, byte lane c: an inclusive warp scan per c, carried from the previous 32 pixels
            uint32_t carry[8] = {0, 0, 0, 0, 0, 0, 0, 0};
            for (uint32_t base = 0; base * bpp < stride; base += 32) {
#pragma unroll
                for (int c = 0; c < 8; ++c) {
                    if (c >= bpp) break;
                    const uint32_t x = (base + lane) * bpp + c;
                    uint32_t s = x < stride ? cur[x] : 0;
                    for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, s, o); if (lane >= o) s += t; }
                    s += carry[c];
                    if (x < stride) cur[x] = (uint8_t)s;
                    carry[c] = __shfl_sync(0xFFFFFFFFu, s, 31) & 0xFF;
                }
            }
        } else if (f == 3 || f == 4) {
            if (lane < bpp) unfilter_chain(cur, prev, stride, bpp, lane, f);
        }
        __syncwarp();
    }
}

__global__ void k_png_rgb(const Pic* __restrict__ pics, const uint8_t* __restrict__ raw, const uint8_t* __restrict__ pal,
                          const int* __restrict__ bad, uint8_t* __restrict__ out)
{
    const Pic& P = pics[blockIdx.y];
    const uint64_t px = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (px >= (uint64_t)P.ow * P.oh) return;
    const int oy = (int)(px / (uint64_t)P.ow), ox = (int)(px - (uint64_t)oy * P.ow);
    uint8_t rgb[3] = {0, 0, 0};
    if (!bad[blockIdx.y]) pixel_rgb(raw + P.raw, pal, P, ox, oy, rgb);
    uint8_t* o = out + P.out + 3 * px;
    o[0] = rgb[0]; o[1] = rgb[1]; o[2] = rgb[2];
}

// the files' chunks, all before any CUDA call: CB200_ERR_ARG naming the picture for a refused file or size
static int parse_files(const uint8_t* const* files, const uint64_t* sizes, int n, std::vector<Parsed>& ps, std::vector<int32_t>& wh)
{
    if (n < 0) return fail(CB200_ERR_ARG, "n < 0");
    if (!files) return fail(CB200_ERR_ARG, "null files");
    if (!sizes) return fail(CB200_ERR_ARG, "null sizes");
    if ((long long)n > 65535) return fail(CB200_ERR_ARG, "more than 65535 pictures in one call");
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

// the decode of parsed files into d_rgb (the packed ragged RGB8 batch), enqueued on the context's stream
static int png_enqueue(cb200_ctx* c, const std::vector<Parsed>& ps, const uint8_t* const* files, uint8_t* d_rgb)
{
    PngState* s = pstate(c);
    const int n = (int)ps.size();
    const Layout L = layout(ps);
    cudaStream_t st = c->stream;
    CK(s->d_blob.ensure(L.bytes), "cudaMalloc PNG upload");
    CK(s->d_raw.ensure(L.raw), "cudaMalloc PNG scanlines");
    CK(s->d_bad.ensure((size_t)n), "cudaMalloc PNG flags");
    int slot, rc;
    uint8_t* h;
    rc = s->up.take(L.bytes, &slot, &h); if (rc) return rc;
    pack(ps, files, L, h);
    rc = s->up.send(st, slot, s->d_blob, L.bytes); if (rc) return rc;
    const uint8_t* b = s->d_blob;
    const Pic* pics = reinterpret_cast<const Pic*>(b + L.pics);
    const Chunk* chunks = reinterpret_cast<const Chunk*>(b + L.chunks);
    CK(cudaMemsetAsync(s->d_bad, 0, sizeof(int) * (size_t)n, st), "memset PNG flags");
    begin_timed_call(c);
    mark(c);
    if (L.nchunks) { k_png_crc<<<L.nchunks, 32, 0, st>>>(chunks, b + L.data, s->d_bad); count_launch(); }
    k_png_inflate<<<n, 32, 0, st>>>(pics, chunks, b + L.data, s->d_raw, s->d_bad);
    count_launch();
    mark(c);
    k_png_unfilter<<<n, 32, 0, st>>>(pics, s->d_raw, s->d_bad);
    count_launch();
    mark(c);
    k_png_rgb<<<dim3((unsigned)((L.max_px + 255) / 256), n), 256, 0, st>>>(pics, s->d_raw, b + L.pal, s->d_bad, d_rgb);
    count_launch();
    mark(c);
    CK(cudaGetLastError(), "PNG launch");
    return CB200_OK;
}

}  // namespace cb200

using namespace cb200;

extern "C" {

int cb200_png_info(const uint8_t* file, uint64_t size, int32_t* w, int32_t* h)
{
    if (!file || !w || !h) return fail(CB200_ERR_ARG, "null argument");
    std::vector<Parsed> ps;
    std::vector<int32_t> wh;
    int rc = parse_files(&file, &size, 1, ps, wh); if (rc) return rc;
    *w = wh[0];
    *h = wh[1];
    return CB200_OK;
}

int cb200_png_decode_dev(cb200_ctx* c, const uint8_t* const* files, const uint64_t* sizes, int n, uint8_t* d_rgb_out, int32_t* d_status)
{
    std::vector<Parsed> ps;
    std::vector<int32_t> wh;
    int rc = parse_files(files, sizes, n, ps, wh); if (rc) return rc;
    if (!c) return fail(CB200_ERR_ARG, "null context");
    if (!d_rgb_out) return fail(CB200_ERR_ARG, "null output");
    if (n == 0) return CB200_OK;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    rc = png_enqueue(c, ps, files, d_rgb_out); if (rc) return rc;
    if (d_status) {
        CK(cudaMemsetAsync(d_status, 0, sizeof(int32_t) * (size_t)n, c->stream), "memset status");
        return file_status(c, c->png->d_bad, n, d_status, nullptr);
    }
    return CB200_OK;
}

int cb200_png_scan_extract_decode_chunks_dev(cb200_ctx* c, const uint8_t* const* files, const uint64_t* sizes, int n, uint32_t flags,
                                             uint8_t* d_chunks, uint32_t* d_chunk_mask, uint8_t* d_frame_flags, int32_t* d_extract_status)
{
    // the decoded pictures are a packed batch of the sizes in the files' headers; where they go is known once they are decoded
    std::vector<Parsed> ps;
    auto build = [&](CameraBatch& b) {
        int rc = parse_files(files, sizes, n, ps, b.wh); if (rc) return rc;
        b.pack(nullptr);
        return CB200_OK;
    };
    CameraBatch b;
    int rc = check_camera_call(c, flags, build, b, d_chunks && d_chunk_mask && d_extract_status ? nullptr : "null output"); if (rc) return rc;
    if (n == 0) return empty_stripe(c, flags, true);
    rc = check_frozen_camera(c, b.wh.data(), n); if (rc) return rc;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    PngState* s = pstate(c);
    uint64_t rgb = 0;
    for (int i = 0; i < n; ++i) rgb += 3 * (uint64_t)b.wh[2 * (size_t)i] * (uint64_t)b.wh[2 * (size_t)i + 1];
    CK(s->d_rgb.ensure(rgb), "cudaMalloc PNG pictures");
    rc = png_enqueue(c, ps, files, s->d_rgb); if (rc) return rc;
    b.pack(s->d_rgb);
    rc = camera_enqueue(c, b, flags, d_chunks, d_chunk_mask, d_frame_flags, d_extract_status); if (rc) return rc;
    return file_status(c, s->d_bad, n, d_extract_status, d_chunk_mask);
}

}  // extern "C"
