// The PNG decode of the camera path (libcimbar_b200/csrc/png_core.cuh: what png.cu's kernels run) compiled for the host, for
// tests/test_png_core_host.py: the same parse, upload layout, CRC pieces, inflate steps, unfilter chains and expand, in the kernels'
// order, with the warp's lanes run one after the other.
#include "../../libcimbar_b200/csrc/png_core.cuh"

#include <stdio.h>

using namespace cb200::png;

namespace {

constexpr int kLanes = 32;

// k_png_inflate for one file: true, or false for corrupt data
bool inflate_file(const Pic& P, const Chunk* chunks, const uint8_t* data, uint8_t* out)
{
    static Huff lit, dist;
    uint8_t lens[320];
    Tok tok[kBatch];
    const uint64_t cap = (uint64_t)P.h * (1 + P.stride);
    const uint8_t* z = data + P.z;
    Inflate I;
    inflate_init(I, P, chunks + P.chunk0, data);
    for (;;) {
        const uint64_t p = I.out;
        if (I.block == kFinished) break;
        if (I.block == kNeedHeader) {
            int nlit = 0, ndist = 0;
            if (!block_header(I, lens, &nlit, &ndist, dist) || consumed(I.b) > 8 * I.b.zlen) return false;
            if (I.block == kStored) {
                uint64_t src;
                uint32_t len;
                if (!stored_step(I, &src, &len)) return false;
                for (int lane = 0; lane < kLanes; ++lane)
                    for (uint32_t i = (uint32_t)lane; i < len; i += kLanes)
                        if (p + i < cap) out[p + i] = z[src + i];
                continue;
            }
            if (!build(lit, lens, nlit, false) || !build(dist, lens + 288, ndist, false)) return false;
            for (uint32_t e = 0; e < (1u << kLookBits); ++e) { fill_look(lit, e); fill_look(dist, e); }
            continue;
        }
        int nt;
        const int st = decode_batch(I, lit, dist, tok, &nt);
        if (st == kEndOfBlock) I.block = I.last ? kFinished : kNeedHeader;
        uint64_t q = p;
        for (int k = 0; k < nt; ++k) {                    // the literals (lane k), then the matches in order, lane by lane
            if (tok[k].len == 1 && q < cap) out[q] = (uint8_t)tok[k].v;
            q += tok[k].len;
        }
        q = p;
        for (int k = 0; k < nt; ++k) {
            if (tok[k].len > 1)
                for (int lane = 0; lane < kLanes; ++lane) copy_match(out, q, tok[k].len, tok[k].v, cap, lane, kLanes);
            q += tok[k].len;
        }
        if (st == kBad) return false;
    }
    uint32_t A = 0, B = 0;
    for (int lane = 0; lane < kLanes; ++lane) {
        uint32_t a, b;
        adler_piece(out, cap, lane, kLanes, &a, &b);
        A = (A + a) % 65521;
        B = (B + b) % 65521;
    }
    return stream_end_ok(I, chunks + P.chunk0, P.nchunks, P.z, adler_of(A, B, cap));
}

}  // namespace

extern "C" {

// w, h of the output (after orientation): 0, or 1 with the refusal reason in why
int pc_info(const uint8_t* file, uint64_t size, int* wh, char* why, int why_cap)
{
    Parsed p;
    const std::string r = parse(file, size, p);
    if (!r.empty()) { snprintf(why, (size_t)why_cap, "%s", r.c_str()); return 1; }
    wh[0] = p.pic.ow; wh[1] = p.pic.oh;
    return 0;
}

// the RGB8 picture into rgb (cap bytes): 0, -2 for corrupt data, 1 refused (why), 2 too small a buffer
int pc_decode(const uint8_t* file, uint64_t size, uint8_t* rgb, uint64_t cap, int* wh, char* why, int why_cap)
{
    std::vector<Parsed> ps(1);
    const std::string r = parse(file, size, ps[0]);
    if (!r.empty()) { snprintf(why, (size_t)why_cap, "%s", r.c_str()); return 1; }
    const Layout L = layout(ps);
    if (L.rgb > cap) return 2;
    std::vector<uint8_t> blob(L.bytes);
    pack(ps, &file, L, blob.data());
    const Pic& P = *reinterpret_cast<const Pic*>(blob.data() + L.pics);
    const Chunk* chunks = reinterpret_cast<const Chunk*>(blob.data() + L.chunks);
    const uint8_t* data = blob.data() + L.data;
    wh[0] = P.ow; wh[1] = P.oh;
    bool bad = false;
    for (uint32_t k = 0; k < L.nchunks; ++k) {            // k_png_crc
        uint32_t x = 0;
        for (int lane = 0; lane < kLanes; ++lane) x ^= crc_piece(data + chunks[k].begin, chunks[k].len, lane, kLanes);
        if (chunk_crc(x, chunks[k].len) != chunks[k].crc) bad = true;
    }
    std::vector<uint8_t> raw(L.raw);
    if (!inflate_file(P, chunks, data, raw.data())) bad = true;
    for (int y = 0; y < P.h && !bad; ++y) {               // k_png_unfilter (Sub as its serial chain: the warp scans give the same)
        uint8_t* row = raw.data() + (uint64_t)y * (1 + P.stride);
        uint8_t* cur = row + 1;
        const uint8_t* prev = y ? cur - (1 + P.stride) : nullptr;
        const int f = row[0];
        if (f > 4) { bad = true; break; }
        if (f == 2 && prev)
            for (uint32_t x = 0; x < P.stride; ++x) cur[x] = (uint8_t)(cur[x] + prev[x]);
        else if (f == 1 || f == 3 || f == 4)
            for (int c = 0; c < P.bpp; ++c) unfilter_chain(cur, prev, P.stride, P.bpp, c, f);
    }
    if (bad) return -2;
    const uint8_t* pal = blob.data() + L.pal;
    for (int y = 0; y < P.oh; ++y)                        // k_png_rgb
        for (int x = 0; x < P.ow; ++x) pixel_rgb(raw.data(), pal, P, x, y, rgb + P.out + 3 * ((size_t)y * P.ow + x));
    return 0;
}

}  // extern "C"
