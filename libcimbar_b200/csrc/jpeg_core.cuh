// jpeg_core.cuh -- the JPEG decode of the camera path, written once for the host (tests/cpp/jpeg_core_host.cpp) and the device
// (jpeg.cu): the header parse and the upload layout (host only), and the per-segment entropy decoder, libjpeg-turbo's JDCT_ISLOW
// integer IDCT, its fancy upsampling, its fixed-point YCbCr -> RGB and cv2.imread's EXIF orientation (host and device).
//
// The goal is the RGB8 picture cv2.cvtColor(cv2.imread(file), COLOR_BGR2RGB) returns, byte for byte (OpenCV's JPEG decoder is
// libjpeg-turbo with its defaults: JDCT_ISLOW, fancy upsampling, no block smoothing on complete files).  What is restated:
//   jdhuff.c  jpeg_make_d_derived_tbl (canonical codes, 9-bit look-ahead), decode_mcu (sequential), HUFF_EXTEND
//   jdphuff.c decode_mcu_DC_first / _AC_first / _DC_refine / _AC_refine (EOBRUN, correction bits), start_pass_phuff_decoder's checks
//   jidctint.c jpeg_idct_islow (CONST_BITS 13, PASS1_BITS 2) with the post-IDCT range limit
//   jdsample.c h2v1_fancy_upsample, h1v2_fancy_upsample, h2v2_fancy_upsample (edge samples replicated, as jdmainct.c's context rows);
//              h2v1_upsample / h2v2_upsample (plain replication) where jinit_upsampler picks them: a component downsampled
//              horizontally whose downsampled_width is 2 or less (pictures up to 4 pixels wide in 4:2:2 and 4:2:0)
//   jdcolor.c  build_ycc_rgb_table + ycc_rgb_convert (SCALEBITS 16), gray_rgb_convert
//   OpenCV     JpegDecoder's first APP1 -> ExifReader orientation -> ApplyExifOrientation (flip / transpose)
// Supported: SOF0/1/2, 8-bit, one component or three YCbCr components, luma 1x1 / 2x1 / 1x2 / 2x2 with chroma 1x1, any restart
// interval.  Everything else is refused by parse() with a reason.  Corrupt entropy-coded data (a code that is not in the table, a
// run past the band, a segment that ends early or carries whole unused bytes) is detected, not repaired: the segment's decode
// reports it and the picture is reported, never decoded approximately.  After the first scan, whatever parse() would refuse (a
// marker that cannot follow a scan, a malformed marker segment, bytes that are not a marker, a scan script cut short) is such
// data too: a lost FF 00 stuffing byte or a flipped bit makes a false marker of any kind.
#pragma once
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#include <string>
#include <vector>

#if defined(__CUDACC__)
#define JD_HD __host__ __device__ __forceinline__
#else
#define JD_HD inline
#endif

namespace cb200 {
namespace jpeg {

constexpr int kLook = 9;                 // look-ahead bits of the Huffman decoder (jdhuff.h HUFF_LOOKAHEAD = 8; any width decodes the same)
constexpr int kMaxBlocks = 10;           // blocks per MCU (D_MAX_BLOCKS_IN_MCU)

// natural (row-major) position of the k-th coefficient in zig-zag order (jutils.c jpeg_natural_order)
#define JD_ZIGZAG {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48, \
                   41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, \
                   30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63}
#if defined(__CUDACC__)
static __device__ const uint8_t kZigzagDev[64] = JD_ZIGZAG;
#endif
static const uint8_t kZigzag[64] = JD_ZIGZAG;

JD_HD int zigzag(int k)
{
#if defined(__CUDA_ARCH__)
    return kZigzagDev[k];
#else
    return kZigzag[k];
#endif
}

struct Huff {                            // one derived table (jpeg_make_d_derived_tbl)
    uint16_t look[1 << kLook];           // (length << 8) | value of the code in the top kLook bits; 0 = a longer code
    int32_t maxcode[18];                 // largest code of each length, -1 = none
    int32_t valoff[18];                  // value index = code + valoff[length]
    uint8_t val[256];
};

struct Comp {
    int h, v;                            // sampling factors
    int bw, bh;                          // blocks of its coefficient and sample planes (whole MCUs)
    int wib, hib;                        // blocks that cover the component: the extent of a non-interleaved scan
    int dw, dh;                          // downsampled_width / downsampled_height
    uint32_t quant;                      // its quantisation table (64 entries, natural order), latched at its first scan
    uint32_t pad;
    uint64_t coef;                       // first coefficient (int16) of its plane in the coefficient buffer
    uint64_t plane;                      // first byte of its sample plane (bw * 8 x bh * 8) in the plane buffer
};

struct Pic {
    int w, h;                            // decoded size
    int ow, oh;                          // output size (after the EXIF orientation)
    int orient;                          // 1..8
    int ncomp, hmax, vmax;
    int bad;                             // the file ends inside its entropy-coded data or before its last scan
    int pad;
    uint64_t out;                        // first byte of its RGB8 picture in the output
    Comp comp[3];
};

enum Kind { kSequential = 0, kDcFirst = 1, kDcRefine = 2, kAcFirst = 3, kAcRefine = 4 };

struct Scan {
    int pic;
    int kind;
    int ncomp;                           // components in the scan (1 = non-interleaved: one block per MCU)
    int blocks;                          // blocks per MCU
    int mcux;                            // MCUs per row
    int ss, se, al;
    uint8_t bcomp[kMaxBlocks];           // per block of an MCU: its component, its position in the MCU, its scan slot
    uint8_t bdx[kMaxBlocks], bdy[kMaxBlocks], bslot[kMaxBlocks];
    uint32_t dc[4], ac[4];               // Huffman tables of each scan slot (indices into the batch's table list)
};

struct Seg {                             // one restart interval (or the whole scan): its MCUs and its entropy-coded bytes
    uint32_t scan;
    uint32_t mcu0, mcus;
    uint32_t pad;
    uint64_t begin, end;                 // byte range in the data section; FF 00 stuffing still in, no marker inside.  The unstuffed
                                         // bytes go to the same offset of the unstuffed buffer
};

// ---- the entropy decoder ----------------------------------------------------------------------------------------------------

struct Bits {                            // a reader over a segment's unstuffed bytes
    const uint8_t* p;
    const uint8_t* end;
    uint64_t acc;                        // next bits, MSB first
    int n;                               // valid bits in acc
    int over;                            // zero bits appended past the end of the data (libjpeg's fill at a marker)
};

JD_HD void fill(Bits& b)
{
    while (b.n <= 56) {
        uint32_t v = 0;
        if (b.p < b.end) {
            v = *b.p++;
        } else {
            b.over += 8;
        }
        b.acc |= (uint64_t)v << (56 - b.n);
        b.n += 8;
    }
}

JD_HD int bits(Bits& b, int s)           // the next s (0..16) bits as an unsigned number
{
    if (s == 0) return 0;
    if (b.n < s) fill(b);
    const int v = (int)(b.acc >> (64 - s));
    b.acc <<= s;
    b.n -= s;
    return v;
}

JD_HD int huff(Bits& b, const Huff& t)   // the next symbol, -1 for a code that is not in the table
{
    if (b.n < 16) fill(b);
    const uint16_t e = t.look[b.acc >> (64 - kLook)];
    if (e) {
        b.acc <<= (e >> 8);
        b.n -= (e >> 8);
        return e & 0xFF;
    }
    const uint32_t c16 = (uint32_t)(b.acc >> 48);
    for (int l = kLook + 1; l <= 16; ++l) {
        const int32_t code = (int32_t)(c16 >> (16 - l));
        if (code <= t.maxcode[l]) {
            b.acc <<= l;
            b.n -= l;
            return t.val[(code + t.valoff[l]) & 0xFF];
        }
    }
    return -1;
}

JD_HD int ctz64(uint64_t v)              // index of the lowest set bit (v != 0)
{
#if defined(__CUDA_ARCH__)
    return __ffsll((long long)v) - 1;
#else
    return __builtin_ctzll(v);
#endif
}

JD_HD int extend(int r, int s) { return r < (1 << (s - 1)) ? r + (int)(~0u << s) + 1 : r; }   // HUFF_EXTEND

// the reader at bit `pos` of unstuffed data u (ulen bytes), and its position
JD_HD void bits_at(Bits& b, const uint8_t* u, uint32_t ulen, uint32_t pos)
{
    b.p = u + (pos >> 3 < ulen ? pos >> 3 : ulen); b.end = u + ulen; b.acc = 0; b.n = 0;
    b.over = pos >> 3 < ulen ? 0 : (int)(8 * ((pos >> 3) - ulen));
    fill(b);
    b.acc <<= (pos & 7);
    b.n -= (int)(pos & 7);
}

JD_HD uint32_t bitpos(const Bits& b, const uint8_t* u) { return (uint32_t)((b.p - u) * 8 + b.over - b.n); }

// the first coefficient (element offset in the coefficient buffer) of block g (in scan order) of a segment
JD_HD uint64_t block_offset(const Pic& P, const Scan& sc, const Seg& sg, uint32_t g)
{
    const uint32_t m = sg.mcu0 + (sc.ncomp == 1 ? g : g / (uint32_t)sc.blocks);
    const int k = sc.ncomp == 1 ? 0 : (int)(g % (uint32_t)sc.blocks);
    const int my = (int)(m / (uint32_t)sc.mcux), mx = (int)m - my * sc.mcux;
    const Comp& C = P.comp[sc.bcomp[k]];
    const int bx = sc.ncomp == 1 ? mx : mx * C.h + sc.bdx[k], by = sc.ncomp == 1 ? my : my * C.v + sc.bdy[k];
    return C.coef + ((uint64_t)by * (uint64_t)C.bw + (uint64_t)bx) * 64;
}

JD_HD int16_t* block_at(const Pic& P, const Scan& sc, const Seg& sg, uint32_t g, int16_t* coef) { return coef + block_offset(P, sc, sg, g); }

// ---- the parallel decode of sequential, DC and AC-first scans (self-synchronisation) --------------------------------------
//
// Weißenberger & Schmidt's scheme (ICPP 2018, HiPC 2021): a segment's bits are cut into T subsequences, one per thread.  Each thread
// decodes its subsequence speculatively from a guessed state at its start; the sync rounds then hand each thread its predecessor's
// end state until no end state changes (Huffman codes resynchronise after a few symbols, so that is typically two or three rounds,
// and at worst T).  Prefix sums of the blocks and DC differences each thread decoded give every thread its first block and its DC
// predictions, and a write pass decodes again from the exact start states into the coefficient buffer.  The state at a block
// boundary is the bit position and, in an interleaved sequential or DC-first scan, the block's place in the MCU (it selects the
// tables); an EOB run of an AC-first scan is taken whole, so no run is ever open at a boundary.

struct Unit {                            // decoder state at a block boundary
    uint32_t pos;                        // bit position in the segment's unstuffed data; kNoState after a decode error
    int32_t j;                           // block within the MCU (interleaved sequential / DC-first scans), else 0
};
constexpr uint32_t kNoState = 0xFFFFFFFFu;

JD_HD bool same(const Unit& a, const Unit& b) { return a.pos == b.pos && a.j == b.j; }

struct Region {                          // what decoding one subsequence gives
    Unit end;                            // state at the first block boundary at or past the subsequence's end
    uint32_t blocks;                     // blocks decoded (an EOB run counts all its blocks)
    int dc[4];                           // count pass: sum of the DC differences per scan slot
    int err;                             // a decode error (or a read past the data)
    uint32_t tail;                       // write pass: bit position after the unit that completes the segment's last block
};

JD_HD uint32_t segment_blocks(const Scan& sc, const Seg& sg) { return sg.mcus * (uint32_t)(sc.ncomp == 1 ? 1 : sc.blocks); }

// decode blocks from state st while the position is below `stop`.  Count pass: coef == nullptr.  Write pass: the blocks are numbered
// from g0, their DC predictions start at pred0, and blocks g0 .. total - 1 are written
JD_HD void run_region(const uint8_t* u, uint32_t ulen, const Pic& P, const Scan& sc, const Seg& sg, const Huff* const* dct,
                      const Huff* const* act, Unit st, uint32_t stop, uint32_t g0, const int* pred0, int16_t* coef, Region& R)
{
    R.end = st; R.blocks = 0; R.err = 0; R.tail = kNoState;
    for (int s = 0; s < 4; ++s) R.dc[s] = 0;
    if (st.pos == kNoState) return;
    const uint32_t L = ulen * 8, total = segment_blocks(sc, sg);
    const bool track_j = sc.ncomp > 1 && (sc.kind == kSequential || sc.kind == kDcFirst);
    int pred[4];
    for (int s = 0; s < 4; ++s) pred[s] = coef ? pred0[s] : 0;
    Bits b;
    bits_at(b, u, ulen, st.pos);
    uint32_t pos = st.pos;
    int j = st.j;
    const int p1 = 1 << sc.al;
    bool err = false;
    while (pos < stop && !err) {
        const uint32_t g = g0 + R.blocks;
        if (coef && g >= total) break;
        int16_t* blk = coef ? block_at(P, sc, sg, g, coef) : nullptr;
        const int slot = track_j ? sc.bslot[j] : 0;
        uint32_t adv = 1;
        if (b.n < 32) fill(b);
        if (sc.kind == kDcRefine) {
            if (bits(b, 1) && blk) blk[0] = (int16_t)(blk[0] | p1);
        } else if (sc.kind == kSequential || sc.kind == kDcFirst) {
            const int s = huff(b, *dct[slot]);
            if (s < 0 || s > 15) { err = true; break; }
            pred[slot] += s ? extend(bits(b, s), s) : 0;
            if (sc.kind == kDcFirst) {
                if (blk) blk[0] = (int16_t)(int)((unsigned)pred[slot] << sc.al);
            } else {
                if (blk) blk[0] = (int16_t)pred[slot];
                const Huff& ac = *act[slot];
                for (int kk = 1; kk < 64; ++kk) {
                    if (b.n < 32) fill(b);
                    const int rs = huff(b, ac);
                    if (rs < 0) { err = true; break; }
                    const int r = rs >> 4, s2 = rs & 15;
                    if (s2) {
                        kk += r;
                        if (kk > 63) { err = true; break; }
                        const int v = extend(bits(b, s2), s2);
                        if (blk) blk[zigzag(kk)] = (int16_t)v;
                    } else {
                        if (r != 15) break;
                        kk += 15;
                    }
                }
            }
        } else {                         // AC first
            const Huff& ac = *act[0];
            for (int kk = sc.ss; kk <= sc.se; ++kk) {
                if (b.n < 32) fill(b);
                const int rs = huff(b, ac);
                if (rs < 0) { err = true; break; }
                const int r = rs >> 4, s = rs & 15;
                if (s) {
                    kk += r;
                    if (kk > sc.se) { err = true; break; }
                    const int v = extend(bits(b, s), s);
                    if (blk) blk[zigzag(kk)] = (int16_t)(int)((unsigned)v << sc.al);
                } else if (r == 15) {
                    kk += 15;
                } else {
                    adv = (1u << r) + (uint32_t)bits(b, r);   // this block and the next adv - 1 end here
                    break;
                }
            }
        }
        if (err) break;
        pos = bitpos(b, u);
        if (pos > L) { err = true; break; }
        if (track_j) j = j + 1 == sc.blocks ? 0 : j + 1;
        if (coef && g + adv >= total) R.tail = pos;
        R.blocks += adv;
    }
    R.err = err;
    R.end.pos = err ? kNoState : pos;
    R.end.j = j;
    for (int s = 0; s < 4; ++s) R.dc[s] = pred[s];
}

// where subsequence t of T begins (the last one runs to the end of the data)
JD_HD uint32_t sub_size(uint32_t ulen, int T) { const uint32_t s = (8 * ulen + (uint32_t)T - 1) / (uint32_t)T; return s < 32 ? 32 : s; }
JD_HD uint32_t sub_begin(uint32_t S, int t, uint32_t ulen) { const uint64_t v = (uint64_t)S * (uint32_t)t; return v < 8ull * ulen ? (uint32_t)v : 8 * ulen; }
JD_HD uint32_t sub_end(uint32_t S, int t, int T, uint32_t ulen) { return t == T - 1 ? kNoState - 1 : sub_begin(S, t + 1, ulen); }

// the write pass's verdict on a thread's region: false if the segment is corrupt there
JD_HD bool region_ok(const Unit& start, const Region& R, uint32_t g0, uint32_t total, uint32_t ulen)
{
    if (g0 < total && (start.pos == kNoState || R.err)) return false;      // blocks of the segment that do not decode
    if (R.tail != kNoState && 8 * ulen - R.tail >= 8) return false;         // a whole unused byte after the last block
    return true;
}

// the parallel decode of one segment with T threads, run one thread after the other (the host's restatement of k_jpeg_decode's
// CTA; the same rounds, prefix sums and write pass)
inline bool decode_segment_sync(int T, const uint8_t* u, uint32_t ulen, const Pic& P, const Scan& sc, const Seg& sg, const Huff* huffs,
                                int16_t* coef)
{
    const Huff* dct[4];
    const Huff* act[4];
    for (int s = 0; s < 4; ++s) { dct[s] = huffs + sc.dc[s]; act[s] = huffs + sc.ac[s]; }
    const uint32_t S = sub_size(ulen, T), total = segment_blocks(sc, sg);
    std::vector<Unit> start((size_t)T);
    std::vector<Region> R((size_t)T);
    for (int t = 0; t < T; ++t) {
        start[(size_t)t] = Unit{sub_begin(S, t, ulen), 0};
        run_region(u, ulen, P, sc, sg, dct, act, start[(size_t)t], sub_end(S, t, T, ulen), 0, nullptr, nullptr, R[(size_t)t]);
    }
    for (bool changed = true; changed;) {
        changed = false;
        std::vector<Unit> in((size_t)T);
        for (int t = 1; t < T; ++t) in[(size_t)t] = R[(size_t)t - 1].end;
        for (int t = 1; t < T; ++t) {
            if (same(in[(size_t)t], start[(size_t)t])) continue;
            start[(size_t)t] = in[(size_t)t];
            const Unit old = R[(size_t)t].end;
            run_region(u, ulen, P, sc, sg, dct, act, start[(size_t)t], sub_end(S, t, T, ulen), 0, nullptr, nullptr, R[(size_t)t]);
            changed = changed || !same(old, R[(size_t)t].end);
        }
    }
    uint32_t g0 = 0;
    int pred[4] = {0, 0, 0, 0};
    bool ok = true, tail = false;
    for (int t = 0; t < T; ++t) {
        Region W;
        run_region(u, ulen, P, sc, sg, dct, act, start[(size_t)t], sub_end(S, t, T, ulen), g0, pred, coef, W);
        ok = ok && region_ok(start[(size_t)t], W, g0, total, ulen);
        tail = tail || W.tail != kNoState;
        g0 += R[(size_t)t].blocks;
        for (int s = 0; s < 4; ++s) pred[s] += R[(size_t)t].dc[s];
    }
    return ok && tail;
}

// FF 00 stuffing out of a segment's bytes: byte i is kept unless the byte before it is FF (no marker lies inside a segment)
JD_HD bool kept(const uint8_t* raw, uint64_t i, uint64_t begin) { return i == begin || raw[i - 1] != 0xFF; }

// ---- AC refinement scans ----------------------------------------------------------------------------------------------
//
// A refinement scan's bit lengths depend on which coefficients of each block are already nonzero, so its segment is decoded in
// order by one thread -- but that thread does bit work only.  Before it, refine_prep records every block's nonzero coefficients as
// a 64-bit mask in zig-zag order (one thread per block); the decode reads one mask per block and records three per block: the
// coefficients whose correction bit is 1, the newly nonzero ones, and their signs; after it, refine_apply updates the
// coefficients (one thread per block).  Each coefficient is corrected at most once per scan, and a new one sits where the block
// had a zero, so applying the masks afterwards gives what decode_mcu_AC_refine gives in place.
// masks: 4 words per block of the coefficient buffer (index = block offset / 64): nonzero, corrected, new, new and negative.

JD_HD void refine_prep(const int16_t* blk, int ss, int se, uint64_t* m)
{
    uint64_t nz = 0;
    for (int k = ss; k <= se; ++k) nz |= (uint64_t)(blk[zigzag(k)] != 0) << k;
    m[0] = nz; m[1] = 0; m[2] = 0; m[3] = 0;
}

JD_HD void refine_apply(int16_t* blk, int al, const uint64_t* m)
{
    const int p1 = 1 << al;
    for (uint64_t c = m[1]; c; c &= c - 1) {
        int16_t& v = blk[zigzag(ctz64(c))];
        if ((v & p1) == 0) v = (int16_t)(v + (v >= 0 ? p1 : -p1));
    }
    for (uint64_t c = m[2]; c; c &= c - 1) {
        const int k = ctz64(c);
        blk[zigzag(k)] = (int16_t)(((m[3] >> k) & 1) ? -p1 : p1);
    }
}

// decode_mcu_AC_refine over one segment (unstuffed bytes u) with the blocks' nonzero masks; false if the data are corrupt
JD_HD bool decode_refine(const uint8_t* u, uint32_t ulen, const Pic& P, const Scan& sc, const Seg& sg, const Huff& ac, uint64_t* masks)
{
    Bits b;
    b.p = u; b.end = u + ulen; b.acc = 0; b.n = 0; b.over = 0;
    unsigned eobrun = 0;
    const uint32_t total = segment_blocks(sc, sg);
    for (uint32_t g = 0; g < total; ++g) {
        uint64_t* m = masks + 4 * (block_offset(P, sc, sg, g) / 64);
        const uint64_t nz = m[0];
        uint64_t cor = 0, nw = 0, neg = 0;
        int kk = sc.ss;
        if (eobrun == 0) {
            for (; kk <= sc.se; ++kk) {
                if (b.n < 32) fill(b);
                const int rs = huff(b, ac);
                if (rs < 0) return false;
                int r = rs >> 4;
                const int s = rs & 15;
                int negative = 0;
                if (s) {
                    if (s != 1) return false;
                    negative = bits(b, 1) ? 0 : 1;
                } else if (r != 15) {
                    eobrun = 1u << r;
                    if (r) eobrun += (unsigned)bits(b, r);
                    break;
                }
                do {
                    if ((nz >> kk) & 1) {
                        if (b.n < 32) fill(b);
                        if (bits(b, 1)) cor |= 1ull << kk;
                    } else if (--r < 0) {
                        break;
                    }
                    ++kk;
                } while (kk <= sc.se);
                if (s) {
                    if (kk > sc.se) return false;
                    nw |= 1ull << kk;
                    neg |= (uint64_t)negative << kk;
                }
            }
        }
        if (eobrun > 0) {
            const uint64_t band = kk > 63 ? 0 : (~0ull << kk) & (sc.se == 63 ? ~0ull : ((1ull << (sc.se + 1)) - 1));
            for (uint64_t c = nz & band; c; c &= c - 1) {
                if (b.n < 32) fill(b);
                if (bits(b, 1)) cor |= c & (~c + 1);
            }
            --eobrun;
        }
        m[1] = cor; m[2] = nw; m[3] = neg;
    }
    return b.n >= b.over && b.p >= b.end && b.n - b.over < 8;
}

// ---- IDCT, upsampling, colour ---------------------------------------------------------------------------------------------

JD_HD uint8_t idct_limit(int64_t v)      // the post-IDCT range limit (v centred on 0)
{
    v += 128;
    return (uint8_t)(v < 0 ? 0 : v > 255 ? 255 : v);
}

JD_HD int wrap32(int64_t v) { return (int)(uint32_t)(uint64_t)v; }   // (int) of a JLONG, as jidctint.c stores its workspace

JD_HD void note_wide(int* wide, int64_t v, int64_t lo, int64_t hi) { if (wide && (v < lo || v > hi)) *wide = 1; }

// jpeg_idct_islow: the 64 coefficients of one block (natural order) with their quantisation table -> 8 x 8 samples at out (stride).
// The arithmetic is jidctint.c's: 64-bit intermediates (JLONG on LP64), an int workspace, so no input overflows.  Where libjpeg-
// turbo's own IDCTs disagree -- a dequantised coefficient or a workspace value beyond 16 bits (its SIMD IDCT's pmullw / packssdw),
// an output beyond [-512, 511] before the range limit (its C IDCT's `& RANGE_MASK` wraps) -- this one clamps, and *wide (when
// given) is set to 1.  No encoder writes such blocks; damaged or hand-made coefficients can
JD_HD void idct_islow(const int16_t* in, const uint16_t* q, uint8_t* out, size_t stride, int* wide = nullptr)
{
    constexpr int CB = 13, P1 = 2;
    constexpr int64_t F0298 = 2446, F0390 = 3196, F0541 = 4433, F0765 = 6270, F0899 = 7373, F1175 = 9633, F1501 = 12299,
                      F1847 = 15137, F1961 = 16069, F2053 = 16819, F2562 = 20995, F3072 = 25172;
    int ws[64];
    for (int c = 0; c < 8; ++c) {
        const int16_t* ip = in + c;
        const uint16_t* qp = q + c;
        int* wp = ws + c;
        int64_t dq[8];                                        // DEQUANTIZE: 16 x 16-bit products (MULTIPLIER short)
        for (int r = 0; r < 8; ++r) {
            dq[r] = (int64_t)((int)ip[8 * r] * (int)(int16_t)qp[8 * r]);
            note_wide(wide, dq[r], -32768, 32767);
        }
        if (!ip[8] && !ip[16] && !ip[24] && !ip[32] && !ip[40] && !ip[48] && !ip[56]) {
            const int64_t dc = dq[0] * (1 << P1);
            note_wide(wide, dc, -32768, 32767);
            for (int r = 0; r < 8; ++r) wp[8 * r] = wrap32(dc);
            continue;
        }
        int64_t z2 = dq[2], z3 = dq[6];
        int64_t z1 = (z2 + z3) * F0541;
        int64_t tmp2 = z1 + z3 * -F1847, tmp3 = z1 + z2 * F0765;
        z2 = dq[0];
        z3 = dq[4];
        int64_t tmp0 = (z2 + z3) * (1 << CB), tmp1 = (z2 - z3) * (1 << CB);
        const int64_t tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
        tmp0 = dq[7]; tmp1 = dq[5]; tmp2 = dq[3]; tmp3 = dq[1];
        z1 = tmp0 + tmp3; z2 = tmp1 + tmp2; z3 = tmp0 + tmp2;
        int64_t z4 = tmp1 + tmp3;
        const int64_t z5 = (z3 + z4) * F1175;
        tmp0 *= F0298; tmp1 *= F2053; tmp2 *= F3072; tmp3 *= F1501;
        z1 *= -F0899; z2 *= -F2562; z3 *= -F1961; z4 *= -F0390;
        z3 += z5; z4 += z5;
        tmp0 += z1 + z3; tmp1 += z2 + z4; tmp2 += z2 + z3; tmp3 += z1 + z4;
        constexpr int S = CB - P1;
        constexpr int64_t R = (int64_t)1 << (S - 1);
        const int64_t v[8] = {tmp10 + tmp3, tmp11 + tmp2, tmp12 + tmp1, tmp13 + tmp0, tmp13 - tmp0, tmp12 - tmp1, tmp11 - tmp2, tmp10 - tmp3};
        for (int r = 0; r < 8; ++r) {
            const int64_t d = (v[r] + R) >> S;
            note_wide(wide, d, -32768, 32767);
            wp[8 * r] = wrap32(d);
        }
    }
    for (int r = 0; r < 8; ++r) {
        const int* wp = ws + 8 * r;
        uint8_t* op = out + (size_t)r * stride;
        if (!wp[1] && !wp[2] && !wp[3] && !wp[4] && !wp[5] && !wp[6] && !wp[7]) {
            const int64_t d = ((int64_t)wp[0] + (1 << (P1 + 2))) >> (P1 + 3);
            note_wide(wide, d, -512, 511);
            const uint8_t v = idct_limit(d);
            for (int c = 0; c < 8; ++c) op[c] = v;
            continue;
        }
        int64_t z2 = wp[2], z3 = wp[6];
        int64_t z1 = (z2 + z3) * F0541;
        int64_t tmp2 = z1 + z3 * -F1847, tmp3 = z1 + z2 * F0765;
        int64_t tmp0 = ((int64_t)wp[0] + wp[4]) * (1 << CB), tmp1 = ((int64_t)wp[0] - wp[4]) * (1 << CB);
        const int64_t tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
        tmp0 = wp[7]; tmp1 = wp[5]; tmp2 = wp[3]; tmp3 = wp[1];
        z1 = tmp0 + tmp3; z2 = tmp1 + tmp2; z3 = tmp0 + tmp2;
        int64_t z4 = tmp1 + tmp3;
        const int64_t z5 = (z3 + z4) * F1175;
        tmp0 *= F0298; tmp1 *= F2053; tmp2 *= F3072; tmp3 *= F1501;
        z1 *= -F0899; z2 *= -F2562; z3 *= -F1961; z4 *= -F0390;
        z3 += z5; z4 += z5;
        tmp0 += z1 + z3; tmp1 += z2 + z4; tmp2 += z2 + z3; tmp3 += z1 + z4;
        constexpr int S = CB + P1 + 3;
        constexpr int64_t R = (int64_t)1 << (S - 1);
        const int64_t v[8] = {tmp10 + tmp3, tmp11 + tmp2, tmp12 + tmp1, tmp13 + tmp0, tmp13 - tmp0, tmp12 - tmp1, tmp11 - tmp2, tmp10 - tmp3};
        for (int c = 0; c < 8; ++c) {
            const int64_t d = (v[c] + R) >> S;
            note_wide(wide, d, -512, 511);
            op[c] = idct_limit(d);
        }
    }
}

// one full-resolution sample (x, y) of component C, upsampled as jdsample.c's jinit_upsampler chooses: a component downsampled
// horizontally (h2v1, h2v2) is filtered only when its downsampled_width is above 2, else replicated (h2v1_upsample /
// h2v2_upsample, which do not filter vertically either); h1v2 is always filtered
JD_HD int sample(const uint8_t* planes, const Pic& P, const Comp& C, int x, int y)
{
    const uint8_t* p = planes + C.plane;
    const size_t st = (size_t)C.bw * 8;
    const int hr = P.hmax / C.h, vr = P.vmax / C.v;
    const int cx = x / hr, cy = y / vr;
    if ((hr == 1 && vr == 1) || (hr == 2 && C.dw <= 2)) return p[(size_t)cy * st + cx];
    if (vr == 1) {                       // h2v1
        const int n = (x & 1) ? (cx + 1 < C.dw ? cx + 1 : cx) : (cx > 0 ? cx - 1 : 0);
        return (3 * p[(size_t)cy * st + cx] + p[(size_t)cy * st + n] + ((x & 1) ? 2 : 1)) >> 2;
    }
    const int ny = (y & 1) ? (cy + 1 < C.dh ? cy + 1 : cy) : (cy > 0 ? cy - 1 : 0);
    const uint8_t* r0 = p + (size_t)cy * st;
    const uint8_t* r1 = p + (size_t)ny * st;
    if (hr == 1) return (3 * r0[cx] + r1[cx] + ((y & 1) ? 2 : 1)) >> 2;   // h1v2
    const int nx = (x & 1) ? (cx + 1 < C.dw ? cx + 1 : cx) : (cx > 0 ? cx - 1 : 0);   // h2v2
    const int t = 3 * r0[cx] + r1[cx], u = 3 * r0[nx] + r1[nx];
    return (3 * t + u + ((x & 1) ? 7 : 8)) >> 4;
}

JD_HD uint8_t clamp255(int v) { return (uint8_t)(v < 0 ? 0 : v > 255 ? 255 : v); }

// the decoded pixel (x, y) of a w x h picture shown at output pixel (ox, oy) under EXIF orientation `orient` (OpenCV's
// ApplyExifOrientation: flips and transposes)
JD_HD void orient_source(int orient, int w, int h, int ox, int oy, int& x, int& y)
{
    switch (orient) {
    case 2: x = w - 1 - ox; y = oy; break;
    case 3: x = w - 1 - ox; y = h - 1 - oy; break;
    case 4: x = ox; y = h - 1 - oy; break;
    case 5: x = oy; y = ox; break;
    case 6: x = oy; y = h - 1 - ox; break;
    case 7: x = w - 1 - oy; y = h - 1 - ox; break;
    case 8: x = w - 1 - oy; y = ox; break;
    default: x = ox; y = oy; break;
    }
}

// output pixel (ox, oy) of picture P: EXIF orientation -> decoded pixel -> RGB (ycc_rgb_convert; gray replicated)
JD_HD void pixel_rgb(const uint8_t* planes, const Pic& P, int ox, int oy, uint8_t* rgb)
{
    int x, y;
    orient_source(P.orient, P.w, P.h, ox, oy, x, y);
    const int Y = sample(planes, P, P.comp[0], x, y);
    if (P.ncomp == 1) { rgb[0] = rgb[1] = rgb[2] = (uint8_t)Y; return; }
    const int cb = sample(planes, P, P.comp[1], x, y) - 128, cr = sample(planes, P, P.comp[2], x, y) - 128;
    // FIX(1.40200) = 91881, FIX(1.77200) = 116130, FIX(0.71414) = 46802, FIX(0.34414) = 22554 (SCALEBITS 16)
    rgb[0] = clamp255(Y + ((91881 * cr + 32768) >> 16));
    rgb[1] = clamp255(Y + ((-22554 * cb + 32768 - 46802 * cr) >> 16));
    rgb[2] = clamp255(Y + ((116130 * cb + 32768) >> 16));
}

// ---- host: the header parse and the upload layout -----------------------------------------------------------------------

struct Parsed {                          // one file as parse() leaves it (offsets relative to the file)
    Pic pic;
    std::vector<uint16_t> quant;         // 64 per component
    std::vector<Huff> huffs;
    std::vector<Scan> scans;             // pic = 0, tables index huffs
    std::vector<Seg> segs;               // scan indexes scans
};

inline unsigned be16(const uint8_t* p) { return (unsigned)p[0] << 8 | p[1]; }

// jpeg_make_d_derived_tbl; "" or why the table is refused
inline std::string derive(const uint8_t* counts, const uint8_t* vals, int nval, bool dc, Huff& t)
{
    memset(&t, 0, sizeof(t));
    memcpy(t.val, vals, (size_t)nval);
    int code = 0, p = 0;
    for (int l = 1; l <= 16; ++l) {
        const int c = counts[l - 1];
        if (c) {
            t.valoff[l] = p - code;
            for (int i = 0; i < c; ++i, ++p, ++code) {
                if (l <= kLook) {
                    const int lo = code << (kLook - l), hi = (code + 1) << (kLook - l);
                    for (int e = lo; e < hi; ++e) t.look[e] = (uint16_t)(l << 8 | vals[p]);
                }
            }
            t.maxcode[l] = code - 1;
        } else {
            t.maxcode[l] = -1;
        }
        if (code >= (1 << l)) return "a Huffman table with more codes than its code lengths allow";
        code <<= 1;
    }
    t.maxcode[17] = 0x7FFFFFFF;
    if (dc)
        for (int i = 0; i < nval; ++i)
            if (vals[i] > 15) return "a DC Huffman table with a symbol above 15";
    return "";
}

// EXIF orientation of the first APP1 segment as OpenCV's ExifReader reads it (TIFF header 6 bytes in), 1 if none
inline int exif_orientation(const uint8_t* d, size_t len)
{
    if (len <= 6) return 1;
    d += 6; len -= 6;
    if (len < 8) return 1;
    const bool le = d[0] == 'I' && d[1] == 'I';
    if (!le && !(d[0] == 'M' && d[1] == 'M')) return 1;
    auto u16 = [&](size_t o) { return le ? (unsigned)d[o] | (unsigned)d[o + 1] << 8 : (unsigned)d[o] << 8 | d[o + 1]; };
    auto u32 = [&](size_t o) { return le ? u16(o) | (size_t)u16(o + 2) << 16 : (size_t)u16(o) << 16 | u16(o + 2); };
    const size_t ifd = u32(4);
    if (ifd + 2 > len) return 1;
    const unsigned cnt = u16(ifd);
    for (unsigned e = 0; e < cnt; ++e) {
        const size_t o = ifd + 2 + 12 * (size_t)e;
        if (o + 12 > len) break;
        if (u16(o) == 0x0112) {
            const unsigned v = u16(o + 8);
            return v >= 1 && v <= 8 ? (int)v : 1;
        }
    }
    return 1;
}

// the markers of one file: "" and P filled, or the reason the file is refused.  Entropy-coded data are only split at their
// restart markers here; a file that ends inside them or before its last scan, or whose markers after its first scan would be
// refused, is accepted with P.pic.bad = 1
inline std::string parse(const uint8_t* f, size_t n, Parsed& P)
{
    P = Parsed();
    Pic& pic = P.pic;
    memset(&pic, 0, sizeof(pic));
    pic.orient = 1;
    if (n < 4 || f[0] != 0xFF || f[1] != 0xD8) return "not a JPEG file (no SOI marker)";
    if (n >= (1u << 28)) return "a file of 256 MB or more";            // bit positions of a segment fit 32 bits
    size_t pos = 2;
    bool frame = false, jfif = false, adobe = false, exif_seen = false, eoi = false;
    int adobe_transform = -1, restart = 0, cid[3] = {0, 0, 0}, cq[3] = {0, 0, 0};
    bool qdef[4] = {false, false, false, false}, latched[3] = {false, false, false};
    uint16_t qtab[4][64];
    int dc_tab[4] = {-1, -1, -1, -1}, ac_tab[4] = {-1, -1, -1, -1};
    int coef_bits[3][64];
    for (auto& cb : coef_bits) for (int& v : cb) v = -1;
    bool progressive = false, in_scan = false;
    // Once a scan has been read, whatever the marker walk would refuse is taken for corrupt data: a lost FF 00 stuffing byte or a
    // flipped bit turns entropy-coded bytes into a false marker of any kind (or into bytes that are not a marker), with any length
    // and contents.  So after the first scan a refusal marks the picture (status -2) instead of failing the whole call
    const auto markers = [&]() -> std::string {
        while (!eoi) {
            // the next marker: FF (fill FFs) code
            if (pos >= n || f[pos] != 0xFF) return "truncated or malformed JPEG header";
            while (pos < n && f[pos] == 0xFF) ++pos;
            if (pos >= n) return "truncated JPEG header";
            const unsigned m = f[pos++];
            if (m == 0xD9) { eoi = true; break; }
            const bool between_scans = m == 0xC4 || m == 0xDA || m == 0xDB || m == 0xDD || (m >= 0xE0 && m <= 0xEF) || m == 0xFE;
            if (!P.scans.empty() && !between_scans) return "a marker that cannot follow a scan";
            if (m == 0xD8 || (m >= 0xD0 && m <= 0xD7) || m == 0x01) return "unexpected marker in the JPEG header";
            if (pos + 2 > n) return "truncated JPEG header";
            const size_t len = be16(f + pos);
            if (len < 2 || pos + len > n) return "truncated JPEG header";
            const uint8_t* d = f + pos + 2;
            const size_t dl = len - 2;
            pos += len;
            if (m == 0xC0 || m == 0xC1 || m == 0xC2) {
                if (frame) return "more than one frame header";
                frame = true;
                progressive = m == 0xC2;
                if (dl < 6) return "truncated frame header";
                if (d[0] != 8) return std::to_string(d[0]) + "-bit samples (only 8-bit JPEG is supported)";
                pic.h = (int)be16(d + 1); pic.w = (int)be16(d + 3); pic.ncomp = d[5];
                if (pic.h == 0) return "a frame header with height 0 (DNL) is not supported";
                if (pic.w == 0) return "a frame header with width 0";
                if (pic.ncomp == 4) return "4 components (CMYK / YCCK) are not supported";
                if (pic.ncomp != 1 && pic.ncomp != 3) return std::to_string(pic.ncomp) + " components (only grey or YCbCr are supported)";
                if (dl < 6 + 3 * (size_t)pic.ncomp) return "truncated frame header";
                for (int c = 0; c < pic.ncomp; ++c) {
                    cid[c] = d[6 + 3 * c];
                    pic.comp[c].h = d[7 + 3 * c] >> 4; pic.comp[c].v = d[7 + 3 * c] & 15;
                    cq[c] = d[8 + 3 * c];
                    if (pic.comp[c].h < 1 || pic.comp[c].h > 4 || pic.comp[c].v < 1 || pic.comp[c].v > 4 || cq[c] > 3)
                        return "a frame header with bad sampling factors or table numbers";
                }
                if (pic.ncomp == 3) {
                    const Comp* c = pic.comp;
                    if (c[1].h != 1 || c[1].v != 1 || c[2].h != 1 || c[2].v != 1 || c[0].h > 2 || c[0].v > 2)
                        return "sampling " + std::to_string(c[0].h) + "x" + std::to_string(c[0].v) + ", " + std::to_string(c[1].h) + "x" +
                               std::to_string(c[1].v) + ", " + std::to_string(c[2].h) + "x" + std::to_string(c[2].v) +
                               " (only 4:4:4, 4:2:2, 4:4:0 and 4:2:0 are supported)";
                    pic.hmax = c[0].h; pic.vmax = c[0].v;
                } else {
                    pic.hmax = pic.comp[0].h; pic.vmax = pic.comp[0].v;
                }
                const int mcux = (pic.w + 8 * pic.hmax - 1) / (8 * pic.hmax), mcuy = (pic.h + 8 * pic.vmax - 1) / (8 * pic.vmax);
                for (int c = 0; c < pic.ncomp; ++c) {
                    Comp& C = pic.comp[c];
                    if (pic.ncomp == 1) { C.h = C.v = 1; pic.hmax = pic.vmax = 1; }   // one component: one block per MCU
                    const int mx = pic.ncomp == 1 ? (pic.w + 7) / 8 : mcux, my = pic.ncomp == 1 ? (pic.h + 7) / 8 : mcuy;
                    C.bw = mx * C.h; C.bh = my * C.v;
                    C.wib = (pic.w * C.h + 8 * pic.hmax - 1) / (8 * pic.hmax);
                    C.hib = (pic.h * C.v + 8 * pic.vmax - 1) / (8 * pic.vmax);
                    C.dw = (pic.w * C.h + pic.hmax - 1) / pic.hmax;
                    C.dh = (pic.h * C.v + pic.vmax - 1) / pic.vmax;
                }
            } else if (m == 0xC3 || (m >= 0xC5 && m <= 0xC7)) {
                return "lossless or hierarchical JPEG (SOF" + std::to_string(m - 0xC0) + ") is not supported";
            } else if ((m >= 0xC9 && m <= 0xCB) || (m >= 0xCD && m <= 0xCF) || m == 0xCC) {
                return "arithmetic-coded JPEG is not supported";
            } else if (m == 0xC8 || (m >= 0xF0 && m <= 0xFD) || m == 0xDE || m == 0xDF) {
                return "unsupported JPEG extension marker";
            } else if (m == 0xC4) {
                size_t o = 0;
                while (o < dl) {
                    if (o + 17 > dl) return "truncated Huffman table";
                    const int tc = d[o] >> 4, th = d[o] & 15;
                    if (tc > 1 || th > 3) return "bad Huffman table number";
                    int cnt = 0;
                    for (int l = 0; l < 16; ++l) cnt += d[o + 1 + l];
                    if (cnt > 256 || o + 17 + (size_t)cnt > dl) return "bad Huffman table";
                    Huff t;
                    const std::string why = derive(d + o + 1, d + o + 17, cnt, tc == 0, t);
                    if (!why.empty()) return why;
                    (tc == 0 ? dc_tab : ac_tab)[th] = (int)P.huffs.size();
                    P.huffs.push_back(t);
                    o += 17 + (size_t)cnt;
                }
            } else if (m == 0xDB) {
                size_t o = 0;
                while (o < dl) {
                    const int pq = d[o] >> 4, tq = d[o] & 15;
                    if (pq > 1 || tq > 3 || o + 1 + 64 * (size_t)(pq + 1) > dl) return "bad quantisation table";
                    for (int k = 0; k < 64; ++k)
                        qtab[tq][zigzag(k)] = (uint16_t)(pq ? be16(d + o + 1 + 2 * k) : d[o + 1 + k]);
                    qdef[tq] = true;
                    o += 1 + 64 * (size_t)(pq + 1);
                }
            } else if (m == 0xDD) {
                if (dl < 2) return "truncated restart interval";
                restart = (int)be16(d);
            } else if (m == 0xDC) {
                return "a DNL marker is not supported";
            } else if (m == 0xE0) {
                if (dl >= 5 && !memcmp(d, "JFIF", 5)) jfif = true;
            } else if (m == 0xE1) {
                if (!exif_seen && P.scans.empty()) { exif_seen = true; pic.orient = exif_orientation(d, dl); }
            } else if (m == 0xEE) {
                if (dl >= 12 && !memcmp(d, "Adobe", 5)) { adobe = true; adobe_transform = d[11]; }
            } else if (m == 0xDA) {
                if (!frame) return "a scan before the frame header";
                if (dl < 1) return "truncated scan header";
                Scan sc;
                memset(&sc, 0, sizeof(sc));
                sc.ncomp = d[0];
                if (sc.ncomp < 1 || sc.ncomp > pic.ncomp || dl < 4 + 2 * (size_t)sc.ncomp) return "bad scan header";
                const uint8_t* e = d + 1 + 2 * sc.ncomp;
                sc.ss = e[0]; sc.se = e[1];
                const int ah = e[2] >> 4;
                sc.al = e[2] & 15;
                int comps[4];
                for (int j = 0; j < sc.ncomp; ++j) {
                    int c = -1;
                    for (int k = 0; k < pic.ncomp; ++k) if (cid[k] == d[1 + 2 * j]) c = k;
                    if (c < 0) return "a scan names a component the frame does not have";
                    comps[j] = c;
                    const int td = d[2 + 2 * j] >> 4, ta = d[2 + 2 * j] & 15;
                    if (td > 3 || ta > 3) return "bad Huffman table number in a scan";
                    const bool need_dc = !progressive || (sc.ss == 0 && ah == 0), need_ac = !progressive || sc.ss > 0;
                    if ((need_dc && dc_tab[td] < 0) || (need_ac && ac_tab[ta] < 0)) return "a scan uses an undefined Huffman table";
                    sc.dc[j] = (uint32_t)(dc_tab[td] < 0 ? 0 : dc_tab[td]);
                    sc.ac[j] = (uint32_t)(ac_tab[ta] < 0 ? 0 : ac_tab[ta]);
                    if (!latched[c]) {
                        if (!qdef[cq[c]]) return "a component's quantisation table is not defined";
                        P.quant.resize(64 * (size_t)pic.ncomp);
                        memcpy(&P.quant[64 * (size_t)c], qtab[cq[c]], sizeof(qtab[0]));
                        latched[c] = true;
                    }
                }
                if (progressive) {
                    bool bad = sc.ss == 0 ? sc.se != 0 : (sc.ss > sc.se || sc.se > 63 || sc.ncomp != 1);
                    if (ah != 0 && sc.al != ah - 1) bad = true;
                    if (sc.al > 13) bad = true;
                    if (bad) return "an invalid progressive scan";
                    for (int j = 0; j < sc.ncomp; ++j) {
                        int* cb = coef_bits[comps[j]];
                        if (sc.ss > 0 && cb[0] < 0) return "an AC scan before the component's DC scan";
                        for (int k = sc.ss; k <= sc.se; ++k) {
                            if (ah != (cb[k] < 0 ? 0 : cb[k])) return "an inconsistent progression sequence";
                            cb[k] = sc.al;
                        }
                    }
                    sc.kind = sc.ss == 0 ? (ah ? kDcRefine : kDcFirst) : (ah ? kAcRefine : kAcFirst);
                } else {
                    sc.kind = kSequential;
                    for (int j = 0; j < sc.ncomp; ++j) for (int k = 0; k < 64; ++k) coef_bits[comps[j]][k] = 0;
                }
                // the MCU
                int mcus;
                if (sc.ncomp == 1) {
                    const Comp& C = pic.comp[comps[0]];
                    sc.blocks = 1; sc.bcomp[0] = (uint8_t)comps[0]; sc.mcux = C.wib;
                    mcus = C.wib * C.hib;
                } else {
                    sc.mcux = (pic.w + 8 * pic.hmax - 1) / (8 * pic.hmax);
                    mcus = sc.mcux * ((pic.h + 8 * pic.vmax - 1) / (8 * pic.vmax));
                    for (int j = 0; j < sc.ncomp; ++j) {
                        const Comp& C = pic.comp[comps[j]];
                        for (int yy = 0; yy < C.v; ++yy)
                            for (int xx = 0; xx < C.h; ++xx) {
                                if (sc.blocks >= kMaxBlocks) return "too many blocks in an MCU";
                                sc.bcomp[sc.blocks] = (uint8_t)comps[j]; sc.bslot[sc.blocks] = (uint8_t)j;
                                sc.bdx[sc.blocks] = (uint8_t)xx; sc.bdy[sc.blocks] = (uint8_t)yy; ++sc.blocks;
                            }
                    }
                }
                const uint32_t si = (uint32_t)P.scans.size();
                P.scans.push_back(sc);
                // the entropy-coded data: split at RSTn, up to the next other marker
                const int nseg = restart ? (mcus + restart - 1) / restart : 1;
                int found = 0;
                size_t begin = pos;
                in_scan = true;
                while (in_scan) {
                    const uint8_t* ff = pos < n ? (const uint8_t*)memchr(f + pos, 0xFF, n - pos) : nullptr;
                    size_t i = ff ? (size_t)(ff - f) : n;
                    size_t j = i + 1;
                    while (j < n && f[j] == 0xFF) ++j;             // fill bytes before a marker
                    if (i >= n || j >= n) {                        // the file ends inside the scan's data
                        if (found < nseg) {
                            Seg s = {si, (uint32_t)(found * restart), (uint32_t)(restart ? (mcus - found * restart < restart ? mcus - found * restart : restart) : mcus), 0, begin, i < n ? i : n};
                            P.segs.push_back(s);
                            ++found;
                        }
                        pic.bad = 1; pos = n; in_scan = false; eoi = true;
                        break;
                    }
                    const unsigned mk = f[j];
                    if (mk == 0x00) {                              // stuffed FF 00 (after fill bytes: not restated)
                        if (j != i + 1) pic.bad = 1;
                        pos = j + 1;
                        continue;
                    }
                    if (found < nseg) {
                        const uint32_t m0 = (uint32_t)(found * restart);
                        Seg s = {si, m0, (uint32_t)(restart ? (mcus - (int)m0 < restart ? mcus - (int)m0 : restart) : mcus), 0, begin, i};
                        P.segs.push_back(s);
                    } else {
                        pic.bad = 1;                               // more intervals than MCUs
                    }
                    ++found;
                    if (mk >= 0xD0 && mk <= 0xD7) {
                        if ((int)(mk - 0xD0) != ((found - 1) & 7) || !restart) pic.bad = 1;
                        pos = begin = j + 1;
                    } else {
                        pos = j - 1;                               // the marker's FF
                        in_scan = false;
                    }
                }
                if (found < nseg) pic.bad = 1;
            }
            // other APPn, COM: skipped
        }
        return "";
    };
    const std::string why = markers();
    if (!why.empty()) {
        if (P.scans.empty()) return why;
        pic.bad = 1;
    }
    if (!frame) return "no frame header";
    if (P.scans.empty()) return "no scan";
    if (pic.ncomp == 3) {
        bool rgb;
        if (jfif) rgb = false;
        else if (adobe) {
            if (adobe_transform != 1) return "an Adobe APP14 colour transform " + std::to_string(adobe_transform) + " (only YCbCr, transform 1, is supported)";
            rgb = false;
        } else rgb = cid[0] == 82 && cid[1] == 71 && cid[2] == 66;
        if (rgb) return "RGB JPEG (component ids 'R', 'G', 'B') is not supported";
    }
    for (int c = 0; c < pic.ncomp; ++c) {
        if (!latched[c]) { pic.bad = 1; P.quant.resize(64 * (size_t)pic.ncomp); }   // a component without its scan: data missing
        // libjpeg smooths blocks whose first coefficients are not at full precision when the output starts, which is not restated.
        // A complete file has them all; a script cut short (a truncated file, or a false EOI: a lost FF 00 before a D9 byte) is
        // corrupt data
        for (int k = 0; k < 10; ++k)
            if (coef_bits[c][k] != 0) { pic.bad = 1; break; }
    }
    pic.ow = pic.orient >= 5 ? pic.h : pic.w;
    pic.oh = pic.orient >= 5 ? pic.w : pic.h;
    return "";
}

// the upload of a batch: [pics | scans | segs (grouped by round) | huffs | quant | data], each section 16-byte aligned.  Round r is
// the r-th scan of every picture: the segments of one round are independent, the rounds run in order
struct Layout {
    size_t pics = 0, scans = 0, segs = 0, huffs = 0, quant = 0, data = 0, bytes = 0;
    std::vector<uint32_t> round0;        // first segment of each round, then the total
    uint64_t coef = 0, planes = 0, rgb = 0;   // int16 coefficients, plane bytes, output bytes
    int max_blocks = 0;                  // blocks of the largest plane
    int max_px = 0;                      // pixels of the largest picture
};

inline size_t al16(size_t v) { return (v + 15) & ~(size_t)15; }

inline Layout layout(const std::vector<Parsed>& ps, const uint64_t* sizes)
{
    Layout L;
    size_t nsc = 0, nseg = 0, nh = 0, nq = 0, nd = 0, rounds = 0;
    for (size_t i = 0; i < ps.size(); ++i) {
        nsc += ps[i].scans.size(); nseg += ps[i].segs.size(); nh += ps[i].huffs.size(); nq += ps[i].quant.size(); nd += sizes[i];
        if (ps[i].scans.size() > rounds) rounds = ps[i].scans.size();
    }
    L.pics = 0;
    L.scans = al16(L.pics + sizeof(Pic) * ps.size());
    L.segs = al16(L.scans + sizeof(Scan) * nsc);
    L.huffs = al16(L.segs + sizeof(Seg) * nseg);
    L.quant = al16(L.huffs + sizeof(Huff) * nh);
    L.data = al16(L.quant + sizeof(uint16_t) * nq);
    L.bytes = al16(L.data + nd);
    std::vector<uint32_t> per(rounds, 0);
    for (const Parsed& p : ps)
        for (const Seg& s : p.segs) ++per[s.scan];
    L.round0.assign(rounds + 1, 0);
    for (size_t r = 0; r < rounds; ++r) L.round0[r + 1] = L.round0[r] + per[r];
    for (const Parsed& p : ps) {
        const Pic& P = p.pic;
        for (int c = 0; c < P.ncomp; ++c) {
            const uint64_t blocks = (uint64_t)P.comp[c].bw * P.comp[c].bh;
            L.coef += 64 * blocks; L.planes += 64 * blocks;
            if ((int)blocks > L.max_blocks) L.max_blocks = (int)blocks;
        }
        L.rgb += 3 * (uint64_t)P.w * P.h;
        if (P.w * P.h > L.max_px) L.max_px = P.w * P.h;
    }
    return L;
}

// the batch into dst (L.bytes): offsets made absolute (coefficients, planes, output, tables, data)
inline void pack(const std::vector<Parsed>& ps, const uint8_t* const* files, const uint64_t* sizes, const Layout& L, uint8_t* dst)
{
    Pic* pics = reinterpret_cast<Pic*>(dst + L.pics);
    Scan* scans = reinterpret_cast<Scan*>(dst + L.scans);
    Seg* segs = reinterpret_cast<Seg*>(dst + L.segs);
    Huff* huffs = reinterpret_cast<Huff*>(dst + L.huffs);
    uint16_t* quant = reinterpret_cast<uint16_t*>(dst + L.quant);
    uint8_t* data = dst + L.data;
    std::vector<uint32_t> next(L.round0.begin(), L.round0.end() - 1);
    uint64_t coef = 0, out = 0, data_off = 0;
    uint32_t sc0 = 0, h0 = 0, q0 = 0;
    for (size_t i = 0; i < ps.size(); ++i) {
        const Parsed& p = ps[i];
        Pic P = p.pic;
        for (int c = 0; c < P.ncomp; ++c) {
            P.comp[c].coef = coef; P.comp[c].plane = coef;    // one plane byte per coefficient
            P.comp[c].quant = q0 + 64 * (uint32_t)c;
            coef += 64 * (uint64_t)P.comp[c].bw * P.comp[c].bh;
        }
        P.out = out;
        out += 3 * (uint64_t)P.w * P.h;
        pics[i] = P;
        for (size_t s = 0; s < p.scans.size(); ++s) {
            Scan S = p.scans[s];
            S.pic = (int)i;
            for (int j = 0; j < 4; ++j) { S.dc[j] += h0; S.ac[j] += h0; }
            scans[sc0 + s] = S;
        }
        for (const Seg& s : p.segs) {
            Seg G = s;
            G.scan = sc0 + s.scan;
            G.begin += data_off; G.end += data_off;
            segs[next[s.scan]++] = G;
        }
        if (!p.huffs.empty()) memcpy(huffs + h0, p.huffs.data(), sizeof(Huff) * p.huffs.size());
        if (!p.quant.empty()) memcpy(quant + q0, p.quant.data(), sizeof(uint16_t) * p.quant.size());
        memcpy(data + data_off, files[i], sizes[i]);
        sc0 += (uint32_t)p.scans.size(); h0 += (uint32_t)p.huffs.size(); q0 += (uint32_t)p.quant.size();
        data_off += sizes[i];
    }
}

}  // namespace jpeg
}  // namespace cb200
