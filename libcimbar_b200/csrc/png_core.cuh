// png_core.cuh -- the PNG decode of the camera path, written once for the host (tests/cpp/png_core_host.cpp) and the device (png.cu):
// the chunk walk and the upload layout (host only), and the IDAT CRC, inflate, unfilter and expand steps (host and device).
//
// The goal is the RGB8 picture cv2.cvtColor(cv2.imread(file, IMREAD_COLOR), COLOR_BGR2RGB) returns, byte for byte.  OpenCV reads PNG
// through libpng with palette expansion, grey 1/2/4 -> 8 expansion, tRNS -> alpha, alpha stripped, grey -> RGB and png_set_strip_16;
// pinned against cv2 4.13 / libpng 1.6.53 (tests/test_png_core_host.py), that is:
//   - grey is replicated to three channels, 1/2/4-bit grey scaled by 255, 85 and 17;
//   - palette entries are looked up; an index past the PLTE entries gives black;
//   - alpha is dropped, never composited: tRNS and bKGD change no pixel;
//   - 16 bit becomes 8 bit by truncation (the high byte);
//   - gAMA, sRGB, iCCP, cHRM and sBIT change no pixel;
//   - an eXIf orientation is applied as for JPEG (jpeg_core.cuh exif_orientation / orient_source).
// libpng's own checks, as they decide between cv2 returning a picture and returning None:
//   - every IDAT chunk's CRC is checked (a mismatch fails the file); ancillary chunks with a bad CRC are dropped;
//   - the zlib stream has to end, Adler-32 included, inside the IDAT chunks, and give at least h x (1 + stride) bytes (more is
//     accepted);
//   - the Adler-32 is compared in the zlib call that completes the last row when the stream's last byte is in the same read slice
//     (8192 bytes of one IDAT chunk, libpng's IDAT_read_size) as that call's input; a mismatch there fails the file.  A mismatch found
//     later, at png_read_end, is only a warning.
#pragma once
#include "jpeg_core.cuh"

#include <stddef.h>
#include <stdint.h>
#include <string.h>

#include <string>
#include <vector>

#if defined(__CUDACC__)
#define PD_HD __host__ __device__ __forceinline__
#else
#define PD_HD inline
#endif

namespace cb200 {
namespace png {

constexpr int kLookBits = 10;            // primary look-up of the Huffman decoder
constexpr uint32_t kSlice = 8192;        // libpng's IDAT read size: the input of one zlib call is at most one slice of one chunk
constexpr int kBatch = 32;               // tokens per warp step of the inflate

struct Pic {
    int w, h;                            // decoded size
    int ow, oh;                          // output size (after the eXIf orientation)
    int orient;                          // 1..8
    int ct, bd;                          // colour type, bit depth
    int bpp;                             // filter distance in bytes (at least 1)
    uint32_t stride;                     // bytes of a row without its filter byte
    uint32_t npal;                       // PLTE entries (colour type 3)
    uint32_t chunk0, nchunks;            // its IDAT chunks in the chunk table
    uint32_t pal;                        // first byte of its palette in the palette section
    uint32_t pad;
    uint64_t z, zlen;                    // its zlib stream (the IDAT payloads back to back) in the data section
    uint64_t raw;                        // first byte of its filtered scanlines (h x (1 + stride)) in the scanline buffer
    uint64_t out;                        // first byte of its RGB8 picture in the output
};

struct Chunk {                           // one IDAT chunk
    uint64_t begin;                      // its payload in the data section
    uint32_t len, crc;                   // payload bytes, the CRC stored in the file
    uint32_t pic;
    uint32_t slice0;                     // libpng read slices of the picture's chunks before this one
};

// ---- CRC-32 of pieces, combined -------------------------------------------------------------------------------------------

constexpr uint32_t kPoly = 0xEDB88320u;  // reflected

PD_HD uint32_t crc_byte(uint32_t c, uint8_t b)          // the register after one byte, bitwise (no table to keep in memory)
{
    c ^= b;
    for (int k = 0; k < 8; ++k) c = (c >> 1) ^ (kPoly & (0u - (c & 1u)));
    return c;
}

PD_HD uint32_t crc_raw(uint32_t c, const uint8_t* p, uint64_t n)   // the register after n bytes from register c (no pre/post xor)
{
    for (uint64_t i = 0; i < n; ++i) c = crc_byte(c, p[i]);
    return c;
}

PD_HD uint32_t mulmod(uint32_t a, uint32_t b)           // a * b mod P, polynomials in reflected form (zlib multmodp)
{
    uint32_t m = 1u << 31, p = 0;
    for (;;) {
        if (a & m) {
            p ^= b;
            if ((a & (m - 1)) == 0) break;
        }
        m >>= 1;
        b = b & 1 ? (b >> 1) ^ kPoly : b >> 1;
    }
    return p;
}

PD_HD uint32_t shift(uint32_t c, uint64_t n)            // the register c followed by n zero bytes: c * x^(8 n) mod P
{
    uint32_t p = 1u << 31, base = 1u << 23;             // x^0, x^8
    for (; n; n >>= 1) {
        if (n & 1) p = mulmod(p, base);
        base = mulmod(base, base);
    }
    return mulmod(p, c);
}

// lane `lane` of `lanes`: its piece of a chunk's payload, as its share of the chunk's CRC register.  XOR over the lanes, then
// chunk_crc, gives the CRC of "IDAT" + payload
PD_HD uint32_t crc_piece(const uint8_t* p, uint32_t len, int lane, int lanes)
{
    const uint32_t per = (len + (uint32_t)lanes - 1) / (uint32_t)lanes;
    const uint32_t b = per * (uint32_t)lane < len ? per * (uint32_t)lane : len, e = b + per < len ? b + per : len;
    return shift(crc_raw(0, p + b, e - b), len - e);
}

PD_HD uint32_t chunk_crc(uint32_t pieces, uint32_t len)
{
    const uint8_t idat[4] = {'I', 'D', 'A', 'T'};
    return ~(shift(crc_raw(0xFFFFFFFFu, idat, 4), len) ^ pieces);
}

// ---- inflate ----------------------------------------------------------------------------------------------------------------

struct Huff {                            // a canonical code (puff.c's count / symbol) with a primary look-up
    uint16_t look[1 << kLookBits];       // by the next kLookBits stream bits: (length << 9) | symbol of a code up to kLookBits long; 0 =
                                         // longer or none
    uint16_t count[16];                  // codes of each length
    uint16_t sym[320];                   // symbols in code order
};

// count / sym from code lengths (puff.c construct): false for an over-subscribed set, or an incomplete one other than a single code
// of length 1 (zlib inflate_table; the code-length code may not be incomplete at all)
PD_HD bool build(Huff& t, const uint8_t* lens, int n, bool code_lengths)
{
    for (int l = 0; l < 16; ++l) t.count[l] = 0;
    for (int s = 0; s < n; ++s) t.count[lens[s]]++;
    if (t.count[0] == n) { t.count[0] = 0; return true; }   // no codes: any symbol read from it is an error
    int left = 1, max = 0;
    for (int l = 1; l < 16; ++l) {
        left = (left << 1) - t.count[l];
        if (left < 0) return false;
        if (t.count[l]) max = l;
    }
    if (left > 0 && (code_lengths || max != 1)) return false;
    uint16_t offs[16];
    offs[1] = 0;
    for (int l = 1; l < 15; ++l) offs[l + 1] = (uint16_t)(offs[l] + t.count[l]);
    for (int s = 0; s < n; ++s)
        if (lens[s]) t.sym[offs[lens[s]]++] = (uint16_t)s;
    t.count[0] = 0;
    return true;
}

// the symbol of the code at the bottom of `bits` (stream order), at most maxlen bits: (length << 9) | symbol, or 0 for none
PD_HD uint32_t canonical(const Huff& t, uint32_t bits, int maxlen)
{
    int code = 0, first = 0, index = 0;
    for (int l = 1; l <= maxlen; ++l) {
        code |= (int)((bits >> (l - 1)) & 1u);
        const int count = t.count[l];
        if (code - count < first) return (uint32_t)l << 9 | t.sym[index + (code - first)];
        index += count;
        first += count;
        first <<= 1;
        code <<= 1;
    }
    return 0;
}

// look-up entry e; the warp fills the table lane by lane
PD_HD void fill_look(Huff& t, uint32_t e) { t.look[e] = (uint16_t)canonical(t, e, kLookBits); }

struct Bits {                            // LSB-first reader over a zlib stream
    const uint8_t* z;
    uint64_t zlen;
    uint64_t next;                       // next byte to load; bytes past zlen read as zero
    uint64_t acc;
    int n;                               // valid bits in acc
};

PD_HD void need(Bits& b, int k)
{
    while (b.n < k) {
        const uint64_t v = b.next < b.zlen ? b.z[b.next] : 0;
        b.acc |= v << b.n;
        b.n += 8;
        b.next++;
    }
}

PD_HD uint32_t getbits(Bits& b, int k)
{
    if (!k) return 0;
    need(b, k);
    const uint32_t v = (uint32_t)(b.acc & ((1ull << k) - 1));
    b.acc >>= k;
    b.n -= k;
    return v;
}

PD_HD uint64_t consumed(const Bits& b) { return 8 * b.next - (uint64_t)b.n; }   // bits read so far

PD_HD int decode(Bits& b, const Huff& t, bool look)     // the next symbol, -1 for a code that is not in the table
{
    need(b, 15);
    uint32_t e = look ? t.look[b.acc & ((1u << kLookBits) - 1)] : 0;
    if (!e) e = canonical(t, (uint32_t)(b.acc & 0x7FFF), 15);
    if (!e) return -1;
    b.acc >>= (e >> 9);
    b.n -= (int)(e >> 9);
    return (int)(e & 511);
}

enum Status { kRun = 0, kEndOfBlock = 1, kBad = 2 };
enum Block { kNeedHeader = 0, kStored = 1, kHuffman = 2, kFinished = 3 };

struct Inflate {                         // the decoder state (one lane of the warp owns it)
    Bits b;
    uint64_t out;                        // bytes produced so far
    uint64_t cap;                        // bytes the rows need: h x (1 + stride)
    uint64_t last_row;                   // first byte of the last row
    uint32_t stored;                     // bytes left in the current stored block
    int block, last;                     // Block, final-block flag of the current block
    int crossed, span;                   // the cap was reached: the byte holding the last bit of that token (b_last), and whether that
    uint64_t b_last;                     // token was a match begun before the last row
    // zlib's window rule as libpng drives it (see window_ok): the window of the zlib header, the row length, the output position
    // of the last zlib call that began inside a row (libpng refilled its input there), and the read slice in use
    uint64_t wsize, rowlen, refill;
    uint64_t slice_end;                  // stream offset of the end of the current read slice (~0 past the last chunk)
    const Chunk* ch;                     // the file's IDAT chunks, their payload offsets relative to z0
    uint64_t z0;
    uint32_t nch, ci;                    // chunks, the chunk of the current slice
};

struct Tok { uint32_t len; uint32_t v; };   // v: a literal (len 1) or a distance

// the next libpng read slice: the next 8 KB of the chunk, or the first of the next non-empty chunk
PD_HD void next_slice(Inflate& I)
{
    if (I.ci < I.nch) {
        const uint64_t e = I.ch[I.ci].begin - I.z0 + I.ch[I.ci].len;
        if (I.slice_end < e) { I.slice_end = I.slice_end + kSlice < e ? I.slice_end + kSlice : e; return; }
        ++I.ci;
    }
    while (I.ci < I.nch && I.ch[I.ci].len == 0) ++I.ci;
    I.slice_end = I.ci < I.nch ? I.ch[I.ci].begin - I.z0 + (I.ch[I.ci].len < kSlice ? I.ch[I.ci].len : kSlice) : ~0ull;
}

// the decoder over picture P's stream in data, whose IDAT chunks are ch[0, P.nchunks)
PD_HD void inflate_init(Inflate& I, const Pic& P, const Chunk* ch, const uint8_t* data)
{
    const uint8_t* z = data + P.z;
    I.b.z = z; I.b.zlen = P.zlen; I.b.next = 2; I.b.acc = 0; I.b.n = 0;   // past the zlib header, checked by parse()
    I.rowlen = 1 + (uint64_t)P.stride;
    I.cap = (uint64_t)P.h * I.rowlen;
    I.out = 0; I.last_row = I.cap - I.rowlen; I.stored = 0; I.block = kNeedHeader; I.last = 0;
    I.crossed = 0; I.span = 0; I.b_last = 0;
    I.wsize = 1ull << ((z[0] >> 4) + 8);                  // CINFO: parse() refused values above 7
    I.refill = 0;
    I.ch = ch; I.z0 = P.z; I.nch = P.nchunks; I.ci = 0; I.slice_end = 0;
    next_slice(I);
}

// after a step that began with `before` bytes out: a step whose bits run past the current slice made zlib return for more input
// there, and libpng's next call begins at that output position
PD_HD void track(Inflate& I, uint64_t before)
{
    while (consumed(I.b) > 8 * I.slice_end) { I.refill = before; next_slice(I); }
}

// zlib's window rule for a match of distance d and length len at output position p, as libpng calls zlib: one call per row (h x
// (1 + stride) bytes in rows), and within a row one more each time the input slice runs out.  zlib keeps min(output before the
// call, window) bytes of history beside what the call has written, so d must be at most (p - c) + min(c, wsize) with c the call's
// first output byte; a match that runs into the next row goes on in a new call, where d must be at most min(c', wsize).  Past the
// rows libpng only warns
PD_HD bool window_ok(const Inflate& I, uint64_t p, uint32_t len, uint32_t d)
{
    if (p >= I.cap) return true;
    const uint64_t row0 = p - p % I.rowlen, c = I.refill > row0 ? I.refill : row0;
    if (d > (p - c) + (c < I.wsize ? c : I.wsize)) return false;
    const uint64_t next = row0 + I.rowlen;
    return !(next < p + len && next < I.cap && d > (next < I.wsize ? next : I.wsize));
}

PD_HD void note_cap(Inflate& I, uint64_t before, uint64_t after, bool match)
{
    if (!I.crossed && before < I.cap && after >= I.cap) {
        I.crossed = 1;
        I.b_last = (consumed(I.b) - 1) >> 3;
        I.span = match && before < I.last_row;
    }
}

// a block header.  Fixed and dynamic blocks leave their code lengths in lens (litlen then dist; *nlit, *ndist) for build(); a stored
// block leaves I.stored.  false for an invalid header (block type 3, LEN / NLEN, bad code-length sets); `cl` is scratch
PD_HD bool block_header_bits(Inflate& I, uint8_t* lens, int* nlit, int* ndist, Huff& cl)
{
    I.last = (int)getbits(I.b, 1);
    const uint32_t type = getbits(I.b, 2);
    if (type == 0) {
        const int drop = I.b.n & 7;                       // to a byte boundary
        I.b.acc >>= drop; I.b.n -= drop;
        const uint32_t len = getbits(I.b, 16), nlen = getbits(I.b, 16);
        if ((len ^ 0xFFFFu) != nlen) return false;
        I.stored = len;
        I.block = kStored;
        return true;
    }
    if (type == 3) return false;
    I.block = kHuffman;
    if (type == 1) {
        for (int s = 0; s < 288; ++s) lens[s] = (uint8_t)(s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : 8);
        for (int s = 0; s < 32; ++s) lens[288 + s] = 5;   // 30 and 31 complete the code and are refused when read
        *nlit = 288; *ndist = 32;
        return true;
    }
    const int hlit = (int)getbits(I.b, 5) + 257, hdist = (int)getbits(I.b, 5) + 1, hclen = (int)getbits(I.b, 4) + 4;
    if (hlit > 286 || hdist > 30) return false;
    const uint8_t order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
    uint8_t cll[19];
    for (int k = 0; k < 19; ++k) cll[order[k]] = k < hclen ? (uint8_t)getbits(I.b, 3) : 0;
    if (!build(cl, cll, 19, true)) return false;
    int k = 0;
    while (k < hlit + hdist) {
        const int s = decode(I.b, cl, false);
        if (s < 0) return false;
        if (s < 16) { lens[k++] = (uint8_t)s; continue; }
        int rep, v = 0;
        if (s == 16) {
            if (k == 0) return false;
            v = lens[k - 1];
            rep = 3 + (int)getbits(I.b, 2);
        } else {
            rep = s == 17 ? 3 + (int)getbits(I.b, 3) : 11 + (int)getbits(I.b, 7);
        }
        if (k + rep > hlit + hdist) return false;
        while (rep--) lens[k++] = (uint8_t)v;
    }
    if (lens[256] == 0) return false;                     // no end-of-block code
    // the distance lengths move up to 288 so that lens has one layout for every block
    for (int d = hdist - 1; d >= 0; --d) lens[288 + d] = lens[hlit + d];
    *nlit = hlit; *ndist = hdist;
    return true;
}

PD_HD bool block_header(Inflate& I, uint8_t* lens, int* nlit, int* ndist, Huff& cl)
{
    const bool ok = block_header_bits(I, lens, nlit, ndist, cl);
    track(I, I.out);
    return ok;
}

// up to kBatch tokens of the current Huffman block into tok (*nt); kEndOfBlock after its end-of-block code, kBad for a code not in
// the tables, a symbol past the alphabet, a distance before the output or past zlib's window (window_ok), or a stream that ran out
PD_HD int decode_batch(Inflate& I, const Huff& lit, const Huff& dist, Tok* tok, int* nt)
{
    const uint16_t lbase[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
    const uint8_t lext[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
    const uint16_t dbase[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073,
                                4097, 6145, 8193, 12289, 16385, 24577};
    int k = 0, st = kRun;
    while (k < kBatch) {
        const int s = decode(I.b, lit, true);
        if (s < 0 || s > 285) { st = kBad; break; }
        if (s == 256) { st = kEndOfBlock; break; }
        const uint64_t before = I.out;
        if (s < 256) {
            tok[k].len = 1; tok[k].v = (uint32_t)s;
        } else {
            const uint32_t len = lbase[s - 257] + getbits(I.b, lext[s - 257]);
            const int ds = decode(I.b, dist, true);
            if (ds < 0 || ds > 29) { st = kBad; break; }
            const uint32_t d = dbase[ds] + getbits(I.b, ds < 4 ? 0 : (ds >> 1) - 1);
            if (d > I.out) { st = kBad; break; }
            track(I, before);
            if (!window_ok(I, before, len, d)) { st = kBad; break; }
            tok[k].len = len; tok[k].v = d;
        }
        track(I, before);
        I.out += tok[k].len;
        note_cap(I, before, I.out, s > 256);
        ++k;
    }
    if (consumed(I.b) > 8 * I.b.zlen) st = kBad;          // the stream ended inside a code
    *nt = k;
    return st;
}

// the current stored block: its bytes at z[*src, *src + *len) go to the output at I.out (before the call); the reader moves past
// them.  false if they run past the stream
PD_HD bool stored_step(Inflate& I, uint64_t* src, uint32_t* len)
{
    const uint64_t q = consumed(I.b) >> 3;                // byte-aligned after LEN / NLEN
    *src = q;
    *len = I.stored;
    if (q + I.stored > I.b.zlen) return false;
    const uint64_t before = I.out;
    while (I.slice_end < q + I.stored) {                  // slices that end inside the block: libpng's next call begins there
        I.refill = before + (I.slice_end > q ? I.slice_end - q : 0);
        next_slice(I);
    }
    I.out += I.stored;
    if (!I.crossed && before < I.cap && I.out >= I.cap) {  // the byte copied to cap - 1 is the last one read for the rows
        I.crossed = 1;
        I.b_last = q + (I.cap - 1 - before);
        I.span = 0;
    }
    I.b.next = q + I.stored; I.b.acc = 0; I.b.n = 0;
    I.stored = 0;
    I.block = I.last ? kFinished : kNeedHeader;
    return true;
}

// the match of token (len, d) whose output starts at p, lane by lane: out[p + i] = out[p - d + i mod d] reads only bytes before p,
// so the lanes of one match are independent.  Bytes at or past cap are not written
PD_HD void copy_match(uint8_t* out, uint64_t p, uint32_t len, uint32_t d, uint64_t cap, int lane, int lanes)
{
    for (uint32_t i = (uint32_t)lane; i < len; i += (uint32_t)lanes)
        if (p + i < cap) out[p + i] = out[p - d + (d >= len ? i : i % d)];
}

// the Adler-32 share of one lane over out[0, n): its sums of b and of (n - i) b, both mod 65521
PD_HD void adler_piece(const uint8_t* out, uint64_t n, int lane, int lanes, uint32_t* a, uint32_t* bsum)
{
    uint64_t s = 0, t = 0;
    for (uint64_t i = (uint64_t)lane; i < n; i += (uint64_t)lanes) {
        s += out[i];
        t += ((n - i) % 65521) * out[i];
        if (t >= (1ull << 62)) { s %= 65521; t %= 65521; }
    }
    *a = (uint32_t)(s % 65521);
    *bsum = (uint32_t)(t % 65521);
}

PD_HD uint32_t adler_of(uint32_t a, uint32_t bsum, uint64_t n)         // the lanes' sums combined (A starts at 1, B at n)
{
    const uint32_t A = (uint32_t)((1 + (uint64_t)a) % 65521), B = (uint32_t)((bsum + n % 65521) % 65521);
    return B << 16 | A;
}

// the read slice of stream byte p (libpng's zlib input at that byte): the slices of the earlier chunks, then p's 8 KB piece of its own
PD_HD uint64_t slice_of(const Chunk* ch, uint32_t nch, uint64_t z, uint64_t p, bool* slice_end)
{
    uint32_t lo = 0, hi = nch;                            // the last chunk whose payload begins at or before p
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) / 2;
        if (ch[mid].begin - z <= p) lo = mid; else hi = mid;
    }
    const uint64_t off = p - (ch[lo].begin - z);
    *slice_end = (off + 1) % kSlice == 0 || off + 1 == ch[lo].len;
    return ch[lo].slice0 + off / kSlice;
}

// the end of the stream: its Adler-32 (the next 4 bytes after the final block, byte-aligned) against the rows.  false where libpng
// fails the file: fewer bytes than the rows, a stream cut short, or an Adler-32 mismatch compared in the call that completed the
// last row (see the header comment)
PD_HD bool stream_end_ok(Inflate& I, const Chunk* ch, uint32_t nch, uint64_t z, uint32_t adler)
{
    const int drop = I.b.n & 7;
    I.b.acc >>= drop; I.b.n -= drop;
    uint32_t stored = 0;                                  // big-endian
    for (int k = 0; k < 4; ++k) stored = stored << 8 | getbits(I.b, 8);
    const uint64_t end = consumed(I.b) >> 3;              // bytes of the stream with its check value
    if (end > I.b.zlen || I.out < I.cap) return false;
    if (I.out > I.cap) return true;                       // the last row's call stopped at the first byte past the rows
    if (stored == adler) return true;
    bool at_end;
    uint64_t s = slice_of(ch, nch, z, I.b_last, &at_end);
    if (I.span && at_end) ++s;                            // a match begun rows earlier: the last row's call refilled its input
    bool unused;
    return slice_of(ch, nch, z, end - 1, &unused) != s;
}

// ---- unfilter ---------------------------------------------------------------------------------------------------------------

PD_HD uint8_t paeth(int a, int b, int c)
{
    const int p = a + b - c, pa = p > a ? p - a : a - p, pb = p > b ? p - b : b - p, pc = p > c ? p - c : c - p;
    return (uint8_t)(pa <= pb && pa <= pc ? a : pb <= pc ? b : c);
}

// the serial chain of filter f (1 Sub, 3 Avg, 4 Paeth) over byte lane c of a row (bytes c, c + bpp, ...), in place.  prev is the
// previous row (unfiltered) or null for the first
PD_HD void unfilter_chain(uint8_t* row, const uint8_t* prev, uint32_t stride, int bpp, int c, int f)
{
    int a = 0, up_left = 0;
    for (uint32_t x = (uint32_t)c; x < stride; x += (uint32_t)bpp) {
        const int b = prev ? prev[x] : 0;
        int v = row[x];
        if (f == 1) v += a;
        else if (f == 3) v += (a + b) >> 1;
        else v += paeth(a, b, up_left);
        a = v & 0xFF;
        up_left = b;
        row[x] = (uint8_t)a;
    }
}

// ---- expand -----------------------------------------------------------------------------------------------------------------

// sample k (0-based, within the row) of depth bd from an unfiltered row
PD_HD int sample_at(const uint8_t* row, int bd, uint32_t k)
{
    if (bd == 8) return row[k];
    if (bd == 16) return row[2 * k];                      // png_set_strip_16: the high byte
    const uint32_t bit = k * (uint32_t)bd;
    return (row[bit >> 3] >> (8 - bd - (int)(bit & 7))) & ((1 << bd) - 1);
}

// output pixel (ox, oy): eXIf orientation, then the decoded pixel's RGB
PD_HD void pixel_rgb(const uint8_t* raw, const uint8_t* pal, const Pic& P, int ox, int oy, uint8_t* rgb)
{
    int x, y;
    jpeg::orient_source(P.orient, P.w, P.h, ox, oy, x, y);
    const uint8_t* row = raw + (uint64_t)y * (1 + P.stride) + 1;
    switch (P.ct) {
    case 0: case 4: {                                     // grey (+ alpha): replicated, sub-byte depths scaled to 8 bit
        const int ch = P.ct == 0 ? 1 : 2;
        int v = sample_at(row, P.bd, (uint32_t)x * ch);
        if (P.bd < 8) v *= P.bd == 1 ? 255 : P.bd == 2 ? 85 : 17;
        rgb[0] = rgb[1] = rgb[2] = (uint8_t)v;
        break;
    }
    case 3: {
        const uint32_t i = (uint32_t)sample_at(row, P.bd, (uint32_t)x);
        for (int k = 0; k < 3; ++k) rgb[k] = i < P.npal ? pal[P.pal + 3 * i + k] : 0;
        break;
    }
    default: {                                            // RGB, RGBA
        const int ch = P.ct == 2 ? 3 : 4;
        for (int k = 0; k < 3; ++k) rgb[k] = (uint8_t)sample_at(row, P.bd, (uint32_t)x * ch + k);
    }
    }
}

// ---- host: the chunk walk and the upload layout ------------------------------------------------------------------------------

struct Parsed {                          // one file as parse() leaves it
    Pic pic;
    std::vector<uint8_t> pal;            // 3 x npal
    std::vector<uint64_t> idat;          // per IDAT chunk: its payload's offset in the file
    std::vector<uint32_t> idat_len, idat_crc;
};

inline uint32_t be32(const uint8_t* p) { return (uint32_t)p[0] << 24 | (uint32_t)p[1] << 16 | (uint32_t)p[2] << 8 | p[3]; }

inline uint32_t crc32_of(const uint8_t* p, size_t n) { return ~crc_raw(0xFFFFFFFFu, p, n); }

inline bool letter(uint8_t c) { return (c >= 'A' && c <= 'Z') || (c >= 'a' && c <= 'z'); }

// the chunks of one file: "" and P filled, or the reason the file is refused.  What the device checks (the IDAT CRCs, the deflate
// data, the filter bytes, the Adler-32) is left to it
inline std::string parse(const uint8_t* f, size_t n, Parsed& out)
{
    static const uint8_t sig[8] = {0x89, 'P', 'N', 'G', 0x0D, 0x0A, 0x1A, 0x0A};
    out = Parsed();
    Pic& P = out.pic;
    memset(&P, 0, sizeof(P));
    P.orient = 1;
    if (n < 8 || memcmp(f, sig, 8) != 0) return "not a PNG file (bad signature)";
    size_t pos = 8;
    bool ihdr = false, plte = false, iend = false, idat_done = false;
    int exifs = 0;
    while (!iend) {
        if (pos + 12 > n) return "a truncated file (no IEND chunk)";
        const uint32_t len = be32(f + pos);
        const uint8_t* type = f + pos + 4;
        const uint8_t* body = f + pos + 8;
        if (len > 0x7FFFFFFFu || (uint64_t)len + 12 > n - pos) return "a truncated file (a chunk runs past its end)";
        const std::string name(reinterpret_cast<const char*>(type), 4);
        // the IDAT CRCs are the device's (k_png_crc); the host checks only the header chunks it reads
        const bool crc_ok = name != "IDAT" && crc32_of(type, (size_t)len + 4) == be32(body + len);
        for (int k = 0; k < 4; ++k)
            if (!letter(type[k])) return "an invalid chunk type";
        if (!ihdr && name != "IHDR") return "IHDR is not the first chunk";
        if (name != "IDAT" && !out.idat.empty()) idat_done = true;
        if (name == "IHDR") {
            if (ihdr) return "a second IHDR chunk";
            if (len != 13) return "an IHDR chunk of " + std::to_string(len) + " bytes";
            if (!crc_ok) return "a bad CRC in IHDR";
            const uint32_t w = be32(body), h = be32(body + 4);
            const int bd = body[8], ct = body[9];
            if (w == 0 || h == 0 || w > 0x7FFFFFFFu || h > 0x7FFFFFFFu) return "an IHDR with an invalid size";
            const bool depth_ok = (ct == 0 && (bd == 1 || bd == 2 || bd == 4 || bd == 8 || bd == 16)) ||
                                  (ct == 3 && (bd == 1 || bd == 2 || bd == 4 || bd == 8)) ||
                                  ((ct == 2 || ct == 4 || ct == 6) && (bd == 8 || bd == 16));
            if (!depth_ok) return "an IHDR with colour type " + std::to_string(ct) + " at bit depth " + std::to_string(bd);
            if (body[10] != 0) return "an IHDR with an unknown compression method";
            if (body[11] != 0) return "an IHDR with an unknown filter method";
            if (body[12] == 1) return "an Adam7-interlaced file (not supported)";
            if (body[12] != 0) return "an IHDR with an unknown interlace method";
            if (w > 1000000 || h > 1000000) return "a width or height above 1000000 (libpng's limit)";
            if ((uint64_t)w * h > (1ull << 30)) return "a picture of more than 2^30 pixels (OpenCV's limit)";
            const int ch = ct == 0 || ct == 3 ? 1 : ct == 4 ? 2 : ct == 2 ? 3 : 4;
            P.w = (int)w; P.h = (int)h; P.ct = ct; P.bd = bd;
            P.stride = (uint32_t)(((uint64_t)w * ch * bd + 7) / 8);
            P.bpp = ch * bd / 8 > 0 ? ch * bd / 8 : 1;
            ihdr = true;
        } else if (name == "PLTE") {
            if (P.ct == 3) {                              // for other colour types libpng ignores PLTE, its CRC included
                if (plte) return "a second PLTE chunk";
                if (!out.idat.empty()) return "PLTE after IDAT";
                if (!crc_ok) return "a bad CRC in PLTE";
                if (len == 0 || len % 3 || len > 768) return "a PLTE chunk of " + std::to_string(len) + " bytes";
                out.pal.assign(body, body + len);
                P.npal = len / 3;
                plte = true;
            }
        } else if (name == "IDAT") {
            if (idat_done) return "IDAT chunks that are not consecutive";
            if (P.ct == 3 && !plte) return "colour type 3 without a PLTE chunk";
            out.idat.push_back(pos + 8);
            out.idat_len.push_back(len);
            out.idat_crc.push_back(be32(body + len));
            P.zlen += len;
        } else if (name == "IEND") {
            iend = true;
        } else if (name == "acTL" || name == "fcTL" || name == "fdAT") {
            return "an animated PNG (APNG, not supported)";
        } else if (!(type[0] & 0x20)) {
            return "an unknown critical chunk " + name;
        } else if (name == "eXIf") {
            if (++exifs > 1) return "more than one eXIf chunk";
            if (crc_ok && len >= 2 && ((body[0] == 'I' && body[1] == 'I') || (body[0] == 'M' && body[1] == 'M'))) {
                std::vector<uint8_t> app1(6, 0);          // exif_orientation reads a JPEG APP1 body: 6 bytes, then the TIFF header
                app1.insert(app1.end(), body, body + len);
                P.orient = jpeg::exif_orientation(app1.data(), app1.size());
            }
        }
        pos += 12 + (size_t)len;
    }
    if (out.idat.empty()) return "no IDAT chunk";
    // the zlib header: the first two bytes of the IDAT payloads
    uint8_t zh[2];
    int got = 0;
    for (size_t k = 0; k < out.idat.size() && got < 2; ++k)
        for (uint32_t i = 0; i < out.idat_len[k] && got < 2; ++i) zh[got++] = f[out.idat[k] + i];
    if (got < 2) return "a truncated zlib header";
    if ((zh[0] & 15) != 8 || (zh[0] >> 4) > 7 || ((unsigned)zh[0] << 8 | zh[1]) % 31) return "an invalid zlib header";
    if (zh[1] & 0x20) return "a zlib stream with a preset dictionary";
    P.ow = P.orient >= 5 ? P.h : P.w;
    P.oh = P.orient >= 5 ? P.w : P.h;
    return "";
}

// the upload of a batch: [pics | chunks | palettes | data], each section 16-byte aligned; data holds each file's IDAT payloads back
// to back (its zlib stream)
struct Layout {
    size_t pics = 0, chunks = 0, pal = 0, data = 0, bytes = 0;
    uint32_t nchunks = 0;
    uint64_t raw = 0, rgb = 0;           // filtered scanline bytes, output bytes
    uint64_t max_px = 0;                 // pixels of the largest picture
};

inline size_t al16(size_t v) { return (v + 15) & ~(size_t)15; }

inline Layout layout(const std::vector<Parsed>& ps)
{
    Layout L;
    size_t np = 0, nd = 0;
    for (const Parsed& p : ps) {
        L.nchunks += (uint32_t)p.idat.size();
        np += p.pal.size();
        nd += p.pic.zlen;
        L.raw += (uint64_t)p.pic.h * (1 + p.pic.stride);
        L.rgb += 3 * (uint64_t)p.pic.w * p.pic.h;
        if ((uint64_t)p.pic.w * p.pic.h > L.max_px) L.max_px = (uint64_t)p.pic.w * p.pic.h;
    }
    L.chunks = al16(sizeof(Pic) * ps.size());
    L.pal = al16(L.chunks + sizeof(Chunk) * L.nchunks);
    L.data = al16(L.pal + np);
    L.bytes = al16(L.data + nd);
    return L;
}

// the batch into dst (L.bytes): offsets made absolute (scanlines, output, palettes, data)
inline void pack(const std::vector<Parsed>& ps, const uint8_t* const* files, const Layout& L, uint8_t* dst)
{
    Pic* pics = reinterpret_cast<Pic*>(dst + L.pics);
    Chunk* chunks = reinterpret_cast<Chunk*>(dst + L.chunks);
    uint8_t* pal = dst + L.pal;
    uint8_t* data = dst + L.data;
    uint64_t raw = 0, out = 0, z = 0;
    uint32_t c0 = 0, p0 = 0;
    for (size_t i = 0; i < ps.size(); ++i) {
        const Parsed& p = ps[i];
        Pic P = p.pic;
        P.raw = raw; P.out = out; P.z = z; P.pal = p0; P.chunk0 = c0; P.nchunks = (uint32_t)p.idat.size();
        raw += (uint64_t)P.h * (1 + P.stride);
        out += 3 * (uint64_t)P.w * P.h;
        uint32_t slices = 0;
        for (size_t k = 0; k < p.idat.size(); ++k) {
            Chunk& C = chunks[c0 + k];
            C.begin = z; C.len = p.idat_len[k]; C.crc = p.idat_crc[k]; C.pic = (uint32_t)i; C.slice0 = slices;
            slices += (C.len + kSlice - 1) / kSlice;
            if (C.len) memcpy(data + z, files[i] + p.idat[k], C.len);
            z += C.len;
        }
        if (!p.pal.empty()) memcpy(pal + p0, p.pal.data(), p.pal.size());
        pics[i] = P;
        c0 += (uint32_t)p.idat.size();
        p0 += (uint32_t)p.pal.size();
    }
}

}  // namespace png
}  // namespace cb200
