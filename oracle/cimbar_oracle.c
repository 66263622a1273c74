/*
 * cimbar_oracle.c -- CPU restatement of libcimbar's per-frame decode hot path.
 *
 * TEST INFRASTRUCTURE ONLY (see cimbar_oracle.h).  Plain C99, no dependencies.
 * Every function cites the reference file:line (relative to /root/reference/) it follows.
 * Build: see oracle/Makefile (-O3 -march=x86-64-v3 -ffp-contract=off: the colour path is float32 and must
 * not be contracted into FMAs; the reference itself is built -O2 for generic x86-64, CMakeLists.txt:22, but its
 * preprocessing runs in OpenCV's SIMD kernels, so the restatement is compiled to vectorise as well).
 */
#define _POSIX_C_SOURCE 200809L
#include "cimbar_oracle.h"

#include <time.h>

#include <float.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

/* ------------------------------------------------------------------------------------------
 * mode table: src/lib/cimb_translator/GridConf.h:8-190, Config.h:20-49
 * ---------------------------------------------------------------------------------------- */
static void conf8x8(cbo_mode* m)
{
    /* GridConf.h:121-141 */
    m->color_bits = 2; m->symbol_bits = 4; m->ecc_bytes = 30; m->ecc_block_size = 155;
    m->image_size_x = 1024; m->image_size_y = 1024;
    m->cell_size = 8; m->cell_spacing_x = 9; m->cell_spacing_y = 9; m->cell_offset = 8;
    m->cells_per_col_x = 112; m->cells_per_col_y = 112;
    m->fountain_chunks_scalar = 2; m->legacy_mode = 0;
}

unsigned cbo_capacity(const cbo_mode* m, unsigned bits_per_cell)
{
    /* GridConf.h:47-52 */
    if (!bits_per_cell) bits_per_cell = m->color_bits + m->symbol_bits;
    return m->total_cells * bits_per_cell / 8;
}

int cbo_mode_init(cbo_mode* m, int mode_val)
{
    memset(m, 0, sizeof(*m));
    m->mode_val = mode_val;
    switch (mode_val) {
    case 4:  /* Config.h:24-29 */
        conf8x8(m); m->color_bits = 2; m->legacy_mode = 1; m->fountain_chunks_scalar = -10; break;
    case 8:  /* Config.h:30-35 */
        conf8x8(m); m->color_bits = 3; m->legacy_mode = 1; m->fountain_chunks_scalar = -10; break;
    case 66: /* Conf8x8_micro, GridConf.h:144-166 */
        conf8x8(m); m->ecc_bytes = 33; m->ecc_block_size = 168; m->image_size_x = 736; m->image_size_y = 637;
        m->cell_offset = 9; m->cells_per_col_x = 80; m->cells_per_col_y = 69; m->fountain_chunks_scalar = 1; break;
    case 67: /* Conf8x8_mini, GridConf.h:168-189 */
        conf8x8(m); m->ecc_bytes = 36; m->ecc_block_size = 179; m->image_size_x = 1024; m->image_size_y = 720;
        m->cell_offset = 9; m->cells_per_col_x = 112; m->cells_per_col_y = 78; m->fountain_chunks_scalar = 2; break;
    case 68:
    default:
        m->mode_val = 68; conf8x8(m); break;
    }
    m->corner_padding_x = (unsigned)lrint(54.0 / m->cell_spacing_x);  /* GridConf.h:32-40 */
    m->corner_padding_y = (unsigned)lrint(54.0 / m->cell_spacing_y);
    m->total_cells = m->cells_per_col_x * m->cells_per_col_y - m->corner_padding_x * m->corner_padding_y * 4;
    m->color_mode = m->legacy_mode ? 0 : 1;
    m->interleave_blocks = m->ecc_block_size;
    m->interleave_partitions = 2;
    {   /* GridConf.h:54-72 */
        unsigned bpc = m->color_bits + m->symbol_bits;
        m->chunks_per_frame = m->fountain_chunks_scalar < 0 ? (unsigned)(-m->fountain_chunks_scalar)
                                                            : bpc * (unsigned)m->fountain_chunks_scalar;
        m->chunk_size = cbo_capacity(m, bpc) * (m->ecc_block_size - m->ecc_bytes) / m->ecc_block_size / m->chunks_per_frame;
    }
    return 0;
}

/* ------------------------------------------------------------------------------------------
 * P2 CellPositions::compute_linear -- CellPositions.cpp:5-50
 * ---------------------------------------------------------------------------------------- */
int cbo_cell_positions(const cbo_mode* m, int padding, int* xs, int* ys)
{
    int sx = (int)m->cell_spacing_x, sy = (int)m->cell_spacing_y;
    int dx = (int)m->cells_per_col_x, dy = (int)m->cells_per_col_y;
    int mx = (int)m->corner_padding_x, my = (int)m->corner_padding_y;
    int offset = (int)m->cell_offset + padding;
    int n = 0;
    int marker_offset_x = sx * mx;
    int top_width = dx - mx - mx;
    int top_cells = top_width * my;
    for (int i = 0; i < top_cells; ++i, ++n) {
        xs[n] = (i % top_width) * sx + marker_offset_x + offset;
        ys[n] = (i / top_width) * sy + offset;
    }
    int mid_y = my * sy;
    int mid_width = dx;
    int mid_cells = mid_width * (dy - my - my);
    for (int i = 0; i < mid_cells; ++i, ++n) {
        xs[n] = (i % mid_width) * sx + offset;
        ys[n] = (i / mid_width) * sy + mid_y + offset;
    }
    int bottom_y = (dy - my) * sy;
    for (int i = 0; i < top_cells; ++i, ++n) {
        xs[n] = (i % top_width) * sx + marker_offset_x + offset;
        ys[n] = (i / top_width) * sy + bottom_y + offset;
    }
    return n;
}

/* ------------------------------------------------------------------------------------------
 * AdjacentCellFinder -- AdjacentCellFinder.cpp:5-105
 * ---------------------------------------------------------------------------------------- */
typedef struct {
    const int* xs; int n; int dim_x; int marker_x; int first_mid; int first_bottom;
} adj_t;

static void adj_init(adj_t* a, const cbo_mode* m, const int* xs, int n)
{
    a->xs = xs; a->n = n; a->dim_x = (int)m->cells_per_col_x; a->marker_x = (int)m->corner_padding_x;
    int mid_height = (int)m->cells_per_col_y - 2 * (int)m->corner_padding_y;
    int mid_cells = a->dim_x * mid_height;
    int edge_cells = (a->dim_x - 2 * a->marker_x) * (int)m->corner_padding_y;
    a->first_mid = edge_cells;
    a->first_bottom = edge_cells + mid_cells;
}
static int adj_margin(const adj_t* a, int index) { return (index < a->first_mid) ? 1 : (index < a->first_bottom ? 0 : 1); }
static int adj_right(const adj_t* a, int index)
{
    if (index < 0 || index >= a->n - 1) return -1;
    int next = index + 1;
    if (a->xs[next] < a->xs[index]) return -1;
    return next;
}
static int adj_left(const adj_t* a, int index)
{
    int next = index - 1;
    if (next < 0) return -1;
    if (a->xs[next] > a->xs[index]) return -1;
    return next;
}
static int adj_bottom(const adj_t* a, int index)
{
    if (index < 0 || index >= a->n) return -1;
    int increment = a->dim_x;
    if (adj_margin(a, index)) increment -= a->marker_x;
    int next = index + increment;
    if (adj_margin(a, next)) next -= a->marker_x;
    if (next < 0 || next >= a->n) return -1;
    if (a->xs[next] != a->xs[index]) return -1;
    return next;
}
static int adj_top(const adj_t* a, int index)
{
    int increment = a->dim_x;
    if (adj_margin(a, index)) increment -= a->marker_x;
    int next = index - increment;
    if (adj_margin(a, next)) next += a->marker_x;
    if (next < 0) return -1;
    if (a->xs[next] != a->xs[index]) return -1;
    return next;
}
void cbo_adjacent(const cbo_mode* m, const int* xs, int ncells, int index, int adj[4])
{
    adj_t a; adj_init(&a, m, xs, ncells);
    adj[0] = adj_right(&a, index); adj[1] = adj_left(&a, index);
    adj[2] = adj_bottom(&a, index); adj[3] = adj_top(&a, index);
}

/* ------------------------------------------------------------------------------------------
 * P7 Interleave -- Interleave.h:8-36
 * ---------------------------------------------------------------------------------------- */
void cbo_interleave_indices(unsigned size, unsigned num_chunks, unsigned partitions, unsigned* idx)
{
    unsigned n = 0;
    if (num_chunks == 0) { for (unsigned i = 0; i < size; ++i) idx[i] = i; return; }
    unsigned partition_size = size / partitions;
    for (unsigned part = 0; part < size; part += partition_size)
        for (unsigned chunk = 0; chunk < num_chunks; ++chunk)
            for (unsigned i = chunk; i < partition_size; i += num_chunks)
                idx[n++] = i + part;
}
void cbo_interleave_reverse(unsigned size, unsigned num_chunks, unsigned partitions, unsigned* inv)
{
    unsigned* idx = (unsigned*)malloc(sizeof(unsigned) * size);
    cbo_interleave_indices(size, num_chunks, partitions, idx);
    memset(inv, 0, sizeof(unsigned) * size);
    for (unsigned src = 0; src < size; ++src) inv[idx[src]] = src;
    free(idx);
}

/* ------------------------------------------------------------------------------------------
 * P1 preprocessSymbolGrid -- CimbReader.cpp:30-46.  OpenCV is a third-party dependency whose
 * source is not under /root/reference; arithmetic pinned against cv2 4.13 (tests/golden/make_fixtures.py):
 *   cvtColor(RGB2GRAY)  == (9798 R + 19235 G + 3735 B + 16384) >> 15
 *   adaptiveThreshold(MEAN_C, BINARY, bs, C=0) == gray > round(boxsum / bs^2), BORDER_REPLICATE
 *   filter2D(3x3 float kernel) == saturate(round_half_even(sum)), BORDER_REFLECT_101
 * ---------------------------------------------------------------------------------------- */
void cbo_rgb_to_gray(const uint8_t* rgb, int w, int h, uint8_t* gray)
{
    size_t n = (size_t)w * h;
    for (size_t i = 0; i < n; ++i) {
        unsigned r = rgb[3 * i], g = rgb[3 * i + 1], b = rgb[3 * i + 2];
        gray[i] = (uint8_t)((9798u * r + 19235u * g + 3735u * b + 16384u) >> 15);
    }
}

static int reflect101(int p, int n)
{
    if (n == 1) return 0;
    while (p < 0 || p >= n) { if (p < 0) p = -p; else p = 2 * n - 2 - p; }
    return p;
}

void cbo_sharpen(const uint8_t* gray, int w, int h, uint8_t* out)
{
    /* kernel (CimbReader.cpp:17-21): [0 -1 0; -1 4.5 -1; 0 -1 0]; all partial sums are multiples
       of 0.5 below 2^11, hence exact in float32 in any order; saturate_cast<uchar>(float) = cvRound
       = round-half-to-even. 2*v = 9*c - 2*(n+s+e+w) is an integer: round-half-even on that. */
    for (int y = 0; y < h; ++y) {
        int yu = reflect101(y - 1, h), yd = reflect101(y + 1, h);
        for (int x = 0; x < w; ++x) {
            int xl = reflect101(x - 1, w), xr = reflect101(x + 1, w);
            int c = gray[(size_t)y * w + x];
            int nb = gray[(size_t)yu * w + x] + gray[(size_t)yd * w + x] + gray[(size_t)y * w + xl] + gray[(size_t)y * w + xr];
            int twice = 9 * c - 2 * nb;       /* = 2 * value */
            int v;
            if (twice & 1) {                  /* value = k + 0.5 -> nearest even */
                int k = (twice - 1) / 2;      /* twice-1 is even: exact, also for negatives */
                v = (k & 1) ? k + 1 : k;
            } else {
                v = twice / 2;
            }
            if (v < 0) v = 0;
            if (v > 255) v = 255;
            out[(size_t)y * w + x] = (uint8_t)v;
        }
    }
}

void cbo_adaptive_threshold(const uint8_t* gray, int w, int h, int block, uint8_t* out)
{
    /* separable box sum with replicate border (boxFilter BORDER_REPLICATE inside cv::adaptiveThreshold), done with
       running sums: a ring of `block` rows of horizontal sums and one array of column sums */
    int r = block / 2;
    unsigned area = (unsigned)(block * block);
    uint16_t* ring = (uint16_t*)malloc(sizeof(uint16_t) * (size_t)w * (size_t)block);
    uint32_t* col = (uint32_t*)calloc((size_t)w, sizeof(uint32_t));
    /* horizontal sums of row yy (clamped) into ring slot */
#define HROW(dst, yy) do { \
        const uint8_t* row_ = gray + (size_t)(yy) * w; uint16_t* d_ = (dst); \
        unsigned s_ = 0; \
        for (int d = -r; d <= r; ++d) { int xx = d < 0 ? 0 : (d >= w ? w - 1 : d); s_ += row_[xx]; } \
        d_[0] = (uint16_t)s_; \
        for (int x = 1; x < w; ++x) { \
            int xin = x + r; if (xin >= w) xin = w - 1; \
            int xout = x - r - 1; if (xout < 0) xout = 0; \
            s_ += row_[xin]; s_ -= row_[xout]; d_[x] = (uint16_t)s_; } \
    } while (0)
    /* prime: rows -r..r (clamped) */
    for (int d = -r; d <= r; ++d) {
        int yy = d < 0 ? 0 : (d >= h ? h - 1 : d);
        uint16_t* slot = ring + (size_t)((d + r) % block) * w;
        HROW(slot, yy);
        for (int x = 0; x < w; ++x) col[x] += slot[x];
    }
    int next_slot = 0;   /* slot holding the oldest row (y - r) */
    for (int y = 0; y < h; ++y) {
        const uint8_t* g = gray + (size_t)y * w;
        uint8_t* o = out + (size_t)y * w;
        for (int x = 0; x < w; ++x) {
            unsigned mean = (2 * col[x] + area) / (2u * area);  /* round to nearest (never a tie: area odd) */
            o[x] = (g[x] > mean) ? 255 : 0;
        }
        if (y + 1 < h) {   /* slide: drop row (y - r) clamped, add row (y + 1 + r) clamped */
            uint16_t* slot = ring + (size_t)next_slot * w;
            for (int x = 0; x < w; ++x) col[x] -= slot[x];
            int yin = y + 1 + r; if (yin >= h) yin = h - 1;
            HROW(slot, yin);
            for (int x = 0; x < w; ++x) col[x] += slot[x];
            next_slot = (next_slot + 1) % block;
        }
    }
#undef HROW
    free(ring); free(col);
}

void cbo_pack_bits(const uint8_t* thr, size_t npix, uint8_t* bits)
{
    /* bitmatrix.h:14-46 -- LSB of each byte, first pixel in the MSB */
    size_t nbytes = npix / 8;
    for (size_t i = 0; i < nbytes; ++i) {
        uint8_t v = 0;
        for (int k = 0; k < 8; ++k) v |= (uint8_t)((thr[8 * i + k] & 1) << (7 - k));
        bits[i] = v;
    }
    size_t rem = npix - nbytes * 8;
    if (rem) {  /* bitmatrix.h:35-45 remainder quirk: val |= (p>0) << size, size counting down */
        uint8_t v = 0; size_t size = rem; const uint8_t* p = thr + nbytes * 8;
        while (size > 0) { v |= (uint8_t)((*p > 0) << size); ++p; --size; }
        bits[nbytes] = v;
    }
}

/* The same preprocessing as the four functions above, fused row by row for speed (the CPU arm of the benchmark should
   not be slower than OpenCV's SIMD passes by construction): gray into a padded row, horizontal box sums as 2r+1 shifted
   adds (vectorisable), a ring of the last 2r+1 rows of horizontal sums with one running column sum, the threshold in its
   integer form  area * g > colsum + (area-1)/2  (== g > round(colsum / area): area is odd, so there is no tie), and the
   MSB-first bit pack eight pixels at a time.  tests/test_oracle_goldens.py asserts this equals the unfused restatement
   (which is what is pinned against cv2) on camera frames, synthetic frames and noise. */
static void gray_row(const uint8_t* rgb, int w, uint8_t* out)
{
    for (int x = 0; x < w; ++x)
        out[x] = (uint8_t)((9798u * rgb[3 * x] + 19235u * rgb[3 * x + 1] + 3735u * rgb[3 * x + 2] + 16384u) >> 15);
}

void cbo_threshold_bits_fast(const uint8_t* gray, int w, int h, int block, uint8_t* bits)
{
    const int r = block / 2;
    const unsigned area = (unsigned)(block * block), half = (area - 1) / 2;
    const int pw = w + 2 * r;
    uint8_t* pad = (uint8_t*)malloc((size_t)pw + 16);
    uint16_t* ring = (uint16_t*)malloc(sizeof(uint16_t) * (size_t)w * (size_t)block);
    uint16_t* col = (uint16_t*)calloc((size_t)w, sizeof(uint16_t));      /* <= 49 * 255 */
    uint8_t* thr = (uint8_t*)malloc((size_t)w + 8);
#define HROW_FAST(dst, yy) do { \
        const uint8_t* row_ = gray + (size_t)(yy) * w; uint16_t* d_ = (dst); \
        memcpy(pad + r, row_, (size_t)w); \
        for (int k_ = 0; k_ < r; ++k_) { pad[k_] = row_[0]; pad[r + w + k_] = row_[w - 1]; } \
        for (int x = 0; x < w; ++x) d_[x] = 0; \
        for (int d = 0; d < block; ++d) { const uint8_t* p_ = pad + d; for (int x = 0; x < w; ++x) d_[x] = (uint16_t)(d_[x] + p_[x]); } \
    } while (0)
    for (int d = -r; d <= r; ++d) {
        int yy = d < 0 ? 0 : (d >= h ? h - 1 : d);
        uint16_t* slot = ring + (size_t)((d + r) % block) * w;
        HROW_FAST(slot, yy);
        for (int x = 0; x < w; ++x) col[x] = (uint16_t)(col[x] + slot[x]);
    }
    int next_slot = 0;
    size_t bitpos = 0;                       /* rows are packed back to back (bitmatrix over the continuous Mat) */
    uint8_t carry = 0; int carry_n = 0;      /* w need not be a multiple of 8 in general; every mode's width is */
    for (int y = 0; y < h; ++y) {
        const uint8_t* g = gray + (size_t)y * w;
        for (int x = 0; x < w; ++x) thr[x] = (uint8_t)(area * g[x] > (unsigned)col[x] + half);
        int x = 0;
        if (carry_n == 0) {
            for (; x + 8 <= w; x += 8) {
                uint64_t v; memcpy(&v, thr + x, 8);
                bits[bitpos >> 3] = (uint8_t)((v * 0x8040201008040201ULL) >> 56);     /* byte k (0/1) -> bit 7-k */
                bitpos += 8;
            }
        }
        for (; x < w; ++x) {                 /* generic tail */
            carry = (uint8_t)((carry << 1) | thr[x]); ++carry_n; ++bitpos;
            if (carry_n == 8) { bits[(bitpos >> 3) - 1] = carry; carry = 0; carry_n = 0; }
        }
        if (y + 1 < h) {
            uint16_t* slot = ring + (size_t)next_slot * w;
            for (int xx = 0; xx < w; ++xx) col[xx] = (uint16_t)(col[xx] - slot[xx]);
            int yin = y + 1 + r; if (yin >= h) yin = h - 1;
            HROW_FAST(slot, yin);
            for (int xx = 0; xx < w; ++xx) col[xx] = (uint16_t)(col[xx] + slot[xx]);
            next_slot = (next_slot + 1) % block;
        }
    }
#undef HROW_FAST
    if (carry_n) {   /* bitmatrix.h:35-45 remainder quirk: val |= (p>0) << size, size counting down from rem */
        uint8_t v = 0; int rem = carry_n;
        for (int k = 0; k < rem; ++k) v |= (uint8_t)(((carry >> (rem - 1 - k)) & 1) << (rem - k));
        bits[bitpos >> 3] = v;
    }
    free(pad); free(ring); free(col); free(thr);
}

void cbo_preprocess(const uint8_t* rgb, int w, int h, int needs_sharpen, uint8_t* bits)
{
    size_t n = (size_t)w * h;
    uint8_t* gray = (uint8_t*)malloc(n);
    for (int y = 0; y < h; ++y) gray_row(rgb + (size_t)y * w * 3, w, gray + (size_t)y * w);
    int block = 5;
    if (needs_sharpen) {
        uint8_t* sh = (uint8_t*)malloc(n);
        cbo_sharpen(gray, w, h, sh);
        free(gray);
        gray = sh;
        block = 7;
    }
    cbo_threshold_bits_fast(gray, w, h, block, bits);
    free(gray);
}

/* the unfused form (cvtColor -> [filter2D] -> adaptiveThreshold -> mat_to_bitbuffer as separate passes) */
void cbo_preprocess_unfused(const uint8_t* rgb, int w, int h, int needs_sharpen, uint8_t* bits)
{
    size_t n = (size_t)w * h;
    uint8_t* gray = (uint8_t*)malloc(n);
    uint8_t* thr = (uint8_t*)malloc(n);
    cbo_rgb_to_gray(rgb, w, h, gray);
    int block = 5;
    if (needs_sharpen) {
        uint8_t* sh = (uint8_t*)malloc(n);
        cbo_sharpen(gray, w, h, sh);
        memcpy(gray, sh, n);
        free(sh);
        block = 7;
    }
    cbo_adaptive_threshold(gray, w, h, block, thr);
    cbo_pack_bits(thr, n, bits);
    free(gray); free(thr);
}

/* ------------------------------------------------------------------------------------------
 * bitbuffer::read / write -- bit_file/bitbuffer.h:62-107 (MSB-first)
 * ---------------------------------------------------------------------------------------- */
static unsigned bb_read(const uint8_t* buf, unsigned index, int length)
{
    int cur_byte = (int)(index / 8), cur_bit = (int)(index % 8);
    unsigned res = 0;
    int next = length < 8 - cur_bit ? length : 8 - cur_bit;
    while (length > 0) {
        unsigned char bits = (unsigned char)(buf[cur_byte] << cur_bit);
        bits = (unsigned char)(bits >> (8 - next));
        res |= (unsigned)bits << (length - next);
        length -= next; cur_bit += next; if (cur_bit >= 8) cur_bit = 0;
        cur_byte += 1;
        next = length < 8 - cur_bit ? length : 8 - cur_bit;
    }
    return res;
}
static void bb_write(uint8_t* buf, unsigned data, unsigned index, int length)
{
    int cur_byte = (int)(index / 8), cur_bit = (int)(index % 8);
    int next = length < 8 - cur_bit ? length : 8 - cur_bit;
    while (length > 0 && next > 0) {
        unsigned char bits = (unsigned char)(data >> (length - next));
        bits = (unsigned char)(bits << (8 - next - cur_bit));
        buf[cur_byte] |= bits;
        length -= next; cur_bit += next; if (cur_bit >= 8) cur_bit = 0;
        cur_byte += 1;
        next = length < 8 - cur_bit ? length : 8 - cur_bit;
    }
}

/* ------------------------------------------------------------------------------------------
 * P5 fuzzy_ahash<8>(bitmatrix) -- average_hash.h:63-75; ahash_result.h:70-106; bit_extractor.h:23-50
 * 10 rows of 10 bits -> 100-bit value, row 0 most significant; hash[id] takes, for k=0..7,
 * the 8 bits at offset (id%3 + (id/3)*10 + 10k) from the top: window row id/3+k, cols id%3..+7.
 * ---------------------------------------------------------------------------------------- */
void cbo_fuzzy_ahash(const uint8_t* bits, int w, int wx, int wy, int all, uint64_t hashes[9])
{
    unsigned rows[10];
    for (int i = 0; i < 10; ++i)
        rows[i] = bb_read(bits, (unsigned)wx + (unsigned)(wy + i) * (unsigned)w, 10);
    for (int id = 0; id < 9; ++id) {
        if (!all && (id == 0 || id == 2 || id == 6 || id == 8)) { hashes[id] = 0; continue; }
        int r0 = id / 3, c0 = id % 3;
        uint64_t h = 0;
        for (int k = 0; k < 8; ++k) {
            unsigned byte = (rows[r0 + k] >> (10 - c0 - 8)) & 0xFFu;
            h = (h << 8) | byte;
        }
        hashes[id] = h;
    }
}

/* tile dictionary = CimbDecoder::_tileHashes (CimbDecoder.cpp:87-99) for symbol_bits=4, dark; dumped from
   /root/reference/bitmap/4/ (the sixteen .png tiles; non-white pixel = 1) and cross-checked with averageHashTest.cpp:43-50 */
static const uint64_t TILE_HASHES[16] = {
    0xfffefcf8f0e0c080ULL, 0x80c0e0f0f8fcfeffULL, 0xff7f3f1f0f070301ULL, 0x0103070f1f3f7fffULL,
    0x181818ffff181818ULL, 0x66e7e70000e7e766ULL, 0x3c7ee7c3c3e77e3cULL, 0x18183c3c7e7effffULL,
    0xc0f0fcfffffcf0c0ULL, 0xfffcf00000f0fcffULL, 0xff3f0f00000f3fffULL, 0xe7e7e7e7c3c38181ULL,
    0x8181c3c3e7e7e7e7ULL, 0x0000c3e77e3c1800ULL, 0x0c1c387070381c0cULL, 0x1e1e38381c1c7878ULL,
};
const uint64_t* cbo_tile_hashes(void) { return TILE_HASHES; }

static unsigned popcnt64(uint64_t v) { return (unsigned)__builtin_popcountll(v); }

/* P6 CimbDecoder::get_best_symbol -- CimbDecoder.cpp:101-132 (order from ahash_result.h:26) */
unsigned cbo_best_symbol(const uint64_t hashes[9], int all, unsigned num_symbols, unsigned cooldown,
                         unsigned* drift_offset, unsigned* best_distance)
{
    static const unsigned ORDER[9] = {4, 5, 7, 3, 1, 8, 0, 2, 6};
    unsigned n = all ? 9 : 5;
    unsigned best_fit = 0;
    *drift_offset = 0;
    *best_distance = 1000;
    for (unsigned o = 0; o < n; ++o) {
        unsigned id = ORDER[o];
        if (id == cooldown && id != 4) continue;
        for (unsigned i = 0; i < num_symbols; ++i) {
            unsigned d = popcnt64(hashes[id] ^ TILE_HASHES[i]);
            if (d < *best_distance) {
                *best_distance = d; best_fit = i; *drift_offset = id;
                if (d == 0) return best_fit;
            }
        }
    }
    return best_fit;
}

/* ------------------------------------------------------------------------------------------
 * P8/P9 colour -- Cell.h:30-62, CimbDecoder.cpp:27-55, :168-217, Common.cpp:21-139
 * ---------------------------------------------------------------------------------------- */
void cbo_palette(unsigned index, unsigned num_colors, unsigned color_mode, uint8_t rgb[3])
{
    static const uint8_t c4[4][3] = {{0, 255, 0}, {0, 255, 255}, {255, 255, 0}, {255, 0, 255}};          /* Common.cpp:21-32 */
    static const uint8_t c4enc[4][3] = {{0, 255, 0}, {0, 255, 255}, {255, 255, 0}, {255, 0x55, 255}};    /* :34-44 */
    static const uint8_t c4old[4][3] = {{0, 255, 255}, {255, 255, 0}, {255, 0, 255}, {0, 255, 0}};       /* :46-55 */
    static const uint8_t c8[8][3] = {{0, 255, 255}, {255, 255, 0}, {0x7F, 0x7F, 255}, {255, 255, 255},
                                     {0, 255, 0}, {255, 0x9F, 0}, {255, 0, 255}, {255, 65, 65}};           /* :57-70 */
    static const uint8_t c8old[8][3] = {{0, 255, 255}, {0x7F, 0x7F, 255}, {255, 0, 255}, {255, 65, 65},
                                        {255, 0x9F, 0}, {255, 255, 0}, {255, 255, 255}, {0, 255, 0}};      /* :72-85 */
    const uint8_t* p;
    if ((color_mode & 0xFF) == 0) p = (num_colors <= 4) ? c4old[index & 3] : c8old[index & 7];           /* :122-139 */
    else if (num_colors > 4) p = c8[index & 7];
    else if (color_mode > 0x100) p = c4enc[index & 3];
    else p = c4[index & 3];
    rgb[0] = p[0]; rgb[1] = p[1]; rgb[2] = p[2];
}

void cbo_avg_color(const uint8_t* rgb, int w, int x, int y, int cell_size, uint8_t out[3])
{
    /* avg_color: crop(1,1,cols-2,rows-2) then mean_rgb_continuous (uint16 sums, integer divide) */
    int xs = x + 1, ys = y + 1, n = cell_size - 2;
    uint16_t r = 0, g = 0, b = 0, count = 0;
    for (int i = 0; i < n; ++i) {
        const uint8_t* p = rgb + ((size_t)(ys + i) * w + xs) * 3;
        for (int j = 0; j < n; ++j, ++count, p += 3) { r += p[0]; g += p[1]; b += p[2]; }
    }
    if (!count) { out[0] = out[1] = out[2] = 0; return; }
    out[0] = (uint8_t)(r / count); out[1] = (uint8_t)(g / count); out[2] = (uint8_t)(b / count);
}

static uint8_t fix_single_color(float c, float adjust_up, float down)
{
    /* CimbDecoder.cpp:27-36 */
    c -= down;
    c *= adjust_up;
    if (c > (245 - down)) c = 255;
    if (c < 0) c = 0;
    return (uint8_t)c;
}

static unsigned color_diff(const uint8_t a[3], const uint8_t b[3])
{
    /* CimbDecoder.cpp:38-55: differences of (r-g, g-b, b-r) */
    int a0 = a[0] - a[1], a1 = a[1] - a[2], a2 = a[2] - a[0];
    int b0 = b[0] - b[1], b1 = b[1] - b[2], b2 = b[2] - b[0];
    return (unsigned)((a0 - b0) * (a0 - b0) + (a1 - b1) * (a1 - b1) + (a2 - b2) * (a2 - b2));
}

unsigned cbo_best_color(float r, float g, float b, unsigned num_colors, unsigned color_mode, const float* ccm)
{
    /* CimbDecoder.cpp:168-200 */
    if (ccm) {  /* color_correction::transform, chromatic_adaptation/color_correction.h:64-68: m * (r,g,b) */
        float rr = ccm[0] * r + ccm[1] * g + ccm[2] * b;
        float gg = ccm[3] * r + ccm[4] * g + ccm[5] * b;
        float bb = ccm[6] * r + ccm[7] * g + ccm[8] * b;
        r = rr; g = gg; b = bb;
    }
    float max = r; if (g > max) max = g; if (b > max) max = b; if (1.0f > max) max = 1.0f;
    float min = r; if (g < min) min = g; if (b < min) min = b; if (48.0f < min) min = 48.0f;
    if (min >= max) min = 0;
    float adjust = (float)(255.0 / (double)(max - min));
    uint8_t c[3];
    c[0] = fix_single_color(r, adjust, min);
    c[1] = fix_single_color(g, adjust, min);
    c[2] = fix_single_color(b, adjust, min);

    unsigned best_fit = 0;
    float best_distance = 1000000;
    for (unsigned i = 0; i < num_colors; ++i) {
        uint8_t cand[3];
        cbo_palette(i, num_colors, color_mode, cand);
        unsigned d = color_diff(c, cand);
        if ((float)d < best_distance) { best_fit = i; best_distance = (float)d; }
    }
    return best_fit;
}

void cbo_best_colors(const uint8_t* means, int n, unsigned num_colors, unsigned color_mode, const float* ccm, uint8_t* out)
{
    for (int i = 0; i < n; ++i)
        out[i] = (uint8_t)cbo_best_color((float)means[3 * i], (float)means[3 * i + 1], (float)means[3 * i + 2], num_colors, color_mode, ccm);
}

/* CimbDecoder's thread_local color_correction (CimbDecoder.cpp:69-85): set by update_color_correction, used by every
   get_best_color until replaced.  NULL deactivates it (TestableCimbDecoder::internal_ccm() = color_correction()). */
static __thread float g_ccm[9];
static __thread int g_ccm_active = 0;
void cbo_set_ccm(const float* m9)
{
    g_ccm_active = m9 != NULL;
    if (m9) memcpy(g_ccm, m9, sizeof(g_ccm));
}
int cbo_get_ccm(float* m9) { if (g_ccm_active && m9) memcpy(m9, g_ccm, sizeof(g_ccm)); return g_ccm_active; }

/* cv::Matx<float,3,3> * cv::Matx<float,3,3> (opencv2/core/matx.hpp Matx_MatMulOp: s = 0; s += a(i,k) * b(k,j), k ascending) */
static void matx33_mul(const float* a, const float* b, float* out)
{
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            float s = 0;
            for (int k = 0; k < 3; ++k) s += a[3 * i + k] * b[3 * k + j];
            out[3 * i + j] = s;
        }
}
/* cv::Matx<float,3,3>::inv() (DECOMP_LU default -> the closed-form 3x3 operator of opencv2/core/operations.hpp:
   determinant in float, d = 1 / d, cofactors * d) */
static int matx33_inv(const float* a, float* b)
{
    float d = a[0] * (a[4] * a[8] - a[7] * a[5]) - a[1] * (a[3] * a[8] - a[6] * a[5]) + a[2] * (a[3] * a[7] - a[6] * a[4]);
    if (d == 0) return 0;
    d = 1 / d;
    b[0] = (a[4] * a[8] - a[5] * a[7]) * d; b[1] = (a[2] * a[7] - a[1] * a[8]) * d; b[2] = (a[1] * a[5] - a[2] * a[4]) * d;
    b[3] = (a[5] * a[6] - a[3] * a[8]) * d; b[4] = (a[0] * a[8] - a[2] * a[6]) * d; b[5] = (a[2] * a[3] - a[0] * a[5]) * d;
    b[6] = (a[3] * a[7] - a[4] * a[6]) * d; b[7] = (a[1] * a[6] - a[0] * a[7]) * d; b[8] = (a[0] * a[4] - a[1] * a[3]) * d;
    return 1;
}
/* color_correction::get_adaptation_matrix<von_kries>(actual, desired), chromatic_adaptation/color_correction.h:12-24,
   von Kries transform adaptation_transform.h:22-33: T.inv() * diag((T*desired) / (T*actual)) * T */
void cbo_adaptation_matrix(const float actual[3], const float desired[3], float out[9])
{
    static const float T[9] = {0.4002400f, 0.7076000f, -0.0808100f, -0.2263000f, 1.1653200f, 0.0457000f, 0.0000000f, 0.0000000f, 0.9182200f};
    float m1[3], m2[3], d[9] = {0}, ti[9], tmp[9];
    for (int i = 0; i < 3; ++i) {
        float s1 = 0, s2 = 0;
        for (int k = 0; k < 3; ++k) { s1 += T[3 * i + k] * actual[k]; s2 += T[3 * i + k] * desired[k]; }
        m1[i] = s1; m2[i] = s2;
    }
    for (int i = 0; i < 3; ++i) d[4 * i] = m2[i] / m1[i];
    if (!matx33_inv(T, ti)) memset(ti, 0, sizeof(ti));
    matx33_mul(ti, d, tmp);
    matx33_mul(tmp, T, out);
}
/* calculateWhite (dark) + simpleColorCorrection, CimbReader.cpp:55-93: max over three anchor 4x4 means, floor (1,1,1) */
void cbo_simple_ccm(const cbo_mode* m, const uint8_t* rgb, int w, int h, float out[9])
{
    int padding = ((w - (int)m->image_size_x) < (h - (int)m->image_size_y) ? (w - (int)m->image_size_x) : (h - (int)m->image_size_y)) / 2;
    unsigned tl = 30 + (unsigned)padding - 2;                                    /* Config::anchor_size() == 30 */
    unsigned right = m->image_size_x + (unsigned)padding - 30 - 2, bottom = m->image_size_y + (unsigned)padding - 30 - 2;
    unsigned ax[3] = {tl, tl, right}, ay[3] = {tl, bottom, tl};
    float white[3] = {1, 1, 1};
    for (int a = 0; a < 3; ++a) {
        double sum[3] = {0, 0, 0};
        for (unsigned y = 0; y < 4; ++y)
            for (unsigned x = 0; x < 4; ++x)
                for (int c = 0; c < 3; ++c) sum[c] += rgb[((size_t)(ay[a] + y) * (size_t)w + (ax[a] + x)) * 3 + c];
        for (int c = 0; c < 3; ++c) { float v = (float)(sum[c] / 16.0); if (v > white[c]) white[c] = v; }   /* cv::mean -> double */
    }
    const float desired[3] = {255.0f, 255.0f, 255.0f};
    cbo_adaptation_matrix(white, desired, out);
}

/* color_correction::get_moore_penrose_lsm(actual, desired), color_correction.h:26-39: x = desired^T, y = actual^T,
   z = cv::invert(y, DECOMP_SVD), result = x * z.  rows = N (5 or 9), row-major N x 3 floats.
   cv::invert(DECOMP_SVD) on the 3 x N float matrix y (OpenCV modules/core/src/lapack.cpp, the build without LAPACK that the
   reference's printed goldens come from): SVD::compute -> _SVDcompute (m < n: works on the rows of y as they are) ->
   JacobiSVDImpl_<float> (one-sided Hestenes rotations, dot products and norms in double, c/s and the rotated values in
   float, eps = 2 FLT_EPSILON, at most max(m, 30) sweeps, singular values sorted descending, rows normalised by 1 / w),
   then SVD::backSubst -> SVBkSbImpl_ (x += v_i * (u_i / w_i)^T, products and sums in double, stored as float after every
   i), then the 3 x N by N x 3 product through cv::gemm (double accumulators).  Reproduces the matrix strings of
   color_correctionTest.cpp:32-84 digit for digit (tests/test_oracle_goldens.py). */
static void jacobi_svd_f32(float* At, int astep, float* Wout, float* Vt, int m, int n)
{
    double W[16];
    const float eps = FLT_EPSILON * 2;
    for (int i = 0; i < n; ++i) {
        double sd = 0;
        for (int k = 0; k < m; ++k) { float t = At[i * astep + k]; sd += (double)t * t; }
        W[i] = sd;
        for (int k = 0; k < n; ++k) Vt[i * n + k] = 0;
        Vt[i * n + i] = 1;
    }
    int max_iter = m > 30 ? m : 30;
    for (int iter = 0; iter < max_iter; ++iter) {
        int changed = 0;
        for (int i = 0; i < n - 1; ++i)
            for (int j = i + 1; j < n; ++j) {
                float *Ai = At + i * astep, *Aj = At + j * astep;
                double a = W[i], p = 0, b = W[j];
                for (int k = 0; k < m; ++k) p += (double)Ai[k] * Aj[k];
                if (fabs(p) <= eps * sqrt((double)a * b)) continue;
                p *= 2;
                double beta = a - b, gamma = hypot((double)p, beta);
                float c, sn;
                if (beta < 0) { double delta = (gamma - beta) * 0.5; sn = (float)sqrt(delta / gamma); c = (float)(p / (gamma * sn * 2)); }
                else { c = (float)sqrt((gamma + beta) / (gamma * 2)); sn = (float)(p / (gamma * c * 2)); }
                a = b = 0;
                for (int k = 0; k < m; ++k) {
                    float t0 = c * Ai[k] + sn * Aj[k];
                    float t1 = -sn * Ai[k] + c * Aj[k];
                    Ai[k] = t0; Aj[k] = t1;
                    a += (double)t0 * t0; b += (double)t1 * t1;
                }
                W[i] = a; W[j] = b;
                changed = 1;
                float *Vi = Vt + i * n, *Vj = Vt + j * n;
                for (int k = 0; k < n; ++k) {
                    float t0 = c * Vi[k] + sn * Vj[k];
                    float t1 = -sn * Vi[k] + c * Vj[k];
                    Vi[k] = t0; Vj[k] = t1;
                }
            }
        if (!changed) break;
    }
    for (int i = 0; i < n; ++i) {
        double sd = 0;
        for (int k = 0; k < m; ++k) { float t = At[i * astep + k]; sd += (double)t * t; }
        W[i] = sqrt(sd);
    }
    for (int i = 0; i < n - 1; ++i) {
        int j = i;
        for (int k = i + 1; k < n; ++k) if (W[j] < W[k]) j = k;
        if (i != j) {
            double tw = W[i]; W[i] = W[j]; W[j] = tw;
            for (int k = 0; k < m; ++k) { float t = At[i * astep + k]; At[i * astep + k] = At[j * astep + k]; At[j * astep + k] = t; }
            for (int k = 0; k < n; ++k) { float t = Vt[i * n + k]; Vt[i * n + k] = Vt[j * n + k]; Vt[j * n + k] = t; }
        }
    }
    for (int i = 0; i < n; ++i) Wout[i] = (float)W[i];
    for (int i = 0; i < n; ++i) {
        /* OpenCV gives a singular value <= FLT_MIN a random unit vector from cv::RNG(0x12345678) as its column of vt.  Grey
           or equal rows do reach it (W = 0 exactly), but the result cannot depend on that vector: backSubst drops every
           w <= threshold = sum(W) * 2^-51, and sum(W) >= |white| >= sqrt(3) (calculateWhite's floor of 1 per channel), so the
           threshold is far above FLT_MIN and the column is never used.  A zero column stands in for it here. */
        double sd = W[i];
        float s = (float)(sd > (double)FLT_MIN ? 1 / sd : 0.);
        for (int k = 0; k < m; ++k) At[i * astep + k] *= s;
    }
}
int cbo_moore_penrose_lsm(const float* actual, const float* desired, int rows, float out[9])
{
    if (rows < 3 || rows > 16) return 0;
    const int N = rows;
    float At[3 * 16], Vt[9], W[3];
    for (int r = 0; r < 3; ++r) for (int k = 0; k < N; ++k) At[r * 16 + k] = actual[k * 3 + r];    /* y = actual^T, 3 x N */
    jacobi_svd_f32(At, 16, W, Vt, N, 3);
    /* SVD of y: u = Vt^T (3 x 3), vt = At (3 x N).  backSubst with no rhs: z (N x 3) = sum_i vt_i^T * (u column i / w_i) */
    float z[16 * 3];
    for (int i = 0; i < N * 3; ++i) z[i] = 0;
    /* SVBkSb's threshold for the float SVD is sum(W) * (float)(DBL_EPSILON * 2) = sum(W) * 2^-51, not FLT_EPSILON's: on grey or
       rank-2 colour rows the Jacobi sweeps leave a residual singular value of ~1e-8 sum(W) that OpenCV inverts (fits of 1e6..1e9) */
    double threshold = 0;
    for (int i = 0; i < 3; ++i) threshold += W[i];
    threshold *= (float)(DBL_EPSILON * 2);
    for (int i = 0; i < 3; ++i) {
        double wi = W[i];
        if (fabs(wi) <= threshold) continue;
        wi = 1 / wi;
        double buffer[3];
        for (int j = 0; j < 3; ++j) buffer[j] = Vt[i * 3 + j] * wi;         /* u(j, i) = Vt(i, j) */
        for (int r = 0; r < N; ++r) {
            float sv = At[i * 16 + r];
            for (int j = 0; j < 3; ++j) z[r * 3 + j] = (float)(z[r * 3 + j] + sv * buffer[j]);
        }
    }
    for (int i = 0; i < 3; ++i)                                             /* x (3 x N) * z (N x 3), x = desired^T */
        for (int j = 0; j < 3; ++j) {
            double acc = 0;
            for (int k = 0; k < N; ++k) acc += (double)desired[k * 3 + i] * z[k * 3 + j];
            out[i * 3 + j] = (float)acc;
        }
    return 1;
}

/* What the aligned_stream callbacks leave in CimbReader::_fountainColorHeader after the symbol stream
   (Decoder.h:171-189, aligned_stream.h:39-116, CimbReader::update_metadata CimbReader.cpp:269-280): the first six bytes
   of the first good chunk, block id incremented once per chunk event from that chunk on (skipping the "radioactive" id).
   blocks/ok = the symbol stream's RS results.  Returns 0 when no header was seen (id() == 0). */
static void md_event(uint8_t hdr[6], int* have, unsigned* radioactive, const uint8_t* buf, unsigned len, unsigned chunk_size)
{   /* CimbReader::update_metadata(buff, len, chunk_size), CimbReader.cpp:269-280 */
    int id_zero = (hdr[0] | hdr[1] | hdr[2] | hdr[3]) == 0;
    if (len == 0 && id_zero) return;
    if (id_zero && buf) { memcpy(hdr, buf, len > 6 ? 6 : len); *have = 1; }
    if (*radioactive == 0) { unsigned fs = cbo_md_file_size(hdr); *radioactive = (fs % chunk_size == 0) ? 0xFFFFFFFFu : fs / chunk_size; }
    unsigned next = cbo_md_block_id(hdr) + 1;
    if (next == *radioactive) next += 1;
    hdr[4] = (uint8_t)((next >> 8) & 0xFF); hdr[5] = (uint8_t)(next & 0xFF);
}

int cbo_header_after_symbols(const uint8_t* blocks, const uint8_t* ok, unsigned nblocks, unsigned msg_len, unsigned chunk_size,
                             uint8_t hdr[6], unsigned* radioactive_out)
{
    uint8_t* buffer = (uint8_t*)calloc(chunk_size, 1);
    unsigned offset = 0, radioactive = 0; int bad_chunk = 0, have = 0;
    memset(hdr, 0, 6);
    for (unsigned b = 0; b < nblocks; ++b) {
        const uint8_t* data = blocks + (size_t)b * msg_len;
        if (!ok[b]) { bad_chunk = 1; offset = (offset + msg_len) % chunk_size; continue; }
        unsigned length = msg_len;
        while (length > 0) {
            unsigned work = length + offset;
            if (work >= chunk_size) {
                unsigned write_len = chunk_size - offset;
                if (bad_chunk) { bad_chunk = 0; offset = 0; md_event(hdr, &have, &radioactive, NULL, 0, chunk_size); }
                else { memcpy(buffer + offset, data, write_len); offset += write_len; md_event(hdr, &have, &radioactive, buffer, offset, chunk_size); offset = 0; }
                length -= write_len; data += write_len;
                continue;
            }
            memcpy(buffer + offset, data, length);
            offset += length; length = 0;
        }
    }
    free(buffer);
    if (radioactive_out) *radioactive_out = radioactive;
    return have && (hdr[0] | hdr[1] | hdr[2] | hdr[3]) != 0;
}

/* CimbReader::init_ccm, CimbReader.cpp:169-267 (color_correction == 2): colours the header predicts at the head of every
   colour-stream chunk -> per-colour average of the observed cell means -> + anchor white -> least-squares 3x3 fit.
   hdr/radioactive as left by the symbol pass.  Returns 1 and fills out when a matrix results, 0 when the reference bails. */
static __thread float g_fit_actual[16 * 3], g_fit_desired[16 * 3];
static __thread int g_fit_rows = 0;
int cbo_last_fit_rows(float* actual, float* desired)
{
    memcpy(actual, g_fit_actual, sizeof(float) * 3 * (size_t)g_fit_rows);
    memcpy(desired, g_fit_desired, sizeof(float) * 3 * (size_t)g_fit_rows);
    return g_fit_rows;
}
int cbo_init_ccm(const cbo_mode* m, const uint8_t* rgb, int w, int h, const uint8_t hdr_in[6], unsigned radioactive, float out[9])
{
    if ((hdr_in[0] | hdr_in[1] | hdr_in[2] | hdr_in[3]) == 0) return 0;
    unsigned ncells = m->total_cells, color_bits = m->color_bits;
    if (color_bits == 0) return 0;
    int padding = ((w - (int)m->image_size_x) < (h - (int)m->image_size_y) ? (w - (int)m->image_size_x) : (h - (int)m->image_size_y)) / 2;
    int* xs = (int*)malloc(sizeof(int) * ncells); int* ys = (int*)malloc(sizeof(int) * ncells);
    unsigned* idx = (unsigned*)malloc(sizeof(unsigned) * ncells);
    cbo_cell_positions(m, padding, xs, ys);
    cbo_interleave_indices(ncells, m->interleave_blocks, m->interleave_partitions, idx);
    unsigned fountain_blocks = m->chunks_per_frame;
    unsigned end = cbo_capacity(m, color_bits) * 8 / color_bits;
    unsigned interval = cbo_capacity(m, m->symbol_bits + color_bits) * 8 / fountain_blocks / color_bits;
    unsigned header_len = 6 * 8 / color_bits;
    uint8_t hdr[6]; memcpy(hdr, hdr_in, 6);
    /* std::unordered_map<uint16_t, ...> of libstdc++: 13 buckets after the first insert, identity hash, every key of 0..7 in
       its own bucket, a new node goes to the front of the list -> iteration runs in reverse order of first appearance */
    unsigned order[8], norder = 0, cnt[8] = {0}, sr[8] = {0}, sg[8] = {0}, sb[8] = {0}; int seen[8] = {0};
    for (unsigned block = 0; block < end; block += interval) {
        for (unsigned s = block, i = 0; s < block + header_len; ++s, i += color_bits) {
            unsigned expected = 0;
            for (unsigned k = 0; k < color_bits; ++k) expected = (expected << 1) | ((hdr[(i + k) >> 3] >> (7 - ((i + k) & 7))) & 1u);
            unsigned cell = idx[s];
            uint8_t avg[3];
            cbo_avg_color(rgb, w, xs[cell], ys[cell], (int)m->cell_size, avg);
            if (!seen[expected]) { seen[expected] = 1; order[norder++] = expected; }
            cnt[expected] += 1; sr[expected] += avg[0]; sg[expected] += avg[1]; sb[expected] += avg[2];
        }
        unsigned next = cbo_md_block_id(hdr) + 1; if (next == radioactive) next += 1;
        hdr[4] = (uint8_t)((next >> 8) & 0xFF); hdr[5] = (uint8_t)(next & 0xFF);
    }
    free(xs); free(ys); free(idx);
    float actual[16 * 3], desired[16 * 3]; int rows = 0;
    for (int k = (int)norder - 1; k >= 0; --k) {
        unsigned c = order[k];
        if (cnt[c] == 0) continue;
        actual[rows * 3] = (float)(sr[c] / cnt[c]); actual[rows * 3 + 1] = (float)(sg[c] / cnt[c]); actual[rows * 3 + 2] = (float)(sb[c] / cnt[c]);
        uint8_t pal[3]; cbo_palette(c, 1u << color_bits, m->color_mode, pal);
        desired[rows * 3] = pal[0]; desired[rows * 3 + 1] = pal[1]; desired[rows * 3 + 2] = pal[2];
        ++rows;
    }
    if (rows < 4) return 0;
    {   /* calculateWhite, dark (CimbReader.cpp:55-72) */
        unsigned tl = 30 + (unsigned)padding - 2, right = m->image_size_x + (unsigned)padding - 30 - 2, bottom = m->image_size_y + (unsigned)padding - 30 - 2;
        unsigned ax[3] = {tl, tl, right}, ay[3] = {tl, bottom, tl};
        float white[3] = {1, 1, 1};
        for (int a = 0; a < 3; ++a) {
            double sum[3] = {0, 0, 0};
            for (unsigned y = 0; y < 4; ++y) for (unsigned x = 0; x < 4; ++x) for (int c = 0; c < 3; ++c)
                sum[c] += rgb[((size_t)(ay[a] + y) * (size_t)w + (ax[a] + x)) * 3 + c];
            for (int c = 0; c < 3; ++c) { float v = (float)(sum[c] / 16.0); if (v > white[c]) white[c] = v; }
        }
        actual[rows * 3] = white[0]; actual[rows * 3 + 1] = white[1]; actual[rows * 3 + 2] = white[2];
        desired[rows * 3] = desired[rows * 3 + 1] = desired[rows * 3 + 2] = 255.0f;
        ++rows;
    }
    g_fit_rows = rows;
    memcpy(g_fit_actual, actual, sizeof(float) * 3 * (size_t)rows);
    memcpy(g_fit_desired, desired, sizeof(float) * 3 * (size_t)rows);
    return cbo_moore_penrose_lsm(actual, desired, rows, out);
}

static unsigned decode_color_at(const cbo_mode* m, const uint8_t* rgb, int w, int x, int y)
{
    /* CimbReader::read_color (CimbReader.cpp:133-137) -> CimbDecoder::decode_color (:211-217) */
    unsigned num_colors = 1u << m->color_bits;
    if (num_colors <= 1) return 0;
    uint8_t avg[3];
    cbo_avg_color(rgb, w, x, y, (int)m->cell_size, avg);
    return cbo_best_color((float)avg[0], (float)avg[1], (float)avg[2], num_colors, m->color_mode, g_ccm_active ? g_ccm : NULL);
}

/* ------------------------------------------------------------------------------------------
 * P3 FloodDecodePositions -- FloodDecodePositions.cpp:17-134, with std::priority_queue restated as
 * libstdc++'s __push_heap/__adjust_heap (bits/stl_heap.h) so ties pop in the same order.
 * ---------------------------------------------------------------------------------------- */
typedef struct { uint16_t idx; uint8_t prio; } heap_elem;
typedef struct { heap_elem* v; int n; int cap; } heap_t;

int cbo_dbg_max_heap = 0, cbo_dbg_pushes = 0;   /* instrumentation for sizing the device heap (tests only) */
static void heap_push(heap_t* h, uint16_t idx, uint8_t prio)
{
    ++cbo_dbg_pushes;
    if (h->n + 1 > cbo_dbg_max_heap) cbo_dbg_max_heap = h->n + 1;
    if (h->n == h->cap) { h->cap *= 2; h->v = (heap_elem*)realloc(h->v, sizeof(heap_elem) * (size_t)h->cap); }
    int hole = h->n++;
    int parent = (hole - 1) / 2;
    while (hole > 0 && h->v[parent].prio > prio) {   /* comp(parent, value): parent.prio > value.prio */
        h->v[hole] = h->v[parent];
        hole = parent; parent = (hole - 1) / 2;
    }
    h->v[hole].idx = idx; h->v[hole].prio = prio;
}
static heap_elem heap_pop(heap_t* h)
{
    heap_elem top = h->v[0];
    heap_elem value = h->v[h->n - 1];
    int len = --h->n;           /* __pop_heap: len = last-1 - first */
    if (len == 0) return top;
    int hole = 0, second = 0;
    while (second < (len - 1) / 2) {
        second = 2 * (second + 1);
        if (h->v[second].prio > h->v[second - 1].prio) second--;   /* comp(right, left) -> take left */
        h->v[hole] = h->v[second];
        hole = second;
    }
    if ((len & 1) == 0 && second == (len - 2) / 2) {
        second = 2 * (second + 1);
        h->v[hole] = h->v[second - 1];
        hole = second - 1;
    }
    int parent = (hole - 1) / 2;     /* __push_heap(first, hole, top=0, value) */
    while (hole > 0 && h->v[parent].prio > value.prio) {
        h->v[hole] = h->v[parent];
        hole = parent; parent = (hole - 1) / 2;
    }
    h->v[hole] = value;
    return top;
}

typedef struct { int8_t dx, dy; uint8_t prio; uint8_t cooldown; } instr_t;

typedef struct {
    heap_t heap; uint8_t* remaining; instr_t* instr; adj_t adj; int n; int count;
} flood_t;

static void flood_update_adjacents(flood_t* f, const int adj[4], int dx, int dy, unsigned err, uint8_t cooldown)
{
    /* FloodDecodePositions.cpp:69-83 */
    for (int k = 0; k < 4; ++k) {
        int next = adj[k];
        if (next < 0 || !f->remaining[next]) continue;
        instr_t* di = &f->instr[next];
        if (di->prio <= err) continue;
        di->dx = (int8_t)dx; di->dy = (int8_t)dy; di->prio = (uint8_t)err; di->cooldown = cooldown;
        heap_push(&f->heap, (uint16_t)next, (uint8_t)err);
    }
}

static void flood_update(flood_t* f, int index, int dx, int dy, unsigned err, uint8_t cooldown)
{
    /* FloodDecodePositions.cpp:86-129 */
    int adj[4] = {adj_right(&f->adj, index), adj_left(&f->adj, index), adj_bottom(&f->adj, index), adj_top(&f->adj, index)};
    flood_update_adjacents(f, adj, dx, dy, err, cooldown);
    instr_t* self = &f->instr[index];
    if (self->prio < 3 && err < 3 && self->cooldown == 4 && cooldown == 4) {
        int rr = adj[0], ll = adj[1];
        if (rr >= 0 && ll >= 0) {
            int hz[4] = {-1, -1, -1, -1};
            hz[0] = adj_right(&f->adj, rr);
            if (hz[0] >= 0) hz[1] = adj_right(&f->adj, hz[0]);
            hz[2] = adj_left(&f->adj, ll);
            if (hz[2] >= 0) hz[3] = adj_left(&f->adj, hz[2]);
            flood_update_adjacents(f, hz, dx, dy, err, cooldown);
        }
        int uu = adj[3], dd = adj[2];
        if (uu >= 0 && dd >= 0) {
            int vt[4] = {-1, -1, -1, -1};
            vt[0] = adj_top(&f->adj, uu);
            if (vt[0] >= 0) vt[1] = adj_top(&f->adj, vt[0]);
            vt[2] = adj_bottom(&f->adj, dd);
            if (vt[2] >= 0) vt[3] = adj_bottom(&f->adj, vt[2]);
            flood_update_adjacents(f, vt, dx, dy, err, cooldown);
        }
    }
    self->prio = (uint8_t)err;
    self->cooldown = cooldown;
}

static void flood_seed(flood_t* f)
{   /* seeds: FloodDecodePositions.cpp:31-41 */
    uint16_t small_row = (uint16_t)(f->adj.dim_x - 2 * f->adj.marker_x);
    uint16_t last = (uint16_t)(f->n - 1);
    heap_push(&f->heap, 0, 0);
    heap_push(&f->heap, (uint16_t)(small_row - 1), 0);
    heap_push(&f->heap, last, 0);
    heap_push(&f->heap, (uint16_t)(last - (small_row - 1)), 0);
    uint16_t bmb = (uint16_t)f->adj.first_mid;
    heap_push(&f->heap, bmb, 1);
    heap_push(&f->heap, (uint16_t)(bmb + f->adj.dim_x - 1), 1);
    heap_push(&f->heap, (uint16_t)(last - bmb), 1);
    heap_push(&f->heap, (uint16_t)(last - (bmb + f->adj.dim_x - 1)), 1);
}

static uint8_t calculate_cooldown(uint8_t previous, uint8_t idx)
{
    /* CellDrift.cpp:34-43 */
    if (idx == 4) return 4;
    if (idx % 2 == 0) return 0xFF;
    if ((previous ^ idx) == 6) return 0xFF;
    return idx;
}

static int clamp7(int v) { if (v > 7) v = 7; if (v < -7) v = -7; return v; }  /* CellDrift.cpp:23-31 */


/* Test hook: run the flood walk with a synthetic, deterministic per-cell decode result so the
   heap/tie-break emulation can be compared with the reference's FloodDecodePositions built on the
   real std::priority_queue (oracle/ref_shim.cpp: ref_flood_walk_synthetic uses the same function). */
static unsigned synth_mix(unsigned a) { a ^= a >> 16; a *= 0x7feb352dU; a ^= a >> 15; a *= 0x846ca68bU; a ^= a >> 16; return a; }
void cbo_synth_result(unsigned seed, unsigned i, int dx, int dy, unsigned cooldown, unsigned noise, unsigned* drift_offset, unsigned* dist)
{
    unsigned h = synth_mix(seed ^ synth_mix(i * 2654435761u ^ (unsigned)((dx + 8) * 17 + (dy + 8)) ^ (cooldown << 20)));
    /* noise in [0,100]: probability (percent) of a non-centre / non-zero result */
    if ((h % 100) < noise) { *drift_offset = (h >> 8) % 9; *dist = (h >> 12) % 20; }
    else { *drift_offset = 4; *dist = (h >> 12) % 3; }
    if (*drift_offset == cooldown && *drift_offset != 4) *drift_offset = 4;
}
int cbo_flood_walk_synthetic(const cbo_mode* m, unsigned seed, unsigned noise, uint16_t* order_out, int8_t* drift_out /*2 per cell*/, uint8_t* cooldown_out)
{
    static const int DP[9][2] = {{-1, -1}, {0, -1}, {1, -1}, {-1, 0}, {0, 0}, {1, 0}, {-1, 1}, {0, 1}, {1, 1}};
    unsigned ncells = m->total_cells;
    int* xs = (int*)malloc(sizeof(int) * ncells); int* ys = (int*)malloc(sizeof(int) * ncells);
    cbo_cell_positions(m, 0, xs, ys);
    flood_t f; f.n = (int)ncells; f.count = 0;
    f.heap.cap = 1024; f.heap.n = 0; f.heap.v = (heap_elem*)malloc(sizeof(heap_elem) * 1024);
    f.remaining = (uint8_t*)malloc(ncells); memset(f.remaining, 1, ncells);
    f.instr = (instr_t*)malloc(sizeof(instr_t) * ncells);
    for (unsigned i = 0; i < ncells; ++i) { f.instr[i].dx = 0; f.instr[i].dy = 0; f.instr[i].prio = 0xFE; f.instr[i].cooldown = 0xFE; }
    adj_init(&f.adj, m, xs, (int)ncells);
    flood_seed(&f);
    int n = 0;
    while (f.count < f.n && f.heap.n > 0) {
        heap_elem e = heap_pop(&f.heap);
        unsigned i = e.idx;
        if (!f.remaining[i]) continue;
        f.remaining[i] = 0; f.count++;
        int ddx = f.instr[i].dx, ddy = f.instr[i].dy; uint8_t cooldown = f.instr[i].cooldown;
        unsigned off, dist;
        cbo_synth_result(seed, i, ddx, ddy, cooldown, noise, &off, &dist);
        int ndx = clamp7(ddx + DP[off][0]), ndy = clamp7(ddy + DP[off][1]);
        flood_update(&f, (int)i, ndx, ndy, dist, calculate_cooldown(cooldown, (uint8_t)off));
        order_out[n] = (uint16_t)i; drift_out[2 * n] = (int8_t)ddx; drift_out[2 * n + 1] = (int8_t)ddy; cooldown_out[n] = cooldown;
        ++n;
    }
    free(f.heap.v); free(f.remaining); free(f.instr); free(xs); free(ys);
    return n;
}

/* ------------------------------------------------------------------------------------------
 * Decoder::do_decode / do_decode_coupled with use_ecc = false -- Decoder.h:60-161
 * ---------------------------------------------------------------------------------------- */
/* per-thread stage timers (benchmark reporting only): 0 preprocess, 1 symbol walk, 2 colour pass, 3 RS */
static __thread int g_stage_on = 0;
static __thread double g_stage_s[4];
static double stage_now(void) { struct timespec ts; clock_gettime(CLOCK_MONOTONIC, &ts); return (double)ts.tv_sec + 1e-9 * (double)ts.tv_nsec; }
void cbo_stage_timing(int enable) { g_stage_on = enable; for (int i = 0; i < 4; ++i) g_stage_s[i] = 0; }
void cbo_stage_times(double out[4]) { for (int i = 0; i < 4; ++i) out[i] = g_stage_s[i]; }
#define STAGE_T0() double st0_ = g_stage_on ? stage_now() : 0
#define STAGE_ADD(i) do { if (g_stage_on) { double t_ = stage_now(); g_stage_s[i] += t_ - st0_; st0_ = t_; } } while (0)

static __thread void (*g_pre_color_hook)(const cbo_mode*, const uint8_t*, int, int, int, const uint8_t*) = NULL;

int cbo_decode_raw(const cbo_mode* m, const uint8_t* rgb, int w, int h, int needs_sharpen,
                   int color_correction, uint8_t* out, cbo_cell* cells)
{
    static const int DRIFT_PAIRS[9][2] = {{-1, -1}, {0, -1}, {1, -1}, {-1, 0}, {0, 0}, {1, 0}, {-1, 1}, {0, 1}, {1, 1}}; /* CellDrift.h:13-15 */
    unsigned bpc = m->symbol_bits + m->color_bits;
    unsigned cap_all = cbo_capacity(m, bpc);
    unsigned cap_sym = cbo_capacity(m, m->symbol_bits);
    unsigned ncells = m->total_cells;
    unsigned num_symbols = 1u << m->symbol_bits;
    memset(out, 0, cap_all);

    int good = (w >= (int)m->image_size_x) && (h >= (int)m->image_size_y);   /* CimbReader.cpp:119 */
    int* xs = (int*)malloc(sizeof(int) * ncells);
    int* ys = (int*)malloc(sizeof(int) * ncells);
    int* cx = (int*)calloc(ncells, sizeof(int));   /* colorPositions x,y (default 0,0) */
    int* cy = (int*)calloc(ncells, sizeof(int));
    uint8_t* have_pos = (uint8_t*)calloc(ncells, 1);
    unsigned* inv = (unsigned*)malloc(sizeof(unsigned) * ncells);
    cbo_interleave_reverse(ncells, m->interleave_blocks, m->interleave_partitions, inv);

    uint8_t* sym_buf = out;                                  /* non-legacy: symbols then colours */
    uint8_t* col_buf = m->legacy_mode ? out : out + cap_sym;
    unsigned sym_stride = m->legacy_mode ? bpc : m->symbol_bits;

    if (good && color_correction == 1) {   /* CimbReader.cpp:124-125: the decoder's CCM is replaced before anything is read */
        float ccm[9];
        cbo_simple_ccm(m, rgb, w, h, ccm);
        cbo_set_ccm(ccm);
    }
    if (good) {
        int padding = ((w - (int)m->image_size_x) < (h - (int)m->image_size_y) ? (w - (int)m->image_size_x) : (h - (int)m->image_size_y)) / 2;
        cbo_cell_positions(m, padding, xs, ys);
        uint8_t* bits = (uint8_t*)malloc((size_t)w * h / 8 + 16);
        STAGE_T0();
        cbo_preprocess(rgb, w, h, needs_sharpen, bits);
        STAGE_ADD(0);

        flood_t f;
        f.n = (int)ncells; f.count = 0;
        f.heap.cap = 1024; f.heap.n = 0; f.heap.v = (heap_elem*)malloc(sizeof(heap_elem) * 1024);
        f.remaining = (uint8_t*)malloc(ncells); memset(f.remaining, 1, ncells);
        f.instr = (instr_t*)malloc(sizeof(instr_t) * ncells);
        for (unsigned i = 0; i < ncells; ++i) { f.instr[i].dx = 0; f.instr[i].dy = 0; f.instr[i].prio = 0xFE; f.instr[i].cooldown = 0xFE; }
        adj_init(&f.adj, m, xs, (int)ncells);
        flood_seed(&f);
        unsigned order = 0;
        while (f.count < f.n && f.heap.n > 0) {
            heap_elem e = heap_pop(&f.heap);                  /* FloodDecodePositions.cpp:49-67 */
            unsigned i = e.idx;
            if (!f.remaining[i]) continue;
            f.remaining[i] = 0; f.count++;
            int ddx = f.instr[i].dx, ddy = f.instr[i].dy; uint8_t cooldown = f.instr[i].cooldown;
            /* CimbReader::read, CimbReader.cpp:139-162 */
            int x = xs[i] + ddx, y = ys[i] + ddy;
            uint64_t hashes[9];
            int all = (cooldown == 0xFE);                     /* CimbDecoder.cpp:144 */
            cbo_fuzzy_ahash(bits, w, x - 1, y - 1, all, hashes);
            unsigned drift_offset, dist;
            unsigned sym = cbo_best_symbol(hashes, all, num_symbols, cooldown, &drift_offset, &dist);
            int bx = DRIFT_PAIRS[drift_offset][0], by = DRIFT_PAIRS[drift_offset][1];
            int ndx = clamp7(ddx + bx), ndy = clamp7(ddy + by);
            flood_update(&f, (int)i, ndx, ndy, dist, calculate_cooldown(cooldown, (uint8_t)drift_offset));
            cx[i] = x + bx; cy[i] = y + by; have_pos[i] = 1;
            bb_write(sym_buf, sym, inv[i] * sym_stride, (int)sym_stride);   /* Decoder.h:91-92 / :147-148 */
            if (cells) {
                cells[i].order = (uint16_t)order; cells[i].symbol = (uint8_t)sym; cells[i].drift_offset = (uint8_t)drift_offset;
                cells[i].distance = (uint8_t)dist; cells[i].x = (int16_t)cx[i]; cells[i].y = (int16_t)cy[i];
                cells[i].drift_x = (int8_t)ddx; cells[i].drift_y = (int8_t)ddy; cells[i].cooldown_in = cooldown; cells[i].color = 0;
            }
            ++order;
        }
        STAGE_ADD(1);
        free(f.heap.v); free(f.remaining); free(f.instr); free(bits);
    }

    /* Decoder.h:104-105: "do color correction init, now that we (hopefully) have some fountain headers from the symbol
       decode" -- only do_decode (not the legacy coupled layout) calls reader.init_ccm */
    if (g_pre_color_hook && !m->legacy_mode) g_pre_color_hook(m, rgb, w, h, good, sym_buf);

    /* colour pass: Decoder.h:107-114 / :153-158.  colorPositions default to {i=0,x=0,y=0} when the reader
       was not good, so every entry ORs the colour at (0,0) into bit position 0. */
    STAGE_T0();
    for (unsigned i = 0; i < ncells; ++i) {
        unsigned bitpos = have_pos[i] ? inv[i] * (m->legacy_mode ? bpc : m->color_bits) : 0;
        unsigned c = decode_color_at(m, rgb, w, cx[i], cy[i]);
        bb_write(col_buf, c, bitpos, (int)m->color_bits);
        if (cells && have_pos[i]) cells[i].color = (uint8_t)c;
    }
    STAGE_ADD(2);
    free(xs); free(ys); free(cx); free(cy); free(have_pos); free(inv);
    return (int)cap_all;
}

/* ------------------------------------------------------------------------------------------
 * P12 Reed-Solomon -- libcorrect (src/third_party_lib/libcorrect/src/reed-solomon/)
 * ---------------------------------------------------------------------------------------- */
struct cbo_rs {
    unsigned min_distance;              /* parity bytes */
    uint8_t exp[512], log[256];         /* field.h:26-62 */
    uint8_t generator[256];             /* coefficients low->high, order = min_distance */
    uint8_t gen_roots[256];
    uint8_t gen_root_exp[64][255];      /* decode.c:279-283 */
    uint8_t element_exp[256][64];       /* decode.c:289-293 */
    /* decoder state (persists across calls exactly as in libcorrect) */
    uint8_t received[512];
    uint8_t syndromes[128];
    uint8_t locator[128]; unsigned locator_order;
    uint8_t last_locator[128]; unsigned last_locator_order;
    uint8_t locator_log[128];
    uint8_t error_roots[256];
    uint8_t error_vals[128];
    uint8_t error_locations[128];
    uint8_t evaluator[128];
    uint8_t derivative[128];
};

static uint8_t f_mul(const cbo_rs* rs, uint8_t l, uint8_t r)
{   /* field.h:92-110 */
    if (l == 0 || r == 0) return 0;
    return rs->exp[(unsigned)rs->log[l] + (unsigned)rs->log[r]];
}
static uint8_t f_div(const cbo_rs* rs, uint8_t l, uint8_t r)
{   /* field.h:112-129: x/0 = 0 */
    if (l == 0) return 0;
    if (r == 0) return 0;
    return rs->exp[255u + (unsigned)rs->log[l] - (unsigned)rs->log[r]];
}
static uint8_t f_mul_log(uint8_t l, uint8_t r)
{   /* field.h:131-145 */
    unsigned res = (unsigned)l + (unsigned)r;
    if (res > 255) return (uint8_t)(res - 255);
    return (uint8_t)res;
}
static uint8_t f_pow(const cbo_rs* rs, uint8_t elem, int pw)
{   /* field.h:156-167 */
    int res_log = (int)rs->log[elem] * pw;
    int mod = res_log % 255;
    if (mod < 0) mod += 255;
    return rs->exp[mod];
}
static void build_exp_lut(const cbo_rs* rs, uint8_t val, unsigned order, uint8_t* val_exp)
{   /* polynomial.c:159-171 */
    uint8_t val_exponentiated = rs->log[1];
    uint8_t val_log = rs->log[val];
    for (unsigned i = 0; i <= order; ++i) {
        if (val == 0) val_exp[i] = 0;
        else { val_exp[i] = val_exponentiated; val_exponentiated = f_mul_log(val_exponentiated, val_log); }
    }
}
static uint8_t poly_eval_lut(const cbo_rs* rs, const uint8_t* coeff, unsigned order, const uint8_t* val_exp)
{   /* polynomial.c:113-132 */
    if (val_exp[0] == 0) return coeff[0];
    uint8_t res = 0;
    for (unsigned i = 0; i <= order; ++i)
        if (coeff[i] != 0) res ^= rs->exp[(unsigned)rs->log[coeff[i]] + (unsigned)val_exp[i]];
    return res;
}
static uint8_t poly_eval_log_lut(const cbo_rs* rs, const uint8_t* coeff_log, unsigned order, const uint8_t* val_exp)
{   /* polynomial.c:134-157 */
    if (val_exp[0] == 0) {
        if (coeff_log[0] == 0) return 0;
        return rs->exp[coeff_log[0]];
    }
    uint8_t res = 0;
    for (unsigned i = 0; i <= order; ++i)
        if (coeff_log[i] != 0) res ^= rs->exp[(unsigned)coeff_log[i] + (unsigned)val_exp[i]];
    return res;
}
static void poly_mul(const cbo_rs* rs, const uint8_t* l, unsigned l_order, const uint8_t* r, unsigned r_order,
                     uint8_t* res, unsigned res_order)
{   /* polynomial.c:17-31 */
    memset(res, 0, res_order + 1);
    for (unsigned i = 0; i <= l_order; ++i) {
        if (i > res_order) continue;
        unsigned j_limit = (r_order > res_order - i) ? res_order - i : r_order;
        for (unsigned j = 0; j <= j_limit; ++j)
            res[i + j] ^= f_mul(rs, l[i], r[j]);
    }
}

cbo_rs* cbo_rs_create(unsigned parity)
{
    /* correct_reed_solomon_create(0x187, 1, 1, parity): ReedSolomon.h:26, reed-solomon.c:14-35 */
    cbo_rs* rs = (cbo_rs*)calloc(1, sizeof(cbo_rs));
    rs->min_distance = parity;
    unsigned element = 1;
    rs->exp[0] = 1; rs->log[0] = 0;
    for (unsigned i = 1; i < 512; ++i) {        /* field.h:48-55 */
        element = element * 2;
        element = (element > 255) ? (element ^ 0x187u) : element;
        rs->exp[i] = (uint8_t)element;
        if (i < 256) rs->log[element] = (uint8_t)i;
    }
    /* generator roots alpha^(1*(i+1)) and generator polynomial (reed-solomon.c:5-12, polynomial.c:215-262) */
    for (unsigned i = 0; i < parity; ++i) rs->gen_roots[i] = rs->exp[(1u * (i + 1u)) % 255u];
    if (parity > 0) {
        uint8_t a[300], b[300];
        memset(a, 0, sizeof(a)); memset(b, 0, sizeof(b));
        uint8_t* cur = a; uint8_t* nxt = b;
        cur[0] = rs->gen_roots[0]; cur[1] = 1;
        unsigned order = 1;
        for (unsigned i = 1; i < parity; ++i) {
            uint8_t l[2] = {rs->gen_roots[i], 1};
            poly_mul(rs, l, 1, cur, order, nxt, i + 1);
            order = i + 1;
            uint8_t* t = cur; cur = nxt; nxt = t;
        }
        memcpy(rs->generator, cur, parity + 1);
    }
    for (unsigned i = 0; i < parity; ++i) build_exp_lut(rs, rs->gen_roots[i], 254, rs->gen_root_exp[i]);
    for (unsigned i = 0; i < 256; ++i) build_exp_lut(rs, (uint8_t)i, parity ? parity - 1 : 0, rs->element_exp[i]);
    return rs;
}
void cbo_rs_destroy(cbo_rs* rs) { free(rs); }

int cbo_rs_encode(cbo_rs* rs, const uint8_t* msg, unsigned msg_len, uint8_t* enc)
{
    /* correct_reed_solomon_encode, encode.c:3-35: systematic, remainder of msg(x)*x^parity mod g(x).
       (Field arithmetic is exact: any correct long division gives the same bytes.) */
    unsigned nroots = rs->min_distance;
    if (msg_len > 255 - nroots) return -1;
    uint8_t rem[256];
    memset(rem, 0, sizeof(rem));
    /* LFSR division, message fed high-order first; generator is monic */
    for (unsigned i = 0; i < msg_len; ++i) {
        uint8_t fb = (uint8_t)(msg[i] ^ rem[nroots - 1]);
        for (unsigned j = nroots - 1; j > 0; --j)
            rem[j] = (uint8_t)(rem[j - 1] ^ f_mul(rs, fb, rs->generator[j]));
        rem[0] = f_mul(rs, fb, rs->generator[0]);
    }
    memmove(enc, msg, msg_len);
    for (unsigned i = 0; i < nroots; ++i) enc[msg_len + i] = rem[nroots - 1 - i];
    return 255;  /* libcorrect returns block_length, not the shortened length (encode.c:33) */
}

static unsigned rs_find_error_locator(cbo_rs* rs)
{
    /* Berlekamp-Massey, decode.c:30-116 (num_erasures = 0) */
    unsigned md = rs->min_distance;
    unsigned numerrors = 0;
    memset(rs->locator, 0, md + 1);
    rs->locator[0] = 1; rs->locator_order = 0;
    memcpy(rs->last_locator, rs->locator, md + 1);
    rs->last_locator_order = rs->locator_order;
    uint8_t discrepancy, last_discrepancy = 1;
    unsigned delay_length = 1;
    for (unsigned i = rs->locator_order; i < md; ++i) {
        discrepancy = rs->syndromes[i];
        for (unsigned j = 1; j <= numerrors; ++j)
            discrepancy ^= f_mul(rs, rs->locator[j], rs->syndromes[i - j]);
        if (!discrepancy) { delay_length++; continue; }
        if (2 * numerrors <= i) {
            for (int j = (int)rs->last_locator_order; j >= 0; --j)
                rs->last_locator[(unsigned)j + delay_length] = f_div(rs, f_mul(rs, rs->last_locator[j], discrepancy), last_discrepancy);
            for (int j = (int)delay_length - 1; j >= 0; --j) rs->last_locator[j] = 0;
            for (unsigned j = 0; j <= rs->last_locator_order + delay_length; ++j) {
                uint8_t temp = rs->locator[j];
                rs->locator[j] ^= rs->last_locator[j];
                rs->last_locator[j] = temp;
            }
            unsigned temp_order = rs->locator_order;
            rs->locator_order = rs->last_locator_order + delay_length;
            rs->last_locator_order = temp_order;
            numerrors = i + 1 - numerrors;
            last_discrepancy = discrepancy;
            delay_length = 1;
            continue;
        }
        for (int j = (int)rs->last_locator_order; j >= 0; --j)
            rs->locator[(unsigned)j + delay_length] ^= f_div(rs, f_mul(rs, rs->last_locator[j], discrepancy), last_discrepancy);
        rs->locator_order = (rs->last_locator_order + delay_length > rs->locator_order)
                                ? rs->last_locator_order + delay_length : rs->locator_order;
        delay_length++;
    }
    return rs->locator_order;
}

int cbo_rs_decode(cbo_rs* rs, const uint8_t* enc, unsigned enc_len, uint8_t* msg)
{
    /* correct_reed_solomon_decode, decode.c:299-379 */
    unsigned md = rs->min_distance;
    if (enc_len > 255) return -1;
    unsigned msg_len = enc_len - md;
    unsigned pad = 255 - enc_len;
    for (unsigned i = 0; i < enc_len; ++i) rs->received[i] = enc[enc_len - (i + 1)];
    for (unsigned i = 0; i < pad; ++i) rs->received[i + enc_len] = 0;

    int all_zero = 1;                                  /* decode.c:12-28 */
    memset(rs->syndromes, 0, md);
    for (unsigned i = 0; i < md; ++i) {
        uint8_t ev = poly_eval_lut(rs, rs->received, 254, rs->gen_root_exp[i]);
        if (ev) all_zero = 0;
        rs->syndromes[i] = ev;
    }
    if (all_zero) {
        for (unsigned i = 0; i < msg_len; ++i) msg[i] = rs->received[enc_len - (i + 1)];
        return (int)msg_len;
    }
    unsigned order = rs_find_error_locator(rs);
    rs->locator_order = order;
    for (unsigned i = 0; i <= order; ++i) rs->locator_log[i] = rs->log[rs->locator[i]];

    {   /* Chien search over all 256 elements, decode.c:120-143 */
        unsigned root = 0;
        memset(rs->error_roots, 0, order);
        for (unsigned i = 0; i < 256; ++i)
            if (!poly_eval_log_lut(rs, rs->locator_log, order, rs->element_exp[i])) rs->error_roots[root++] = (uint8_t)i;
        if (root != order) return -1;
    }
    for (unsigned i = 0; i < order; ++i) {             /* decode.c:198-222, generator_root_gap = 1 */
        if (rs->error_roots[i] == 0) continue;
        unsigned loc = f_div(rs, 1, rs->error_roots[i]);
        for (unsigned j = 0; j < 256; ++j)
            if (f_pow(rs, (uint8_t)j, 1) == loc) { rs->error_locations[i] = rs->log[j]; break; }
    }
    {   /* Forney, decode.c:163-194 */
        poly_mul(rs, rs->locator, order, rs->syndromes, md - 1, rs->evaluator, md - 1);
        unsigned der_order = order - 1;
        memset(rs->derivative, 0, der_order + 1);
        for (unsigned i = 0; i <= der_order; ++i)    /* polynomial.c:97-111, field_sum */
            rs->derivative[i] = ((i + 1) % 2) ? rs->locator[i + 1] : 0;
        for (unsigned i = 0; i < order; ++i) {
            if (rs->error_roots[i] == 0) continue;
            const uint8_t* ee = rs->element_exp[rs->error_roots[i]];
            rs->error_vals[i] = f_mul(rs, f_pow(rs, rs->error_roots[i], 0),
                                      f_div(rs, poly_eval_lut(rs, rs->evaluator, md - 1, ee),
                                                poly_eval_lut(rs, rs->derivative, der_order, ee)));
        }
    }
    for (unsigned i = 0; i < order; ++i)               /* decode.c:369-372; location 255 is out of range in libcorrect */
        rs->received[rs->error_locations[i]] ^= rs->error_vals[i];
    for (unsigned i = 0; i < msg_len; ++i) msg[i] = rs->received[enc_len - (i + 1)];
    return (int)msg_len;
}

/* P11 reed_solomon_stream::write into a plain stream -- reed_solomon_stream.h:54-76, :96-107 */
int cbo_rs_stream(unsigned parity, unsigned block, const uint8_t* raw, unsigned raw_len, uint8_t* out, uint8_t* ok)
{
    cbo_rs* rs = cbo_rs_create(parity);
    unsigned msg = block - parity;
    int good = 0;
    unsigned b = 0;
    while (raw_len >= block) {
        int n = cbo_rs_decode(rs, raw, block, out);
        if (n <= 0) { memset(out, 0, msg); if (ok) ok[b] = 0; }
        else { if (ok) ok[b] = 1; ++good; }
        raw += block; raw_len -= block; out += msg; ++b;
    }
    cbo_rs_destroy(rs);
    return good;
}

/* P13 aligned_stream + escrow_buffer_writer -- aligned_stream.h:39-116, escrow_buffer_writer.h:44-60,
   reed_solomon_stream.h:109-114.  align_offset = 0. */
unsigned cbo_align_chunks(const uint8_t* blocks, const uint8_t* ok, unsigned nblocks, unsigned msg_len,
                          unsigned chunk_size, uint8_t* chunks_out, uint32_t* mask)
{
    uint8_t* buffer = (uint8_t*)calloc(chunk_size, 1);
    unsigned offset = 0; int bad_chunk = 0; unsigned total = 0; unsigned emitted = 0;
    unsigned consumed = 0;   /* bytes of the frame's post-ECC stream consumed so far -> chunk index */
    if (mask) *mask = 0;
    for (unsigned b = 0; b < nblocks; ++b) {
        const uint8_t* data = blocks + (size_t)b * msg_len;
        if (!ok[b]) {                                   /* mark_bad_chunk(msg_len) */
            bad_chunk = 1;
            offset = (offset + msg_len) % chunk_size;
            consumed += msg_len;
            continue;
        }
        unsigned length = msg_len;
        while (length > 0) {
            unsigned work = length + offset;
            if (work >= chunk_size) {
                unsigned write_len = chunk_size - offset;
                if (bad_chunk) { bad_chunk = 0; offset = 0; }
                else {
                    memcpy(buffer + offset, data, write_len);
                    offset += write_len;
                    /* flush(): one full chunk goes to the escrow writer */
                    unsigned chunk_idx = (consumed + write_len) / chunk_size - 1;
                    memcpy(chunks_out + (size_t)emitted * chunk_size, buffer, offset);
                    if (mask) *mask |= 1u << chunk_idx;
                    ++emitted; total += offset; offset = 0;
                }
                length -= write_len; data += write_len; consumed += write_len;
                continue;
            }
            memcpy(buffer + offset, data, length);
            offset += length; consumed += length; length = 0;
        }
    }
    free(buffer);
    return total;
}

int cbo_decode(const cbo_mode* m, const uint8_t* rgb, int w, int h, int needs_sharpen, int use_ecc,
               uint8_t* out, uint8_t* block_ok)
{
    unsigned bpc = m->symbol_bits + m->color_bits;
    unsigned cap_all = cbo_capacity(m, bpc);
    uint8_t* raw = (uint8_t*)malloc(cap_all);
    cbo_decode_raw(m, rgb, w, h, needs_sharpen, 0, raw, NULL);
    if (!use_ecc || m->ecc_bytes == 0) { memcpy(out, raw, cap_all); free(raw); return (int)cap_all; }
    unsigned msg = m->ecc_block_size - m->ecc_bytes;
    unsigned total = 0;
    STAGE_T0();
    if (m->legacy_mode) {
        unsigned nb = cap_all / m->ecc_block_size;
        cbo_rs_stream(m->ecc_bytes, m->ecc_block_size, raw, cap_all, out, block_ok);
        total = nb * msg;
    } else {
        unsigned cap_sym = cbo_capacity(m, m->symbol_bits), cap_col = cbo_capacity(m, m->color_bits);
        unsigned nbs = cap_sym / m->ecc_block_size, nbc = cap_col / m->ecc_block_size;
        cbo_rs_stream(m->ecc_bytes, m->ecc_block_size, raw, cap_sym, out, block_ok);
        cbo_rs_stream(m->ecc_bytes, m->ecc_block_size, raw + cap_sym, cap_col, out + (size_t)nbs * msg, block_ok ? block_ok + nbs : NULL);
        total = (nbs + nbc) * msg;
    }
    STAGE_ADD(3);
    free(raw);
    return (int)total;
}

/* the symbol pass of a fountain decode with color_correction == 2: RS the symbol stream, replay the aligned_stream
   callbacks, fit the CCM (CimbReader::init_ccm) and install it before the colour pass */
static void fountain_ccm_hook(const cbo_mode* m, const uint8_t* rgb, int w, int h, int good, const uint8_t* sym_buf)
{
    if (!good || m->ecc_bytes == 0) return;
    unsigned cap_sym = cbo_capacity(m, m->symbol_bits), msg = m->ecc_block_size - m->ecc_bytes;
    unsigned nbs = cap_sym / m->ecc_block_size;
    uint8_t* data = (uint8_t*)malloc((size_t)nbs * msg); uint8_t* ok = (uint8_t*)malloc(nbs);
    cbo_rs_stream(m->ecc_bytes, m->ecc_block_size, sym_buf, cap_sym, data, ok);
    uint8_t hdr[6]; unsigned radioactive = 0; float ccm[9];
    if (cbo_header_after_symbols(data, ok, nbs, msg, m->chunk_size, hdr, &radioactive) &&
        cbo_init_ccm(m, rgb, w, h, hdr, radioactive, ccm))
        cbo_set_ccm(ccm);
    free(data); free(ok);
}

int cbo_decode_fountain_cc(const cbo_mode* m, const uint8_t* rgb, int w, int h, int needs_sharpen, int color_correction,
                           uint8_t* chunks_out, uint32_t* mask)
{
    /* Decoder::decode_fountain, Decoder.h:171-189: one aligned_stream spans the symbol and colour RS streams */
    unsigned bpc = m->symbol_bits + m->color_bits;
    unsigned cap_all = cbo_capacity(m, bpc);
    unsigned msg = m->ecc_block_size - m->ecc_bytes;
    unsigned nblocks = cap_all / m->ecc_block_size;
    uint8_t* data = (uint8_t*)malloc((size_t)nblocks * msg);
    uint8_t* ok = (uint8_t*)malloc(nblocks);
    uint8_t* raw = (uint8_t*)malloc(cap_all);
    g_pre_color_hook = (color_correction == 2) ? fountain_ccm_hook : NULL;
    cbo_decode_raw(m, rgb, w, h, needs_sharpen, color_correction, raw, NULL);
    g_pre_color_hook = NULL;
    if (m->legacy_mode) cbo_rs_stream(m->ecc_bytes, m->ecc_block_size, raw, cap_all, data, ok);
    else {
        unsigned cap_sym = cbo_capacity(m, m->symbol_bits), cap_col = cbo_capacity(m, m->color_bits);
        unsigned nbs = cap_sym / m->ecc_block_size;
        cbo_rs_stream(m->ecc_bytes, m->ecc_block_size, raw, cap_sym, data, ok);
        cbo_rs_stream(m->ecc_bytes, m->ecc_block_size, raw + cap_sym, cap_col, data + (size_t)nbs * msg, ok + nbs);
    }
    free(raw);
    unsigned good = cbo_align_chunks(data, ok, nblocks, msg, m->chunk_size, chunks_out, mask);
    free(data); free(ok);
    return (int)good;
}

int cbo_decode_fountain(const cbo_mode* m, const uint8_t* rgb, int w, int h, int needs_sharpen,
                        uint8_t* chunks_out, uint32_t* mask)
{
    /* Decoder::decode_fountain, Decoder.h:171-189: one aligned_stream spans the symbol and colour RS streams */
    unsigned bpc = m->symbol_bits + m->color_bits;
    unsigned cap_all = cbo_capacity(m, bpc);
    unsigned msg = m->ecc_block_size - m->ecc_bytes;
    unsigned nblocks = cap_all / m->ecc_block_size;
    uint8_t* data = (uint8_t*)malloc((size_t)nblocks * msg);
    uint8_t* ok = (uint8_t*)malloc(nblocks);
    cbo_decode(m, rgb, w, h, needs_sharpen, 1, data, ok);
    unsigned good = cbo_align_chunks(data, ok, nblocks, msg, m->chunk_size, chunks_out, mask);
    free(data); free(ok);
    return (int)good;
}

/* P14 FountainMetadata -- FountainMetadata.h:16-90 */
void cbo_md_pack(uint8_t encode_id, unsigned size, uint16_t block_id, uint8_t out[6])
{
    out[0] = (uint8_t)((encode_id & 0x7F) | ((size >> 17) & 0x80));
    out[1] = (uint8_t)((size >> 16) & 0xFF); out[2] = (uint8_t)((size >> 8) & 0xFF); out[3] = (uint8_t)(size & 0xFF);
    out[4] = (uint8_t)((block_id >> 8) & 0xFF); out[5] = (uint8_t)(block_id & 0xFF);
}
unsigned cbo_md_file_size(const uint8_t md[6])
{
    return (unsigned)md[3] | ((unsigned)md[2] << 8) | ((unsigned)md[1] << 16) | (((unsigned)md[0] & 0x80u) << 17);
}
unsigned cbo_md_block_id(const uint8_t md[6]) { return ((unsigned)md[4] << 8) | md[5]; }
unsigned cbo_md_encode_id(const uint8_t md[6]) { return md[0] & 0x7Fu; }

/* ------------------------------------------------------------------------------------------
 * Encoder side (synthetic-input generator) -- Encoder.h:69-129 / :131-165, CimbWriter.cpp:84-95
 * ---------------------------------------------------------------------------------------- */
void cbo_payload_to_cells(const cbo_mode* m, const uint8_t* payload, unsigned payload_len, uint8_t* cellvals)
{
    unsigned bpc = m->symbol_bits + m->color_bits;
    unsigned ncells = m->total_cells;
    unsigned cap_all = cbo_capacity(m, bpc);
    unsigned msg = m->ecc_block_size - m->ecc_bytes;
    unsigned nblocks = cap_all / m->ecc_block_size;
    /* RS-encode consecutive msg-byte pieces (reed_solomon_stream::readsome, reed_solomon_stream.h:32-52) */
    uint8_t* enc = (uint8_t*)calloc((size_t)nblocks * m->ecc_block_size + 256, 1);
    cbo_rs* rs = cbo_rs_create(m->ecc_bytes);
    uint8_t piece[256];
    for (unsigned b = 0; b < nblocks; ++b) {
        memset(piece, 0, sizeof(piece));
        unsigned off = b * msg;
        unsigned n = 0;
        if (off < payload_len) n = (payload_len - off < msg) ? payload_len - off : msg;
        memcpy(piece, payload + off, n);
        if (m->ecc_bytes) cbo_rs_encode(rs, piece, msg, enc + (size_t)b * m->ecc_block_size);
        else memcpy(enc + (size_t)b * m->ecc_block_size, piece, msg);
    }
    cbo_rs_destroy(rs);
    unsigned* idx = (unsigned*)malloc(sizeof(unsigned) * ncells);
    cbo_interleave_indices(ncells, m->interleave_blocks, m->interleave_partitions, idx);
    memset(cellvals, 0, ncells);
    if (m->legacy_mode) {
        for (unsigned s = 0; s < ncells; ++s)                   /* encode_next_coupled */
            cellvals[idx[s]] = (uint8_t)bb_read(enc, s * bpc, (int)bpc);
    } else {
        unsigned cap_sym = cbo_capacity(m, m->symbol_bits);
        for (unsigned s = 0; s < ncells; ++s) {                 /* symbol pass then colour pass */
            unsigned sym = bb_read(enc, s * m->symbol_bits, (int)m->symbol_bits);
            unsigned col = m->color_bits ? bb_read(enc + cap_sym, s * m->color_bits, (int)m->color_bits) : 0;
            cellvals[idx[s]] = (uint8_t)((col << m->symbol_bits) | sym);
        }
    }
    free(idx); free(enc);
}

void cbo_render_frame(const cbo_mode* m, const uint8_t* cellvals, uint8_t* rgb)
{
    /* dark mode: black canvas (CimbWriter.cpp:54-55); tile = palette colour where the tile bitmap is set,
       background black (Common.cpp:141-171, getBgColor with color_mode <= 0x100). Anchors/guides are not
       drawn: they lie outside every cell's 5x5-mean support (CimbWriter.cpp:61-78). */
    unsigned w = m->image_size_x, h = m->image_size_y;
    unsigned ncells = m->total_cells;
    unsigned num_symbols = 1u << m->symbol_bits, num_colors = 1u << m->color_bits;
    int* xs = (int*)malloc(sizeof(int) * ncells);
    int* ys = (int*)malloc(sizeof(int) * ncells);
    cbo_cell_positions(m, 0, xs, ys);
    memset(rgb, 0, (size_t)w * h * 3);
    for (unsigned i = 0; i < ncells; ++i) {
        unsigned v = cellvals[i] % (num_symbols * num_colors);   /* CimbEncoder.cpp:39-42 */
        unsigned sym = v % num_symbols, col = v / num_symbols;  /* CimbEncoder.cpp:20-25 */
        uint8_t c[3];
        cbo_palette(col, num_colors, m->color_mode, c);
        uint64_t tile = TILE_HASHES[sym];
        for (int r = 0; r < 8; ++r)
            for (int cc = 0; cc < 8; ++cc)
                if ((tile >> (63 - (8 * r + cc))) & 1) {
                    uint8_t* p = rgb + ((size_t)(ys[i] + r) * w + (size_t)(xs[i] + cc)) * 3;
                    p[0] = c[0]; p[1] = c[1]; p[2] = c[2];
                }
    }
    free(xs); free(ys);
}
