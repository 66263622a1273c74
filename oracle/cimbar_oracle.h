/*
 * cimbar_oracle.h -- CPU restatement of libcimbar's per-frame decode hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under oracle/ is part of the product: only
 * tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
 * legs may build, load or call it, and there only as the checker / CPU baseline.
 * The product path (libcimbar_b200/) never links or falls back to this code.
 *
 * Each function cites the reference file:line (relative to /root/reference/) it
 * restates.  Parity is PINNED: tests/test_oracle_goldens.py checks this code
 * against the reference's own SHA-256 goldens (src/lib/encoder/test/DecoderTest.cpp:26-106),
 * per-cell known answers (cimb_translator/test/CimbReaderTest.cpp:37-163,
 * CimbDecoderTest.cpp:77-131), RS known answers (encoder/test/reed_solomon_streamTest.cpp:23)
 * and against the reference's own OpenCV-free sources compiled unmodified into
 * oracle/_ref/ (libcorrect RS, flood walk, interleave, aligned_stream).
 */
#ifndef CIMBAR_ORACLE_H
#define CIMBAR_ORACLE_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CBO_MAX_CELLS 16384

/* mirrors cimbar::conf (src/lib/cimb_translator/GridConf.h:8-77) + Config.h accessors */
typedef struct cbo_mode {
    int mode_val;          /* 68=B, 67=Bm, 66=Bu, 4=4C, 8=8C (Config.h:20-43) */
    unsigned color_bits;
    unsigned symbol_bits;
    unsigned ecc_bytes;
    unsigned ecc_block_size;
    unsigned image_size_x;
    unsigned image_size_y;
    unsigned cell_size;
    unsigned cell_spacing_x;
    unsigned cell_spacing_y;
    unsigned cell_offset;
    unsigned cells_per_col_x;
    unsigned cells_per_col_y;
    int fountain_chunks_scalar;
    int legacy_mode;
    /* derived */
    unsigned corner_padding_x;
    unsigned corner_padding_y;
    unsigned total_cells;
    unsigned color_mode;            /* Config.h:61-64: legacy ? 0 : 1 */
    unsigned interleave_blocks;     /* = ecc_block_size (Config.h:157-160) */
    unsigned interleave_partitions; /* = 2 (Config.h:162-165) */
    unsigned chunks_per_frame;      /* fountain_chunks_per_frame() */
    unsigned chunk_size;            /* fountain_chunk_size() */
} cbo_mode;

/* per-cell trace of the symbol walk (for the reference's CimbReaderTest-style checks) */
typedef struct cbo_cell {
    uint16_t order;        /* position in the flood-walk order */
    uint8_t  symbol;
    uint8_t  color;
    uint8_t  drift_offset; /* 0..8, 4 = centre */
    uint8_t  distance;
    int16_t  x, y;         /* drift-adjusted top-left used for the colour read */
    int8_t   drift_x, drift_y; /* accumulated drift when the cell was decoded */
    uint8_t  cooldown_in;
} cbo_cell;

int  cbo_mode_init(cbo_mode* m, int mode_val);
unsigned cbo_capacity(const cbo_mode* m, unsigned bits_per_cell);

/* P2: CellPositions::compute_linear (CellPositions.cpp:5-50). returns count */
int  cbo_cell_positions(const cbo_mode* m, int padding, int* xs, int* ys);
/* AdjacentCellFinder::find (AdjacentCellFinder.cpp:54-105): right,left,bottom,top */
void cbo_adjacent(const cbo_mode* m, const int* xs, int ncells, int index, int adj[4]);
/* P7: Interleave::interleave_reverse (Interleave.h:8-36) */
void cbo_interleave_reverse(unsigned size, unsigned num_chunks, unsigned partitions, unsigned* inv);
void cbo_interleave_indices(unsigned size, unsigned num_chunks, unsigned partitions, unsigned* idx);

/* P1: cv::cvtColor(RGB2GRAY) as pinned against cv2 4.13 (CimbReader.cpp:35) */
void cbo_rgb_to_gray(const uint8_t* rgb, int w, int h, uint8_t* gray);
/* sharpen: cv::filter2D with the 3x3 kernel of CimbReader.cpp:17-27 (8-bit saturating, BORDER_REFLECT_101) */
void cbo_sharpen(const uint8_t* gray, int w, int h, uint8_t* out);
/* cv::adaptiveThreshold(MEAN_C, THRESH_BINARY, block, C=0) (CimbReader.cpp:41): out 0/255 per pixel */
void cbo_adaptive_threshold(const uint8_t* gray, int w, int h, int block, uint8_t* out);
/* bitmatrix::mat_to_bitbuffer (bitmatrix.h:14-46): MSB-first, 8 px / byte */
void cbo_pack_bits(const uint8_t* thr, size_t npix, uint8_t* bits);
/* whole P1 */
void cbo_preprocess(const uint8_t* rgb, int w, int h, int needs_sharpen, uint8_t* bits /* w*h/8 */);   /* fused, fast */
void cbo_preprocess_unfused(const uint8_t* rgb, int w, int h, int needs_sharpen, uint8_t* bits);          /* pass by pass */
/* per-thread stage timers for the benchmark's per-stage split: [0] preprocess, [1] symbol walk, [2] colour, [3] RS (seconds) */
void cbo_stage_timing(int enable);
void cbo_stage_times(double out[4]);
void cbo_threshold_bits_fast(const uint8_t* gray, int w, int h, int block, uint8_t* bits);

/* P5: fuzzy_ahash<8>(bitmatrix) + ahash_result (average_hash.h:63-75, ahash_result.h:70-106).
   window origin (wx,wy) = (x-1,y-1); hashes[9], FAST leaves corners 0 */
void cbo_fuzzy_ahash(const uint8_t* bits, int w, int wx, int wy, int all, uint64_t hashes[9]);
/* P6: CimbDecoder::get_best_symbol (CimbDecoder.cpp:101-132) */
unsigned cbo_best_symbol(const uint64_t hashes[9], int all, unsigned num_symbols, unsigned cooldown,
                         unsigned* drift_offset, unsigned* best_distance);
const uint64_t* cbo_tile_hashes(void);

/* P8: Cell::mean_rgb_continuous over the inner 6x6 (Cell.h:30-62, CimbDecoder.cpp:202-209) */
void cbo_avg_color(const uint8_t* rgb, int w, int x, int y, int cell_size, uint8_t out[3]);
/* P9: CimbDecoder::get_best_color (CimbDecoder.cpp:168-200); ccm = 9 floats row-major or NULL */
unsigned cbo_best_color(float r, float g, float b, unsigned num_colors, unsigned color_mode, const float* ccm);
/* cbo_best_color of n integer means (r, g, b bytes), one call for a batch */
void cbo_best_colors(const uint8_t* means, int n, unsigned num_colors, unsigned color_mode, const float* ccm, uint8_t* out);
void cbo_palette(unsigned index, unsigned num_colors, unsigned color_mode, uint8_t rgb[3]);

/* P3+P4+P5+P6+P8+P9+P7+P10: Decoder::do_decode / do_decode_coupled with use_ecc=false
   (Decoder.h:60-161): raw cell bits.  out must hold capacity(bits_per_cell) bytes.
   cells (optional) gets ncells entries indexed by cell index.  Returns bytes written
   (capacity), also when the image is too small (zero-filled, CimbReader.cpp:119,141). */
int  cbo_decode_raw(const cbo_mode* m, const uint8_t* rgb, int w, int h, int needs_sharpen,
                    int color_correction /* 0, or 1 = simpleColorCorrection; 2 (header fit) is not restated */, uint8_t* out, cbo_cell* cells);
/* the decoder's thread-local CCM (CimbDecoder::update_color_correction, CimbDecoder.cpp:82-85); NULL = inactive */
void cbo_set_ccm(const float* m9);
int cbo_get_ccm(float* m9);
/* color_correction::get_adaptation_matrix<von_kries> (color_correction.h:12-24) and simpleColorCorrection (CimbReader.cpp:55-93) */
void cbo_adaptation_matrix(const float actual[3], const float desired[3], float out[9]);
void cbo_simple_ccm(const cbo_mode* m, const uint8_t* rgb, int w, int h, float out[9]);
/* color_correction::get_moore_penrose_lsm (color_correction.h:26-39): rows x 3 row-major inputs; returns 1 on success */
int cbo_moore_penrose_lsm(const float* actual, const float* desired, int rows, float out[9]);
/* CimbReader::_fountainColorHeader after the symbol stream's chunk callbacks (CimbReader.cpp:269-280) */
int cbo_header_after_symbols(const uint8_t* blocks, const uint8_t* ok, unsigned nblocks, unsigned msg_len, unsigned chunk_size,
                             uint8_t hdr[6], unsigned* radioactive_out);
/* CimbReader::init_ccm (CimbReader.cpp:169-267); returns 1 when a matrix was fitted */
int cbo_init_ccm(const cbo_mode* m, const uint8_t* rgb, int w, int h, const uint8_t hdr[6], unsigned radioactive, float out[9]);
/* the N x 3 actual / desired rows the calling thread's last cbo_init_ccm fitted (white last); returns N (0 before any fit) */
int cbo_last_fit_rows(float* actual, float* desired);
/* Decoder::decode_fountain(img, stream, should_preprocess, color_correction) incl. color_correction == 2 */
int cbo_decode_fountain_cc(const cbo_mode* m, const uint8_t* rgb, int w, int h, int needs_sharpen, int color_correction,
                           uint8_t* chunks_out, uint32_t* mask);

/* test hooks for the flood-walk / heap emulation (compared with the reference's FloodDecodePositions in oracle/_ref) */
void cbo_synth_result(unsigned seed, unsigned i, int dx, int dy, unsigned cooldown, unsigned noise, unsigned* drift_offset, unsigned* dist);
int  cbo_flood_walk_synthetic(const cbo_mode* m, unsigned seed, unsigned noise, uint16_t* order_out, int8_t* drift_out, uint8_t* cooldown_out);

/* P12: correct_reed_solomon_decode / _encode (libcorrect decode.c:299-379, encode.c:3-35),
   poly 0x187, fcr 1, gap 1.  decode returns msg_len or -1; encode writes msg+parity */
typedef struct cbo_rs cbo_rs;
cbo_rs* cbo_rs_create(unsigned parity);
void    cbo_rs_destroy(cbo_rs*);
int     cbo_rs_decode(cbo_rs*, const uint8_t* enc, unsigned enc_len, uint8_t* msg);
int     cbo_rs_encode(cbo_rs*, const uint8_t* msg, unsigned msg_len, uint8_t* enc);

/* P11: reed_solomon_stream::write into a plain stream (reed_solomon_stream.h:54-76, :96-107):
   failed block -> zeros.  raw: nblocks*block bytes; out: nblocks*(block-parity); ok[nblocks].
   returns number of good blocks */
int  cbo_rs_stream(unsigned parity, unsigned block, const uint8_t* raw, unsigned raw_len,
                   uint8_t* out, uint8_t* ok);
/* P13: aligned_stream chunking of a sequence of RS block results (aligned_stream.h:39-116,
   reed_solomon_stream.h:109-114).  blocks: nblocks*(msg) bytes, ok flags.  Emits good chunks
   densely into chunks_out (escrow_buffer_writer order), mask bit q set if chunk q emitted.
   returns good bytes (aligned_stream::tellp) */
unsigned cbo_align_chunks(const uint8_t* blocks, const uint8_t* ok, unsigned nblocks, unsigned msg_len,
                          unsigned chunk_size, uint8_t* chunks_out, uint32_t* mask);

/* Decoder::decode (ofstream semantics): raw -> RS -> bytes (7500 for mode B).  returns bytes */
int  cbo_decode(const cbo_mode* m, const uint8_t* rgb, int w, int h, int needs_sharpen,
                int use_ecc, uint8_t* out, uint8_t* block_ok);
/* Decoder::decode_fountain into an escrow_buffer_writer: returns good bytes, fills chunks densely */
int  cbo_decode_fountain(const cbo_mode* m, const uint8_t* rgb, int w, int h, int needs_sharpen,
                         uint8_t* chunks_out, uint32_t* mask);

/* P14: FountainMetadata (FountainMetadata.h:16-90) */
void     cbo_md_pack(uint8_t encode_id, unsigned size, uint16_t block_id, uint8_t out[6]);
unsigned cbo_md_file_size(const uint8_t md[6]);
unsigned cbo_md_block_id(const uint8_t md[6]);
unsigned cbo_md_encode_id(const uint8_t md[6]);

/* Encoder side (input generator; Encoder.h:69-129, CimbWriter.cpp:84-95, CimbEncoder.cpp:22-42):
   cellvals[i] = (color << symbol_bits) | symbol for linear cell i -> RGB frame (no anchors unless
   assets given).  payload -> cellvals via RS encode + bit striping. */
void cbo_payload_to_cells(const cbo_mode* m, const uint8_t* payload, unsigned payload_len, uint8_t* cellvals);
void cbo_render_frame(const cbo_mode* m, const uint8_t* cellvals, uint8_t* rgb /* image_size_x*image_size_y*3 */);

#ifdef __cplusplus
}
#endif
#endif
