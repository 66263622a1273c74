/*
 * cb200.h -- C ABI of libcb200.so: the H100 (sm_90a) implementation of libcimbar's per-frame decode hot path.
 *
 * Drop-in boundary (SURVEY.md section 8b).  The reference (sz3/libcimbar) has no plugin registry: the path sits
 * behind header-only C++ templates (Decoder / CimbReader / CimbDecoder) and one facade C ABI (cimbard_*,
 * src/lib/cimbar_js/cimbar_recv_js.h:11-39).  These entry points are what a binding for this path would call;
 * each cites the reference interface it replaces (paths relative to the libcimbar checkout).  The header-compatible
 * C++ shims that route libcimbar's own class names here are in libcimbar_b200/host/ (see INTEGRATION.md).
 *
 * Conventions: plain pointers and sizes, no exceptions, int return (0 = CB200_OK, negative = error, see
 * cb200_last_error()).  A context is bound to one GPU and one CUDA stream and is NOT thread-safe -- same model as
 * the reference's "one Decoder per thread" (thread_local Config, src/lib/cimb_translator/Config.h:11-15).
 * Buffers are caller-owned.  `_dev` entry points take device pointers and only enqueue work on the context's
 * stream (call cb200_sync before reading results); the others take host pointers and return when results are in
 * host memory.  Frames are tightly packed RGB8, image_size_y rows x image_size_x px x 3 bytes, already extracted
 * (the output of the reference's Extractor / `--no-deskew` input).
 */
#ifndef CB200_H
#define CB200_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CB200_OK            0
#define CB200_ERR_ARG      -1   /* bad argument (null pointer, n out of range, ...) */
#define CB200_ERR_CUDA     -2   /* CUDA runtime error, text in cb200_last_error() */
#define CB200_ERR_MODE     -3   /* unknown / unsupported mode_val */
#define CB200_ERR_NOMEM    -4
#define CB200_ERR_NODEVICE -5   /* no usable CUDA device: the library never falls back to a CPU path */

/* decode flags */
#define CB200_FLAG_NO_FALLBACK  0x1u  /* do not run the exact flood-walk kernel on frames K1 flags as inexact (bench only) */
#define CB200_FLAG_SHARPEN      0x2u  /* needs_sharpen / should_preprocess=true: 3x3 sharpen + block 7 (CimbReader.cpp:17-40) */
#define CB200_FLAG_CC_SIMPLE    0x4u  /* color_correction == 1: every frame gets the von Kries matrix of its own anchor white
                                         before anything is read (simpleColorCorrection, CimbReader.cpp:55-93, :124-125);
                                         afterwards the context's CCM is the last frame's, as in the reference's decoder.
                                         Without a CC flag the colour pass uses the context's CCM if one is set (below). */
#define CB200_FLAG_CC_FIT       0x8u  /* color_correction == 2 (the reference's default) with the output stream of
                                         Decoder::decode_fountain, whose chunk callback hands the decoder the fountain
                                         headers (Decoder.h:171-189): honoured by the RS entry points (cb200_decode,
                                         cb200_decode_chunks_dev, cb200_decode_fountain); a caller that mirrors
                                         Decoder::decode on a plain stream must not set it (no callback, no fit), and the
                                         raw entry points ignore it.  After the symbol stream's RS pass the fountain
                                         header of the frame predicts the colours at the head of every colour-stream chunk,
                                         a 3x3 least-squares CCM is fitted from them and the anchor white
                                         (CimbReader::init_ccm, CimbReader.cpp:169-267; OpenCV's float Jacobi SVD restated),
                                         and the frame's colours are decided with it.  A frame without a usable header keeps
                                         the CCM of the frame before it (frame 0: the context's), exactly like the
                                         reference's thread-local decoder state when frames are decoded in order; the
                                         context's CCM afterwards is the last frame's.  Mutually exclusive with CC_SIMPLE:
                                         every entry point that honours CC_FIT refuses the pair with CB200_ERR_ARG before
                                         any CUDA call, whatever n is. */

#define CB200_FLAG_NO_INTERLEAVE 0x10u /* Decoder(use_ecc, interleave=false): cells map to stream slots in linear order
                                         (Interleave::interleave_indices with num_chunks == 0, Interleave.h:10-16; Decoder.h:68) */
#define CB200_FLAG_SHARPEN_IF_NEEDED 0x20u /* the cimbar CLI's `--preprocess -1` (its default, src/exe/cimbar/cimbar.cpp:124-160):
                                         camera picture i is decoded with should_preprocess = true iff Extractor::extract returns
                                         NEEDS_SHARPEN for it, i.e. its corners fail Corners::is_granular_scale (Extractor.h:30-46),
                                         and without sharpening otherwise, all in one batch, in order (the CCM of CC_FIT still
                                         carries from picture to picture).  Honoured by the camera entry points
                                         (cb200_scan_extract_decode_fountain, cb200_extract_decode_fountain[_dev]); with
                                         CB200_FLAG_SHARPEN, or on an entry point that takes extracted frames, CB200_ERR_ARG. */

/* per-frame status bits written to frame_flags[] */
#define CB200_FRAME_FALLBACK    0x1u  /* frame was decoded by the exact flood-walk kernel (drift tracking needed) */
#define CB200_FRAME_INEXACT     0x2u  /* K1 could not prove the drift-0 decode exact and no fallback was run */

typedef struct cb200_ctx cb200_ctx;

/* geometry of the active mode == the cimbar::Config accessors (src/lib/cimb_translator/Config.h:51-175) */
typedef struct cb200_info {
    int mode_val;            /* 68 = B, 67 = Bm, 66 = Bu, 4 = 4C, 8 = 8C (Config.h:20-43) */
    int image_size_x, image_size_y;
    int frame_bytes;         /* image_size_x * image_size_y * 3 */
    int total_cells;         /* Config::total_cells() */
    int symbol_bits, color_bits;
    int raw_bytes;           /* Config::capacity(): bytes of cell bits per frame (9300) */
    int raw_symbol_bytes;    /* capacity(symbol_bits): 6200; == raw_bytes for the legacy coupled modes */
    int ecc_bytes, ecc_block_size;
    int rs_blocks;           /* RS blocks per frame (60) */
    int data_bytes;          /* bytes after ECC per frame (7500) */
    int chunk_size;          /* Config::fountain_chunk_size() (625) */
    int chunks_per_frame;    /* Config::fountain_chunks_per_frame() (12) */
    int legacy_mode;
    int max_frames;          /* batch capacity of this context */
    int sm_count;
} cb200_info;

const char* cb200_last_error(void);   /* thread-local text of the last error */
int cb200_version(void);

/* Replaces: Config::update(mode_val) + Decoder::Decoder() -> CimbDecoder::CimbDecoder()/load_tiles()
   (src/lib/cimb_translator/Config.h:46-49, src/lib/encoder/Decoder.h:40-45, CimbDecoder.cpp:57-99).
   Allocates device workspaces for up to max_frames frames per call. device < 0: current device. */
int cb200_create(cb200_ctx** out, int device, int mode_val, int max_frames);
int cb200_destroy(cb200_ctx* ctx);
int cb200_get_info(const cb200_ctx* ctx, cb200_info* out);
/* run on a caller-provided cudaStream_t (e.g. a torch stream); NULL restores the context's own stream
   (to select the legacy default stream pass cudaStreamLegacy = (void*)0x1, not 0) */
int cb200_set_stream(cb200_ctx* ctx, void* cuda_stream);
int cb200_sync(cb200_ctx* ctx);

/* ---- device-pointer entry points: enqueue only -------------------------------------------------------------- */

/* Replaces: CimbReader::CimbReader (preprocessSymbolGrid) + Decoder::do_decode with use_ecc=false:
   the flood walk CimbReader::read / read_color over all cells and the de-interleaved MSB-first bit packing
   (src/lib/cimb_translator/CimbReader.cpp:30-46,:107-162; src/lib/encoder/Decoder.h:60-161).
   d_rgb: n frames; d_raw_out: n * raw_bytes (symbol stream then colour stream; one coupled stream in legacy modes);
   d_frame_flags: n bytes or NULL. */
int cb200_decode_raw_dev(cb200_ctx* ctx, const uint8_t* d_rgb, int n, uint32_t flags,
                         uint8_t* d_raw_out, uint8_t* d_frame_flags);

/* Replaces: reed_solomon_stream::write + ReedSolomon::decode -> correct_reed_solomon_decode
   (src/lib/encoder/reed_solomon_stream.h:54-76; src/third_party_lib/libcorrect/src/reed-solomon/decode.c:299-379).
   d_raw: n * raw_bytes; d_data_out: n * data_bytes (a failed block is zero-filled, reed_solomon_stream.h:96-107);
   d_block_ok: n * rs_blocks (1 = decoded) or NULL. */
int cb200_rs_correct_dev(cb200_ctx* ctx, const uint8_t* d_raw, int n, uint8_t* d_data_out, uint8_t* d_block_ok);

/* Replaces: Decoder::decode_fountain into an escrow_buffer_writer, kept in fixed slots
   (src/lib/encoder/Decoder.h:171-189, aligned_stream.h:39-116, escrow_buffer_writer.h:44-60).
   d_chunks: n * chunks_per_frame * chunk_size (slot q of frame f valid iff bit q of d_chunk_mask[f] is set:
   a chunk is dropped when any of its RS blocks failed); d_chunk_mask: n words. */
int cb200_decode_chunks_dev(cb200_ctx* ctx, const uint8_t* d_rgb, int n, uint32_t flags,
                            uint8_t* d_chunks, uint32_t* d_chunk_mask, uint8_t* d_frame_flags);

/* The same with a per-frame choice of preprocessing: frame f is decoded with should_preprocess = (sharpen[f] != 0), exactly as
   Decoder::decode_fountain(img_f, stream, sharpen[f], color_correction) decodes it, and everything that depends on order (the
   CCM carry of CC_FIT, the outputs) stays in batch order.  sharpen: n bytes in HOST memory, read before the call returns (the
   caller may reuse it at once); the call stays enqueue-only.  `flags` must not contain CB200_FLAG_SHARPEN.  A batch of both
   kinds runs K1 twice, once over each kind's frames; a selection of one kind only is the call without / with CB200_FLAG_SHARPEN. */
int cb200_decode_chunks_sharpen_dev(cb200_ctx* ctx, const uint8_t* d_rgb, int n, uint32_t flags, const uint8_t* sharpen,
                                    uint8_t* d_chunks, uint32_t* d_chunk_mask, uint8_t* d_frame_flags);

/* ---- host-pointer entry points: H2D + kernels + D2H, synchronous ---------------------------------------------- */

/* == Decoder(false).decode(img, stream): raw cell bits (Decoder.h:163-168 with _useEcc=false) */
int cb200_decode_raw(cb200_ctx* ctx, const uint8_t* rgb, int n, uint32_t flags, uint8_t* raw_out, uint8_t* frame_flags);
/* == Decoder().decode(img, ofstream): RS-corrected bytes, zeros for failed blocks; returns good bytes per frame in
   good_bytes[n] (may be NULL) */
int cb200_decode(cb200_ctx* ctx, const uint8_t* rgb, int n, uint32_t flags, uint8_t* data_out, uint8_t* block_ok,
                 uint8_t* frame_flags);
/* == Decoder().decode_fountain(img, escrow_buffer_writer): per frame, the good chunks packed densely at
   chunks_out + f * chunks_per_frame * chunk_size, their count in chunk_count[f], bit mask in chunk_mask[f] (may be
   NULL); good bytes = count * chunk_size == the reference's return value (aligned_stream::tellp) */
int cb200_decode_fountain(cb200_ctx* ctx, const uint8_t* rgb, int n, uint32_t flags, uint8_t* chunks_out,
                          uint32_t* chunk_count, uint32_t* chunk_mask, uint8_t* frame_flags);

/* cb200_decode_fountain with a per-frame sharpen selection (n host bytes, as cb200_decode_chunks_sharpen_dev): the batched
   form of the loop `for f: decoder.decode_fountain(img_f, stream, should_preprocess_f, color_correction)` */
int cb200_decode_fountain_sharpen(cb200_ctx* ctx, const uint8_t* rgb, int n, uint32_t flags, const uint8_t* sharpen, uint8_t* chunks_out,
                                  uint32_t* chunk_count, uint32_t* chunk_mask, uint8_t* frame_flags);

/* the same with frames that are already in device memory (the output of cb200_deskew_dev): results to host memory */
int cb200_decode_fountain_from_dev(cb200_ctx* ctx, const uint8_t* d_rgb, int n, uint32_t flags, uint8_t* chunks_out,
                                   uint32_t* chunk_count, uint32_t* chunk_mask, uint8_t* frame_flags);

/* ---- extractor: deskew in front of the decode (SURVEY 8f-2) -------------------------------------------------------

   Replaces: Deskewer::deskew (src/lib/extractor/Deskewer.h:25-40) = cv::getPerspectiveTransform(corners, outputPoints) +
   cv::warpPerspective(img, out, transform, size, cv::INTER_LINEAR) to the mode's image size, as Extractor::extract calls it
   with the four anchor centres Scanner found (src/lib/extractor/Extractor.h:30-46).  Here the caller supplies the corners
   (cb200_scan below finds them on the device) (order: top-left, top-right, bottom-left, bottom-right, as Corners::all()).
   OpenCV's arithmetic is restated bit for bit (pinned against cv2 in tests/test_deskew.py). */

/* cv::getPerspectiveTransform(src, dst): 4 points each (x, y pairs) -> 3x3 double, row-major.  Host only. */
int cb200_perspective_transform(const float* src_xy, const float* dst_xy, double* m9_out);
/* cv::warpPerspective(src, dst, M, Size(image_size_x, image_size_y), INTER_LINEAR) (border constant 0) for n source images of
   src_w x src_h RGB8 in device memory, tightly packed; m9: n x 9 doubles on the HOST (the forward transforms, inverted here as
   warpPerspective does); d_dst: n frames of the context's mode, ready for the cb200_decode_*_dev entry points. */
int cb200_deskew_dev(cb200_ctx* ctx, const uint8_t* d_src, int src_w, int src_h, int n, const double* m9, uint8_t* d_dst);
/* host pointers in and out (H2D + kernel + D2H): what Deskewer::deskew returns */
int cb200_deskew(cb200_ctx* ctx, const uint8_t* src, int src_w, int src_h, int n, const double* m9, uint8_t* dst);
/* Extractor's deskew + Decoder::decode_fountain in one call: camera images (host) and their four anchor centres
   (n x 8 floats) in, fountain chunks out; the deskewed frames stay on the device.  Outputs as cb200_decode_fountain.
   With CB200_FLAG_SHARPEN_IF_NEEDED picture i is sharpened iff its corners fail Corners::is_granular_scale (some side of the
   quadrilateral spans no more than the frame's width in x and its height in y, Corners.h:57-75). */
int cb200_extract_decode_fountain(cb200_ctx* ctx, const uint8_t* src, int src_w, int src_h, int n, const float* corners, uint32_t flags,
                                  uint8_t* chunks_out, uint32_t* chunk_count, uint32_t* chunk_mask, uint8_t* frame_flags);

/* the same with the camera images already in device memory */
int cb200_extract_decode_fountain_dev(cb200_ctx* ctx, const uint8_t* d_src, int src_w, int src_h, int n, const float* corners, uint32_t flags,
                                      uint8_t* chunks_out, uint32_t* chunk_count, uint32_t* chunk_mask, uint8_t* frame_flags);

/* ---- extractor: the anchor scan (SURVEY 8f-2) -------------------------------------------------------------------------

   Replaces: Scanner(img).scan() (src/lib/extractor/Scanner.h:168-174 constructor = preprocess_image(fast): cvtColor(RGB2GRAY) +
   GaussianBlur + Otsu threshold, :146-166, :124-128; Scanner.cpp:182-199 scan = scan_primary + add_bottom_right_corner) for a batch
   of n camera pictures of w x h RGB8, tightly packed.  Results in host memory:
     anchors: n x 4 x 4 int32 = (x, xmax, y, ymax) of each Anchor (Anchor.h:13-18) in the reference's order top-left, top-right,
              bottom-left, bottom-right; entries beyond count[i] are zero.  May be NULL.
     count:   n int32: anchors found (0..4; Extractor::extract needs 4), or -1 if one of the scan's fixed-capacity lists
              overflowed on that picture (thousands of pattern hits: not a photograph of a cimbar code) -- reported, never guessed
     cutoff:  n uint32: filter_candidates' size cutoff (Scanner.cpp:83-105).  May be NULL.
   OpenCV's arithmetic (8-bit GaussianBlur in fixed point with the 3/5/7/9-tap table, Otsu in double precision) and libstdc++'s
   std::sort are restated bit for bit (tests/test_scan_oracle.py pins the CPU restatement to cv2 and to every golden string of
   extractor/test/ScannerTest.cpp; tests/test_gpu_scan.py compares the device with it).  Pictures whose short side is 4500 pixels
   or more (a 17-tap Gaussian) or less than 60 are rejected with CB200_ERR_ARG. */
int cb200_scan(cb200_ctx* ctx, const uint8_t* pictures, int w, int h, int n, int32_t* anchors, int32_t* count, uint32_t* cutoff);
int cb200_scan_dev(cb200_ctx* ctx, const uint8_t* d_pictures, int w, int h, int n, int32_t* anchors, int32_t* count, uint32_t* cutoff);
/* what the last scan call of this context computed on the way: the blurred gray pictures (n x h x w bytes) and their Otsu
   thresholds (Scanner's binarised image is blurred > threshold).  Either pointer may be NULL.  For tests and diagnostics. */
int cb200_scan_blurred(cb200_ctx* ctx, uint8_t* blurred_out, int32_t* thresholds_out, int w, int h, int n);
/* Extractor::extract (src/lib/extractor/Extractor.h:30-46) + Decoder::decode_fountain for n camera pictures in host memory:
   scan -> Corners (the anchors' centres) -> deskew to the mode's frame size -> decode; one H2D copy of the pictures, nothing
   but anchors and chunks comes back.  extract_status: n int32 with the reference's return values -- 0 FAILURE (fewer than four
   anchors; no chunks), 1 SUCCESS, 2 NEEDS_SHARPEN (Corners::is_granular_scale false: the reference's CLI then decodes that
   picture with should_preprocess = true) -- or -1 for a capacity overflow (see cb200_scan).  CB200_FLAG_SHARPEN_IF_NEEDED does
   exactly that per picture (sharpen iff status 2); CB200_FLAG_SHARPEN sharpens every picture.  The other flags apply to the
   whole batch.  The other outputs are as cb200_decode_fountain. */
int cb200_scan_extract_decode_fountain(cb200_ctx* ctx, const uint8_t* pictures, int w, int h, int n, uint32_t flags,
                                       uint8_t* chunks_out, uint32_t* chunk_count, uint32_t* chunk_mask, uint8_t* frame_flags,
                                       int32_t* extract_status);

/* ---- ragged batches: n camera pictures, each of its own size ----------------------------------------------------------

   The reference CLI's decode loop (src/exe/cimbar/cimbar.cpp:124-160) takes files of any sizes -- landscape and portrait photographs
   alternate -- and runs Extractor::extract + Decoder::decode_fountain on each, in order, with one decoder.  These entry points do
   the same in one call.  wh: n x 2 int32 in HOST memory, (w_i, h_i) of picture i; the pictures are tightly packed RGB8.  The host
   entry points take n host pointers (one buffer per picture, e.g. per file; packed into the library's staging buffer with one copy
   each); the _dev entry points take one packed device buffer in which picture i starts at byte 3 * sum_{j<i} w_j h_j.  A uniform
   batch gives exactly what the uniform entry point gives.  CB200_ERR_ARG, before any CUDA call, for n < 0, a null wh or pictures
   (or a null picture pointer), a picture whose short side is under 60 or 4500 and up (the message names the picture's index),
   n > max_frames on the decoding calls, and both sharpen flags together; a bad picture fails the whole call. */

/* cb200_scan for a ragged batch: outputs as cb200_scan, one entry per picture */
int cb200_scan_ragged(cb200_ctx* ctx, const uint8_t* const* pictures, const int32_t* wh, int n, int32_t* anchors, int32_t* count, uint32_t* cutoff);
int cb200_scan_ragged_dev(cb200_ctx* ctx, const uint8_t* d_pictures, const int32_t* wh, int n, int32_t* anchors, int32_t* count, uint32_t* cutoff);
/* cb200_scan_blurred after a ragged scan: the blurred gray pictures back to back (sum_i w_i h_i bytes) and n thresholds */
int cb200_scan_blurred_ragged(cb200_ctx* ctx, uint8_t* blurred_out, int32_t* thresholds_out, const int32_t* wh, int n);
/* cb200_extract_decode_fountain_dev for a ragged batch in device memory, with the caller's corners (n x 8 floats); honours
   CB200_FLAG_SHARPEN_IF_NEEDED as that call does (sharpen iff the corners fail Corners::is_granular_scale) */
int cb200_extract_decode_fountain_ragged_dev(cb200_ctx* ctx, const uint8_t* d_pictures, const int32_t* wh, int n, const float* corners,
                                             uint32_t flags, uint8_t* chunks_out, uint32_t* chunk_count, uint32_t* chunk_mask,
                                             uint8_t* frame_flags);
/* the CLI's decode loop in one call: cb200_scan_extract_decode_fountain for a ragged batch.  Outputs, extract_status and every flag
   behave as there: CB200_FLAG_SHARPEN_IF_NEEDED sharpens exactly the NEEDS_SHARPEN pictures, and the CCM of CB200_FLAG_CC_FIT
   carries from picture to picture in batch order. */
int cb200_scan_extract_decode_fountain_ragged(cb200_ctx* ctx, const uint8_t* const* pictures, const int32_t* wh, int n, uint32_t flags,
                                              uint8_t* chunks_out, uint32_t* chunk_count, uint32_t* chunk_mask, uint8_t* frame_flags,
                                              int32_t* extract_status);

/* ---- enqueue-only camera decode -----------------------------------------------------------------------------------------

   The camera path on the device from end to end: scan, Extractor::extract (one thread per picture), deskew and decode are only
   enqueued on the context's stream, and the call returns without waiting for the device -- so a caller can queue a batch behind
   other work, overlap the copy of the next batch with this one's decode, and hand the records to cb200_gather_push.
     d_pictures: a ragged batch packed in device memory as for cb200_scan_ragged_dev; wh: n x 2 int32 in HOST memory, read before
                 the call returns.
     d_chunks, d_chunk_mask, d_frame_flags (may be NULL): the fixed-slot layout of cb200_decode_chunks_dev -- data_bytes per picture,
                 slot q valid iff bit q of the mask is set.  A picture with status <= 0 gets mask 0.
     d_extract_status: n int32 (4-byte aligned) with cb200_scan_extract_decode_fountain's statuses: -1, 0, 1 or 2.
   Every flag behaves as on cb200_scan_extract_decode_fountain_ragged: CB200_FLAG_SHARPEN_IF_NEEDED sharpens exactly the
   NEEDS_SHARPEN pictures, the CCM of CB200_FLAG_CC_FIT (and CC_SIMPLE's last matrix) carries in batch order, and from one call to
   the next: a call enqueued while an earlier one that may change the CCM is still running takes that CCM from the device.
   CB200_ERR_ARG before any CUDA call, with the checks and messages of the ragged entry points, for null outputs, and for
   CC_SIMPLE with CC_FIT.
   The call never waits for the device, with two exceptions:
     1. a call that has to grow one of the context's buffers waits for the device (cudaFree synchronises); after one call with the
        same or a larger batch (and the same pictures' sizes or smaller) nothing grows;
     2. each call uploads one pinned table (its picture table) from a ring of three slots: a fourth call in flight waits until the
        upload of the first has run.
   The outputs, and the context's scratch buffers, belong to the stream: read them after cb200_sync or an event on that stream. */
int cb200_scan_extract_decode_chunks_ragged_dev(cb200_ctx* ctx, const uint8_t* d_pictures, const int32_t* wh, int n, uint32_t flags,
                                                uint8_t* d_chunks, uint32_t* d_chunk_mask, uint8_t* d_frame_flags, int32_t* d_extract_status);
/* the same for n pictures of one size w x h */
int cb200_scan_extract_decode_chunks_dev(cb200_ctx* ctx, const uint8_t* d_pictures, int w, int h, int n, uint32_t flags, uint8_t* d_chunks,
                                         uint32_t* d_chunk_mask, uint8_t* d_frame_flags, int32_t* d_extract_status);

/* ---- camera pictures in the caller's layout ----------------------------------------------------------------------------------

   One descriptor per picture, so a batch needs no packing: each picture may sit in its own allocation, at any byte address, with
   padding at the end of its rows.  Pixel (x, y) of an interleaved layout starts at data + y * row_pitch + x * channels; in the
   planar layout its R, G and B bytes are at data + y * row_pitch + x, plus 0, 1 and 2 plane_pitch.  A picture decodes exactly as its
   packed RGB copy (cvtColor's BGR2RGB, RGBA2RGB or BGRA2RGB) does: alpha is ignored. */
#define CB200_LAYOUT_RGB        0     /* R G B, 3 bytes per pixel (OpenCV after cvtColor(BGR2RGB), numpy / torch HWC) */
#define CB200_LAYOUT_BGR        1     /* B G R, 3 bytes per pixel (an OpenCV Mat as imread gives it) */
#define CB200_LAYOUT_RGBA       2     /* R G B A, 4 bytes per pixel (browser ImageData, Android RGBA_8888) */
#define CB200_LAYOUT_BGRA       3     /* B G R A, 4 bytes per pixel (capture and interop surfaces) */
#define CB200_LAYOUT_RGB_PLANAR 4     /* three planes R, G, B of 1 byte per pixel (torch CHW, torchvision.io.decode_jpeg) */
typedef struct cb200_picture {
    const uint8_t* data;              /* device address of pixel (0, 0) (of the R plane for CB200_LAYOUT_RGB_PLANAR) */
    int32_t w, h;
    int64_t row_pitch;                /* bytes from one row to the next: >= w x channels (3, 4, or 1 per plane) */
    int64_t plane_pitch;              /* CB200_LAYOUT_RGB_PLANAR: bytes from one plane to the next, >= h x row_pitch; otherwise ignored */
    int32_t layout;                   /* CB200_LAYOUT_* */
} cb200_picture;
/* cb200_scan_extract_decode_chunks_ragged_dev for n pictures described by pics[0 .. n) (HOST memory, read before the call returns):
   the outputs, the flags, the CCM carry, cb200_camera_transforms, the sharpen selection and the statuses are exactly those of that
   call on the packed RGB batch, and it waits for the device only as that call does (one picture table through the upload ring).
   The pictures belong to the stream until it passes the call.  CB200_ERR_ARG, before any CUDA call, naming the picture: n < 0 or
   n > max_frames, a null pics or data pointer, an unknown layout, a size the scan does not take (short side 60 .. 4499), a negative
   pitch, a row pitch below w x channels, planes that overlap (plane pitch below h x row pitch), a picture that spans 4 GB or more,
   and the flags and outputs cb200_scan_extract_decode_chunks_ragged_dev refuses. */
int cb200_scan_extract_decode_chunks_pictures_dev(cb200_ctx* ctx, const cb200_picture* pics, int n, uint32_t flags, uint8_t* d_chunks,
                                                  uint32_t* d_chunk_mask, uint8_t* d_frame_flags, int32_t* d_extract_status);
/* ---- receivers: pictures of many decoders in one batch ------------------------------------------------------------------------

   A batch of the calls above is one decoder: under CC_FIT a picture without a usable header takes the matrix of the picture before
   it, and CC_SIMPLE leaves the last picture's matrix as the context's CCM.  The _receivers_dev calls decode pictures of many
   independent decoders ("receivers", e.g. the users of a decode service) in one batch, each with its own colour-correction state.
   cb200_receiver_state is the state one decoder carries from picture to picture (its CimbDecoder's CCM, CimbDecoder.cpp:69-85): the
   matrix, row-major, and whether it is active.  The caller keeps one per receiver in device memory. */
typedef struct cb200_receiver_state {
    float ccm[9];
    uint32_t active;                  /* nonzero: the matrix is used; 0: no CCM (cb200_set_ccm(NULL)) */
} cb200_receiver_state;               /* 40 bytes */
/* Picture i belongs to receiver receiver_of[i] (HOST memory, n entries, read before the call returns).  For every receiver r, the
   outputs for r's pictures equal, bit for bit, those of the matching direct call on a context whose CCM was set to d_states[r]
   (cb200_set_ccm(ccm), or NULL when active == 0) run on r's pictures alone, in batch order: cb200_decode_chunks_dev for the frame
   call, cb200_scan_extract_decode_chunks_pictures_dev for the camera call (records, masks, frame flags, extract statuses,
   cb200_camera_transforms).  After the call d_states[r] holds what cb200_get_ccm of that context would return:
     CC_FIT (a mode that fits): r's last fit in this call, else its entry matrix, with the activity of r's last picture;
     CC_SIMPLE: the matrix of r's last picture, active;
     no CC flag, or CC_FIT in a legacy mode (which never fits): unchanged.
   Receivers without a picture in the call are neither read nor written.  The call neither reads nor changes the context's own CCM
   (cb200_get_ccm and the next direct call are as if it had not run); cb200_get_frame_ccms reports the matrix each picture was decoded
   with.  Enqueue-only like the calls they mirror: the camera call makes one upload (the receiver map travels with the picture table),
   the frame call one (the map).  d_states belongs to the stream until it passes the call.
   CB200_ERR_ARG, before any CUDA call: a null receiver_of, a null d_states or one not 4-byte aligned, n_receivers < 1, a receiver
   index outside [0, n_receivers) (naming the picture), a context linked to a CCM chain (the chain carries one decoder's CCM across
   ranks), and everything the mirrored call refuses.  Several modes in one call: use one context per mode. */
int cb200_decode_chunks_receivers_dev(cb200_ctx* ctx, const uint8_t* d_rgb, int n, uint32_t flags, const int32_t* receiver_of,
                                      int n_receivers, cb200_receiver_state* d_states, uint8_t* d_chunks, uint32_t* d_chunk_mask,
                                      uint8_t* d_frame_flags);
int cb200_scan_extract_decode_chunks_receivers_dev(cb200_ctx* ctx, const cb200_picture* pics, int n, uint32_t flags,
                                                   const int32_t* receiver_of, int n_receivers, cb200_receiver_state* d_states,
                                                   uint8_t* d_chunks, uint32_t* d_chunk_mask, uint8_t* d_frame_flags,
                                                   int32_t* d_extract_status);
/* ---- camera plans: the enqueue-only camera call captured once in a CUDA graph ----------------------------------------------

   A plan is cb200_scan_extract_decode_chunks_ragged_dev for n pictures of sizes wh, with these flags and these device buffers,
   captured once: each cb200_camera_plan_launch is one cudaGraphLaunch on the context's current stream, with no host work per batch,
   and the graph itself (cb200_camera_plan_graph) can be embedded in a larger one.  The buffers are bound when the plan is created:
   the caller writes each batch's pictures into d_pictures in stream order before the launch; two plans on one context double-buffer.
   A launch gives what the direct call would give at that point of the context's call sequence: records, masks, frame flags, statuses,
   cb200_camera_transforms, cb200_get_ccm and cb200_get_frame_ccms.  Its CCM always comes from the device (the last matrix the context
   kept or was given, which the context keeps current there while plans exist); CC_SIMPLE's last matrix and CC_FIT's carry reach the
   host as after an enqueue-only call, pending behind an event.
     create: the argument checks and messages of cb200_scan_extract_decode_chunks_ragged_dev, all before any CUDA call, and
             CB200_ERR_ARG for n == 0 and for a context attached to a CCM chain.  Every context buffer the graph uses is grown to this
             batch's size here; with the buffers already that large, create does not wait for the device.
     launch: outside a capture, the context's host state (pending CCM, the transforms' picture count) follows each launch as it
             follows a direct call.  Inside a stream capture of the context's stream (torch.cuda.graph), the graph goes into that
             capture as a child node and the host state is left alone: replays of an enclosing graph, or of one the plan's graph was
             added to, update device memory only.  Such a graph reads the plan's buffers, so the plan must outlive it.
   While a plan exists, the buffers its graph uses are frozen: a call on the context that would grow one fails with CB200_ERR_ARG
   before any CUDA call, naming the buffer.  cb200_destroy destroys the context's plans; cb200_set_timing does not time launches,
   and cb200_launch_count counts a launch as the kernels in its graph. */
typedef struct cb200_camera_plan cb200_camera_plan;
int cb200_camera_plan_create(cb200_ctx* ctx, const int32_t* wh, int n, uint32_t flags, const uint8_t* d_pictures, uint8_t* d_chunks,
                             uint32_t* d_chunk_mask, uint8_t* d_frame_flags, int32_t* d_extract_status, cb200_camera_plan** out);
/* one cudaGraphLaunch on the context's current stream (or a child node in its capture) */
int cb200_camera_plan_launch(cb200_camera_plan* plan);
/* the plan's cudaGraph_t, owned by the plan (for cudaGraphAddChildGraphNode, which copies it) */
int cb200_camera_plan_graph(cb200_camera_plan* plan, void** cuda_graph);
int cb200_camera_plan_destroy(cb200_camera_plan* plan);
/* ---- receivers camera plans: cb200_scan_extract_decode_chunks_receivers_dev captured once ---------------------------------------

   A camera plan (above) over pictures of many receivers, for a decode service that replays fixed-size batches.  The pictures are
   bound as descriptors (pics, HOST memory, read at create: any layout and pitch, one allocation per picture; the caller writes each
   batch's pixels into them in stream order before the launch).  d_receiver_of: n int32 in DEVICE memory, bound at create and read
   when each launch runs, so the caller rewrites it per batch (a copy on the stream, or a kernel in the same capture).  d_states
   (n_receivers entries, cb200_receiver_state) and n_receivers are bound at create.
   At each launch, let P be the slots whose d_receiver_of lies in [0, n_receivers).  Every output for P, and every receiver's state
   afterwards, equals bit for bit what cb200_scan_extract_decode_chunks_receivers_dev gives on the pictures of P alone, in batch
   order, with the same receivers and states: records, masks, frame flags, extract statuses, cb200_camera_transforms and
   cb200_get_frame_ccms.  A slot whose receiver lies outside [0, n_receivers) (-1 by convention) is EMPTY: it is still scanned and
   decoded (it costs GPU time), but it reads and writes no state, its mask is 0 and its extract status CB200_EXTRACT_EMPTY.  So a
   plan of n slots runs part-full batches, and an index that is out of range at replay time -- which no check at create can see --
   leaves its slot empty instead of touching memory outside d_states.  The map is grouped by receiver on the device at each launch:
   one kernel more than the direct call, with work and memory that depend on n, not on n_receivers.
   Like the receivers calls, a launch neither reads nor changes the context's own CCM (the plan keeps no CCM); it sets the
   transforms' picture count and cb200_get_frame_ccms's frame count as the direct call does.  Launched, embedded, frozen, counted
   and destroyed as every camera plan.
   CB200_ERR_ARG, before any CUDA call: a null d_receiver_of or one not 4-byte aligned, a null d_states or one not 4-byte aligned,
   n_receivers < 1, everything else cb200_scan_extract_decode_chunks_receivers_dev refuses, n == 0 and a context attached to a CCM
   chain. */
#define CB200_EXTRACT_EMPTY (-3)      /* extract status of an empty slot of a receivers plan */
int cb200_camera_plan_create_receivers(cb200_ctx* ctx, const cb200_picture* pics, int n, uint32_t flags, const int32_t* d_receiver_of,
                                       int n_receivers, cb200_receiver_state* d_states, uint8_t* d_chunks, uint32_t* d_chunk_mask,
                                       uint8_t* d_frame_flags, int32_t* d_extract_status, cb200_camera_plan** out);
/* ---- receivers camera plans over device descriptors: any sizes, layouts and buffers per batch ------------------------------------

   cb200_camera_plan_create_receivers with the picture descriptors in DEVICE memory too: d_pics is n descriptors of type
   cb200_picture, 40 bytes each, 8-byte aligned, read when each launch runs, like d_receiver_of.  So every slot may hold a picture of another size, layout and
   buffer at every launch (torchvision.io.decode_jpeg outputs where they lie, say); the caller writes the descriptors in stream order
   before the launch (one n x 40-byte copy, or a kernel in the same capture).  bounds (HOST, read at create) is the range of pictures
   the plan is sized for: short side in [min_short, max_short], long side at most max_long.  Everything else is as for
   cb200_camera_plan_create_receivers.  At each launch:
     EMPTY slot: its receiver lies outside [0, n_receivers), exactly as there.  Its descriptor is not read (unused slots need not be
             filled); status CB200_EXTRACT_EMPTY, mask 0, no state read or written.
     REFUSED slot: a non-empty slot whose descriptor a direct call would refuse (a null data pointer, an unknown layout, a negative
             pitch, a row pitch below w x channels, overlapping planes, a span of 4 GB or more) or that lies outside the bounds.  Status
             CB200_EXTRACT_REFUSED, and otherwise as an empty slot.  No memory behind a refused or empty descriptor is read: the plan
             scans a small black picture of its own in that slot's place.
     the others: every output and every state afterwards equal bit for bit what cb200_scan_extract_decode_chunks_receivers_dev gives
             on those descriptors alone, in slot order (records, masks, frame flags, statuses, cb200_camera_transforms).
   The graph is the same for every descriptor set: a kernel at its head checks the descriptors and builds the picture table, and the
   blur reads its tile lists from there.  The scan's buffers are sized from the bounds: n x max_long x max_short blurred bytes.
   CB200_ERR_ARG, before any CUDA call, naming the cause: the receiver arguments as for cb200_camera_plan_create_receivers; the flags;
   n < 0; a null d_pics or one not 8-byte aligned; null bounds; min_short < 60; max_short > 4499 (the scan's 9-tap limit);
   min_short > max_short; max_long < max_short; bounds whose blur tiles or scan rows would not fit 31 bits; then everything else
   cb200_camera_plan_create_receivers refuses except the descriptors' contents. */
typedef struct cb200_picture_bounds { int32_t min_short, max_short, max_long; } cb200_picture_bounds;
#define CB200_EXTRACT_REFUSED (-4)    /* extract status of a plan slot whose descriptor the launch refused */
int cb200_camera_plan_create_receivers_pictures_dev(cb200_ctx* ctx, const cb200_picture* d_pics, int n, const cb200_picture_bounds* bounds,
                                                    uint32_t flags, const int32_t* d_receiver_of, int n_receivers,
                                                    cb200_receiver_state* d_states, uint8_t* d_chunks, uint32_t* d_chunk_mask,
                                                    uint8_t* d_frame_flags, int32_t* d_extract_status, cb200_camera_plan** out);
/* ---- per-receiver decode flags: each receiver's sharpen policy and colour correction from a device table -----------------------

   A decode service whose sessions differ in their settings (the web receiver sharpens every picture with CC_FIT, the CLI guesses
   sharpening, CB200_FLAG_SHARPEN_IF_NEEDED, with any colour correction) decodes them in one batch with a receiver flags table:
   d_receiver_flags, n_receivers uint32 words in DEVICE memory, 4-byte aligned, read in stream order by the direct call and when each
   launch runs by the plan (it is bound at create, so a session changes its settings between launches by writing its own word).
   Word r holds receiver r's per-receiver bits: at most one of CB200_FLAG_SHARPEN / CB200_FLAG_SHARPEN_IF_NEEDED and at most one of
   CB200_FLAG_CC_SIMPLE / CB200_FLAG_CC_FIT.  The call's own flags keep every other bit (CB200_FLAG_NO_INTERLEAVE, NO_FALLBACK) and
   may hold none of those four.
     valid word: receiver r's pictures get, bit for bit, what the mirrored call gives on r's pictures alone, in batch order, with
             flags | d_receiver_flags[r]: records, masks, frame flags, extract statuses, cb200_camera_transforms,
             cb200_get_frame_ccms, and d_states[r] afterwards.
     invalid word (any other bit, or both bits of one pair): r's pictures get status CB200_EXTRACT_REFUSED, mask 0 and a zeroed
             record; d_states[r] is neither read nor written.
   Everything else is as for the mirrored function: empty slots in the plan, receivers without a picture, the context's CCM.  Every
   picture takes the fitted-CCM route (mean colours, then the colour decision per picture with its receiver's matrix), so a uniform
   table costs about one CC_FIT call.
   CB200_ERR_ARG, before any CUDA call, naming the cause: a null d_receiver_flags or one not 4-byte aligned; a per-receiver bit in
   flags; then everything the mirrored function refuses, in its order.
   cb200_scan_extract_decode_chunks_receivers_flags_dev mirrors cb200_scan_extract_decode_chunks_receivers_dev;
   cb200_camera_plan_create_receivers_pictures_flags_dev mirrors cb200_camera_plan_create_receivers_pictures_dev;
   cb200_detect_scan_extract_decode_chunks_receivers_flags_dev mirrors cb200_detect_scan_extract_decode_chunks_receivers_dev, and
   cb200_camera_plan_create_detect_receivers_pictures_flags_dev mirrors cb200_camera_plan_create_detect_receivers_pictures_dev (below):
   one table serves every candidate mode, and for a valid word the contract also covers modes, mode masks and every mode's table.  A
   refused receiver's pictures also get mode -1 and a zeroed mode-mask row, and no mode's table is read or written for it. */
int cb200_scan_extract_decode_chunks_receivers_flags_dev(cb200_ctx* ctx, const cb200_picture* pics, int n, uint32_t flags,
                                                         const int32_t* receiver_of, int n_receivers, cb200_receiver_state* d_states,
                                                         const uint32_t* d_receiver_flags, uint8_t* d_chunks, uint32_t* d_chunk_mask,
                                                         uint8_t* d_frame_flags, int32_t* d_extract_status);
int cb200_camera_plan_create_receivers_pictures_flags_dev(cb200_ctx* ctx, const cb200_picture* d_pics, int n, const cb200_picture_bounds* bounds,
                                                          uint32_t flags, const int32_t* d_receiver_of, int n_receivers,
                                                          cb200_receiver_state* d_states, const uint32_t* d_receiver_flags, uint8_t* d_chunks,
                                                          uint32_t* d_chunk_mask, uint8_t* d_frame_flags, int32_t* d_extract_status,
                                                          cb200_camera_plan** out);
/* cb200_camera_plan_create_detect_receivers (below) with its descriptors in DEVICE memory too, read at each launch within bounds, as
   above.  A slot is EMPTY exactly as in that plan (receiver out of range, or no candidate bit below n_modes): its descriptor is not
   read.  A non-empty slot whose descriptor is refused as above gets status CB200_EXTRACT_REFUSED and otherwise what an empty slot
   gets: mode -1, mask 0, a zeroed record and mode-mask row, no state of any mode read or written.  The other slots equal bit for bit
   what cb200_detect_scan_extract_decode_chunks_receivers_dev gives on those descriptors alone, in slot order: records, masks,
   statuses, modes, mode masks and every mode's table.  CB200_ERR_ARG, before any CUDA call: n_modes, the flags, then d_pics and
   bounds as above, then everything else cb200_camera_plan_create_detect_receivers refuses except the descriptors' contents. */
int cb200_camera_plan_create_detect_receivers_pictures_dev(cb200_ctx* const* ctxs, int n_modes, const cb200_picture* d_pics, int n,
                                                           const cb200_picture_bounds* bounds, uint32_t flags, const uint32_t* d_candidates,
                                                           const int32_t* d_receiver_of, int n_receivers, cb200_receiver_state* const* d_states,
                                                           uint8_t* d_chunks, uint32_t* d_chunk_mask, int32_t* d_extract_status,
                                                           int32_t* d_mode, uint32_t* d_mode_masks, cb200_camera_plan** out);
/* the receiver flags forms of the detect receivers call and its plan over device descriptors (see "per-receiver decode flags" above):
   d_receiver_flags follows d_states */
int cb200_detect_scan_extract_decode_chunks_receivers_flags_dev(cb200_ctx* const* ctxs, int n_modes, const cb200_picture* pics, int n,
                                                                uint32_t flags, const uint32_t* candidates, const int32_t* receiver_of,
                                                                int n_receivers, cb200_receiver_state* const* d_states,
                                                                const uint32_t* d_receiver_flags, uint8_t* d_chunks, uint32_t* d_chunk_mask,
                                                                int32_t* d_extract_status, int32_t* d_mode, uint32_t* d_mode_masks);
int cb200_camera_plan_create_detect_receivers_pictures_flags_dev(cb200_ctx* const* ctxs, int n_modes, const cb200_picture* d_pics, int n,
                                                                 const cb200_picture_bounds* bounds, uint32_t flags, const uint32_t* d_candidates,
                                                                 const int32_t* d_receiver_of, int n_receivers,
                                                                 cb200_receiver_state* const* d_states, const uint32_t* d_receiver_flags,
                                                                 uint8_t* d_chunks, uint32_t* d_chunk_mask, int32_t* d_extract_status,
                                                                 int32_t* d_mode, uint32_t* d_mode_masks, cb200_camera_plan** out);
/* ---- auto mode: the sender's mode detected by decoding ----------------------------------------------------------------------

   The receiver's auto mode (the reference's web receiver tries 66, 68, 67 and 4 and keeps the first mode under which a frame gives
   a chunk): the camera path of cb200_scan_extract_decode_chunks_ragged_dev under several candidate modes in one enqueue-only call.
     ctxs, n_modes: 1 .. 5 contexts the caller created, one per mode, in priority order.  Each keeps its own CCM
                 (cb200_get_ccm / cb200_set_ccm / cb200_get_frame_ccms work on it as before).
     d_pictures, wh, n, flags: as on cb200_scan_extract_decode_chunks_ragged_dev; the call runs on the contexts' stream.
     d_mode:     n int32: the index into ctxs of the first context whose decode of picture i accepted a chunk (mask != 0), or -1 when
                 no mode did (a picture that fails extraction included).
     d_chunks:   n fixed slots of the largest data_bytes of the set (8750 with mode 8, 7500 with 68 or 4): slot i holds picture
                 i's record under its detected mode in that mode's fixed-slot layout, zeros after it and in the whole slot for -1.
     d_chunk_mask: that mode's mask (0 for -1); d_extract_status: the extract status under the detected mode, under ctxs[0] for -1.
     d_mode_masks: NULL, or n x n_modes uint32: every mode's mask of every picture (picture-major).
   Exactness: every context is left where cb200_scan_extract_decode_chunks_ragged_dev on it with these pictures and flags would
   leave it -- records, masks, statuses, transforms, CCM carry (a wrong-mode decode moves that mode's CCM as a direct call would).
   The output only selects among those results.
   Sharing: the anchor scan runs once (on ctxs[0]'s scratch); each frame geometry (68 / 4 / 8: 1024 x 1024; 67; 66) is deskewed and
   walked once, on the group's first context, and the other modes of the geometry colour that walk's positions with their own
   palette and CCM.  K1, colours, RS and the masks run per mode.  With more than one geometry the geometries run on side streams
   forked from the contexts' stream and joined back into it before the selection, so their walks overlap on the device.
   CB200_ERR_ARG before any CUDA call, naming the violation: n_modes outside 1 .. 5, a null context, two contexts of one mode, contexts
   on different devices or streams, a context attached to a CCM chain or with live camera plans, n above a context's max_frames, a
   null output other than d_mode_masks, and the flag and picture checks of cb200_scan_extract_decode_chunks_ragged_dev.  Waits for
   the device as that call does (a buffer that grows, the upload ring of ctxs[0]).  Not capturable in a camera plan; graph replay
   of auto mode is cb200_camera_plan_create_detect_receivers, over receiver tables instead of the contexts' own CCM. */
int cb200_detect_scan_extract_decode_chunks_dev(cb200_ctx* const* ctxs, int n_modes, const uint8_t* d_pictures, const int32_t* wh, int n,
                                                uint32_t flags, uint8_t* d_chunks, uint32_t* d_chunk_mask, int32_t* d_extract_status,
                                                int32_t* d_mode, uint32_t* d_mode_masks);
/* ---- auto mode for receivers: each picture under its receiver's candidate modes ------------------------------------------------

   The auto-mode call for a batch of many receivers (a decode service's sessions, some still detecting their sender's mode, others
   locked to one), in one enqueue-only call.
     ctxs, n_modes: as on cb200_detect_scan_extract_decode_chunks_dev (1 .. 5 contexts, one per mode, priority order).
     pics, n, flags: as on cb200_scan_extract_decode_chunks_receivers_dev (descriptors in any layout and pitch).
     candidates: HOST, n entries, read before the call returns: picture i is decoded under ctxs[k] when bit k is set.  NULL: every
                 picture under every mode.
     receiver_of, n_receivers: HOST, n entries in [0, n_receivers), as on the receivers calls.
     d_states:   a HOST array of n_modes pointers, each to a DEVICE table of n_receivers cb200_receiver_state: mode k's state of every
                 receiver.  The n_modes tables must not overlap.
     d_chunks, d_chunk_mask, d_extract_status, d_mode, d_mode_masks: as on the detect call.
   Contract.  Let P_k be the pictures whose candidates have bit k set, in batch order.  For every k, every output for the pictures of
   P_k, and d_states[k] afterwards, equals bit for bit what cb200_scan_extract_decode_chunks_receivers_dev(ctxs[k], P_k's
   descriptors, P_k's receivers, d_states[k]) gives: records, masks, frame flags, extract statuses, states.  d_mode[i] is the first k
   in priority order with i in P_k and a nonzero mask, or -1; d_chunks slot i holds that mode's record as on the detect call;
   d_extract_status[i] is the status under d_mode[i], or under picture i's first candidate for -1; d_mode_masks[i][k] is 0 when i is
   not in P_k.  As on the receivers calls, no context's own CCM is read or changed; as on the detect call, a wrong-mode decode moves
   that mode's receiver state (a receiver with every candidate bit advances every mode's table).  cb200_camera_transforms and
   cb200_get_frame_ccms on the contexts are not part of the contract after this call.
   Sharing: one anchor scan over all n pictures; each frame geometry extracts, deskews and walks only the pictures that some of its
   modes decode, once, on side streams as in the detect call, and a geometry none of whose modes has pictures launches nothing.  So a
   batch locked to one mode pays for that mode's geometry only.  K1, colours, CCM, RS and masks run per mode with that mode's receiver
   table; a picture of the geometry's sub-batch that the mode does not decode is an empty slot of that table, as in a receivers plan.
   The lists travel in the one upload of the picture table.
   CB200_ERR_ARG before any CUDA call, naming the violation: everything the detect call refuses (n_modes, flags, null outputs and the
   context checks); everything cb200_scan_extract_decode_chunks_receivers_dev refuses on the pictures and receivers (descriptors,
   sizes, spans, a null receiver_of, n_receivers < 1, a receiver out of range, naming the picture); a candidates entry that is 0 or
   has a bit at or above n_modes (naming the picture); a null d_states, a null or not 4-byte aligned table (naming it); two tables
   whose n_receivers-entry ranges overlap (their modes may run on different streams).  Not capturable in a camera plan itself: its
   plan is cb200_camera_plan_create_detect_receivers, below. */
int cb200_detect_scan_extract_decode_chunks_receivers_dev(cb200_ctx* const* ctxs, int n_modes, const cb200_picture* pics, int n,
                                                          uint32_t flags, const uint32_t* candidates, const int32_t* receiver_of,
                                                          int n_receivers, cb200_receiver_state* const* d_states, uint8_t* d_chunks,
                                                          uint32_t* d_chunk_mask, int32_t* d_extract_status, int32_t* d_mode,
                                                          uint32_t* d_mode_masks);
/* ---- detect receivers camera plans: the auto mode for receivers captured once ---------------------------------------------------

   cb200_detect_scan_extract_decode_chunks_receivers_dev captured once over n fixed slots, for a decode service whose sessions are
   partly in auto mode and which replays its batches from a graph.
     bound at create: ctxs, n_modes, the picture descriptors (pics, HOST, read at create; the caller writes each batch's pixels into
                 them in stream order before the launch), flags, n_receivers, the n_modes state tables (d_states: a HOST array of
                 DEVICE pointers, read at create) and the outputs.
     d_candidates: n uint32 in DEVICE memory, or NULL for every mode; d_receiver_of: n int32 in DEVICE memory.  Both are read when
                 each launch runs, so the caller rewrites them per batch (a copy on the stream, or a kernel in the same capture).
   At a launch, slot i is EMPTY when its receiver lies outside [0, n_receivers) or its candidates have no bit below n_modes (higher
   bits are ignored).  For every mode k let P_k be the non-empty slots with bit k set, in slot order.  Every output for the non-empty
   slots, and every mode's state table afterwards, equals bit for bit what the direct call gives on the non-empty slots alone, in
   order: records, masks, extract statuses, d_mode, d_mode_masks.  An empty slot gets mode -1, mask 0, a zeroed record slot, a
   d_mode_masks row of zeros and status CB200_EXTRACT_EMPTY, and reads and writes no state: an index that is out of range at replay
   time never reaches memory outside a table.  A launch neither reads nor changes any context's own CCM or host CCM state.
   How: a kernel at the head of the graph builds every list of the direct call from the two device arrays, over all n slots (slot i is
   picture i in every geometry, and a slot a mode does not decode is an empty slot of that mode's receiver map).  A slot that no mode
   of a geometry decodes is skipped by that geometry's exact walk, so a batch locked to one geometry walks that geometry only; its
   K1, RS and list kernels still run on the absent slots (deskew included), which costs little next to a walk.  The geometries are
   parallel branches of the graph.
   The plan is registered with every one of its contexts: each freezes the buffers the graph uses (the detect call's own included),
   cb200_destroy on any of them destroys the plan, and cb200_camera_plan_destroy unregisters it from all.  Launched (on ctxs[0]'s
   stream), embedded, counted and destroyed as every camera plan; cb200_launch_count counts a launch as the kernels of its graph, the
   same for every map and every candidate pattern.
   CB200_ERR_ARG, before any CUDA call, naming the cause: everything the direct call refuses except the contents of the candidates
   and of the map; a null d_receiver_of or one not 4-byte aligned; a d_candidates not 4-byte aligned; n == 0 and a null out; any
   context attached to a CCM chain.  Unlike the direct call, contexts with live camera plans are accepted when no buffer has to grow
   (so two plans on the same contexts double-buffer the pixel uploads); a buffer that would grow is refused, naming it. */
int cb200_camera_plan_create_detect_receivers(cb200_ctx* const* ctxs, int n_modes, const cb200_picture* pics, int n, uint32_t flags,
                                              const uint32_t* d_candidates, const int32_t* d_receiver_of, int n_receivers,
                                              cb200_receiver_state* const* d_states, uint8_t* d_chunks, uint32_t* d_chunk_mask,
                                              int32_t* d_extract_status, int32_t* d_mode, uint32_t* d_mode_masks,
                                              cb200_camera_plan** out);
/* ---- JPEG files in: the CLI's input, decoded on the device ---------------------------------------------------------------

   Replaces: cv::imread(file) + cv::cvtColor(BGR2RGB) (src/exe/cimbar/cimbar.cpp:132-133) for a batch of JPEG files in host memory:
   the output is byte for byte the RGB8 picture cv2.imread + cvtColor(BGR2RGB) returns (libjpeg-turbo's JDCT_ISLOW IDCT, fancy
   upsampling and fixed-point YCbCr -> RGB, and the EXIF orientation as imread applies it).
     files, sizes: n pointers to whole JPEG files and their sizes in bytes, in HOST memory; read before the call returns.
   Supported: baseline, extended-sequential Huffman and progressive (SOF0 / SOF1 / SOF2), 8-bit samples, one component (grey: the
   three channels are equal) or three YCbCr components (JFIF, no APP marker, or Adobe APP14 with transform 1), luma sampling 1x1,
   2x1, 1x2 or 2x2 with chroma 1x1 (4:4:4, 4:2:2, 4:4:0, 4:2:0), any restart interval, EXIF orientation 1-8, and output sizes the
   camera path accepts (short side 60 .. 4499).  Anything else -- arithmetic coding, 12-bit, lossless, hierarchical, CMYK, Adobe
   transform 0 / 2, other sampling layouts such as 4:1:1, a progressive script that leaves the first coefficients incomplete,
   truncated headers, bytes that are not a JPEG file -- fails the whole call with CB200_ERR_ARG before any CUDA call, and
   cb200_last_error names the picture and the reason.  Entropy-coded data that turn out corrupt or truncated are found on the
   device: that picture gets status -2 (and is written black); the other pictures are unaffected. */

/* the output size of one file (after the EXIF orientation), or CB200_ERR_ARG with the refusal reason.  Host only: no context,
   no CUDA call */
int cb200_jpeg_info(const uint8_t* file, uint64_t size, int32_t* w, int32_t* h);
/* enqueue-only decode of n files into d_rgb_out, the packed ragged RGB8 batch of the _ragged_dev entry points: picture i at byte
   3 * sum_{j<i} w_j h_j (sizes as cb200_jpeg_info).  d_status (may be NULL): n int32 in device memory, 0 = decoded, -2 = corrupt
   data.  Waits for the device only as cb200_scan_extract_decode_chunks_ragged_dev does (a buffer that grows, the upload ring). */
int cb200_jpeg_decode_dev(cb200_ctx* ctx, const uint8_t* const* files, const uint64_t* sizes, int n, uint8_t* d_rgb_out, int32_t* d_status);
/* cb200_jpeg_decode_dev into a context buffer, then exactly cb200_scan_extract_decode_chunks_ragged_dev on the decoded pictures:
   the same flags, CCM carry across calls, fixed-slot records, statuses and wait rules, plus extract status -2 and mask 0 for a
   picture with corrupt data (which is otherwise treated as the black picture it decodes to: a status-0 picture).  Checks as
   cb200_scan_extract_decode_chunks_ragged_dev, all before any CUDA call.  The files and their descriptors go up from a ring of
   three pinned buffers of the JPEG calls (each grows to the largest batch's compressed size), the scan's picture table from the
   context's ring: one slot of each per call, so, as on the RGB call, a fourth call in flight waits until the first one's
   uploads have run. */
int cb200_jpeg_scan_extract_decode_chunks_dev(cb200_ctx* ctx, const uint8_t* const* files, const uint64_t* sizes, int n, uint32_t flags,
                                              uint8_t* d_chunks, uint32_t* d_chunk_mask, uint8_t* d_frame_flags, int32_t* d_extract_status);

/* ---- PNG files decoded on the device (cv::imread + cvtColor(BGR2RGB) of the reference CLI, for PNG) -------------------------
   The same three entry points for PNG files, byte for byte cv2.cvtColor(cv2.imread(file, IMREAD_COLOR), COLOR_BGR2RGB) as
   OpenCV 4.13 with libpng 1.6 gives it: grey replicated, palettes looked up (an index past PLTE is black), alpha dropped (tRNS and
   bKGD change nothing), 16 bit truncated to its high byte, gAMA / sRGB / iCCP ignored, the eXIf orientation applied as for JPEG.
   Supported: non-interlaced files of colour type 0 (1, 2, 4, 8, 16 bit), 2 (8, 16), 3 (1, 2, 4, 8), 4 (8, 16) and 6 (8, 16), any
   number and size of consecutive IDAT chunks, every deflate block type, ancillary chunks (skipped), and output sizes the camera path
   accepts (short side 60 .. 4499).  Refused with CB200_ERR_ARG before any CUDA call, cb200_last_error naming the picture and the
   reason: a bad signature; a missing, repeated, misplaced or invalid IHDR or a bad CRC in it; colour type 3 without PLTE, a repeated
   PLTE, a PLTE after IDAT, of a bad size or with a bad CRC; an unknown critical chunk or an invalid chunk type; Adam7 interlace;
   APNG (acTL, fcTL, fdAT); IDAT chunks that are not consecutive; more than one eXIf chunk; an invalid zlib header or a preset
   dictionary; a truncated file (no IEND); a width or height above 1 000 000 (libpng's limit) or more than 2^30 pixels (OpenCV's).
   Found on the device, status -2 and a black picture, the other pictures unaffected: an IDAT CRC mismatch, an invalid block type,
   stored LEN / NLEN that do not match, bad code lengths, a code not in the table, a distance before the output or past zlib's
   window as libpng calls zlib (the window of the zlib header, row by row), a stream that ends before its Adler-32 or gives fewer
   bytes than the rows, a filter type above 4, and an Adler-32 mismatch where libpng fails the file for it (the check value read in
   the same 8 KB read of the last IDAT data as the last row).  Corrupt data after the last row that libpng reads in a later zlib
   call (where it only warns) are also reported -2.

   Extracted frames (the encoder's output, the CLI's --no-deskew input) need no entry point of their own: when every file has the
   mode's frame size, the packed ragged batch of cb200_png_decode_dev is the frame batch of cb200_decode_chunks_dev, so
   cb200_png_decode_dev followed by cb200_decode_chunks_dev on the same stream is the CLI's --no-deskew loop on the device. */

/* the output size of one file (after the eXIf orientation), or CB200_ERR_ARG with the refusal reason.  Host only */
int cb200_png_info(const uint8_t* file, uint64_t size, int32_t* w, int32_t* h);
/* enqueue-only decode of n files into d_rgb_out, the packed ragged RGB8 batch: picture i at byte 3 * sum_{j<i} w_j h_j (sizes as
   cb200_png_info).  d_status (may be NULL): n int32 in device memory, 0 = decoded, -2 = corrupt data.  Waits for the device only
   as cb200_jpeg_decode_dev does (a buffer that grows, the upload ring of the PNG calls). */
int cb200_png_decode_dev(cb200_ctx* ctx, const uint8_t* const* files, const uint64_t* sizes, int n, uint8_t* d_rgb_out, int32_t* d_status);
/* cb200_png_decode_dev into a context buffer, then exactly cb200_scan_extract_decode_chunks_ragged_dev on the decoded pictures, with
   extract status -2 and mask 0 for a picture with corrupt data; arguments, flags and wait rules as
   cb200_jpeg_scan_extract_decode_chunks_dev (the PNG calls have a ring of three pinned upload buffers of their own). */
int cb200_png_scan_extract_decode_chunks_dev(cb200_ctx* ctx, const uint8_t* const* files, const uint64_t* sizes, int n, uint32_t flags,
                                             uint8_t* d_chunks, uint32_t* d_chunk_mask, uint8_t* d_frame_flags, int32_t* d_extract_status);

/* diagnostic: the forward transforms (getPerspectiveTransform(corners, output points), n x 9 doubles, row-major) of the first n
   pictures of the last camera call of this context; a picture with status <= 0 has the transform of the output points onto
   themselves.  Synchronises the context's stream. */
int cb200_camera_transforms(cb200_ctx* ctx, double* m9_out, int n);

/* per-cell record of the exact flood walk: what CimbReader::read() hands back, step by step
   (src/lib/cimb_translator/CimbReader.cpp:139-162, PositionData.h:4-9) */
typedef struct cb200_cell_trace {
    uint16_t order;        /* position of this cell in the walk order (0 = first read) */
    int16_t  x, y;         /* drift-adjusted position = PositionData.x / .y */
    uint8_t  drift_offset; /* winning hash id 0..8, 4 = centre */
    uint8_t  distance;     /* best Hamming distance */
} cb200_cell_trace;

/* Replaces: the loop `while (!reader.done()) reader.read(pos)` + `reader.read_color(pos)` of a CimbReader
   (CimbReader.cpp:133-162), always through the exact flood-walk kernel.  Host pointers.
   cellvals_out: n * total_cells bytes (symbol | colour << symbol_bits, linear cell index);
   trace_out: n * total_cells records indexed by cell. */
int cb200_decode_cells(cb200_ctx* ctx, const uint8_t* rgb, int n, uint32_t flags, uint8_t* cellvals_out,
                       cb200_cell_trace* trace_out);

/* Same, for a host that mirrors CimbReader call by call: with means_out != NULL (n * total_cells words, r | g << 8 | b << 16 =
   Cell::mean_rgb of the inner 6x6 at the cell's drift-adjusted position, Cell.h:30-62) the colours are NOT decided here --
   cellvals_out carries the symbols only -- so that CimbReader::read_color can classify them later with the CCM the decoder
   holds by then (after CimbReader::init_ccm): cb200_best_colors on the stored means is CimbDecoder::decode_color.
   CB200_FLAG_CC_SIMPLE still installs the frame's von Kries matrix as the context's CCM (CimbReader.cpp:124-125). */
int cb200_decode_cells_means(cb200_ctx* ctx, const uint8_t* rgb, int n, uint32_t flags, uint8_t* cellvals_out,
                             cb200_cell_trace* trace_out, uint32_t* means_out);

/* ---- single-cell entry points (CimbDecoder API parity; run one tiny kernel) ------------------------------------- */

/* Replaces: CimbDecoder::decode_symbol(const bitmatrix&, drift_offset, best_distance, cooldown)
   (src/lib/cimb_translator/CimbDecoder.cpp:142-147 -> fuzzy_ahash<8> + get_best_symbol :101-132).
   windows: n x 10 rows of 10 bits (uint16 each, bit 9 = leftmost column), cooldown[n] (0xFE = ALL, 0xFF = none).
   out: symbol[n], drift_offset[n], distance[n]. Host pointers. */
int cb200_decode_symbols(cb200_ctx* ctx, const uint16_t* windows, const uint8_t* cooldown, int n,
                         uint8_t* symbol, uint8_t* drift_offset, uint8_t* distance);
/* Replaces: CimbDecoder::get_best_color(r, g, b, color_mode) (CimbDecoder.cpp:168-200) for integer means.
   rgb: n x 3 bytes; out: color[n]. Host pointers. */
int cb200_best_colors(cb200_ctx* ctx, const uint8_t* rgb_means, int n, uint8_t* color);

/* ---- colour correction matrix (the decoder's CCM state) -------------------------------------------------------- */

/* Replaces: CimbDecoder::update_color_correction(cv::Matx<float,3,3>&&) (src/lib/cimb_translator/CimbDecoder.cpp:82-85),
   also what DecoderPlus::load_ccm feeds (src/lib/encoder/DecoderPlus.h:31-42).  m9 = 9 floats, row-major; NULL deactivates
   the CCM (TestableCimbDecoder: internal_ccm() = color_correction()).  While a CCM is active every colour decision of this
   context (all decode entry points and cb200_best_colors) runs color_correction::transform + get_best_color in the
   reference's float32 operation order (chromatic_adaptation/color_correction.h:64-68, CimbDecoder.cpp:168-200). */
int cb200_set_ccm(cb200_ctx* ctx, const float* m9);
/* Replaces: CimbDecoder::get_ccm() (CimbDecoder.cpp:76-80): returns 1 and fills m9 when a CCM is active, else 0.
   After a CB200_FLAG_CC_SIMPLE call this is the last frame's matrix (synchronises the context's stream). */
int cb200_get_ccm(cb200_ctx* ctx, float* m9);

/* Replaces: CimbReader::init_ccm (src/lib/cimb_translator/CimbReader.cpp:169-267) for a host that tracked the fountain header
   itself (CimbReader::update_metadata, CimbReader.cpp:269-280): header6 = _fountainColorHeader as it stands (block id already
   "+1"), radioactive_block_id = _radioactiveBlockId.  rgb: one frame (host pointer), or NULL = the frame the last host-pointer
   call of this context uploaded.  flags: CB200_FLAG_NO_INTERLEAVE or 0.  Samples the header cells of every colour-stream chunk
   and the anchor white on the device and runs the Moore-Penrose fit (OpenCV's float Jacobi SVD restated).  Returns 1 when a
   matrix was fitted -- it is then the context's CCM and copied to m9_out (may be NULL) --, 0 when the reference would have
   returned without one (no header, fewer than four colours seen), negative on error. */
/* the matrices the first n frames of the last call that fitted CCMs (CB200_FLAG_CC_FIT, or a call reading a CCM still in flight)
   were decoded with: n x 9 floats, row-major, and n activity bytes (0: that frame had no CCM).  Synchronises.  CB200_ERR_ARG for
   n beyond that call's frames */
int cb200_get_frame_ccms(cb200_ctx* ctx, int n, float* m9n, uint8_t* active);
int cb200_fit_ccm(cb200_ctx* ctx, const uint8_t* rgb, const uint8_t* header6, uint32_t radioactive_block_id, uint32_t flags, float* m9_out);

/* Replaces: CimbDecoder::get_color(i, color_mode) -> cimbar::getColor(i, num_colors, color_mode)
   (src/lib/cimb_translator/CimbDecoder.cpp:149-152, Common.cpp:122-139): decode palette entry i for 1 << color_bits colours. */
int cb200_palette_color(int color_bits, unsigned color_mode, int i, uint8_t* rgb_out /* 3 bytes */);

/* ---- synthetic input (benchmark support; the inverse of the path) ---------------------------------------------- */

/* cellvals: n * total_cells bytes on the device, value = (colour << symbol_bits) | symbol of linear cell i
   (what CimbWriter::write pastes, src/lib/cimb_translator/CimbWriter.cpp:84-95); d_rgb_out: n frames. */
int cb200_render_frames_dev(cb200_ctx* ctx, const uint8_t* d_cellvals, int n, uint8_t* d_rgb_out);

/* payload: n * data_bytes bytes on the device -> RS-encoded (correct_reed_solomon_encode, libcorrect encode.c:3-35),
   bit-striped (Encoder::encode_next, src/lib/encoder/Encoder.h:69-129) and interleaved cell values, n * total_cells. */
int cb200_encode_cells_dev(cb200_ctx* ctx, const uint8_t* d_payload, int n, uint8_t* d_cellvals);

/* ---- per-kernel timing (measurement support) --------------------------------------------------------------------- */

/* when enabled, CUDA events are recorded on the context's stream around every kernel of every pipeline call (a ring of
   the last 64 calls).  cb200_get_timing returns the milliseconds of the call `calls_back` calls ago (0 = last) in launch
   order: [0] K1 fused decode (both K1 launches of a batch with a per-frame sharpen choice), [1] K1x exact-walk kernel, [2] pack, [3] RS, [4] chunk mask (decode_raw_dev stops after [2]);
   a scan call: [0] blur + histogram (all blur launches of a ragged batch), [1] Otsu, [2] anchors */
int cb200_set_timing(cb200_ctx* ctx, int enable);
/* kernels launched by this library in this process so far (every launch site counts itself): bench.py reports the
   difference across its timed region as "gpu_launches" */
unsigned long long cb200_launch_count(void);
int cb200_get_timing(cb200_ctx* ctx, int calls_back, float* ms, int max_entries, int* n_entries);

/* ---- multi-GPU: the chunk records of all ranks -> rank 0 ------------------------------------------------------------

   Replaces: the many-decoders -> one-sink hand-over of concurrent_fountain_decoder_sink
   (src/lib/fountain/concurrent_fountain_decoder_sink.h:58-84), for one process per GPU (frames shard f % world).

   (1) NVLink window.  Rank 0 allocates a double-buffered window in its HBM (cb200_gather_root_create) and hands the 64-byte
   CUDA IPC handle to the other ranks by any host channel; they map it (cb200_gather_peer_open: peer access over NVLink).
   cb200_gather_slot returns, per buffer, where THIS rank's decode must write: pass the pointers to cb200_decode_chunks_dev and
   the RS / chunk-mask kernels store their results straight into rank 0's memory while they compute -- no separate copy or
   collective.  After the decode a rank publishes an epoch (cb200_gather_publish: system-scope release store, enqueued on the
   context's stream); rank 0 enqueues cb200_gather_wait(buffer, epoch) (system-scope acquire spin over all ranks, bounded by
   timeout_s; cb200_gather_status reports a rank that never arrived) and then reads the window: cb200_gather_slot(ctx, buffer,
   rank, ...) on rank 0 addresses any rank's records.  Frames per rank must be <= the max_frames the contexts were created with
   (the same on every rank).  Back-pressure for the double buffer, also on the device: when rank 0 is done with buffer b of
   epoch e it enqueues cb200_gather_release(b, e); a rank enqueues cb200_gather_acquire(b, e) before the decode that overwrites
   buffer b (epochs are the caller's step counter, starting at 1 and increasing; step s uses buffer s & 1). */
#define CB200_IPC_HANDLE_BYTES 64
int cb200_gather_root_create(cb200_ctx* ctx, int nranks, uint8_t* handle_out /* CB200_IPC_HANDLE_BYTES */);
int cb200_gather_peer_open(cb200_ctx* ctx, int nranks, int rank, const uint8_t* handle);
int cb200_gather_slot(cb200_ctx* ctx, int buffer /* 0 | 1 */, int rank /* < 0: this rank */, uint8_t** d_chunks, uint32_t** d_mask);
int cb200_gather_publish(cb200_ctx* ctx, int buffer, uint32_t epoch);
/* the push form: n records that the decode wrote into LOCAL buffers travel to this rank's slot by a copy-engine transfer on a
   side stream (ordered after everything enqueued on the context's stream so far, and -- acquire_epoch != 0 -- after rank 0 has
   released that slot up to acquire_epoch), then the epoch is published from the side stream.  The decode stream does not
   wait; before the local buffers are written again: cb200_gather_chunks_wait(ctx, buffer). */
int cb200_gather_push(cb200_ctx* ctx, int buffer, const uint8_t* d_chunks, const uint32_t* d_mask, int n, uint32_t epoch,
                      uint32_t acquire_epoch);
int cb200_gather_wait(cb200_ctx* ctx, int buffer, uint32_t epoch, double timeout_s /* <= 0: 30 s */);
int cb200_gather_release(cb200_ctx* ctx, int buffer, uint32_t epoch);                    /* rank 0 */
int cb200_gather_acquire(cb200_ctx* ctx, int buffer, uint32_t epoch, double timeout_s);  /* any rank (no-op on rank 0) */
int cb200_gather_status(cb200_ctx* ctx);   /* rank 0, synchronises: 0, or an error naming the rank that timed out */

/* (2) NCCL.  cb200_gather_chunks sends n records of this rank to rank 0 (ncclSend / ncclRecv, grouped) on a side stream of
   the context, ordered after the work already enqueued on the context's stream; the next decode can be enqueued at once and
   overlaps the exchange.  cb200_gather_chunks_wait(buffer) makes the context's stream wait for the last exchange issued with that
   buffer index (before its send buffers are reused / its gathered data is read): with two buffers the exchange of step s
   overlaps the decode of step s + 1.  nccl_comm: the host's ncclComm_t, or NULL to use the communicator made by
   cb200_comm_init (ncclGetUniqueId on rank 0 -> out-of-band broadcast -> ncclCommInitRank on every rank).  NCCL is bound at
   run time (dlopen libnccl.so.2); d_all_chunks / d_all_masks (rank 0): nranks x n records, rank-major. */
#define CB200_UNIQUE_ID_BYTES 128
int cb200_comm_unique_id(uint8_t* id_out /* CB200_UNIQUE_ID_BYTES */);
int cb200_comm_init(cb200_ctx* ctx, const uint8_t* id, int nranks, int rank);
int cb200_gather_chunks(cb200_ctx* ctx, void* nccl_comm, int nranks, int rank, int buffer /* 0 | 1 */, const uint8_t* d_chunks,
                        const uint32_t* d_mask, int n, uint8_t* d_all_chunks, uint32_t* d_all_masks);
int cb200_gather_chunks_wait(cb200_ctx* ctx, int buffer);

/* ---- multi-GPU: the CC_FIT colour correction chained across ranks ------------------------------------------------

   Under CB200_FLAG_CC_FIT a frame without a usable fountain header takes the CCM of the frame before it: the one state that
   crosses frames.  When a batch is cut into contiguous stripes, one per rank in rank order, linking the ranks' contexts to a chain
   makes every rank's records equal those of one context decoding the whole batch: the CCM entering rank r's stripe is the last fit
   of the stripes of ranks 0 .. r-1 in the same step, or, when none of them fit, the CCM rank 0 entered the step with.
   Rank 0 allocates a small region (cb200_ccm_chain_root_create) and hands the IPC handle to the other ranks
   (cb200_ccm_chain_peer_open); every rank then links its context (cb200_ccm_chain_attach) and, before each CC_FIT call, sets the
   call's step (cb200_ccm_chain_step: epochs start at >= 1 and increase; every rank uses the same epoch for the same step; a rank
   with no frames in a step still makes the call with n = 0: every entry point that honours CB200_FLAG_CC_FIT, host-pointer and
   camera ones included, then takes part in the step).  A chained call enqueues, with no host wait, a publish of the stripe's
   last fit after its fit kernel, a bounded system-scope wait for the lower ranks' publishes of the step before its colour
   decisions, and at its end a bounded wait for all ranks' publishes: afterwards the context's CCM (cb200_get_ccm, and the next
   call) is the step's global exit on every rank.  A wait that gives up after 30 s records the missing rank;
   cb200_ccm_chain_status (synchronises, any rank) reports it.  Calls without CB200_FLAG_CC_FIT are not chained.
   CB200_ERR_ARG, before any CUDA call: a CC_FIT call on a linked context without a step set, cb200_set_ccm / cb200_fit_ccm on a
   linked context, a step on a context that is not linked, rank >= nranks or values that differ from the region's. */
int cb200_ccm_chain_root_create(cb200_ctx* ctx, int nranks, uint8_t* handle_out /* CB200_IPC_HANDLE_BYTES */);
int cb200_ccm_chain_peer_open(cb200_ctx* ctx, int nranks, int rank, const uint8_t* handle);
int cb200_ccm_chain_attach(cb200_ctx* ctx, int rank, int nranks);
int cb200_ccm_chain_step(cb200_ctx* ctx, uint32_t epoch);
int cb200_ccm_chain_status(cb200_ctx* ctx);
/* with cb200_set_timing on: the milliseconds the last chained call's link kernel took (its wait for the lower ranks' fits) */
int cb200_ccm_chain_link_ms(cb200_ctx* ctx, float* ms);

/* ---- rank-0 fountain ingest (host only, no GPU) ------------------------------------------------------------------

   Replaces: fountain_decoder_sink::decode_frame -> fountain_decoder_stream::write -> FountainDecoder::decode
   (src/lib/fountain/fountain_decoder_sink.h:133-166, fountain_decoder_stream.h:45-79, FountainDecoder.h:48-60) and the
   FountainMetadata header parse (FountainMetadata.h:16-90).  The fountain codec is wirehair and stays what it is in the
   reference: the four callbacks have wirehair's C API signatures (wirehair_decoder_create, wirehair_decode,
   wirehair_recover, wirehair_free), so an integrated build passes those symbols. */
typedef struct cb200_sink cb200_sink;
typedef void* (*cb200_codec_create_fn)(void* reuse, uint64_t message_bytes, uint32_t block_bytes);
typedef int (*cb200_codec_decode_fn)(void* codec, unsigned block_id, const void* block_data, uint32_t data_bytes);
typedef int (*cb200_codec_recover_fn)(void* codec, void* message_out, uint64_t message_bytes);
typedef void (*cb200_codec_free_fn)(void* codec);

cb200_sink* cb200_sink_create(unsigned chunk_size, cb200_codec_create_fn create_fn, cb200_codec_decode_fn decode_fn,
                              cb200_codec_recover_fn recover_fn, cb200_codec_free_fn free_fn);
/* same, with the codec taken from a shared library that exports wirehair's C API (wirehair_init_, wirehair_decoder_create,
   wirehair_decode, wirehair_recover, wirehair_free): the reference's third-party codec compiled unmodified
   (libcimbar_b200/build.py build_wirehair -> libcimbar_b200/lib/libwirehair.so).  NULL on failure. */
cb200_sink* cb200_sink_create_wirehair(unsigned chunk_size, const char* wirehair_library);
void cb200_sink_destroy(cb200_sink* sink);
/* one chunk (6-byte header + payload): > 0 = file id (encode_id|size word) when the file completed, 0 = progress,
   -1 = already done, -10/-11/-12 = malformed (same values as the reference) */
int64_t cb200_sink_decode_frame(cb200_sink* sink, const uint8_t* chunk, unsigned size);
/* the fixed-slot output of cb200_decode_chunks_dev (or the records gathered from all ranks): feeds every chunk whose
   mask bit is set; returns the last completed file id or 0 */
int64_t cb200_sink_ingest(cb200_sink* sink, const uint8_t* chunks, const uint32_t* masks, int n_frames, int chunks_per_frame);
int64_t cb200_sink_file_size(const cb200_sink* sink, uint32_t id);                     /* -1 if not complete */
int cb200_sink_file_read(const cb200_sink* sink, uint32_t id, uint8_t* out, uint64_t size);

/* ---- host-side helpers that need no GPU ------------------------------------------------------------------------ */

/* geometry without a context (for sizing buffers before a device exists) */
int cb200_mode_info(int mode_val, cb200_info* out);
/* host-side consistency checks of the mode tables the kernels rely on (cell adjacency in closed form vs the literal
   AdjacentCellFinder evaluation); 0 = consistent */
int cb200_selfcheck(int mode_val);
/* Interleave::interleave_indices (Interleave.h:8-24): slot -> linear cell index; idx has total_cells entries */
int cb200_interleave_indices(int mode_val, uint16_t* idx);

#ifdef __cplusplus
}
#endif
#endif /* CB200_H */
