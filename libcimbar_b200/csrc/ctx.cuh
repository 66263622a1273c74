// ctx.cuh -- the context object behind the C ABI (include/cb200.h) and the error helpers, shared by api.cu / gather.cu / deskew.cu
#pragma once
#include "../../include/cb200.h"
#include "cb200_common.cuh"
#include "k1x_flood.cuh"
#include "ccm.cuh"

#include <string>
#include <vector>

namespace cb200 {
// thread-local error text behind cb200_last_error(); both return `code`
int fail(int code, const std::string& msg);
int fail_cuda(cudaError_t e, const char* what);
struct GatherState;      // gather.cu
struct DeskewState;      // deskew.cu
struct ScanScratch;      // scan.cu
struct JpegState;        // jpeg.cu
struct PngState;         // png.cu
struct ChainState;       // chain.cu
void gather_destroy(GatherState* g);
void chain_destroy(ChainState* s);
void deskew_destroy(DeskewState* d);     // delete: its buffers free themselves
void scan_destroy(ScanScratch* s);       // likewise
void jpeg_destroy(JpegState* j);         // likewise
void png_destroy(PngState* p);           // likewise
// the uploads of the file calls (descriptors + compressed data, jpeg.cu / png.cu): a ring of pinned buffers, each reused once the
// copy enqueued from it has run -- one per call, so, as on the RGB camera call, a fourth call in flight waits until the first
// one's upload has run.  take() hands out the next slot with room for `bytes`; send() enqueues the copy of its first `bytes` to
// d_dst and records the slot's event
struct FileUpload {
    static constexpr int kSlots = 3;
    PinnedBuf<uint8_t> h[kSlots];
    cudaEvent_t ev[kSlots] = {};
    int next = 0;
    ~FileUpload() { for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e); }
    int take(size_t bytes, int* slot, uint8_t** host);
    int send(cudaStream_t st, int slot, void* d_dst, size_t bytes);
};
// status -2 (and, when d_mask is given, mask 0) for every picture whose flag in d_bad is set: the corrupt files of a file call
// (files.cu, like FileUpload's members)
int file_status(cb200_ctx* c, const int* d_bad, int n, int32_t* d_status, uint32_t* d_mask);
// cb200_decode_fountain_from_dev with an optional per-frame sharpen selection: `sharpen` = n host bytes (nonzero =
// should_preprocess) or NULL (the batch-wide CB200_FLAG_SHARPEN decides).  The flags are checked by the caller (api.cu)
int decode_fountain_to_host(cb200_ctx* c, const uint8_t* d_rgb, int n, uint32_t flags, const uint8_t* sharpen, uint8_t* chunks_out,
                            uint32_t* chunk_count, uint32_t* chunk_mask, uint8_t* frame_flags);
// CB200_ERR_ARG for CB200_FLAG_SHARPEN together with CB200_FLAG_SHARPEN_IF_NEEDED (deskew.cu)
int check_camera_flags(uint32_t flags);
// one camera picture of a batch as the extractor kernels (scan.cu, deskew.cu) read it.  The host builds the table per call, for
// uniform batches too: picture i of a packed batch starts at byte 3 * sum_{j<i} w_j h_j, its blurred gray at sum_{j<i} w_j h_j
struct PicDesc {
    uint64_t src;        // byte offset of the RGB8 picture in the source buffer
    uint64_t blur;       // byte offset of its blurred gray picture in the scan's buffer (k_scan_blur4 / k_scan_anchors)
    int w, h;
    int words;           // k_scan_blur4's word path: w % 4 == 0 and both bases 4-byte aligned
    int tile0;           // first tile of the picture in the blur launch of its radius
};
// wh: n x (w, h) on the host.  CB200_ERR_ARG naming the picture if a size is outside what the scan restates (short side 60 ..
// 4499) (scan.cu); no CUDA call
int check_picture_sizes(const int32_t* wh, int n);
// the uniform batch as a ragged one: n x (w, h)
std::vector<int32_t> uniform_sizes(int w, int h, int n);
// cb200_extract_decode_fountain_dev with the same selection, for pictures of sizes wh (n x (w, h)) packed in d_src (deskew.cu)
int extract_decode_to_host(cb200_ctx* c, const uint8_t* d_src, const int32_t* wh, int n, const float* corners, uint32_t flags,
                           const uint8_t* sharpen, uint8_t* chunks_out, uint32_t* chunk_count, uint32_t* chunk_mask, uint8_t* frame_flags);
// CB200_FLAG_SHARPEN_IF_NEEDED on given corners: sharpen[i] = 1 iff picture i's corners fail Corners::is_granular_scale (deskew.cu)
std::vector<uint8_t> sharpen_from_corners(const cb200_ctx* c, const float* corners, int n);
// room for n deskewed frames in the context's frame buffer, *frames = its base (deskew.cu)
int deskew_frames(cb200_ctx* c, int n, uint8_t** frames);
// k_deskew over n pictures described by d_desc (src, w, h; src_bytes in all) with the inverse maps d_minv (n x 9) into d_dst (deskew.cu)
int deskew_launch(cb200_ctx* c, const uint8_t* d_src, size_t src_bytes, const double* d_minv, const PicDesc* d_desc, int n, uint8_t* d_dst);
// the enqueue-only decode of n extracted frames (api.cu): cb200_decode_chunks_dev, but the sharpen selection, if any, is n bytes in
// device memory (d_sharp, at c->d_sel + 4 n: k_select builds the frame lists there; NULL = as the flags say) and a CCM that an earlier call still in flight may
// change is taken from the device (c->d_carry) instead of waiting for it
int decode_chunks_enqueue(cb200_ctx* c, const uint8_t* d_rgb, int n, uint32_t flags, const uint8_t* d_sharp, uint8_t* d_chunks,
                          uint32_t* d_chunk_mask, uint8_t* d_frame_flags);
// the argument checks of cb200_scan_extract_decode_chunks_ragged_dev beyond its pictures, all before any CUDA call (scan.cu): the
// flags (both sharpen flags, CC_SIMPLE with CC_FIT), then the context, the outputs and n against max_frames
int check_camera_dev_flags(uint32_t flags);
int check_camera_dev_outputs(cb200_ctx* c, int n, const uint8_t* d_chunks, const uint32_t* d_chunk_mask, const int32_t* d_extract_status);
// the enqueue-only camera path (scan, k_extract, deskew, decode, failed pictures' masks cleared) for n pictures of sizes wh packed
// in device memory, arguments checked (scan.cu)
int camera_enqueue(cb200_ctx* c, const uint8_t* d, const int32_t* wh, int n, uint32_t flags, uint8_t* d_chunks, uint32_t* d_mask,
                   uint8_t* d_frame_flags, int32_t* d_status);
// the results of the last decode (c->d_data, c->d_mask, c->d_flags, and d_status when given) to host memory with one synchronise,
// the good chunks of each frame packed densely (api.cu)
int fetch_fountain(cb200_ctx* c, int n, const int32_t* d_status, uint8_t* chunks_out, uint32_t* chunk_count, uint32_t* chunk_mask,
                   uint8_t* frame_flags, int32_t* extract_status);
// the CCM chain across ranks (chain.cu).  chain_linked: a call with these flags on this context runs the chain (attached, CC_FIT).
// check_chain_call: CB200_ERR_ARG for such a call without a step set; check_host_ccm: CB200_ERR_ARG for cb200_set_ccm /
// cb200_fit_ccm on an attached context (both without CUDA calls).  chain_publish_link enqueues, after k_ccm_fit, the publish of
// the stripe's n fits (d_fit / d_valid; n = 0: an empty stripe, no fit) and, with entry given, the link that leaves the stripe's
// entry CCM on the device and points *entry at it; own = the CCM this context would enter the stripe with.  chain_settle enqueues
// the global exit of the step into d_carry (9 floats + activity byte) and ends the step
bool chain_linked(const cb200_ctx* c, uint32_t flags);
int check_chain_call(const cb200_ctx* c, uint32_t flags);
int check_host_ccm(const cb200_ctx* c);
int chain_publish_link(cb200_ctx* c, int n, const float* d_fit, const uint8_t* d_valid, const CcmArg& own, CcmArg* entry);
int chain_settle(cb200_ctx* c, float* d_carry);
// a camera call with no pictures: on a chained CC_FIT call the empty stripe's part of the step, else nothing (scan.cu)
int camera_empty(cb200_ctx* c, uint32_t flags);
// camera plans (plan.cu).  Every context buffer a plan's graph uses is grown through grow(): while plans exist a call that needs
// more fails with CB200_ERR_ARG (plan_frozen) instead.  Called with plans, the *_reserve functions below therefore make no CUDA
// call, and an entry point runs them first (check_frozen*) so that a frozen buffer refuses the call before any CUDA call
int plan_frozen(const cb200_ctx* c, const char* buffer, size_t have, size_t need);
// the camera path's buffers for n pictures of sizes wh: the scan's (scan_reserve), the transforms, the selection, the deskewed
// frames and the exact walk's (scan.cu, deskew.cu, api.cu)
int scan_reserve(cb200_ctx* c, const int32_t* wh, int n);
int camera_reserve(cb200_ctx* c, const int32_t* wh, int n);
int deskew_reserve(cb200_ctx* c, int n);
int flood_reserve(cb200_ctx* c, int n);
// the decode's buffers sized by max_frames, the CCM event and the slot map of these flags (api.cu): no CUDA call after the first time
int decode_reserve(cb200_ctx* c, uint32_t flags);
// CB200_ERR_ARG, before any CUDA call, when live plans freeze a buffer this call would grow; nothing without plans (plan.cu).
// frames: n decoded frames (the exact walk); deskew: n deskewed frames too; camera / scan: n camera pictures of sizes wh
int check_frozen_frames(cb200_ctx* c, int n);
int check_frozen_deskew(cb200_ctx* c, int n);
int check_frozen_camera(cb200_ctx* c, const int32_t* wh, int n);
int check_frozen_scan(cb200_ctx* c, const int32_t* wh, int n);
// the CCM a plan's graph starts from is d_carry: with plans, a matrix the host sets (cb200_set_ccm, cb200_fit_ccm, a new plan) is
// copied there in stream order (api.cu)
int carry_from_host(cb200_ctx* c);
// a CC_FIT call in this mode fits matrices (init_ccm needs a header from the RS stream, not the legacy coupled layout) (api.cu)
bool ccm_fits(const Mode& m, uint32_t flags);
// the camera path with the picture table given in device memory (a plan's), so nothing is uploaded (scan.cu)
int camera_enqueue_table(cb200_ctx* c, const uint8_t* d, const int32_t* wh, int n, uint32_t flags, uint8_t* d_chunks, uint32_t* d_mask,
                         uint8_t* d_frame_flags, int32_t* d_status, const PicDesc* d_table);
// the pictures of the last camera call (cb200_camera_transforms reads that many) (scan.cu)
int camera_pictures(cb200_ctx* c);
void set_camera_pictures(cb200_ctx* c, int n);
// the picture table of that call for n pictures of sizes wh at d_pics, built on the host (scan.cu): PicDesc n, then the order
int camera_table(cb200_ctx* c, const uint8_t* d_pics, const int32_t* wh, int n, std::vector<uint8_t>& table);
}  // namespace cb200
#define CK(call, what) do { cudaError_t e__ = (call); if (e__ != cudaSuccess) return cb200::fail_cuda(e__, what); } while (0)

// Every buffer of the context is a cb200::Buffer and frees itself; cb200_destroy only destroys the streams and events
struct cb200_ctx {
    cb200::Mode mode;
    int device = 0, max_frames = 0, sm_count = 0;
    cudaStream_t own_stream = nullptr, stream = nullptr;
    // device workspaces
    cb200::DevBuf<uint8_t> d_rgb;           // host-pointer entry points only: max_frames frames
    cb200::DevBuf<uint8_t> d_cellvals;      // max_frames * num_cells
    cb200::DevBuf<uint32_t> d_dirty;        // max_frames
    cb200::DevBuf<uint8_t> d_raw;           // max_frames * cap_all
    cb200::DevBuf<uint8_t> d_data;          // max_frames * data_bytes
    cb200::DevBuf<uint8_t> d_ok;            // max_frames * nblocks
    cb200::DevBuf<uint32_t> d_mask;         // max_frames
    cb200::DevBuf<uint8_t> d_flags;         // max_frames
    cb200::DevBuf<uint16_t> d_idx;          // num_cells: slot -> cell (Interleave::interleave_indices)
    cb200::DevBuf<uint16_t> d_inv;          // num_cells: cell -> slot (Interleave::interleave_reverse)
    cb200::DevBuf<uint16_t> d_idx_ident;    // identity map for CB200_FLAG_NO_INTERLEAVE (created on first use)
    cb200::DevBuf<uint8_t> d_gen;           // RS generator polynomial, ecc_bytes+1 coefficients
    cb200::DevBuf<uint8_t> d_rho;           // 4 x 64 bytes: x^(D+j) mod x^pad g, the basis of K2's remainder tables (k2_remainder_basis)
    // per-kernel timing (cb200_set_timing): events around every launch of the last pipeline call
    bool timing = false;
    static constexpr int kEvSets = 64;
    cudaEvent_t ev[kEvSets][8] = {};
    int ev_count[kEvSets] = {};
    long calls = 0;                  // pipeline calls since timing was enabled
    int cur = 0;                     // event set of the call in progress
    cb200::FloodWorkspace flood;            // exact-walk fallback scratch
    // small scratch for the single-cell entry points
    cb200::DevBuf<uint8_t> d_scratch;
    // pinned host staging for results of the host-pointer entry points
    cb200::PinnedBuf<uint8_t> h_pinned;
    // host-built tables of a call (sharpen selections, picture tables, inverse maps) on their way to the device: a ring of pinned
    // slots, each reused once the copy enqueued from it has run (stage_take / stage_send).  A call uploads at most two tables
    // (cb200_deskew_dev: its table; a frame call with a mixed selection: the selection), so no call waits for a copy it enqueued
    // itself; a camera call uploads one (its picture table), so three camera calls can be in flight before the fourth waits
    struct StageSlot { cb200::PinnedBuf<uint8_t> h; cudaEvent_t ev = nullptr; };
    static constexpr int kStageSlots = 3;
    StageSlot stage[kStageSlots];
    int stage_next = 0;
    // a sharpen selection of n frames: the plain frames' batch indices, then the sharpened ones' (both in batch order, 4 n bytes),
    // then one sharpen byte per frame (n bytes); built from the bytes by k_select (api.cu), which also leaves the launch schedule
    // of each list in d_sched: {count, K1 bands, first entry} for the plain and for the sharpened frames
    cb200::DevBuf<uint8_t> d_sel;           // max_frames x (4 + 1)
    cb200::DevBuf<int> d_sched;             // 6
    // colour correction (the reference's thread-local CimbDecoder CCM, CimbDecoder.cpp:69-85)
    float ccm[9] = {};               // active matrix, row-major
    bool ccm_active = false;
    bool ccm_pending = false;        // the last CC_SIMPLE batch's final matrix is still on its way to h_ccm
    bool ccm_pending_flag = false;   // ... and so is whether that frame had a CCM at all (CC_FIT batches)
    cb200::DevBuf<float> d_ccm;             // per-frame matrices of a CC_SIMPLE / CC_FIT batch (the ones used): max_frames x 9
    cb200::DevBuf<float> d_carry;           // the last such batch's final matrix + activity byte (at float index 9), stream-ordered
    cb200::PinnedBuf<float> h_ccm;          // d_carry's copy on the host
    // CC_FIT scratch: per-cell mean colours of the first pass, per-frame fits
    cb200::DevBuf<uint32_t> d_means;        // max_frames x num_cells
    cb200::DevBuf<float> d_fit;             // max_frames x 9
    cb200::DevBuf<uint8_t> d_fit_valid;     // max_frames
    cb200::DevBuf<uint8_t> d_ccm_active;    // max_frames: the frame is decoded with d_ccm[f]
    int ccm_frames = 0;              // frames of the last call that took the fitted-CCM route (cb200_get_frame_ccms)
    cudaEvent_t ccm_ev = nullptr;    // recorded after the D2H copies of the last batch's CCM (ccm_resolve waits on it)
    cb200::GatherState* gather = nullptr;   // multi-GPU chunk-record window (gather.cu)
    cb200::ChainState* chain = nullptr;     // multi-GPU CC_FIT chain (chain.cu)
    cb200::DeskewState* deskew = nullptr;   // extractor scratch (deskew.cu)
    cb200::ScanScratch* scan = nullptr;     // anchor-scan scratch (scan.cu)
    cb200::JpegState* jpeg = nullptr;       // JPEG decode scratch (jpeg.cu)
    cb200::PngState* png = nullptr;         // PNG decode scratch (png.cu)
    std::vector<cb200_camera_plan*> plans;  // live camera plans (plan.cu): they freeze the buffers their graphs use
    bool capturing = false;                 // a plan's capture is in progress: the CCM always comes from d_carry
};

namespace cb200 {
template <typename B> int grow(cb200_ctx* c, B& b, size_t count, const char* buffer)
{
    if (count <= b.capacity()) return CB200_OK;
    if (!c->plans.empty()) return plan_frozen(c, buffer, b.capacity(), count);
    const cudaError_t e = b.ensure(count);
    if (e != cudaSuccess) return fail_cuda(e, (std::string("cudaMalloc ") + buffer).c_str());
    return CB200_OK;
}
}  // namespace cb200

namespace cb200 {
// cb200_set_timing: begin_timed_call starts the event set of a pipeline call, mark records its next event on the call's stream
inline void begin_timed_call(cb200_ctx* c) { if (c->timing) { c->cur = (int)(c->calls % cb200_ctx::kEvSets); c->calls++; c->ev_count[c->cur] = 0; } }
inline void mark(cb200_ctx* c) { if (c->timing && c->ev_count[c->cur] < 8) cudaEventRecord(c->ev[c->cur][c->ev_count[c->cur]++], c->stream); }
// a host-built table for this call: stage_take hands out the next pinned slot with room for `bytes` (after the copy last
// enqueued from it has run); the caller fills *h, and stage_send enqueues the copy of its first `bytes` to d_dst on the call's
// stream and records the slot's event.  The caller's own host inputs are free again when the call returns
int stage_take(cb200_ctx* c, size_t bytes, int* slot, uint8_t** h);
int stage_send(cb200_ctx* c, int slot, void* d_dst, size_t bytes, const char* what);
}  // namespace cb200
