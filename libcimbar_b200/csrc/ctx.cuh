// ctx.cuh -- the context object behind the C ABI (include/cb200.h) and the error helpers, shared by api.cu / gather.cu / deskew.cu
#pragma once
#include "../../include/cb200.h"
#include "cb200_common.cuh"
#include "k1x_flood.cuh"
#include "ccm.cuh"
#include "pic_desc.cuh"

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
struct DetectState;      // detect.cu
void gather_destroy(GatherState* g);
void chain_destroy(ChainState* s);
void detect_destroy(DetectState* d);
// the exact walk of a detect call (detect.cu), shared by the modes of one frame geometry: `lead` walks (flood_launch, the walk's
// records kept in `kept`), every other context of the geometry takes its frame flags and colours that walk's positions in its own
// palette and CCM (flood_colour_launch).  The walk reads only the geometry, the frames and their sharpen bytes, and K1's dirty
// flag is a symbol decision, so each mode's cells equal what its own walk would give.  present: NULL, or (a detect receivers plan,
// whose geometries work on every slot) one device byte per frame, 0 for a slot no mode of the geometry decodes: the lead walks
// only the others
struct SharedWalk { cb200_ctx* lead; uint32_t* kept; const uint8_t* present; };
void deskew_destroy(DeskewState* d);     // delete: its buffers free themselves
void scan_destroy(ScanScratch* s);       // likewise
void jpeg_destroy(JpegState* j);         // likewise
void png_destroy(PngState* p);           // likewise
// host-built data of a call on its way to the device: a ring of pinned buffers, each reused once the copy enqueued from it has run.
// take() hands out the next slot with room for `bytes` (after the copy last enqueued from it has run); the caller fills *host, and
// send() enqueues the copy of its first `bytes` to d_dst on stream st and records the slot's event.  The caller's own host inputs
// are free again when the call returns.  Instances: the context's (cb200_ctx::upload), the JPEG calls' and the PNG calls'
struct UploadRing {
    static constexpr int kSlots = 3;
    PinnedBuf<uint8_t> h[kSlots];
    cudaEvent_t ev[kSlots] = {};
    int next = 0;
    ~UploadRing() { for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e); }
    int take(size_t bytes, int* slot, uint8_t** host);
    int send(cudaStream_t st, int slot, void* d_dst, size_t bytes);
};
// status -2 (and, when d_mask is given, mask 0) for every picture whose flag in d_bad is set: the corrupt files of a file call
// (files.cu, like UploadRing's members)
int file_status(cb200_ctx* c, const int* d_bad, int n, int32_t* d_status, uint32_t* d_mask);
// the decode of n extracted frames (n = 0: a chained call's empty stripe) that every frame, corner, camera and detect call runs
// once, after its own checks (n <= max_frames, chain step, frozen walk workspace, non-null buffers): it checks nothing (api.cu).
// Selection: n host bytes (sharpen), n device bytes at c->d_sel + 4 n (d_sel_bytes), or neither (CB200_FLAG_SHARPEN decides).
// enqueue_only: a CCM still on its way from an earlier batch is not waited for but read from c->d_carry on the device (k_ccm_carry:
// a batch without a fit then takes the fitted-CCM route with no fits, deciding every colour as K1 would with that matrix)
// recv: a _receivers_dev call's receivers (the CCM of each picture is its receiver's; the context's CCM is neither read nor changed)
struct Receivers;
int decode_chunks(cb200_ctx* c, const uint8_t* d_rgb, int n, uint32_t flags, const uint8_t* sharpen, uint8_t* d_chunks,
                  uint32_t* d_chunk_mask, uint8_t* d_frame_flags, const uint8_t* d_sel_bytes = nullptr, bool enqueue_only = false,
                  Receivers* recv = nullptr);
// decode_chunks into the context's buffers, then fetch_fountain (api.cu)
int decode_fountain_to_host(cb200_ctx* c, const uint8_t* d_rgb, int n, uint32_t flags, const uint8_t* sharpen, uint8_t* chunks_out,
                            uint32_t* chunk_count, uint32_t* chunk_mask, uint8_t* frame_flags);
// CB200_ERR_ARG for CB200_FLAG_SHARPEN together with CB200_FLAG_SHARPEN_IF_NEEDED, or CB200_FLAG_CC_SIMPLE with CB200_FLAG_CC_FIT
// (scan.cu)
int check_camera_flags(uint32_t flags);
// CB200_ERR_ARG for a receiver flags table that is null or not 4-byte aligned, or call flags with a per-receiver bit (scan.cu)
int check_receiver_flags(const uint32_t* d_receiver_flags, uint32_t flags);
// PicDesc, one camera picture as the extractor kernels read it: pic_desc.cuh.
// The pictures of one camera, corner or deskew call, whatever the caller passed in (scan.cu): one descriptor per picture, their
// sizes n x (w, h) (what scan_reserve and check_frozen_* take), and `packed`: every picture is RGB with row pitch 3 w, so the
// kernels run their packed (kLayouts = false) instantiations.  `host`: the pictures are still in host memory, stage_batch takes
// them to the device.  One builder per kind of input applies that kind's per-picture rules, all before any CUDA call.
// A plan over device descriptors (device_batch) has neither pics nor wh: d_pics holds dev_n descriptors the plan reads at each
// launch, and `bounds` the sizes it is built for (what its buffers are sized from: the CameraBatch overloads of the reserve
// functions below)
struct CameraBatch {
    std::vector<cb200_picture> pics;
    std::vector<int32_t> wh;
    bool packed = true, host = false;
    const cb200_picture* d_pics = nullptr;
    int dev_n = 0;
    cb200_picture_bounds bounds = {};
    int n() const { return d_pics ? dev_n : (int)(wh.size() / 2); }
    void pack(const uint8_t* d);       // the pictures of sizes wh back to back from d in packed RGB
};
// wh: n x (w, h) on the host.  CB200_ERR_ARG naming the picture if a size is outside what the scan restates (short side 60 ..
// 4499) (scan.cu); no CUDA call
int check_picture_sizes(const int32_t* wh, int n);
// the uniform batch as a ragged one: n x (w, h)
std::vector<int32_t> uniform_sizes(int w, int h, int n);
// the builders (scan.cu): n packed pictures of sizes wh from the device buffer d (the _dev entry points, plans, detect; a file
// call's decoded pictures are packed this way too, with the sizes parse_files gives); n packed pictures of w x h from d (host or
// device: the uniform entry points, which then take the ragged path); n host pointers, packed when staged; n picture descriptors
// in the caller's layouts.  The scan's size rule (check_picture_sizes) applies to all four
int packed_batch(const uint8_t* d, const int32_t* wh, int n, CameraBatch& b);
int uniform_batch(const uint8_t* d, int w, int h, int n, CameraBatch& b);
int host_batch(const uint8_t* const* pictures, const int32_t* wh, int n, CameraBatch& b);
int picture_batch(const cb200_picture* pics, int n, CameraBatch& b);
// n descriptors in device memory within bounds (cb200_camera_plan_create_receivers_pictures_dev): the pointer (null, 8-byte
// alignment) and the bounds are checked, none of the descriptors is read
int device_batch(const cb200_picture* d_pics, int n, const cb200_picture_bounds* bounds, CameraBatch& b);
// The device table of a plan over device descriptors, which k_plan_pictures writes at each launch (scan.cu): n PicDesc; three lists of
// n slots, the slots of blur radius group 0, 1, 2 in slot order; the groups' slot counts and tile counts (6 int); the effective
// receiver map (n int32: the caller's, -1 for a refused slot); one refused byte per slot; the stand-in picture's row (zeros).
// plan_pictures_launch enqueues k_plan_pictures on the context's stream; a detect plan passes its candidates (NULL: every mode)
// and n_modes, and a slot without a candidate below n_modes is empty like one whose receiver is out of range
struct PlanTable {
    size_t order, groups, of, refused, standin, bytes;
    explicit PlanTable(const CameraBatch& b);
};
int plan_pictures_launch(cb200_ctx* c, const CameraBatch& b, const int32_t* d_receiver_of, int receivers, uint8_t* d_table,
                         const uint32_t* d_cand = nullptr, int n_modes = 1);
// CB200_ERR_ARG naming the first picture that spans 4 GB or more: k_deskew's offsets inside a picture are 32-bit (scan.cu)
int check_spans(const CameraBatch& b);
// a host batch packed into the context's one staging buffer for host pictures, with one copy per run of adjacent pictures; the
// batch then describes the staged pictures.  Nothing for a device batch (scan.cu)
int stage_batch(cb200_ctx* c, CameraBatch& b);
// room for n deskewed frames in the context's frame buffer, *frames = its base (deskew.cu)
int deskew_frames(cb200_ctx* c, int n, uint8_t** frames);
// k_deskew over the pictures of b described by d_desc, with the inverse maps d_minv (n x 9), into d_dst (deskew.cu)
int deskew_launch(cb200_ctx* c, const CameraBatch& b, const double* d_minv, const PicDesc* d_desc, uint8_t* d_dst);
// the enqueue-only camera path (reserve, scan, k_extract, deskew, decode, failed pictures' masks cleared) for a device batch,
// arguments checked (scan.cu).  The picture table is this call's one upload, unless d_table holds it already (a camera plan's); a
// receivers call's map goes up with it
int camera_enqueue(cb200_ctx* c, const CameraBatch& b, uint32_t flags, uint8_t* d_chunks, uint32_t* d_mask, uint8_t* d_frame_flags,
                   int32_t* d_status, const PicDesc* d_table = nullptr, Receivers* recv = nullptr);
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
// a frame or camera call with no frames, checked: on a chained CC_FIT call the empty stripe's part of the step (it publishes "no fit"
// and settles), else nothing.  enqueue_only as for decode_chunks (the camera calls) (api.cu)
int empty_stripe(cb200_ctx* c, uint32_t flags, bool enqueue_only);
// camera plans (plan.cu).  Every context buffer a plan's graph uses is grown through grow(): while plans exist a call that needs
// more fails with CB200_ERR_ARG (plan_frozen) instead.  Called with plans, the *_reserve functions below therefore make no CUDA
// call, and an entry point runs them first (check_frozen*) so that a frozen buffer refuses the call before any CUDA call
int plan_frozen(const cb200_ctx* c, const char* buffer, size_t have, size_t need);
// the camera path's buffers for n pictures of sizes wh: the scan's (scan_reserve), the transforms, the selection, the deskewed
// frames and the exact walk's (scan.cu, deskew.cu, api.cu)
int scan_reserve(cb200_ctx* c, const int32_t* wh, int n);
int camera_reserve(cb200_ctx* c, const int32_t* wh, int n);
// the same for a batch: its sizes, or a device batch's bounds
int scan_reserve(cb200_ctx* c, const CameraBatch& b);
int camera_reserve(cb200_ctx* c, const CameraBatch& b);
int deskew_reserve(cb200_ctx* c, int n);
int flood_reserve(cb200_ctx* c, int n);
// the decode's buffers sized by max_frames, the CCM event and the slot map of these flags, and with `receivers` a receivers call's
// (api.cu): no CUDA call after the first time
int decode_reserve(cb200_ctx* c, uint32_t flags, bool receivers = false);
// CB200_ERR_ARG, before any CUDA call, when live plans freeze a buffer this call would grow; nothing without plans (plan.cu).
// frames: n decoded frames (the exact walk); deskew: n deskewed frames too; camera / scan: n camera pictures of sizes wh
int check_frozen_frames(cb200_ctx* c, int n);
int check_frozen_deskew(cb200_ctx* c, int n);
int check_frozen_camera(cb200_ctx* c, const int32_t* wh, int n);
int check_frozen_camera(cb200_ctx* c, const CameraBatch& b);
int check_frozen_scan(cb200_ctx* c, const int32_t* wh, int n);
// the CCM a plan's graph starts from is d_carry: with plans, a matrix the host sets (cb200_set_ccm, cb200_fit_ccm, a new plan) is
// copied there in stream order (api.cu)
int carry_from_host(cb200_ctx* c);
// a CC_FIT call in this mode fits matrices (init_ccm needs a header from the RS stream, not the legacy coupled layout) (api.cu)
bool ccm_fits(const Mode& m, uint32_t flags);
// the pictures of the last camera call (cb200_camera_transforms reads that many) (scan.cu)
int camera_pictures(cb200_ctx* c);
void set_camera_pictures(cb200_ctx* c, int n);
// the picture table of a batch as the scan reads it, built on the host (scan.cu): n PicDesc, then the pictures grouped by blur
// radius (n int); a camera plan builds its own with it
int pic_table(cb200_ctx* c, const CameraBatch& b, std::vector<uint8_t>& table);
// the stages of camera_enqueue, for the detect call (scan.cu).  camera_reserve_for: camera_reserve without the scan's buffers
// (scans = false) or the deskewed frames' and the walk's (walks = false).  camera_scan: the scan of the batch on this context's
// scratch (the table from d_table, else uploaded), *d_desc = its picture table.  camera_after_scan: k_extract on `scanned`'s
// anchors into this context's transforms and d_status, the deskew into `frames` (deskew = false: `frames` holds them already,
// deskewed for this geometry), the decode and the failed pictures' masks.  A detect receivers call's geometry runs camera_after_scan
// on a sub-batch: b and d_desc describe its pictures, and d_slots (device) names each one's picture in the scanned batch; its host
// lists (tail) travel with camera_scan's upload
int camera_reserve_for(cb200_ctx* c, const int32_t* wh, int n, bool scans, bool walks);
int camera_scan(cb200_ctx* c, const CameraBatch& b, const PicDesc* d_table, const PicDesc** d_desc, Receivers* recv = nullptr,
                const std::vector<uint8_t>* tail = nullptr, const uint8_t** d_tail = nullptr);
int camera_after_scan(cb200_ctx* c, const cb200_ctx* scanned, const CameraBatch& b, const PicDesc* d_desc, uint32_t flags, uint8_t* frames,
                      bool deskew, uint8_t* d_chunks, uint32_t* d_mask, uint8_t* d_frame_flags, int32_t* d_status,
                      Receivers* recv = nullptr, const int32_t* d_slots = nullptr);
// the receivers of a _receivers_dev call (include/cb200.h).  check_receivers: CB200_ERR_ARG, before any CUDA call, for a null
// receiver map, null or misaligned states, n_receivers < 1, a receiver index out of range, a context linked to a CCM chain (api.cu).
// Receivers(...) then builds `map` on the host: the n receiver indices, then the receiver-major order (receivers_core.cuh); d_map is
// its device copy once uploaded (the camera calls: behind the picture table; the frame call: in cb200_ctx::d_recv).
// A receivers camera plan reads its map on the device: check_receivers with on_device checks the pointer (null, 4-byte alignment)
// instead of the indices.  Receivers(d_map, states) has no host map: d_map is a device map already, the plan's (built by
// k_receivers_order at each launch) or a detect call's mode's.  In every map receiver -1 marks an empty slot, which reads and
// writes no state, gets mask 0 and status CB200_EXTRACT_EMPTY
int check_receivers(const cb200_ctx* c, const int32_t* receiver_of, int n, int n_receivers, const cb200_receiver_state* d_states,
                    bool on_device = false);
// d_refused: NULL, or (a plan over device descriptors) one byte per slot, set where the launch refused the slot's descriptor: its
// status becomes CB200_EXTRACT_REFUSED instead of CB200_EXTRACT_EMPTY.
// d_words: NULL, or a receiver flags table (the _receivers_flags_dev calls; receivers_core.cuh, word_refused): k_extract empties the
// map entry of every slot whose receiver's word is invalid and sets its refused byte, and writes every slot's sharpen byte from its
// receiver's word; every frame takes the fitted-CCM route, with the CCM kind of its receiver's word (decode_chunks).  The direct call's
// refused bytes travel zeroed behind its map (refused_bytes), so d_refused is always set with d_words.  A refused receiver's slots
// become runs of receiver -1 that may sit in the middle of the order; the carry and the masks compare neighbours and read no state
// for them
struct Receivers {
    std::vector<int32_t> map;
    const int32_t* d_map = nullptr;
    cb200_receiver_state* d_states = nullptr;
    const uint8_t* d_refused = nullptr;
    const uint32_t* d_words = nullptr;
    // with d_words: the table's size, and each scanned picture's receiver (NULL: d_map's, the map of a call without sub-batches; a
    // detect call's caller map, whose pictures each mode's sub-batch or empty slots leave out)
    int receivers = 0;
    const int32_t* d_pic_of = nullptr;
    Receivers(const int32_t* receiver_of, int n, int n_receivers, cb200_receiver_state* states);
    // a direct call with a flags table: n zero bytes behind the map, d_refused once the map is on the device
    void refused_bytes(int n) { map.resize(2 * (size_t)n + ((size_t)n + 3) / 4, 0); }
    void map_on_device(const int32_t* d, int n)
    {
        d_map = d;
        if (d_words) d_refused = reinterpret_cast<const uint8_t*>(d + 2 * (size_t)n);
    }
    Receivers(const int32_t* d_map_, cb200_receiver_state* states) : d_map(d_map_), d_states(states) {}
    size_t bytes() const { return map.size() * sizeof(int32_t); }
};
// a camera plan's own rules, checked after its batch's: n > 0, a non-null `out` (set to NULL) (plan.cu)
int plan_rules(int n, cb200_camera_plan** out);
// A detect receivers camera plan (plan.cu) is the detect receivers call's geometry loop (detect.cu) captured over n fixed slots.
// DetectPlan: what its graph reads -- the plan's picture table, the caller's candidates (NULL: every mode) and map, read at each
// launch, and one state table per mode; the lists the graph builds (detect_plan_words(n_modes, n) words: the modes' raw receivers,
// maps and positions) and the geometries' present bytes (n_modes x n).  check_detect_plan: every argument check of
// cb200_camera_plan_create_detect_receivers, before any CUDA call.  detect_plan_reserve: every buffer of the contexts the graph uses,
// at b's size; frozen_only: only on the contexts with live plans, where it makes no CUDA call and refuses what would grow.
// detect_plan_enqueue: the whole call on ctxs[0]'s stream, for the capture
// d_pics_table: a plan over device descriptors, its table for k_plan_pictures (PlanTable, = d_table), else NULL
struct DetectPlan {
    const PicDesc* d_table;
    const uint32_t* d_cand;
    const int32_t* d_of;
    int receivers;
    cb200_receiver_state* const* d_states;
    int32_t* d_lists;
    uint8_t* d_present;
    uint8_t* d_pics_table;
    const uint32_t* d_words;         // a receiver flags table (plans over device descriptors only), else NULL
};
size_t detect_plan_words(int n_modes, int n);
// bounds: NULL for cb200_camera_plan_create_detect_receivers (pics on the host), else the plan's bounds and pics in device memory
// (device_batch's checks; a null bounds is refused there)
int check_detect_plan(cb200_ctx* const* ctxs, int n_modes, const cb200_picture* pics, bool dev_pics, const cb200_picture_bounds* bounds,
                      int n, uint32_t flags, const uint32_t* d_candidates,
                      const int32_t* d_receiver_of, int n_receivers, cb200_receiver_state* const* d_states, const uint8_t* d_chunks,
                      const uint32_t* d_chunk_mask, const int32_t* d_extract_status, const int32_t* d_mode, cb200_camera_plan** out,
                      CameraBatch& b);
int detect_plan_reserve(cb200_ctx* const* ctxs, int n_modes, const CameraBatch& b, uint32_t flags, bool frozen_only);
int detect_plan_enqueue(cb200_ctx* const* ctxs, int n_modes, const CameraBatch& b, uint32_t flags, uint8_t* d_chunks, uint32_t* d_chunk_mask,
                        int32_t* d_extract_status, int32_t* d_mode, uint32_t* d_mode_masks, const DetectPlan& dp);
// the context is attached to a CCM chain (chain.cu)
bool chain_attached(const cb200_ctx* c);
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
    // host-built tables of a call (sharpen selections, picture tables, inverse maps) on their way to the device.  A call uploads at
    // most two tables (a corner call: its table; a frame call with a mixed selection: the selection), so no call waits for a copy it
    // enqueued itself; a camera call uploads one (its picture table), so three camera calls can be in flight before the fourth waits
    cb200::UploadRing upload;
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
    cb200::DevBuf<int32_t> d_recv;          // a receivers frame call's map (Receivers::map): max_frames x 2
    int ccm_frames = 0;              // frames of the last call that took the fitted-CCM route (cb200_get_frame_ccms)
    cudaEvent_t ccm_ev = nullptr;    // recorded after the D2H copies of the last batch's CCM (ccm_resolve waits on it)
    cb200::GatherState* gather = nullptr;   // multi-GPU chunk-record window (gather.cu)
    cb200::ChainState* chain = nullptr;     // multi-GPU CC_FIT chain (chain.cu)
    cb200::DetectState* detect = nullptr;   // side streams and buffers of detect calls led by this context (detect.cu)
    const cb200::SharedWalk* shared_walk = nullptr;   // set only while a detect call decodes this context's mode
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

// the checks every camera and corner call shares, in this order and before any CUDA call: the flags; the batch, from the call's
// builder `build` (which may add the call's own checks that come before the context), and the 4 GB span rule of the deskew; the
// context; `missing` (the message for a null output, or nullptr); n against max_frames; the CCM chain.  The frozen buffers the
// call would grow are checked by the caller (check_frozen_*), which knows which ones it uses
template <class Build>
int check_camera_call(cb200_ctx* c, uint32_t flags, Build&& build, CameraBatch& b, const char* missing)
{
    int rc = check_camera_flags(flags); if (rc) return rc;
    if ((rc = build(b)) || (rc = check_spans(b))) return rc;
    if (!c) return fail(CB200_ERR_ARG, "null context");
    if (missing) return fail(CB200_ERR_ARG, missing);
    if (b.n() > c->max_frames) return fail(CB200_ERR_ARG, "n = " + std::to_string(b.n()) + " > max_frames = " + std::to_string(c->max_frames));
    return check_chain_call(c, flags);
}
}  // namespace cb200
