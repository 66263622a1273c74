// detect.cu -- the receiver's auto mode on the device (cb200_detect_scan_extract_decode_chunks_dev), sm_90a.
//
// The reference's web receiver (web/recv.js) starts without a mode, tries 66, 68, 67 and 4 one per camera frame and keeps the first
// under which a frame gives a chunk.  Here every candidate decodes every picture of one batch, and the work that does not depend on
// the mode is done once:
//   the anchor scan        never reads the mode: it runs once, on the first context's scratch, and every mode's k_extract reads it
//   extract, deskew, sharpen decision and exact walk
//                          depend on the frame geometry only (Extractor / Deskewer take image_size_x / y, is_granular_scale the
//                          size, CimbReader::read decodes symbols and drift on the grey threshold raster): one deskew and one walk
//                          per geometry, on the first context of that geometry; its other modes colour the walk's positions
//                          (SharedWalk, ctx.cuh).  68, 4 and 8 share the 1024 x 1024 geometry; 67 and 66 have their own
//   K1, colours, RS, masks per mode, under that mode's palette and CCM rules (none, CC_SIMPLE, CC_FIT with its carry)
// Geometries run on side streams forked from the contexts' stream, so their walks overlap; k_detect_select joins the results.
//
// cb200_detect_scan_extract_decode_chunks_receivers_dev adds receivers (a decode service's sessions): picture i is decoded only
// under its candidate modes, each mode keeps one state table of receivers, and each geometry extracts, deskews and walks only the
// pictures some of its modes decode (receivers_core.cuh: detect_lists).  A mode's other pictures of that sub-batch are empty slots,
// as in a receivers plan: decoded, masked, reading and writing no state.  k_detect_select_at joins the results.
#include "ctx.cuh"
#include "receivers_core.cuh"

#include <cstring>
#include <string>
#include <vector>

namespace cb200 {

constexpr int kDetectModes = receivers::kMaxModes;

struct DetectState {                 // on the first context of a detect call
    cudaStream_t side[kDetectModes] = {};
    cudaEvent_t fork = nullptr, join[kDetectModes] = {};
    DevBuf<uint32_t> kept[kDetectModes];     // per geometry: the walk's records of every listed frame (SharedWalk::kept)
    DevBuf<int32_t> status;                  // n_modes x n: every mode's extract status
    ~DetectState()
    {
        for (cudaStream_t s : side) if (s) cudaStreamDestroy(s);
        for (cudaEvent_t e : join) if (e) cudaEventDestroy(e);
        if (fork) cudaEventDestroy(fork);
    }
};

void detect_destroy(DetectState* d) { delete d; }

struct DetectArgs {
    int n_modes, slot;                       // slot: the largest data_bytes of the set
    const uint8_t* data[kDetectModes];       // every mode's fixed-slot records (its context's d_data), data_bytes[k] per picture
    int data_bytes[kDetectModes];
    const uint32_t* mask[kDetectModes];
    const int32_t* status[kDetectModes];
};

// one CTA per picture: the first mode with a chunk, its record, mask and status
__global__ void __launch_bounds__(256)
k_detect_select(const DetectArgs a, uint8_t* __restrict__ chunks, uint32_t* __restrict__ mask, int32_t* __restrict__ status,
                int32_t* __restrict__ mode, uint32_t* __restrict__ mode_masks)
{
    const int i = blockIdx.x;
    int sel = -1;
    for (int k = 0; k < a.n_modes; ++k)
        if (sel < 0 && a.mask[k][i] != 0) sel = k;
    if (threadIdx.x == 0) {
        mode[i] = sel;
        mask[i] = sel < 0 ? 0u : a.mask[sel][i];
        status[i] = a.status[sel < 0 ? 0 : sel][i];
        if (mode_masks)
            for (int k = 0; k < a.n_modes; ++k) mode_masks[(size_t)i * a.n_modes + k] = a.mask[k][i];
    }
    const int have = sel < 0 ? 0 : a.data_bytes[sel];
    const uint8_t* src = sel < 0 ? nullptr : a.data[sel] + (size_t)i * have;
    uint8_t* dst = chunks + (size_t)i * a.slot;
    for (int b = threadIdx.x; b < a.slot; b += blockDim.x) dst[b] = b < have ? src[b] : 0;
}

// k_detect_select of a detect receivers call: mode k decoded picture i at position at[k * n + i] of its geometry's sub-batch, or not at
// all (-1: its mask there counts as 0).  The status of a picture no mode took is its first candidate's
__global__ void __launch_bounds__(256)
k_detect_select_at(const DetectArgs a, const int32_t* __restrict__ at, int n, uint8_t* __restrict__ chunks, uint32_t* __restrict__ mask,
                   int32_t* __restrict__ status, int32_t* __restrict__ mode, uint32_t* __restrict__ mode_masks)
{
    const int i = blockIdx.x;
    int sel = -1, first = -1, p_sel = 0, p_first = 0;
    for (int k = 0; k < a.n_modes; ++k) {
        const int p = at[(size_t)k * n + i];
        if (p < 0) continue;
        if (first < 0) { first = k; p_first = p; }
        if (sel < 0 && a.mask[k][p] != 0) { sel = k; p_sel = p; }
    }
    if (threadIdx.x == 0) {
        mode[i] = sel;
        mask[i] = sel < 0 ? 0u : a.mask[sel][p_sel];
        status[i] = sel < 0 ? a.status[first][p_first] : a.status[sel][p_sel];
        if (mode_masks)
            for (int k = 0; k < a.n_modes; ++k) {
                const int p = at[(size_t)k * n + i];
                mode_masks[(size_t)i * a.n_modes + k] = p < 0 ? 0u : a.mask[k][p];
            }
    }
    const int have = sel < 0 ? 0 : a.data_bytes[sel];
    const uint8_t* src = sel < 0 ? nullptr : a.data[sel] + (size_t)p_sel * have;
    uint8_t* dst = chunks + (size_t)i * a.slot;
    for (int b = threadIdx.x; b < a.slot; b += blockDim.x) dst[b] = b < have ? src[b] : 0;
}

static bool same_geometry(const Mode& a, const Mode& b)
{
    return a.width == b.width && a.height == b.height && a.cells_x == b.cells_x && a.cells_y == b.cells_y && a.cell_offset == b.cell_offset &&
           a.corner == b.corner;
}

static std::string ctx_name(int k) { return "context " + std::to_string(k); }

// the receivers checks of a detect receivers call, which need no context
static int check_detect_receivers(int n_modes, int n, const uint32_t* candidates, const int32_t* receiver_of, int n_receivers,
                                  cb200_receiver_state* const* d_states)
{
    for (int i = 0; candidates && i < n; ++i) {
        if (!candidates[i]) return fail(CB200_ERR_ARG, "picture " + std::to_string(i) + " has no candidate mode (candidates = 0)");
        if (candidates[i] >> n_modes)
            return fail(CB200_ERR_ARG, "picture " + std::to_string(i) + ": candidates = " + std::to_string(candidates[i]) + " has a bit at or above n_modes = " +
                                           std::to_string(n_modes));
    }
    if (!receiver_of) return fail(CB200_ERR_ARG, "null receiver_of");
    if (n_receivers < 1) return fail(CB200_ERR_ARG, "n_receivers < 1");
    for (int i = 0; i < n; ++i)
        if (receiver_of[i] < 0 || receiver_of[i] >= n_receivers)
            return fail(CB200_ERR_ARG, "picture " + std::to_string(i) + ": receiver " + std::to_string(receiver_of[i]) + " outside [0, " +
                                       std::to_string(n_receivers) + ")");
    if (!d_states) return fail(CB200_ERR_ARG, "null d_states");
    const size_t span = sizeof(cb200_receiver_state) * (size_t)n_receivers;
    for (int k = 0; k < n_modes; ++k) {
        const uintptr_t p = reinterpret_cast<uintptr_t>(d_states[k]);
        const std::string name = "d_states[" + std::to_string(k) + "]";
        if (!p) return fail(CB200_ERR_ARG, name + " (the state table of context " + std::to_string(k) + ") is null");
        if (p % 4) return fail(CB200_ERR_ARG, name + " (the state table of context " + std::to_string(k) + ") is not 4-byte aligned");
        for (int j = 0; j < k; ++j) {
            const uintptr_t q = reinterpret_cast<uintptr_t>(d_states[j]);
            if (p < q + span && q < p + span)
                return fail(CB200_ERR_ARG, "d_states[" + std::to_string(j) + "] and " + name + " overlap: each candidate mode needs its own " +
                                               std::to_string(n_receivers) + "-entry table");
        }
    }
    return CB200_OK;
}

// the checks that read the contexts, after every other one
static int check_detect_contexts(cb200_ctx* const* ctxs, int n_modes, int n)
{
    if (!ctxs) return fail(CB200_ERR_ARG, "null context list");
    for (int k = 0; k < n_modes; ++k)
        if (!ctxs[k]) return fail(CB200_ERR_ARG, ctx_name(k) + " is null");
    for (int k = 0; k < n_modes; ++k) {
        const cb200_ctx* c = ctxs[k];
        for (int j = 0; j < k; ++j)
            if (ctxs[j]->mode.mode_val == c->mode.mode_val)
                return fail(CB200_ERR_ARG, "contexts " + std::to_string(j) + " and " + std::to_string(k) + " are both mode " + std::to_string(c->mode.mode_val) +
                                               ": the candidate modes must be distinct");
        if (c->device != ctxs[0]->device)
            return fail(CB200_ERR_ARG, ctx_name(k) + " is on device " + std::to_string(c->device) + ", context 0 on device " + std::to_string(ctxs[0]->device) +
                                           ": the candidates must share one device");
        if (c->stream != ctxs[0]->stream) return fail(CB200_ERR_ARG, ctx_name(k) + " is on another stream than context 0: the candidates must share one stream");
        if (chain_attached(c)) return fail(CB200_ERR_ARG, ctx_name(k) + " is linked to a CCM chain: chained contexts cannot be detect candidates");
        if (!c->plans.empty()) return fail(CB200_ERR_ARG, ctx_name(k) + " has live camera plans: destroy them before a detect call");
        if (n > c->max_frames)
            return fail(CB200_ERR_ARG, "n = " + std::to_string(n) + " > max_frames = " + std::to_string(c->max_frames) + " of " + ctx_name(k));
    }
    return CB200_OK;
}

// every argument check, before any CUDA call: the ones that need no context first.  build: the call's batch builder; more: the
// call's own checks that need no context (a detect receivers call's receivers)
template <class Build, class More>
static int check_detect(cb200_ctx* const* ctxs, int n_modes, uint32_t flags, Build&& build, const uint8_t* d_chunks, const uint32_t* d_chunk_mask,
                        const int32_t* d_extract_status, const int32_t* d_mode, CameraBatch& b, More&& more)
{
    if (n_modes < 1 || n_modes > kDetectModes)
        return fail(CB200_ERR_ARG, "n_modes = " + std::to_string(n_modes) + ": between 1 and " + std::to_string(kDetectModes) + " candidate modes");
    int rc = check_camera_flags(flags); if (rc) return rc;
    if ((rc = build(b)) || (rc = check_spans(b))) return rc;
    if (!d_chunks || !d_chunk_mask || !d_extract_status || !d_mode) return fail(CB200_ERR_ARG, "null output");
    if ((rc = more())) return rc;
    return check_detect_contexts(ctxs, n_modes, b.n());
}

// a context's stream for the duration of one geometry's work, restored on every path out
struct StreamSwap {
    cb200_ctx* c; cudaStream_t was;
    StreamSwap(cb200_ctx* c_, cudaStream_t st, const SharedWalk* sw) : c(c_), was(c_->stream) { c->stream = st; c->shared_walk = sw; }
    ~StreamSwap() { c->stream = was; c->shared_walk = nullptr; }
};

// a detect receivers call's receivers: the candidate modes and the receiver map of every picture (host), one state table per mode
struct DetectReceivers { const uint32_t* cand; const int32_t* of; int count; cb200_receiver_state* const* d_states; };

// With dr (a detect receivers call), geometry g decodes only its sub-batch U_g (receivers_core.cuh: detect_lists), each of its modes
// with its own receiver map over U_g and state table; a geometry or mode without pictures launches nothing.  The sub-batches' picture
// tables (the scan table's entries, so their blurred offsets keep pointing into ctxs[0]'s scan), scan slots, maps and the selection's
// positions travel behind the scan's picture table: one upload per call
static int detect_enqueue(cb200_ctx* const* ctxs, int n_modes, const CameraBatch& b, uint32_t flags, uint8_t* d_chunks, uint32_t* d_chunk_mask,
                          int32_t* d_extract_status, int32_t* d_mode, uint32_t* d_mode_masks, const DetectReceivers* dr = nullptr)
{
    cb200_ctx* c0 = ctxs[0];
    const int n = b.n();
    int rc;
    // geometries: lead[g] = the first context of geometry g in priority order (with dr: the first that decodes pictures, or -1)
    int group[kDetectModes], lead[kDetectModes], ng = 0;
    for (int k = 0; k < n_modes; ++k) {
        int g = 0;
        while (g < ng && !same_geometry(ctxs[lead[g]]->mode, ctxs[k]->mode)) ++g;
        if (g == ng) lead[ng++] = k;
        group[k] = g;
    }
    receivers::DetectLists lists;
    CameraBatch sub[kDetectModes];
    if (dr) {
        receivers::detect_lists(dr->cand, dr->of, n, dr->count, n_modes, group, lists);
        for (int g = 0; g < ng; ++g) lead[g] = -1;
        for (int k = n_modes - 1; k >= 0; --k) if (lists.count[k]) lead[group[k]] = k;
        for (int g = 0; g < ng; ++g) {
            sub[g].packed = b.packed;
            for (const int32_t i : lists.slots[g]) {
                sub[g].pics.push_back(b.pics[(size_t)i]);
                sub[g].wh.push_back(b.wh[2 * (size_t)i]); sub[g].wh.push_back(b.wh[2 * (size_t)i + 1]);
            }
        }
    }
    auto batch = [&](int g) -> const CameraBatch& { return dr ? sub[g] : b; };
    auto decodes = [&](int k) { return !dr || lists.count[k] > 0; };
    int live = 0;                            // geometries with pictures
    for (int g = 0; g < ng; ++g) live += lead[g] >= 0;
    if (!c0->detect) c0->detect = new DetectState();
    DetectState* ds = c0->detect;
    if (dr) { rc = scan_reserve(c0, b.wh.data(), n); if (rc) return rc; }
    for (int k = 0; k < n_modes; ++k) {
        if (!decodes(k)) continue;
        const CameraBatch& bk = batch(group[k]);
        rc = camera_reserve_for(ctxs[k], bk.wh.data(), bk.n(), !dr && k == 0, lead[group[k]] == k); if (rc) return rc;
    }
    CK(ds->status.ensure((size_t)n_modes * n), "cudaMalloc detect statuses");
    uint8_t* frames[kDetectModes];
    for (int g = 0; g < ng; ++g) {
        if (lead[g] < 0) continue;
        const cb200_ctx* L = ctxs[lead[g]];
        CK(ds->kept[g].ensure((size_t)batch(g).n() * L->mode.num_cells), "cudaMalloc detect walk records");
        rc = deskew_frames(ctxs[lead[g]], batch(g).n(), &frames[g]); if (rc) return rc;
    }
    if (live > 1) {
        if (!ds->fork) CK(cudaEventCreateWithFlags(&ds->fork, cudaEventDisableTiming), "cudaEventCreate detect fork");
        for (int g = 0; g < ng; ++g) {
            if (!ds->side[g]) CK(cudaStreamCreateWithFlags(&ds->side[g], cudaStreamNonBlocking), "cudaStreamCreate detect side stream");
            if (!ds->join[g]) CK(cudaEventCreateWithFlags(&ds->join[g], cudaEventDisableTiming), "cudaEventCreate detect join");
        }
    }
    // dr's lists, in byte offsets from the tail's start: per geometry its picture table and scan slots, per mode its map, the positions
    std::vector<uint8_t> tail;
    size_t desc_at[kDetectModes] = {}, slots_at[kDetectModes] = {}, map_at[kDetectModes] = {}, pos_at = 0;
    if (dr) {
        static_assert(sizeof(PicDesc) % 8 == 0, "the sub-batch tables follow each other 8-byte aligned");
        std::vector<uint8_t> table;
        rc = pic_table(c0, b, table); if (rc) return rc;
        const PicDesc* desc = reinterpret_cast<const PicDesc*>(table.data());
        size_t at = 0;
        for (int g = 0; g < ng; ++g) { desc_at[g] = at; at += sizeof(PicDesc) * lists.slots[g].size(); }
        for (int g = 0; g < ng; ++g) { slots_at[g] = at; at += sizeof(int32_t) * lists.slots[g].size(); }
        for (int k = 0; k < n_modes; ++k) { map_at[k] = at; at += sizeof(int32_t) * lists.map[k].size(); }
        pos_at = at; at += sizeof(int32_t) * lists.pos.size();
        tail.resize(at);
        for (int g = 0; g < ng; ++g) {
            PicDesc* d = reinterpret_cast<PicDesc*>(tail.data() + desc_at[g]);
            for (size_t j = 0; j < lists.slots[g].size(); ++j) d[j] = desc[lists.slots[g][j]];
            memcpy(tail.data() + slots_at[g], lists.slots[g].data(), sizeof(int32_t) * lists.slots[g].size());
        }
        for (int k = 0; k < n_modes; ++k) memcpy(tail.data() + map_at[k], lists.map[k].data(), sizeof(int32_t) * lists.map[k].size());
        memcpy(tail.data() + pos_at, lists.pos.data(), sizeof(int32_t) * lists.pos.size());
    }
    const PicDesc* d_desc;
    const uint8_t* d_tail = nullptr;
    rc = camera_scan(c0, b, nullptr, &d_desc, nullptr, dr ? &tail : nullptr, &d_tail); if (rc) return rc;
    cudaStream_t main = c0->stream;
    if (live > 1) {
        CK(cudaEventRecord(ds->fork, main), "record detect fork");
        for (int g = 0; g < ng; ++g) if (lead[g] >= 0) CK(cudaStreamWaitEvent(ds->side[g], ds->fork, 0), "wait detect fork");
    }
    // every geometry's modes in priority order, the lead first; every side stream is joined back even when one fails
    for (int g = 0; g < ng && !rc; ++g) {
        if (lead[g] < 0) continue;
        const SharedWalk sw{ctxs[lead[g]], ds->kept[g].get()};
        const PicDesc* desc_g = dr ? reinterpret_cast<const PicDesc*>(d_tail + desc_at[g]) : d_desc;
        const int32_t* slots_g = dr ? reinterpret_cast<const int32_t*>(d_tail + slots_at[g]) : nullptr;
        for (int k = 0; k < n_modes && !rc; ++k) {
            if (group[k] != g || !decodes(k)) continue;
            cb200_ctx* c = ctxs[k];
            StreamSwap on(c, live > 1 ? ds->side[g] : main, &sw);
            if (!dr) {
                rc = camera_after_scan(c, c0, b, d_desc, flags, frames[g], k == lead[g], c->d_data, c->d_mask, nullptr, ds->status + (size_t)k * n);
                continue;
            }
            Receivers r(reinterpret_cast<const int32_t*>(d_tail + map_at[k]), dr->d_states[k]);
            r.empty_slots = lists.count[k] < batch(g).n();       // without empty slots, the direct receivers call's kernels
            rc = camera_after_scan(c, c0, batch(g), desc_g, flags, frames[g], k == lead[g], c->d_data, c->d_mask, nullptr, ds->status + (size_t)k * n,
                                   &r, slots_g);
        }
    }
    if (live > 1) {
        for (int g = 0; g < ng; ++g) {
            if (lead[g] < 0) continue;
            CK(cudaEventRecord(ds->join[g], ds->side[g]), "record detect join");
            CK(cudaStreamWaitEvent(main, ds->join[g], 0), "wait detect join");
        }
    }
    if (rc) return rc;
    DetectArgs a;
    memset(&a, 0, sizeof(a));
    a.n_modes = n_modes;
    for (int k = 0; k < n_modes; ++k) {
        const cb200_ctx* c = ctxs[k];
        a.data[k] = c->d_data; a.data_bytes[k] = c->mode.data_bytes; a.mask[k] = c->d_mask; a.status[k] = ds->status + (size_t)k * n;
        if (a.data_bytes[k] > a.slot) a.slot = a.data_bytes[k];
    }
    if (dr) k_detect_select_at<<<n, 256, 0, main>>>(a, reinterpret_cast<const int32_t*>(d_tail + pos_at), n, d_chunks, d_chunk_mask, d_extract_status,
                                                    d_mode, d_mode_masks);
    else k_detect_select<<<n, 256, 0, main>>>(a, d_chunks, d_chunk_mask, d_extract_status, d_mode, d_mode_masks);
    count_launch();
    CK(cudaGetLastError(), "detect select launch");
    return CB200_OK;
}

}  // namespace cb200

using namespace cb200;

extern "C" int cb200_detect_scan_extract_decode_chunks_dev(cb200_ctx* const* ctxs, int n_modes, const uint8_t* d_pictures, const int32_t* wh,
                                                           int n, uint32_t flags, uint8_t* d_chunks, uint32_t* d_chunk_mask,
                                                           int32_t* d_extract_status, int32_t* d_mode, uint32_t* d_mode_masks)
{
    CameraBatch b;
    auto build = [&](CameraBatch& bb) { return packed_batch(d_pictures, wh, n, bb); };
    int rc = check_detect(ctxs, n_modes, flags, build, d_chunks, d_chunk_mask, d_extract_status, d_mode, b, [] { return CB200_OK; });
    if (rc) return rc;
    if (n == 0) return CB200_OK;
    CK(cudaSetDevice(ctxs[0]->device), "cudaSetDevice");
    return detect_enqueue(ctxs, n_modes, b, flags, d_chunks, d_chunk_mask, d_extract_status, d_mode, d_mode_masks);
}

extern "C" int cb200_detect_scan_extract_decode_chunks_receivers_dev(cb200_ctx* const* ctxs, int n_modes, const cb200_picture* pics, int n,
                                                                     uint32_t flags, const uint32_t* candidates, const int32_t* receiver_of,
                                                                     int n_receivers, cb200_receiver_state* const* d_states, uint8_t* d_chunks,
                                                                     uint32_t* d_chunk_mask, int32_t* d_extract_status, int32_t* d_mode,
                                                                     uint32_t* d_mode_masks)
{
    CameraBatch b;
    auto build = [&](CameraBatch& bb) { return picture_batch(pics, n, bb); };
    auto more = [&] { return check_detect_receivers(n_modes, n, candidates, receiver_of, n_receivers, d_states); };
    int rc = check_detect(ctxs, n_modes, flags, build, d_chunks, d_chunk_mask, d_extract_status, d_mode, b, more); if (rc) return rc;
    if (n == 0) return CB200_OK;
    CK(cudaSetDevice(ctxs[0]->device), "cudaSetDevice");
    std::vector<uint32_t> all;
    if (!candidates) all.assign((size_t)n, (1u << n_modes) - 1);
    const DetectReceivers dr = {candidates ? candidates : all.data(), receiver_of, n_receivers, d_states};
    return detect_enqueue(ctxs, n_modes, b, flags, d_chunks, d_chunk_mask, d_extract_status, d_mode, d_mode_masks, &dr);
}
