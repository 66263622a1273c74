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
// as in a receivers plan: decoded, masked, reading and writing no state.  k_detect_select joins the results at each picture's
// position in the sub-batches.
//
// A detect receivers plan (cb200_camera_plan_create_detect_receivers, plan.cu) captures the same geometry loop once over n fixed
// slots.  Its candidates and map are read at each launch, so it has no sub-batches: every geometry works on all n slots, slot i is
// picture i, and k_detect_plan_lists at the head of the graph builds from the two device arrays what detect_lists builds on the host
// (receivers_core.cuh: plan_slot).  A slot that no mode of a geometry decodes is an empty slot of each of its modes, and the
// geometry's walk skips it (SharedWalk::present), so a batch locked to one geometry walks that geometry only.
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

// one CTA per picture: the first mode with a chunk, its record, mask and status.  at: NULL (mode k decoded picture i at position i),
// or (a detect receivers call or plan) mode k decoded picture i at position at[k * n + i] of its geometry's sub-batch, or not at all
// (-1: its mask there counts as 0).  The status of a picture no mode took is its first candidate's; a detect receivers plan's empty
// slot, which has no candidate, gets CB200_EXTRACT_EMPTY (and mode -1, mask 0, a zeroed record).  refused: NULL, or (a plan over
// device descriptors) one byte per slot, set where the launch refused the slot's descriptor: that slot, empty otherwise, reports
// CB200_EXTRACT_REFUSED
__global__ void __launch_bounds__(256)
k_detect_select(const DetectArgs a, const int32_t* __restrict__ at, const uint8_t* __restrict__ refused, int n, uint8_t* __restrict__ chunks,
                uint32_t* __restrict__ mask, int32_t* __restrict__ status, int32_t* __restrict__ mode, uint32_t* __restrict__ mode_masks)
{
    const int i = blockIdx.x;
    int sel = -1, first = -1, p_sel = 0, p_first = 0;
    for (int k = 0; k < a.n_modes; ++k) {
        const int p = at ? at[(size_t)k * n + i] : i;
        if (p < 0) continue;
        if (first < 0) { first = k; p_first = p; }
        if (sel < 0 && a.mask[k][p] != 0) { sel = k; p_sel = p; }
    }
    if (threadIdx.x == 0) {
        mode[i] = sel;
        mask[i] = sel < 0 ? 0u : a.mask[sel][p_sel];
        status[i] = refused && refused[i] ? CB200_EXTRACT_REFUSED : sel >= 0 ? a.status[sel][p_sel] : first >= 0 ? a.status[first][p_first] : CB200_EXTRACT_EMPTY;
        if (mode_masks)
            for (int k = 0; k < a.n_modes; ++k) {
                const int p = at ? at[(size_t)k * n + i] : i;
                mode_masks[(size_t)i * a.n_modes + k] = p < 0 ? 0u : a.mask[k][p];
            }
    }
    const int have = sel < 0 ? 0 : a.data_bytes[sel];
    const uint8_t* src = sel < 0 ? nullptr : a.data[sel] + (size_t)p_sel * have;
    uint8_t* dst = chunks + (size_t)i * a.slot;
    for (int b = threadIdx.x; b < a.slot; b += blockDim.x) dst[b] = b < have ? src[b] : 0;
}

// a detect receivers plan's lists at one launch, one thread per slot (receivers_core.cuh: plan_slot): every mode's raw receivers
// (k_receivers_order then orders each), every geometry's present bytes and every mode's positions.  cand NULL: every mode
struct PlanListArgs { int n_modes, n_geoms, receivers; int group[kDetectModes]; };
__global__ void k_detect_plan_lists(const uint32_t* __restrict__ cand, const int32_t* __restrict__ receiver_of, int n, const PlanListArgs a,
                                    int32_t* __restrict__ raw, uint8_t* __restrict__ present, int32_t* __restrict__ at)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    receivers::plan_slot(cand ? cand[i] : ~0u, receiver_of[i], a.receivers, a.n_modes, a.group, a.n_geoms, n, i, raw, present, at);
}

// a detect receivers plan's list words (DetectPlan::d_lists): n_modes x n raw receivers, n_modes x 2 n maps ([of | order]), then
// n_modes x n positions
size_t detect_plan_words(int n_modes, int n) { return 4 * (size_t)n_modes * (size_t)n; }
static int32_t* plan_map(const DetectPlan& dp, int n_modes, int n, int k) { return dp.d_lists + (size_t)n_modes * n + 2 * (size_t)n * k; }
static int32_t* plan_at(const DetectPlan& dp, int n_modes, int n) { return dp.d_lists + 3 * (size_t)n_modes * n; }

static bool same_geometry(const Mode& a, const Mode& b)
{
    return a.width == b.width && a.height == b.height && a.cells_x == b.cells_x && a.cells_y == b.cells_y && a.cell_offset == b.cell_offset &&
           a.corner == b.corner;
}

// the frame geometries of a set of contexts: group[k], and lead[g] = the first context of geometry g in priority order; returns
// their count
static int geometries(cb200_ctx* const* ctxs, int n_modes, int* group, int* lead)
{
    int ng = 0;
    for (int k = 0; k < n_modes; ++k) {
        int g = 0;
        while (g < ng && !same_geometry(ctxs[lead[g]]->mode, ctxs[k]->mode)) ++g;
        if (g == ng) lead[ng++] = k;
        group[k] = g;
    }
    return ng;
}

// the side streams and events of ng geometries running at once
static int detect_streams(DetectState* ds, int ng)
{
    if (!ds->fork) CK(cudaEventCreateWithFlags(&ds->fork, cudaEventDisableTiming), "cudaEventCreate detect fork");
    for (int g = 0; g < ng; ++g) {
        if (!ds->side[g]) CK(cudaStreamCreateWithFlags(&ds->side[g], cudaStreamNonBlocking), "cudaStreamCreate detect side stream");
        if (!ds->join[g]) CK(cudaEventCreateWithFlags(&ds->join[g], cudaEventDisableTiming), "cudaEventCreate detect join");
    }
    return CB200_OK;
}

static std::string ctx_name(int k) { return "context " + std::to_string(k); }

// the receivers checks of a detect receivers call, which need no context.  on_device (a plan): candidates and receiver_of are device
// arrays that only a launch reads, so their pointers are checked instead of their entries
static int check_detect_receivers(int n_modes, int n, const uint32_t* candidates, const int32_t* receiver_of, int n_receivers,
                                  cb200_receiver_state* const* d_states, bool on_device = false)
{
    if (on_device && reinterpret_cast<uintptr_t>(candidates) % 4) return fail(CB200_ERR_ARG, "d_candidates is not 4-byte aligned");
    for (int i = 0; candidates && !on_device && i < n; ++i) {
        if (!candidates[i]) return fail(CB200_ERR_ARG, "picture " + std::to_string(i) + " has no candidate mode (candidates = 0)");
        if (candidates[i] >> n_modes)
            return fail(CB200_ERR_ARG, "picture " + std::to_string(i) + ": candidates = " + std::to_string(candidates[i]) + " has a bit at or above n_modes = " +
                                           std::to_string(n_modes));
    }
    if (!receiver_of) return fail(CB200_ERR_ARG, on_device ? "null d_receiver_of" : "null receiver_of");
    if (on_device && reinterpret_cast<uintptr_t>(receiver_of) % 4) return fail(CB200_ERR_ARG, "d_receiver_of is not 4-byte aligned");
    if (n_receivers < 1) return fail(CB200_ERR_ARG, "n_receivers < 1");
    for (int i = 0; !on_device && i < n; ++i)
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

// the checks that read the contexts, after every other one.  A plan accepts contexts with live plans (their frozen buffers are
// checked when it is made)
static int check_detect_contexts(cb200_ctx* const* ctxs, int n_modes, int n, bool plan)
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
        if (!plan && !c->plans.empty()) return fail(CB200_ERR_ARG, ctx_name(k) + " has live camera plans: destroy them before a detect call");
        if (n > c->max_frames)
            return fail(CB200_ERR_ARG, "n = " + std::to_string(n) + " > max_frames = " + std::to_string(c->max_frames) + " of " + ctx_name(k));
    }
    return CB200_OK;
}

// every argument check, before any CUDA call: the ones that need no context first.  build: the call's batch builder; more: the
// call's own checks that need no context (a detect receivers call's receivers); plan: a plan's checks
template <class Build, class More>
static int check_detect(cb200_ctx* const* ctxs, int n_modes, uint32_t flags, Build&& build, const uint8_t* d_chunks, const uint32_t* d_chunk_mask,
                        const int32_t* d_extract_status, const int32_t* d_mode, CameraBatch& b, More&& more, bool plan = false)
{
    if (n_modes < 1 || n_modes > kDetectModes)
        return fail(CB200_ERR_ARG, "n_modes = " + std::to_string(n_modes) + ": between 1 and " + std::to_string(kDetectModes) + " candidate modes");
    int rc = check_camera_flags(flags); if (rc) return rc;
    if ((rc = build(b)) || (rc = check_spans(b))) return rc;
    if (!d_chunks || !d_chunk_mask || !d_extract_status || !d_mode) return fail(CB200_ERR_ARG, "null output");
    if ((rc = more())) return rc;
    return check_detect_contexts(ctxs, n_modes, b.n(), plan);
}

// a context's stream for the duration of one geometry's work, restored on every path out
struct StreamSwap {
    cb200_ctx* c; cudaStream_t was;
    StreamSwap(cb200_ctx* c_, cudaStream_t st, const SharedWalk* sw) : c(c_), was(c_->stream) { c->stream = st; c->shared_walk = sw; }
    ~StreamSwap() { c->stream = was; c->shared_walk = nullptr; }
};

// a detect receivers call's receivers: the candidate modes and the receiver map of every picture (host), one state table per mode
// (and a receiver flags table, else NULL: every mode reads it, each scanned picture's receiver travels with the lists, and every mode
// has refused bytes of its own over its geometry's sub-batch)
struct DetectReceivers { const uint32_t* cand; const int32_t* of; int count; cb200_receiver_state* const* d_states; const uint32_t* words; };

// With dr (a detect receivers call), geometry g decodes only its sub-batch U_g (receivers_core.cuh: detect_lists), each of its modes
// with its own receiver map over U_g and state table; a geometry or mode without pictures launches nothing.  The sub-batches' picture
// tables (the scan table's entries, so their blurred offsets keep pointing into ctxs[0]'s scan), scan slots, maps and the selection's
// positions travel behind the scan's picture table: one upload per call.
// With dp (a detect receivers plan's capture), every geometry and mode works on all n slots with the plan's picture table, and the
// lists come from k_detect_plan_lists at the head of the work, on the device
static int detect_enqueue(cb200_ctx* const* ctxs, int n_modes, const CameraBatch& b, uint32_t flags, uint8_t* d_chunks, uint32_t* d_chunk_mask,
                          int32_t* d_extract_status, int32_t* d_mode, uint32_t* d_mode_masks, const DetectReceivers* dr = nullptr,
                          const DetectPlan* dp = nullptr)
{
    cb200_ctx* c0 = ctxs[0];
    const int n = b.n();
    int rc;
    // geometries: lead[g] = the first context of geometry g in priority order (with dr: the first that decodes pictures, or -1)
    int group[kDetectModes], lead[kDetectModes];
    const int ng = geometries(ctxs, n_modes, group, lead);
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
        // (a device batch's scan buffers: camera_scan reserves them from the bounds)
        rc = camera_reserve_for(ctxs[k], bk.wh.data(), bk.n(), !dr && k == 0 && !b.d_pics, lead[group[k]] == k); if (rc) return rc;
    }
    // grown through grow(): a live detect plan's graph reads them
    if ((rc = grow(c0, ds->status, (size_t)n_modes * n, "detect statuses"))) return rc;
    uint8_t* frames[kDetectModes];
    for (int g = 0; g < ng; ++g) {
        if (lead[g] < 0) continue;
        const cb200_ctx* L = ctxs[lead[g]];
        if ((rc = grow(c0, ds->kept[g], (size_t)batch(g).n() * L->mode.num_cells, "detect walk records"))) return rc;
        rc = deskew_frames(ctxs[lead[g]], batch(g).n(), &frames[g]); if (rc) return rc;
    }
    if (live > 1 && (rc = detect_streams(ds, ng))) return rc;
    // dr's lists, in byte offsets from the tail's start: per geometry its picture table and scan slots, per mode its map, the positions
    std::vector<uint8_t> tail;
    size_t desc_at[kDetectModes] = {}, slots_at[kDetectModes] = {}, map_at[kDetectModes] = {}, pos_at = 0, of_at = 0, refused_at = 0;
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
        if (dr->words) { of_at = at; at += sizeof(int32_t) * (size_t)n; refused_at = at; at += (size_t)n_modes * n; }
        tail.assign(at, 0);
        for (int g = 0; g < ng; ++g) {
            PicDesc* d = reinterpret_cast<PicDesc*>(tail.data() + desc_at[g]);
            for (size_t j = 0; j < lists.slots[g].size(); ++j) d[j] = desc[lists.slots[g][j]];
            memcpy(tail.data() + slots_at[g], lists.slots[g].data(), sizeof(int32_t) * lists.slots[g].size());
        }
        for (int k = 0; k < n_modes; ++k) memcpy(tail.data() + map_at[k], lists.map[k].data(), sizeof(int32_t) * lists.map[k].size());
        memcpy(tail.data() + pos_at, lists.pos.data(), sizeof(int32_t) * lists.pos.size());
        if (dr->words) memcpy(tail.data() + of_at, dr->of, sizeof(int32_t) * (size_t)n);
    }
    // a plan over device descriptors: this launch's picture table first, and its map (refused slots emptied) in place of the caller's
    const int32_t* d_of = dp ? dp->d_of : nullptr;
    const uint8_t* d_refused = nullptr;
    if (dp && dp->d_pics_table) {
        rc = plan_pictures_launch(c0, b, dp->d_of, dp->receivers, dp->d_pics_table, dp->d_cand, n_modes); if (rc) return rc;
        const PlanTable t(b);
        d_of = reinterpret_cast<const int32_t*>(dp->d_pics_table + t.of);
        d_refused = dp->d_pics_table + t.refused;
    }
    const PicDesc* d_desc;
    const uint8_t* d_tail = nullptr;
    rc = camera_scan(c0, b, dp ? dp->d_table : nullptr, &d_desc, nullptr, dr ? &tail : nullptr, &d_tail); if (rc) return rc;
    cudaStream_t main = c0->stream;
    if (dp) {                                // this launch's lists, then each mode's [of | order]
        PlanListArgs la;
        memset(&la, 0, sizeof(la));
        la.n_modes = n_modes; la.n_geoms = ng; la.receivers = dp->receivers;
        for (int k = 0; k < n_modes; ++k) la.group[k] = group[k];
        k_detect_plan_lists<<<(n + 127) / 128, 128, 0, main>>>(dp->d_cand, d_of, n, la, dp->d_lists, dp->d_present, plan_at(*dp, n_modes, n));
        count_launch();
        CK(cudaGetLastError(), "detect plan lists launch");
        for (int k = 0; k < n_modes; ++k)
            CK(receivers_order_launch(n, dp->d_lists + (size_t)k * n, dp->receivers, plan_map(*dp, n_modes, n, k), main), "receivers order launch");
    }
    if (live > 1) {
        CK(cudaEventRecord(ds->fork, main), "record detect fork");
        for (int g = 0; g < ng; ++g) if (lead[g] >= 0) CK(cudaStreamWaitEvent(ds->side[g], ds->fork, 0), "wait detect fork");
    }
    // every geometry's modes in priority order, the lead first; every side stream is joined back even when one fails
    for (int g = 0; g < ng && !rc; ++g) {
        if (lead[g] < 0) continue;
        const SharedWalk sw{ctxs[lead[g]], ds->kept[g].get(), dp ? dp->d_present + (size_t)g * n : nullptr};
        const PicDesc* desc_g = dr ? reinterpret_cast<const PicDesc*>(d_tail + desc_at[g]) : d_desc;
        const int32_t* slots_g = dr ? reinterpret_cast<const int32_t*>(d_tail + slots_at[g]) : nullptr;
        for (int k = 0; k < n_modes && !rc; ++k) {
            if (group[k] != g || !decodes(k)) continue;
            cb200_ctx* c = ctxs[k];
            StreamSwap on(c, live > 1 ? ds->side[g] : main, &sw);
            // a plan or a receivers call decodes under mode k's map, in which a slot the mode does not decode is empty
            const int32_t* map_k = dp ? plan_map(*dp, n_modes, n, k) : dr ? reinterpret_cast<const int32_t*>(d_tail + map_at[k]) : nullptr;
            Receivers r(map_k, dp ? dp->d_states[k] : dr ? dr->d_states[k] : nullptr);
            if (dp && dp->d_words) {           // the launch's map, refused descriptors emptied; refused bytes shared by the modes
                r.d_words = dp->d_words; r.receivers = dp->receivers; r.d_pic_of = d_of;
                r.d_refused = d_refused;
            } else if (dr && dr->words) {
                r.d_words = dr->words; r.receivers = dr->count; r.d_pic_of = reinterpret_cast<const int32_t*>(d_tail + of_at);
                r.d_refused = d_tail + refused_at + (size_t)k * n;
            }
            rc = camera_after_scan(c, c0, batch(g), desc_g, flags, frames[g], k == lead[g], c->d_data, c->d_mask, nullptr, ds->status + (size_t)k * n,
                                   map_k ? &r : nullptr, slots_g);
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
    const int32_t* at = dp ? plan_at(*dp, n_modes, n) : dr ? reinterpret_cast<const int32_t*>(d_tail + pos_at) : nullptr;
    k_detect_select<<<n, 256, 0, main>>>(a, at, d_refused, n, d_chunks, d_chunk_mask, d_extract_status, d_mode, d_mode_masks);
    count_launch();
    CK(cudaGetLastError(), "detect select launch");
    return CB200_OK;
}

int check_detect_plan(cb200_ctx* const* ctxs, int n_modes, const cb200_picture* pics, bool dev_pics, const cb200_picture_bounds* bounds,
                      int n, uint32_t flags, const uint32_t* d_candidates, const int32_t* d_receiver_of, int n_receivers,
                      cb200_receiver_state* const* d_states, const uint8_t* d_chunks, const uint32_t* d_chunk_mask,
                      const int32_t* d_extract_status, const int32_t* d_mode, cb200_camera_plan** out, CameraBatch& b)
{
    auto build = [&](CameraBatch& bb) {
        const int rc = dev_pics ? device_batch(pics, n, bounds, bb) : picture_batch(pics, n, bb);
        return rc ? rc : plan_rules(n, out);
    };
    auto more = [&] { return check_detect_receivers(n_modes, n, d_candidates, d_receiver_of, n_receivers, d_states, true); };
    return check_detect(ctxs, n_modes, flags, build, d_chunks, d_chunk_mask, d_extract_status, d_mode, b, more, true);
}

int detect_plan_reserve(cb200_ctx* const* ctxs, int n_modes, const CameraBatch& b, uint32_t flags, bool frozen_only)
{
    int group[kDetectModes], lead[kDetectModes];
    const int ng = geometries(ctxs, n_modes, group, lead), n = b.n();
    int rc;
    for (int k = 0; k < n_modes; ++k) {      // what detect_enqueue reserves with every geometry live, and the decode's own buffers
        cb200_ctx* c = ctxs[k];
        if (frozen_only && c->plans.empty()) continue;
        if ((rc = camera_reserve_for(c, b.wh.data(), n, k == 0 && !b.d_pics, lead[group[k]] == k))) return rc;
        if (k == 0 && b.d_pics && (rc = scan_reserve(c, b))) return rc;      // sized from the bounds
        if (!frozen_only && (rc = decode_reserve(c, flags, true))) return rc;
    }
    cb200_ctx* c0 = ctxs[0];
    if (frozen_only && c0->plans.empty()) return CB200_OK;
    if (!c0->detect) c0->detect = new DetectState();
    DetectState* ds = c0->detect;
    if ((rc = grow(c0, ds->status, (size_t)n_modes * n, "detect statuses"))) return rc;
    for (int g = 0; g < ng; ++g)
        if ((rc = grow(c0, ds->kept[g], (size_t)n * ctxs[lead[g]]->mode.num_cells, "detect walk records"))) return rc;
    return frozen_only || ng < 2 ? CB200_OK : detect_streams(ds, ng);
}

int detect_plan_enqueue(cb200_ctx* const* ctxs, int n_modes, const CameraBatch& b, uint32_t flags, uint8_t* d_chunks, uint32_t* d_chunk_mask,
                        int32_t* d_extract_status, int32_t* d_mode, uint32_t* d_mode_masks, const DetectPlan& dp)
{
    return detect_enqueue(ctxs, n_modes, b, flags, d_chunks, d_chunk_mask, d_extract_status, d_mode, d_mode_masks, nullptr, &dp);
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

static int detect_receivers_call(cb200_ctx* const* ctxs, int n_modes, const cb200_picture* pics, int n, uint32_t flags,
                                 const uint32_t* candidates, const int32_t* receiver_of, int n_receivers, cb200_receiver_state* const* d_states,
                                 const uint32_t* words, uint8_t* d_chunks, uint32_t* d_chunk_mask, int32_t* d_extract_status, int32_t* d_mode,
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
    const DetectReceivers dr = {candidates ? candidates : all.data(), receiver_of, n_receivers, d_states, words};
    return detect_enqueue(ctxs, n_modes, b, flags, d_chunks, d_chunk_mask, d_extract_status, d_mode, d_mode_masks, &dr);
}

extern "C" int cb200_detect_scan_extract_decode_chunks_receivers_dev(cb200_ctx* const* ctxs, int n_modes, const cb200_picture* pics, int n,
                                                                     uint32_t flags, const uint32_t* candidates, const int32_t* receiver_of,
                                                                     int n_receivers, cb200_receiver_state* const* d_states, uint8_t* d_chunks,
                                                                     uint32_t* d_chunk_mask, int32_t* d_extract_status, int32_t* d_mode,
                                                                     uint32_t* d_mode_masks)
{
    return detect_receivers_call(ctxs, n_modes, pics, n, flags, candidates, receiver_of, n_receivers, d_states, nullptr, d_chunks, d_chunk_mask,
                                 d_extract_status, d_mode, d_mode_masks);
}

extern "C" int cb200_detect_scan_extract_decode_chunks_receivers_flags_dev(cb200_ctx* const* ctxs, int n_modes, const cb200_picture* pics,
                                                                           int n, uint32_t flags, const uint32_t* candidates,
                                                                           const int32_t* receiver_of, int n_receivers,
                                                                           cb200_receiver_state* const* d_states, const uint32_t* d_receiver_flags,
                                                                           uint8_t* d_chunks, uint32_t* d_chunk_mask, int32_t* d_extract_status,
                                                                           int32_t* d_mode, uint32_t* d_mode_masks)
{
    const int rc = check_receiver_flags(d_receiver_flags, flags); if (rc) return rc;
    return detect_receivers_call(ctxs, n_modes, pics, n, flags, candidates, receiver_of, n_receivers, d_states, d_receiver_flags, d_chunks,
                                 d_chunk_mask, d_extract_status, d_mode, d_mode_masks);
}
