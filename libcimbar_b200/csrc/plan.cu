// plan.cu -- camera plans: the enqueue-only camera call (scan.cu camera_enqueue) captured once in a CUDA graph and replayed with one
// cudaGraphLaunch per batch (include/cb200.h, "camera plans").
//
// What the direct call decides on the host per call, a plan decides once:
//   - the picture table is built at creation into the plan's own device memory (a captured copy from the context's pinned upload
//     ring would read the slot at replay time, after later calls rewrote it);
//   - every context buffer the path uses is grown before the capture, and frozen while the plan lives (grow(), ctx.cuh): a graph
//     keeps the pointers it was captured with, and growing frees them;
//   - the CCM always comes from the device (c->d_carry, which carry_from_host keeps current while plans exist) instead of
//     cudaEventQuery choosing between the host matrix and the carry, a choice a graph would freeze at capture time.
// The kernels are the direct call's, launched by the same code on a private capture stream.
//
// A receivers plan (cb200_camera_plan_create_receivers) is the receivers camera call captured so.  Its receiver map is the one
// input the direct call builds on the host per batch: here k_receivers_order, captured at the head of the graph, builds it at each
// launch from the caller's d_receiver_of into the plan's own d_map, and the rest of the graph reads it from there.
//
// A receivers plan over device descriptors (cb200_camera_plan_create_receivers_pictures_dev) reads the picture descriptors at each
// launch too: k_plan_pictures (scan.cu), ahead of k_receivers_order, checks them and writes the picture table the host builds for the
// other plans, and the plan's map with its refused slots emptied; the scan's buffers are sized from the plan's bounds.
//
// A detect receivers plan (cb200_camera_plan_create_detect_receivers) is the detect receivers call captured so, over several
// contexts: detect.cu's geometry loop on every context's buffers, with every context's stream swapped to the capture stream, and
// the side streams' forks and joins becoming parallel branches of the graph.  Its candidates and map are read at each launch
// (k_detect_plan_lists at the head of the graph builds every list into d_map and d_present).  It is registered in the plans of every
// one of its contexts, so each of them freezes the buffers the graph uses, and destroying any of them destroys the plan.  Over device
// descriptors (cb200_camera_plan_create_detect_receivers_pictures_dev), k_plan_pictures comes first and k_detect_plan_lists reads its
// map, and the selection gives the refused slots their status.
#include "ctx.cuh"

#include <memory>
#include <string>
#include <vector>

using namespace cb200;

struct cb200_camera_plan {
    cb200_ctx* ctx = nullptr;               // the context whose stream launches the plan (a detect plan: its first)
    std::vector<cb200_ctx*> ctxs;           // every context whose buffers the graph uses: ctx, or a detect plan's candidates
    int n = 0;
    uint32_t flags = 0;
    DevBuf<uint8_t> d_table;                // n PicDesc, then the pictures grouped by blur radius
    // a receivers plan: the caller's map and states, and the map the graph builds from it (n receivers, -1 = empty, then the order).
    // A detect receivers plan: the caller's map and candidates, each mode's state table, and d_map holds the lists the graph builds
    // (detect_plan_words), d_present the geometries' present bytes
    const int32_t* d_receiver_of = nullptr;
    int n_receivers = 0;
    cb200_receiver_state* d_states = nullptr;
    DevBuf<int32_t> d_map;
    const uint32_t* d_candidates = nullptr;
    std::vector<cb200_receiver_state*> d_mode_states;
    DevBuf<uint8_t> d_present;
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t exec = nullptr;
    int kernels = 0;                        // kernel nodes of the graph (cb200_launch_count)
    bool keeps_ccm = false;                 // CC_SIMPLE, or CC_FIT where it fits: a launch leaves a new CCM in d_carry / h_ccm
};

namespace cb200 {

int plan_frozen(const cb200_ctx* c, const char* buffer, size_t have, size_t need)
{
    return fail(CB200_ERR_ARG, std::string("the ") + buffer + " would grow from " + std::to_string(have) + " to " + std::to_string(need) +
                                   " elements, but " + std::to_string(c->plans.size()) +
                                   " camera plan(s) of this context use it: destroy the plans first");
}

int check_frozen_frames(cb200_ctx* c, int n) { return c->plans.empty() ? CB200_OK : flood_reserve(c, n); }

int check_frozen_deskew(cb200_ctx* c, int n)
{
    if (c->plans.empty()) return CB200_OK;
    int rc = deskew_reserve(c, n); if (rc) return rc;
    return flood_reserve(c, n);
}

int check_frozen_camera(cb200_ctx* c, const int32_t* wh, int n) { return c->plans.empty() ? CB200_OK : camera_reserve(c, wh, n); }

int check_frozen_camera(cb200_ctx* c, const CameraBatch& b) { return c->plans.empty() ? CB200_OK : camera_reserve(c, b); }

int check_frozen_scan(cb200_ctx* c, const int32_t* wh, int n) { return c->plans.empty() ? CB200_OK : scan_reserve(c, wh, n); }

int plan_rules(int n, cb200_camera_plan** out)
{
    if (n == 0) return fail(CB200_ERR_ARG, "n = 0: a camera plan needs at least one picture");
    if (!out) return fail(CB200_ERR_ARG, "null plan");
    *out = nullptr;
    return CB200_OK;
}

}  // namespace cb200

namespace {

int count_kernel_nodes(cudaGraph_t g, int* kernels)
{
    size_t count = 0;
    CK(cudaGraphGetNodes(g, nullptr, &count), "cudaGraphGetNodes");
    std::vector<cudaGraphNode_t> nodes(count);
    CK(cudaGraphGetNodes(g, nodes.data(), &count), "cudaGraphGetNodes");
    *kernels = 0;
    for (cudaGraphNode_t nd : nodes) {
        cudaGraphNodeType t;
        CK(cudaGraphNodeGetType(nd, &t), "cudaGraphNodeGetType");
        *kernels += t == cudaGraphNodeTypeKernel;
    }
    return CB200_OK;
}

// enqueue(): the plan's work on the private stream `cap`, captured into p->graph.  Every context's stream, timing and host CCM state
// are set aside for the duration and restored: a capture runs nothing, so it changes nothing the host can observe
template <class Enqueue>
int capture(cb200_camera_plan* p, cudaStream_t cap, Enqueue&& enqueue)
{
    struct Saved {
        cudaStream_t stream; bool timing, pending, pending_flag, active; int ccm_frames, camera_n;
        cudaEvent_t ccm_ev, scratch_ev;     // ccm_keep_last records c->ccm_ev: inside a capture that record joins the graph
    };
    std::vector<Saved> saved(p->ctxs.size());
    for (size_t i = 0; i < saved.size(); ++i) {
        const cudaError_t e = cudaEventCreateWithFlags(&saved[i].scratch_ev, cudaEventDisableTiming);
        if (e != cudaSuccess) { while (i > 0) cudaEventDestroy(saved[--i].scratch_ev); return fail_cuda(e, "cudaEventCreate"); }
    }
    for (size_t i = 0; i < saved.size(); ++i) {
        cb200_ctx* c = p->ctxs[i];
        Saved& s = saved[i];
        s.stream = c->stream; s.timing = c->timing; s.pending = c->ccm_pending; s.pending_flag = c->ccm_pending_flag; s.active = c->ccm_active;
        s.ccm_frames = c->ccm_frames; s.camera_n = camera_pictures(c); s.ccm_ev = c->ccm_ev;
        c->ccm_ev = s.scratch_ev;
        c->stream = cap;
        c->timing = false;
        c->capturing = true;
    }
    const unsigned long long launches = cb200_launch_count();
    int rc = CB200_OK;
    cudaError_t e = cudaStreamBeginCapture(cap, cudaStreamCaptureModeThreadLocal);
    if (e != cudaSuccess) rc = fail_cuda(e, "cudaStreamBeginCapture");
    if (!rc) {
        rc = enqueue();
        cudaGraph_t g = nullptr;
        e = cudaStreamEndCapture(cap, &g);
        if (!rc && e != cudaSuccess) rc = fail_cuda(e, "cudaStreamEndCapture");
        if (rc) { if (g) cudaGraphDestroy(g); } else p->graph = g;
    }
    for (size_t i = 0; i < saved.size(); ++i) {
        cb200_ctx* c = p->ctxs[i];
        const Saved& s = saved[i];
        c->capturing = false;
        c->timing = s.timing;
        c->stream = s.stream;
        c->ccm_ev = s.ccm_ev;
        c->ccm_pending = s.pending; c->ccm_pending_flag = s.pending_flag; c->ccm_active = s.active;
        c->ccm_frames = s.ccm_frames;
        set_camera_pictures(c, s.camera_n);
        cudaEventDestroy(s.scratch_ev);
    }
    // the captured launches did not run: launch() counts them each time the graph does
    count_launch(-(int)(cb200_launch_count() - launches));
    return rc;
}

// a plan for the checked batch b (after every argument check), in p (its contexts, size, flags and bound pointers set; owned here):
// the freeze check -- reserve(true), no CUDA call --, every buffer the graph uses grown -- reserve(false) --, the table uploaded, the
// capture of enqueue(table), the graph instantiated, the plan registered with every one of its contexts
template <class Reserve, class Enqueue>
int make_plan(cb200_camera_plan* plan, const CameraBatch& b, Reserve&& reserve, Enqueue&& enqueue, cb200_camera_plan** out)
{
    std::unique_ptr<cb200_camera_plan> own(plan);
    cb200_camera_plan* p = plan;
    cb200_ctx* c = p->ctx;
    int rc = reserve(true); if (rc) return rc;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    // with plans already there, the freeze check above guarantees this grows nothing
    rc = reserve(false); if (rc) return rc;
    std::vector<uint8_t> table;
    cudaStream_t cap = nullptr;
    // a plan over device descriptors: its graph writes the table at each launch, and only the stand-in picture's row (zeros) is set here
    if (!rc && !b.d_pics) rc = pic_table(c, b, table);
    const size_t bytes = b.d_pics ? PlanTable(b).bytes : table.size();
    if (!rc) { const cudaError_t e = p->d_table.ensure(bytes); if (e != cudaSuccess) rc = fail_cuda(e, "cudaMalloc plan picture table"); }
    if (!rc) { const cudaError_t e = cudaStreamCreateWithFlags(&cap, cudaStreamNonBlocking); if (e != cudaSuccess) rc = fail_cuda(e, "cudaStreamCreate"); }
    if (!rc) {   // the table goes up once, on the private stream, before anything can replay
        cudaError_t e = b.d_pics ? cudaMemsetAsync(p->d_table, 0, bytes, cap) : cudaMemcpyAsync(p->d_table, table.data(), bytes, cudaMemcpyHostToDevice, cap);
        if (e == cudaSuccess) e = cudaStreamSynchronize(cap);
        if (e != cudaSuccess) rc = fail_cuda(e, "H2D plan picture table");
    }
    if (!rc) rc = capture(p, cap, [&] { return enqueue(reinterpret_cast<const PicDesc*>(p->d_table.get())); });
    if (cap) cudaStreamDestroy(cap);
    if (!rc) rc = count_kernel_nodes(p->graph, &p->kernels);
    if (!rc) { const cudaError_t e = cudaGraphInstantiate(&p->exec, p->graph, 0); if (e != cudaSuccess) rc = fail_cuda(e, "cudaGraphInstantiate"); }
    if (rc) {
        const std::string why = cb200_last_error();
        if (p->graph) cudaGraphDestroy(p->graph);
        return fail(rc, why);
    }
    own.release();
    // the graph starts from d_carry: unless a CCM is on its way there from the device, the host's goes there now (a receivers plan
    // reads no context CCM, but while plans exist d_carry mirrors the host's matrix for every plain one)
    for (cb200_ctx* x : p->ctxs) x->plans.push_back(p);
    for (cb200_ctx* x : p->ctxs)
        if (!x->ccm_pending && (rc = carry_from_host(x)) != CB200_OK) { cb200_camera_plan_destroy(p); return rc; }
    *out = p;
    return CB200_OK;
}

// a plain or receivers plan on context c (recv: the bound map and states; its d_map is allocated here) over the batch `build`
// makes: the direct camera call's checks, with the plan's own after the batch's and after the CCM chain's, then the plan
struct PlanReceivers { const int32_t* d_receiver_of; int n_receivers; cb200_receiver_state* d_states; const uint32_t* d_words; };

template <class Build>
int make_camera_plan(cb200_ctx* c, Build&& build, uint32_t flags, uint8_t* d_chunks, uint32_t* d_chunk_mask, uint8_t* d_frame_flags,
                     int32_t* d_extract_status, const PlanReceivers* recv, cb200_camera_plan** out)
{
    auto plan_build = [&](CameraBatch& b) { const int rc = build(b); return rc ? rc : plan_rules(b.n(), out); };
    CameraBatch b;
    int rc = check_camera_call(c, flags, plan_build, b, d_chunks && d_chunk_mask && d_extract_status ? nullptr : "null output"); if (rc) return rc;
    if (check_host_ccm(c))
        return fail(CB200_ERR_ARG, "the context is linked to a CCM chain, whose step the host sets per call: no camera plan");
    const int n = b.n();
    cb200_camera_plan* p = new cb200_camera_plan();
    p->ctx = c; p->ctxs.assign(1, c); p->n = n; p->flags = flags;
    p->keeps_ccm = !recv && ((flags & CB200_FLAG_CC_SIMPLE) || ccm_fits(c->mode, flags));
    if (recv) { p->d_receiver_of = recv->d_receiver_of; p->n_receivers = recv->n_receivers; p->d_states = recv->d_states; }
    auto reserve = [&](bool frozen_only) {
        if (frozen_only) return check_frozen_camera(c, b);
        int rc = camera_reserve(c, b); if (rc) return rc;
        if ((rc = decode_reserve(c, flags, recv != nullptr))) return rc;
        if (recv) CK(p->d_map.ensure(2 * (size_t)n), "cudaMalloc plan receiver map");
        return CB200_OK;
    };
    auto enqueue = [&](const PicDesc* table) {
        if (!recv) return camera_enqueue(c, b, flags, d_chunks, d_chunk_mask, d_frame_flags, d_extract_status, table);
        Receivers r(p->d_map.get(), p->d_states);
        r.d_words = recv->d_words;
        r.receivers = p->n_receivers;
        const int32_t* of = p->d_receiver_of;
        if (b.d_pics) {   // device descriptors: k_plan_pictures first, and the order from its map, in which refused slots are empty
            int rc = plan_pictures_launch(c, b, p->d_receiver_of, p->n_receivers, p->d_table); if (rc) return rc;
            const PlanTable t(b);
            of = reinterpret_cast<const int32_t*>(p->d_table + t.of);
            r.d_refused = p->d_table + t.refused;
        }
        CK(receivers_order_launch(n, of, p->n_receivers, p->d_map, c->stream), "receivers order launch");
        return camera_enqueue(c, b, flags, d_chunks, d_chunk_mask, d_frame_flags, d_extract_status, table, &r);
    };
    return make_plan(p, b, reserve, enqueue, out);
}

// a detect receivers plan for the checked batch b (descriptors on the host, or in device memory within bounds)
int make_detect_plan(cb200_ctx* const* ctxs, int n_modes, const CameraBatch& b, uint32_t flags, const uint32_t* d_candidates,
                     const int32_t* d_receiver_of, int n_receivers, cb200_receiver_state* const* d_states, uint8_t* d_chunks,
                     uint32_t* d_chunk_mask, int32_t* d_extract_status, int32_t* d_mode, uint32_t* d_mode_masks, cb200_camera_plan** out,
                     const uint32_t* d_words = nullptr)
{
    const int n = b.n();
    cb200_camera_plan* p = new cb200_camera_plan();
    p->ctx = ctxs[0]; p->ctxs.assign(ctxs, ctxs + n_modes); p->n = n; p->flags = flags;
    p->d_receiver_of = d_receiver_of; p->n_receivers = n_receivers; p->d_candidates = d_candidates;
    p->d_mode_states.assign(d_states, d_states + n_modes);
    auto reserve = [&](bool frozen_only) {
        int rc = detect_plan_reserve(ctxs, n_modes, b, flags, frozen_only);
        if (rc || frozen_only) return rc;
        CK(p->d_map.ensure(detect_plan_words(n_modes, n)), "cudaMalloc plan lists");
        CK(p->d_present.ensure((size_t)n_modes * n), "cudaMalloc plan present slots");
        return CB200_OK;
    };
    auto enqueue = [&](const PicDesc* table) {
        const DetectPlan dp = {table, d_candidates, d_receiver_of, n_receivers, p->d_mode_states.data(), p->d_map.get(), p->d_present.get(),
                               b.d_pics ? p->d_table.get() : nullptr, d_words};
        return detect_plan_enqueue(ctxs, n_modes, b, flags, d_chunks, d_chunk_mask, d_extract_status, d_mode, d_mode_masks, dp);
    };
    return make_plan(p, b, reserve, enqueue, out);
}


}  // namespace

extern "C" {

int cb200_camera_plan_create(cb200_ctx* c, const int32_t* wh, int n, uint32_t flags, const uint8_t* d_pictures, uint8_t* d_chunks,
                             uint32_t* d_chunk_mask, uint8_t* d_frame_flags, int32_t* d_extract_status, cb200_camera_plan** out)
{
    // the checks of cb200_scan_extract_decode_chunks_ragged_dev, then the plan's own
    auto build = [&](CameraBatch& b) { return packed_batch(d_pictures, wh, n, b); };
    return make_camera_plan(c, build, flags, d_chunks, d_chunk_mask, d_frame_flags, d_extract_status, nullptr, out);
}

int cb200_camera_plan_create_receivers(cb200_ctx* c, const cb200_picture* pics, int n, uint32_t flags, const int32_t* d_receiver_of,
                                       int n_receivers, cb200_receiver_state* d_states, uint8_t* d_chunks, uint32_t* d_chunk_mask,
                                       uint8_t* d_frame_flags, int32_t* d_extract_status, cb200_camera_plan** out)
{
    // the checks of cb200_scan_extract_decode_chunks_receivers_dev (the map's pointer in place of its indices, which only a launch
    // reads), then the plan's own as cb200_camera_plan_create makes them
    int rc = check_receivers(c, d_receiver_of, n, n_receivers, d_states, true); if (rc) return rc;
    auto build = [&](CameraBatch& b) { return picture_batch(pics, n, b); };
    const PlanReceivers recv = {d_receiver_of, n_receivers, d_states, nullptr};
    return make_camera_plan(c, build, flags, d_chunks, d_chunk_mask, d_frame_flags, d_extract_status, &recv, out);
}

int cb200_camera_plan_create_receivers_pictures_dev(cb200_ctx* c, const cb200_picture* d_pics, int n, const cb200_picture_bounds* bounds,
                                                    uint32_t flags, const int32_t* d_receiver_of, int n_receivers,
                                                    cb200_receiver_state* d_states, uint8_t* d_chunks, uint32_t* d_chunk_mask,
                                                    uint8_t* d_frame_flags, int32_t* d_extract_status, cb200_camera_plan** out)
{
    // cb200_camera_plan_create_receivers' checks, with the descriptors' pointer and bounds in place of their contents (which each
    // launch checks on the device)
    int rc = check_receivers(c, d_receiver_of, n, n_receivers, d_states, true); if (rc) return rc;
    auto build = [&](CameraBatch& b) { return device_batch(d_pics, n, bounds, b); };
    const PlanReceivers recv = {d_receiver_of, n_receivers, d_states, nullptr};
    return make_camera_plan(c, build, flags, d_chunks, d_chunk_mask, d_frame_flags, d_extract_status, &recv, out);
}

int cb200_camera_plan_create_receivers_pictures_flags_dev(cb200_ctx* c, const cb200_picture* d_pics, int n, const cb200_picture_bounds* bounds,
                                                          uint32_t flags, const int32_t* d_receiver_of, int n_receivers,
                                                          cb200_receiver_state* d_states, const uint32_t* d_receiver_flags, uint8_t* d_chunks,
                                                          uint32_t* d_chunk_mask, uint8_t* d_frame_flags, int32_t* d_extract_status,
                                                          cb200_camera_plan** out)
{
    // the table's own checks, then cb200_camera_plan_create_receivers_pictures_dev's
    int rc = check_receiver_flags(d_receiver_flags, flags); if (rc) return rc;
    if ((rc = check_receivers(c, d_receiver_of, n, n_receivers, d_states, true))) return rc;
    auto build = [&](CameraBatch& b) { return device_batch(d_pics, n, bounds, b); };
    const PlanReceivers recv = {d_receiver_of, n_receivers, d_states, d_receiver_flags};
    return make_camera_plan(c, build, flags, d_chunks, d_chunk_mask, d_frame_flags, d_extract_status, &recv, out);
}

int cb200_camera_plan_create_detect_receivers(cb200_ctx* const* ctxs, int n_modes, const cb200_picture* pics, int n, uint32_t flags,
                                              const uint32_t* d_candidates, const int32_t* d_receiver_of, int n_receivers,
                                              cb200_receiver_state* const* d_states, uint8_t* d_chunks, uint32_t* d_chunk_mask,
                                              int32_t* d_extract_status, int32_t* d_mode, uint32_t* d_mode_masks, cb200_camera_plan** out)
{
    // the checks of cb200_detect_scan_extract_decode_chunks_receivers_dev (the pointers of the candidates and the map in place of
    // their entries, which only a launch reads; live plans allowed), with the plan's own after the batch's
    CameraBatch b;
    int rc = check_detect_plan(ctxs, n_modes, pics, false, nullptr, n, flags, d_candidates, d_receiver_of, n_receivers, d_states, d_chunks,
                               d_chunk_mask, d_extract_status, d_mode, out, b);
    if (rc) return rc;
    return make_detect_plan(ctxs, n_modes, b, flags, d_candidates, d_receiver_of, n_receivers, d_states, d_chunks, d_chunk_mask,
                            d_extract_status, d_mode, d_mode_masks, out);
}

int cb200_camera_plan_create_detect_receivers_pictures_dev(cb200_ctx* const* ctxs, int n_modes, const cb200_picture* d_pics, int n,
                                                           const cb200_picture_bounds* bounds, uint32_t flags, const uint32_t* d_candidates,
                                                           const int32_t* d_receiver_of, int n_receivers, cb200_receiver_state* const* d_states,
                                                           uint8_t* d_chunks, uint32_t* d_chunk_mask, int32_t* d_extract_status,
                                                           int32_t* d_mode, uint32_t* d_mode_masks, cb200_camera_plan** out)
{
    // cb200_camera_plan_create_detect_receivers' checks, with the descriptors' pointer and bounds in place of their contents
    CameraBatch b;
    int rc = check_detect_plan(ctxs, n_modes, d_pics, true, bounds, n, flags, d_candidates, d_receiver_of, n_receivers, d_states, d_chunks,
                               d_chunk_mask, d_extract_status, d_mode, out, b);
    if (rc) return rc;
    return make_detect_plan(ctxs, n_modes, b, flags, d_candidates, d_receiver_of, n_receivers, d_states, d_chunks, d_chunk_mask,
                            d_extract_status, d_mode, d_mode_masks, out);
}


int cb200_camera_plan_create_detect_receivers_pictures_flags_dev(cb200_ctx* const* ctxs, int n_modes, const cb200_picture* d_pics, int n,
                                                                 const cb200_picture_bounds* bounds, uint32_t flags, const uint32_t* d_candidates,
                                                                 const int32_t* d_receiver_of, int n_receivers,
                                                                 cb200_receiver_state* const* d_states, const uint32_t* d_receiver_flags,
                                                                 uint8_t* d_chunks, uint32_t* d_chunk_mask, int32_t* d_extract_status,
                                                                 int32_t* d_mode, uint32_t* d_mode_masks, cb200_camera_plan** out)
{
    // the table's own checks, then cb200_camera_plan_create_detect_receivers_pictures_dev's
    int rc = check_receiver_flags(d_receiver_flags, flags); if (rc) return rc;
    CameraBatch b;
    rc = check_detect_plan(ctxs, n_modes, d_pics, true, bounds, n, flags, d_candidates, d_receiver_of, n_receivers, d_states, d_chunks,
                           d_chunk_mask, d_extract_status, d_mode, out, b);
    if (rc) return rc;
    return make_detect_plan(ctxs, n_modes, b, flags, d_candidates, d_receiver_of, n_receivers, d_states, d_chunks, d_chunk_mask,
                            d_extract_status, d_mode, d_mode_masks, out, d_receiver_flags);
}


int cb200_camera_plan_launch(cb200_camera_plan* p)
{
    if (!p) return fail(CB200_ERR_ARG, "null plan");
    cb200_ctx* c = p->ctx;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    cudaStreamCaptureStatus status;
    cudaGraph_t outer = nullptr;
    const cudaGraphNode_t* deps = nullptr;
    size_t ndeps = 0;
    CK(cudaStreamGetCaptureInfo(c->stream, &status, nullptr, &outer, &deps, &ndeps), "cudaStreamGetCaptureInfo");
    if (status == cudaStreamCaptureStatusActive) {      // torch.cuda.graph and the like: the plan becomes a child node of that capture
        cudaGraphNode_t node;
        CK(cudaGraphAddChildGraphNode(&node, outer, deps, ndeps, p->graph), "cudaGraphAddChildGraphNode");
        CK(cudaStreamUpdateCaptureDependencies(c->stream, &node, 1, cudaStreamSetCaptureDependencies), "cudaStreamUpdateCaptureDependencies");
        return CB200_OK;                                // nothing runs yet: the host state stays as it is
    }
    CK(cudaGraphLaunch(p->exec, c->stream), "cudaGraphLaunch");
    count_launch(p->kernels);
    // the host state the direct call leaves behind (a receivers call reports every picture's matrix, CC_SIMPLE too; a detect plan's
    // contexts each decoded all n slots)
    for (cb200_ctx* x : p->ctxs) {
        set_camera_pictures(x, p->n);
        if (p->d_receiver_of || !(p->flags & CB200_FLAG_CC_SIMPLE)) x->ccm_frames = p->n;
    }
    if (p->keeps_ccm) {
        CK(cudaEventRecord(c->ccm_ev, c->stream), "record ccm");
        c->ccm_pending = true;
        c->ccm_pending_flag = !(p->flags & CB200_FLAG_CC_SIMPLE);
        if (p->flags & CB200_FLAG_CC_SIMPLE) c->ccm_active = true;
    }
    return CB200_OK;
}

int cb200_camera_plan_graph(cb200_camera_plan* p, void** cuda_graph)
{
    if (!p || !cuda_graph) return fail(CB200_ERR_ARG, "bad arguments");
    *cuda_graph = p->graph;
    return CB200_OK;
}

int cb200_camera_plan_destroy(cb200_camera_plan* p)
{
    if (!p) return CB200_OK;
    cb200_ctx* c = p->ctx;
    cudaSetDevice(c->device);
    // a replay still in flight reads the plan's table: the graph and the table go once the device has passed it (as cudaFree
    // would wait anyway)
    cudaDeviceSynchronize();
    if (p->exec) cudaGraphExecDestroy(p->exec);
    if (p->graph) cudaGraphDestroy(p->graph);
    for (cb200_ctx* x : p->ctxs)             // a detect plan is registered with each of its contexts
        for (size_t i = 0; i < x->plans.size(); ++i)
            if (x->plans[i] == p) { x->plans.erase(x->plans.begin() + (long)i); break; }
    delete p;
    return CB200_OK;
}

}  // extern "C"
