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
#include "ctx.cuh"

#include <string>
#include <vector>

using namespace cb200;

struct cb200_camera_plan {
    cb200_ctx* ctx = nullptr;
    int n = 0;
    uint32_t flags = 0;
    DevBuf<uint8_t> d_table;                // n PicDesc, then the pictures grouped by blur radius
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

int check_frozen_scan(cb200_ctx* c, const int32_t* wh, int n) { return c->plans.empty() ? CB200_OK : scan_reserve(c, wh, n); }

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

// camera_enqueue on the private stream `cap`, captured into p->graph.  The context's stream, timing and host CCM state are set aside
// for the duration and restored: a capture runs nothing, so it changes nothing the host can observe
int capture(cb200_camera_plan* p, cudaStream_t cap, const uint8_t* d_pictures, const int32_t* wh, uint8_t* d_chunks, uint32_t* d_mask,
            uint8_t* d_frame_flags, int32_t* d_status)
{
    cb200_ctx* c = p->ctx;
    cudaEvent_t scratch_ev;                 // ccm_keep_last records c->ccm_ev: inside a capture that record joins the graph
    CK(cudaEventCreateWithFlags(&scratch_ev, cudaEventDisableTiming), "cudaEventCreate");
    const cudaStream_t stream = c->stream;
    const bool timing = c->timing, pending = c->ccm_pending, pending_flag = c->ccm_pending_flag, active = c->ccm_active;
    const int ccm_frames = c->ccm_frames, camera_n = camera_pictures(c);
    const unsigned long long launches = cb200_launch_count();
    cudaEvent_t ccm_ev = c->ccm_ev;
    c->ccm_ev = scratch_ev;
    c->stream = cap;
    c->timing = false;
    c->capturing = true;
    int rc = CB200_OK;
    cudaError_t e = cudaStreamBeginCapture(cap, cudaStreamCaptureModeThreadLocal);
    if (e != cudaSuccess) rc = fail_cuda(e, "cudaStreamBeginCapture");
    if (!rc) {
        rc = camera_enqueue_table(c, d_pictures, wh, p->n, p->flags, d_chunks, d_mask, d_frame_flags, d_status,
                                  reinterpret_cast<const PicDesc*>(p->d_table.get()));
        cudaGraph_t g = nullptr;
        e = cudaStreamEndCapture(cap, &g);
        if (!rc && e != cudaSuccess) rc = fail_cuda(e, "cudaStreamEndCapture");
        if (rc) { if (g) cudaGraphDestroy(g); } else p->graph = g;
    }
    c->capturing = false;
    c->timing = timing;
    c->stream = stream;
    c->ccm_ev = ccm_ev;
    c->ccm_pending = pending; c->ccm_pending_flag = pending_flag; c->ccm_active = active;
    c->ccm_frames = ccm_frames;
    set_camera_pictures(c, camera_n);
    cudaEventDestroy(scratch_ev);
    // the captured launches did not run: launch() counts them each time the graph does
    count_launch(-(int)(cb200_launch_count() - launches));
    return rc;
}

}  // namespace

extern "C" {

int cb200_camera_plan_create(cb200_ctx* c, const int32_t* wh, int n, uint32_t flags, const uint8_t* d_pictures, uint8_t* d_chunks,
                             uint32_t* d_chunk_mask, uint8_t* d_frame_flags, int32_t* d_extract_status, cb200_camera_plan** out)
{
    // the checks of cb200_scan_extract_decode_chunks_ragged_dev, in its order, then the plan's own
    int rc = check_camera_dev_flags(flags); if (rc) return rc;
    if (n < 0) return fail(CB200_ERR_ARG, "n < 0");
    if (!wh) return fail(CB200_ERR_ARG, "null wh");
    if (!d_pictures) return fail(CB200_ERR_ARG, "null pictures");
    rc = check_picture_sizes(wh, n); if (rc) return rc;
    if (n == 0) return fail(CB200_ERR_ARG, "n = 0: a camera plan needs at least one picture");
    if (!out) return fail(CB200_ERR_ARG, "null plan");
    *out = nullptr;
    rc = check_camera_dev_outputs(c, n, d_chunks, d_chunk_mask, d_extract_status); if (rc) return rc;
    if (check_host_ccm(c))
        return fail(CB200_ERR_ARG, "the context is linked to a CCM chain, whose step the host sets per call: no camera plan");
    for (int i = 0; i < n; ++i)
        if ((size_t)wh[2 * i] * (size_t)wh[2 * i + 1] * 3 >= ((size_t)1 << 32))
            return fail(CB200_ERR_ARG, "source picture " + std::to_string(i) + " of 4 GB or more");
    rc = check_frozen_camera(c, wh, n); if (rc) return rc;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    // every buffer the graph uses, at this batch's size (with plans already there, the freeze check above guarantees this grows nothing)
    rc = camera_reserve(c, wh, n); if (rc) return rc;
    rc = decode_reserve(c, flags); if (rc) return rc;
    cb200_camera_plan* p = new cb200_camera_plan();
    p->ctx = c; p->n = n; p->flags = flags;
    p->keeps_ccm = (flags & CB200_FLAG_CC_SIMPLE) || ccm_fits(c->mode, flags);
    std::vector<uint8_t> table;
    cudaStream_t cap = nullptr;
    rc = camera_table(c, d_pictures, wh, n, table);
    if (!rc) { const cudaError_t e = p->d_table.ensure(table.size()); if (e != cudaSuccess) rc = fail_cuda(e, "cudaMalloc plan picture table"); }
    if (!rc) { const cudaError_t e = cudaStreamCreateWithFlags(&cap, cudaStreamNonBlocking); if (e != cudaSuccess) rc = fail_cuda(e, "cudaStreamCreate"); }
    if (!rc) {   // the table goes up once, on the private stream, before anything can replay
        cudaError_t e = cudaMemcpyAsync(p->d_table, table.data(), table.size(), cudaMemcpyHostToDevice, cap);
        if (e == cudaSuccess) e = cudaStreamSynchronize(cap);
        if (e != cudaSuccess) rc = fail_cuda(e, "H2D plan picture table");
    }
    if (!rc) rc = capture(p, cap, d_pictures, wh, d_chunks, d_chunk_mask, d_frame_flags, d_extract_status);
    if (cap) cudaStreamDestroy(cap);
    if (!rc) rc = count_kernel_nodes(p->graph, &p->kernels);
    if (!rc) { const cudaError_t e = cudaGraphInstantiate(&p->exec, p->graph, 0); if (e != cudaSuccess) rc = fail_cuda(e, "cudaGraphInstantiate"); }
    if (rc) {
        const std::string why = cb200_last_error();
        if (p->graph) cudaGraphDestroy(p->graph);
        delete p;
        return fail(rc, why);
    }
    // the graph starts from d_carry: unless a CCM is on its way there from the device, the host's goes there now
    c->plans.push_back(p);
    if (!c->ccm_pending && (rc = carry_from_host(c)) != CB200_OK) { cb200_camera_plan_destroy(p); return rc; }
    *out = p;
    return CB200_OK;
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
    // the host state the direct call leaves behind
    set_camera_pictures(c, p->n);
    if (!(p->flags & CB200_FLAG_CC_SIMPLE)) c->ccm_frames = p->n;
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
    for (size_t i = 0; i < c->plans.size(); ++i)
        if (c->plans[i] == p) { c->plans.erase(c->plans.begin() + (long)i); break; }
    delete p;
    return CB200_OK;
}

}  // extern "C"
