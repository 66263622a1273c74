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
#include "ctx.cuh"

#include <cstring>
#include <string>

namespace cb200 {

constexpr int kDetectModes = 5;

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

static bool same_geometry(const Mode& a, const Mode& b)
{
    return a.width == b.width && a.height == b.height && a.cells_x == b.cells_x && a.cells_y == b.cells_y && a.cell_offset == b.cell_offset &&
           a.corner == b.corner;
}

static std::string ctx_name(int k) { return "context " + std::to_string(k); }

// every argument check, before any CUDA call: the ones that need no context first
static int check_detect(cb200_ctx* const* ctxs, int n_modes, const uint8_t* d_pictures, const int32_t* wh, int n, uint32_t flags,
                        const uint8_t* d_chunks, const uint32_t* d_chunk_mask, const int32_t* d_extract_status, const int32_t* d_mode,
                        CameraBatch& b)
{
    if (n_modes < 1 || n_modes > kDetectModes)
        return fail(CB200_ERR_ARG, "n_modes = " + std::to_string(n_modes) + ": between 1 and " + std::to_string(kDetectModes) + " candidate modes");
    int rc = check_camera_flags(flags); if (rc) return rc;
    if ((rc = packed_batch(d_pictures, wh, n, b)) || (rc = check_spans(b))) return rc;
    if (!d_chunks || !d_chunk_mask || !d_extract_status || !d_mode) return fail(CB200_ERR_ARG, "null output");
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

// a context's stream for the duration of one geometry's work, restored on every path out
struct StreamSwap {
    cb200_ctx* c; cudaStream_t was;
    StreamSwap(cb200_ctx* c_, cudaStream_t st, const SharedWalk* sw) : c(c_), was(c_->stream) { c->stream = st; c->shared_walk = sw; }
    ~StreamSwap() { c->stream = was; c->shared_walk = nullptr; }
};

static int detect_enqueue(cb200_ctx* const* ctxs, int n_modes, const CameraBatch& b, uint32_t flags, uint8_t* d_chunks, uint32_t* d_chunk_mask,
                          int32_t* d_extract_status, int32_t* d_mode, uint32_t* d_mode_masks)
{
    cb200_ctx* c0 = ctxs[0];
    const int n = b.n();
    int rc;
    // geometries: lead[g] = the first context of geometry g in priority order
    int group[kDetectModes], lead[kDetectModes], ng = 0;
    for (int k = 0; k < n_modes; ++k) {
        int g = 0;
        while (g < ng && !same_geometry(ctxs[lead[g]]->mode, ctxs[k]->mode)) ++g;
        if (g == ng) lead[ng++] = k;
        group[k] = g;
    }
    if (!c0->detect) c0->detect = new DetectState();
    DetectState* ds = c0->detect;
    for (int k = 0; k < n_modes; ++k) { rc = camera_reserve_for(ctxs[k], b.wh.data(), n, k == 0, lead[group[k]] == k); if (rc) return rc; }
    CK(ds->status.ensure((size_t)n_modes * n), "cudaMalloc detect statuses");
    uint8_t* frames[kDetectModes];
    for (int g = 0; g < ng; ++g) {
        const cb200_ctx* L = ctxs[lead[g]];
        CK(ds->kept[g].ensure((size_t)n * L->mode.num_cells), "cudaMalloc detect walk records");
        rc = deskew_frames(ctxs[lead[g]], n, &frames[g]); if (rc) return rc;
    }
    if (ng > 1) {
        if (!ds->fork) CK(cudaEventCreateWithFlags(&ds->fork, cudaEventDisableTiming), "cudaEventCreate detect fork");
        for (int g = 0; g < ng; ++g) {
            if (!ds->side[g]) CK(cudaStreamCreateWithFlags(&ds->side[g], cudaStreamNonBlocking), "cudaStreamCreate detect side stream");
            if (!ds->join[g]) CK(cudaEventCreateWithFlags(&ds->join[g], cudaEventDisableTiming), "cudaEventCreate detect join");
        }
    }
    const PicDesc* d_desc;
    rc = camera_scan(c0, b, nullptr, &d_desc); if (rc) return rc;
    cudaStream_t main = c0->stream;
    if (ng > 1) {
        CK(cudaEventRecord(ds->fork, main), "record detect fork");
        for (int g = 0; g < ng; ++g) CK(cudaStreamWaitEvent(ds->side[g], ds->fork, 0), "wait detect fork");
    }
    // every geometry's modes in priority order, the lead first; every side stream is joined back even when one fails
    for (int g = 0; g < ng && !rc; ++g) {
        const SharedWalk sw{ctxs[lead[g]], ds->kept[g].get()};
        for (int k = 0; k < n_modes && !rc; ++k) {
            if (group[k] != g) continue;
            cb200_ctx* c = ctxs[k];
            StreamSwap on(c, ng > 1 ? ds->side[g] : main, &sw);
            rc = camera_after_scan(c, c0, b, d_desc, flags, frames[g], k == lead[g], c->d_data, c->d_mask, nullptr, ds->status + (size_t)k * n);
        }
    }
    if (ng > 1) {
        for (int g = 0; g < ng; ++g) {
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
    k_detect_select<<<n, 256, 0, main>>>(a, d_chunks, d_chunk_mask, d_extract_status, d_mode, d_mode_masks);
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
    int rc = check_detect(ctxs, n_modes, d_pictures, wh, n, flags, d_chunks, d_chunk_mask, d_extract_status, d_mode, b); if (rc) return rc;
    if (n == 0) return CB200_OK;
    CK(cudaSetDevice(ctxs[0]->device), "cudaSetDevice");
    return detect_enqueue(ctxs, n_modes, b, flags, d_chunks, d_chunk_mask, d_extract_status, d_mode, d_mode_masks);
}
