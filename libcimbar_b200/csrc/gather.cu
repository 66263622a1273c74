// gather.cu -- the one exchange of the decode path: the decoded fountain chunk records of every rank -> rank 0.
//
// Replaces the many-decoders -> one-sink role of concurrent_fountain_decoder_sink (reference:
// src/lib/fountain/concurrent_fountain_decoder_sink.h:58-84: decoder threads push chunks, one thread drains them into the
// fountain_decoder_sink) for one process per GPU on an NVLink / NVSwitch box.
//
// Primary path -- a window in rank 0's HBM that every rank maps (CUDA IPC, NVLink peer access).  A rank's records reach its
// slot of the window in one of two ways:
//   push   (cb200_gather_push, the default of the drivers): the decode writes into local buffers, and a copy-engine transfer on
//          a side stream of the context moves them through the peer mapping -- no SM is involved, the transfer of step i runs
//          under the decode of step i + 1, and eight ranks finishing their RS kernels at the same moment do not pile their
//          stores up on rank 0's NVLink ingress;
//   direct (cb200_gather_slot gives the pointers to hand to cb200_decode_chunks_dev): the RS kernel of rank r writes its
//          corrected bytes, and the chunk-mask kernel its masks, STRAIGHT INTO rank 0's memory, tile by tile while the decode
//          runs.  Fine for two to four ranks.
// Either way the rank then publishes an epoch with a system-scope release store into a flag word of the window; rank 0 waits
// for the epochs of all ranks with a system-scope acquire spin (bounded).  The window is double buffered: rank 0 may still be
// draining buffer b while everybody works on buffer b ^ 1; a rank re-uses a slot only after rank 0 has released it.
//
// Second path -- cb200_gather_chunks(ctx, ncclComm_t, ...): ncclSend / ncclRecv (grouped) on a side stream of the context,
// ordered after the decode by an event, so that the exchange of step i overlaps the decode of step i + 1.  NCCL is bound at
// run time (dlopen of libnccl.so.2 -- the copy already loaded in the process when there is one), the library does not link it.
#include "ctx.cuh"

#include <dlfcn.h>
#include <cstdio>
#include <cstring>

namespace cb200 {

struct Uid { char internal[CB200_UNIQUE_ID_BYTES]; };   // == ncclUniqueId

struct NcclApi {
    void* lib = nullptr;
    int (*GetUniqueId)(void*) = nullptr;
    int (*CommInitRank)(void**, int, Uid /* by value, as in nccl.h */, int) = nullptr;
    int (*CommDestroy)(void*) = nullptr;
    int (*Send)(const void*, size_t, int, int, void*, cudaStream_t) = nullptr;
    int (*Recv)(void*, size_t, int, int, void*, cudaStream_t) = nullptr;
    int (*GroupStart)() = nullptr;
    int (*GroupEnd)() = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
};

struct GatherState {
    int nranks = 0, rank = 0;
    // ---- P2P window (owned by rank 0, IPC-mapped by the others)
    uint8_t* win = nullptr;            // base of the window as this process sees it
    bool win_owner = false;
    size_t chunk_bytes = 0;            // max_frames * data_bytes
    size_t slot_bytes = 0;             // one rank's share of one buffer: chunks + masks, 256-byte aligned
    size_t buffer_bytes = 0;           // nranks * slot_bytes
    size_t flags_off = 0;              // after the two buffers, 128 words: [32 b + r] epoch published by rank r for buffer b,
                                       // [64] error word, [65 + b] epoch up to which rank 0 has released buffer b
    // ---- NCCL path
    NcclApi nccl;
    void* own_comm = nullptr;          // created by cb200_comm_init
    cudaStream_t side = nullptr;
    cudaEvent_t ev_ready = nullptr, ev_done[2] = {nullptr, nullptr};   // one completion event per send buffer
};

static const char* nccl_load(NcclApi& a)
{
    if (a.lib) return nullptr;
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char* n : names) { a.lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL); if (a.lib) break; }
    if (!a.lib) return "libnccl.so.2 not found (dlopen)";
#define CB200_SYM(field, name) *reinterpret_cast<void**>(&a.field) = dlsym(a.lib, name); if (!a.field) return "missing NCCL symbol " name;
    CB200_SYM(GetUniqueId, "ncclGetUniqueId") CB200_SYM(CommInitRank, "ncclCommInitRank") CB200_SYM(CommDestroy, "ncclCommDestroy")
    CB200_SYM(Send, "ncclSend") CB200_SYM(Recv, "ncclRecv") CB200_SYM(GroupStart, "ncclGroupStart") CB200_SYM(GroupEnd, "ncclGroupEnd")
    CB200_SYM(GetErrorString, "ncclGetErrorString")
#undef CB200_SYM
    return nullptr;
}

void gather_destroy(GatherState* g)
{
    if (!g) return;
    if (g->win) { if (g->win_owner) cudaFree(g->win); else cudaIpcCloseMemHandle(g->win); }
    if (g->own_comm && g->nccl.CommDestroy) g->nccl.CommDestroy(g->own_comm);
    if (g->side) cudaStreamDestroy(g->side);
    if (g->ev_ready) cudaEventDestroy(g->ev_ready);
    for (cudaEvent_t e : g->ev_done) if (e) cudaEventDestroy(e);
    delete g;
}

static GatherState* state(cb200_ctx* c)
{
    if (!c->gather) c->gather = new GatherState();
    return c->gather;
}

static cudaError_t ensure_side(GatherState* g)
{
    if (g->side) return cudaSuccess;
    cudaError_t e = cudaStreamCreateWithFlags(&g->side, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&g->ev_ready, cudaEventDisableTiming);
    for (cudaEvent_t& ev : g->ev_done) if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ev, cudaEventDisableTiming);
    return e;
}

static void layout(GatherState* g, const cb200_ctx* c, int nranks)
{
    g->nranks = nranks;
    g->chunk_bytes = (size_t)c->max_frames * (size_t)c->mode.data_bytes;
    g->slot_bytes = (g->chunk_bytes + (size_t)c->max_frames * sizeof(uint32_t) + 255) & ~size_t(255);
    g->buffer_bytes = g->slot_bytes * (size_t)nranks;
    g->flags_off = 2 * g->buffer_bytes;
}

// ---------------------------------------------------------------------------------------------- flag kernels
__global__ void k_gather_publish(uint32_t* flag, uint32_t epoch)
{
    // everything this rank wrote into the window before (earlier kernels of the stream) is ordered before the flag
    __threadfence_system();
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(flag), "r"(epoch) : "memory");
}

// lane r waits until flags[r] has reached `epoch` (rank 0: the epoch rank r published for this buffer; a peer, with one lane:
// the epoch up to which rank 0 released the buffer); gives up after ~timeout_ns and reports through *error
__global__ void k_gather_wait(const uint32_t* flags, int nranks, uint32_t epoch, unsigned long long timeout_ns, uint32_t* error)
{
    const int r = threadIdx.x;
    if (r >= nranks) return;
    unsigned long long t0;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
    while (true) {
        uint32_t v;
        asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(flags + r) : "memory");
        if ((int32_t)(v - epoch) >= 0) break;
        unsigned long long t1;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
        if (t1 - t0 > timeout_ns) { atomicExch(error, 1u + (uint32_t)r); break; }
        __nanosleep(200);
    }
}

}  // namespace cb200

using namespace cb200;

extern "C" {

int cb200_gather_root_create(cb200_ctx* c, int nranks, uint8_t* handle_out)
{
    if (!c || nranks < 1 || nranks > 32 || !handle_out) return fail(CB200_ERR_ARG, "bad arguments");
    static_assert(sizeof(cudaIpcMemHandle_t) == CB200_IPC_HANDLE_BYTES, "IPC handle size");
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    GatherState* g = state(c);
    if (g->win) return fail(CB200_ERR_ARG, "gather window already exists");
    layout(g, c, nranks);
    g->rank = 0; g->win_owner = true;
    const size_t total = g->flags_off + 128 * sizeof(uint32_t);
    CK(cudaMalloc(&g->win, total), "cudaMalloc gather window");
    CK(cudaMemset(g->win, 0, total), "memset gather window");
    cudaIpcMemHandle_t h;
    CK(cudaIpcGetMemHandle(&h, g->win), "cudaIpcGetMemHandle");
    memcpy(handle_out, &h, sizeof(h));
    return CB200_OK;
}

int cb200_gather_peer_open(cb200_ctx* c, int nranks, int rank, const uint8_t* handle)
{
    if (!c || nranks < 2 || nranks > 32 || rank < 1 || rank >= nranks || !handle) return fail(CB200_ERR_ARG, "bad arguments");
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    GatherState* g = state(c);
    if (g->win) return fail(CB200_ERR_ARG, "gather window already exists");
    layout(g, c, nranks);
    g->rank = rank; g->win_owner = false;
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, sizeof(h));
    void* p = nullptr;
    CK(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess), "cudaIpcOpenMemHandle (NVLink peer mapping of rank 0's window)");
    g->win = static_cast<uint8_t*>(p);
    return CB200_OK;
}

int cb200_gather_slot(cb200_ctx* c, int buffer, int rank, uint8_t** d_chunks, uint32_t** d_mask)
{
    if (!c || !c->gather || !c->gather->win || buffer < 0 || buffer > 1) return fail(CB200_ERR_ARG, "no gather window");
    GatherState* g = c->gather;
    if (rank < 0) rank = g->rank;
    if (rank >= g->nranks) return fail(CB200_ERR_ARG, "rank out of range");
    if (!g->win_owner && rank != g->rank) return fail(CB200_ERR_ARG, "a peer only addresses its own slot");
    uint8_t* base = g->win + (size_t)buffer * g->buffer_bytes + (size_t)rank * g->slot_bytes;
    if (d_chunks) *d_chunks = base;
    if (d_mask) *d_mask = reinterpret_cast<uint32_t*>(base + g->chunk_bytes);
    return CB200_OK;
}

int cb200_gather_publish(cb200_ctx* c, int buffer, uint32_t epoch)
{
    if (!c || !c->gather || !c->gather->win || buffer < 0 || buffer > 1) return fail(CB200_ERR_ARG, "no gather window");
    GatherState* g = c->gather;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    uint32_t* flag = reinterpret_cast<uint32_t*>(g->win + g->flags_off) + buffer * 32 + g->rank;
    k_gather_publish<<<1, 1, 0, c->stream>>>(flag, epoch); count_launch();
    CK(cudaGetLastError(), "publish launch");
    return CB200_OK;
}

int cb200_gather_wait(cb200_ctx* c, int buffer, uint32_t epoch, double timeout_s)
{
    if (!c || !c->gather || !c->gather->win || buffer < 0 || buffer > 1) return fail(CB200_ERR_ARG, "no gather window");
    GatherState* g = c->gather;
    if (!g->win_owner) return fail(CB200_ERR_ARG, "only rank 0 waits on the window");
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    uint32_t* flags = reinterpret_cast<uint32_t*>(g->win + g->flags_off);
    if (timeout_s <= 0) timeout_s = 30.0;
    k_gather_wait<<<1, 32, 0, c->stream>>>(flags + buffer * 32, g->nranks, epoch, (unsigned long long)(timeout_s * 1e9), flags + 64); count_launch();
    CK(cudaGetLastError(), "wait launch");
    return CB200_OK;
}

int cb200_gather_release(cb200_ctx* c, int buffer, uint32_t epoch)
{
    if (!c || !c->gather || !c->gather->win || buffer < 0 || buffer > 1) return fail(CB200_ERR_ARG, "no gather window");
    GatherState* g = c->gather;
    if (!g->win_owner) return fail(CB200_ERR_ARG, "only rank 0 releases a buffer");
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    uint32_t* flags = reinterpret_cast<uint32_t*>(g->win + g->flags_off);
    k_gather_publish<<<1, 1, 0, c->stream>>>(flags + 65 + buffer, epoch); count_launch();
    CK(cudaGetLastError(), "release launch");
    return CB200_OK;
}

int cb200_gather_acquire(cb200_ctx* c, int buffer, uint32_t epoch, double timeout_s)
{
    if (!c || !c->gather || !c->gather->win || buffer < 0 || buffer > 1) return fail(CB200_ERR_ARG, "no gather window");
    GatherState* g = c->gather;
    if (g->win_owner) return CB200_OK;             // rank 0's own decode is ordered after its release by its stream
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    uint32_t* flags = reinterpret_cast<uint32_t*>(g->win + g->flags_off);
    if (timeout_s <= 0) timeout_s = 30.0;
    // (a timeout lands in the window's error word, which rank 0 reports)
    k_gather_wait<<<1, 32, 0, c->stream>>>(flags + 65 + buffer, 1, epoch, (unsigned long long)(timeout_s * 1e9), flags + 64); count_launch();
    CK(cudaGetLastError(), "acquire launch");
    return CB200_OK;
}

int cb200_gather_push(cb200_ctx* c, int buffer, const uint8_t* d_chunks, const uint32_t* d_mask, int n, uint32_t epoch, uint32_t acquire_epoch)
{
    if (!c || !c->gather || !c->gather->win || buffer < 0 || buffer > 1 || !d_chunks || !d_mask || n < 0 || n > c->max_frames)
        return fail(CB200_ERR_ARG, "no gather window / bad arguments");
    GatherState* g = c->gather;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    CK(ensure_side(g), "side stream (gather)");
    uint32_t* flags = reinterpret_cast<uint32_t*>(g->win + g->flags_off);
    // after everything enqueued on the decode stream so far ...
    CK(cudaEventRecord(g->ev_ready, c->stream), "record");
    CK(cudaStreamWaitEvent(g->side, g->ev_ready, 0), "wait");
    // ... and after rank 0 has let go of what this slot held two steps ago
    if (!g->win_owner && acquire_epoch) {
        k_gather_wait<<<1, 32, 0, g->side>>>(flags + 65 + buffer, 1, acquire_epoch, 30000000000ull, flags + 64); count_launch();
        CK(cudaGetLastError(), "acquire launch");
    }
    uint8_t* base = g->win + (size_t)buffer * g->buffer_bytes + (size_t)g->rank * g->slot_bytes;
    CK(cudaMemcpyAsync(base, d_chunks, (size_t)n * (size_t)c->mode.data_bytes, cudaMemcpyDeviceToDevice, g->side), "push chunks (peer copy)");
    CK(cudaMemcpyAsync(base + g->chunk_bytes, d_mask, (size_t)n * sizeof(uint32_t), cudaMemcpyDeviceToDevice, g->side), "push masks (peer copy)");
    k_gather_publish<<<1, 1, 0, g->side>>>(flags + buffer * 32 + g->rank, epoch); count_launch();
    CK(cudaGetLastError(), "publish launch");
    CK(cudaEventRecord(g->ev_done[buffer], g->side), "record");
    return CB200_OK;
}

int cb200_gather_status(cb200_ctx* c)
{
    if (!c || !c->gather || !c->gather->win || !c->gather->win_owner) return fail(CB200_ERR_ARG, "no gather window");
    GatherState* g = c->gather;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    uint32_t err = 0;
    CK(cudaStreamSynchronize(c->stream), "sync");
    CK(cudaMemcpy(&err, g->win + g->flags_off + 64 * sizeof(uint32_t), sizeof(err), cudaMemcpyDeviceToHost), "read gather status");
    if (err) { char msg[96]; snprintf(msg, sizeof(msg), "gather: rank %u did not publish in time", err - 1); return fail(CB200_ERR_CUDA, msg); }
    return CB200_OK;
}

// ---------------------------------------------------------------------------------------------- NCCL path
int cb200_comm_unique_id(uint8_t* id_out)
{
    if (!id_out) return fail(CB200_ERR_ARG, "null id");
    static NcclApi api;
    if (const char* e = nccl_load(api)) return fail(CB200_ERR_CUDA, e);
    Uid id;
    int rc = api.GetUniqueId(&id);
    if (rc) return fail(CB200_ERR_CUDA, std::string("ncclGetUniqueId: ") + api.GetErrorString(rc));
    memcpy(id_out, &id, sizeof(id));
    return CB200_OK;
}

int cb200_comm_init(cb200_ctx* c, const uint8_t* id, int nranks, int rank)
{
    if (!c || !id || nranks < 1 || rank < 0 || rank >= nranks) return fail(CB200_ERR_ARG, "bad arguments");
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    GatherState* g = state(c);
    if (const char* e = nccl_load(g->nccl)) return fail(CB200_ERR_CUDA, e);
    if (g->own_comm) return fail(CB200_ERR_ARG, "communicator already created");
    Uid u;
    memcpy(&u, id, sizeof(u));
    int rc = g->nccl.CommInitRank(&g->own_comm, nranks, u, rank);
    if (rc) return fail(CB200_ERR_CUDA, std::string("ncclCommInitRank: ") + g->nccl.GetErrorString(rc));
    if (!g->nranks) { g->nranks = nranks; g->rank = rank; }
    return CB200_OK;
}

int cb200_gather_chunks(cb200_ctx* c, void* nccl_comm, int nranks, int rank, int buffer, const uint8_t* d_chunks, const uint32_t* d_mask, int n,
                        uint8_t* d_all_chunks, uint32_t* d_all_masks)
{
    if (!c || n < 0 || n > c->max_frames || nranks < 1 || rank < 0 || rank >= nranks || buffer < 0 || buffer > 1 || !d_chunks || !d_mask)
        return fail(CB200_ERR_ARG, "bad arguments");
    if (rank == 0 && (!d_all_chunks || !d_all_masks)) return fail(CB200_ERR_ARG, "rank 0 needs the gather buffers");
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    GatherState* g = state(c);
    if (const char* e = nccl_load(g->nccl)) return fail(CB200_ERR_CUDA, e);
    void* comm = nccl_comm ? nccl_comm : g->own_comm;
    if (!comm) return fail(CB200_ERR_ARG, "no communicator: pass an ncclComm_t or call cb200_comm_init");
    CK(ensure_side(g), "side stream (gather)");
    // the exchange runs on the side stream, after everything enqueued on the decode stream so far
    CK(cudaEventRecord(g->ev_ready, c->stream), "record");
    CK(cudaStreamWaitEvent(g->side, g->ev_ready, 0), "wait");
    const size_t cb = (size_t)n * (size_t)c->mode.data_bytes, mb = (size_t)n * sizeof(uint32_t);
    const int kU8 = 1;   // ncclUint8
    int rc = g->nccl.GroupStart();
    if (!rc && rank == 0) {
        for (int r = 1; r < nranks && !rc; ++r) {
            rc = g->nccl.Recv(d_all_chunks + (size_t)r * cb, cb, kU8, r, comm, g->side);
            if (!rc) rc = g->nccl.Recv(reinterpret_cast<uint8_t*>(d_all_masks) + (size_t)r * mb, mb, kU8, r, comm, g->side);
        }
    } else if (!rc) {
        rc = g->nccl.Send(d_chunks, cb, kU8, 0, comm, g->side);
        if (!rc) rc = g->nccl.Send(d_mask, mb, kU8, 0, comm, g->side);
    }
    int rc2 = g->nccl.GroupEnd();
    if (rc || rc2) return fail(CB200_ERR_CUDA, std::string("nccl send/recv: ") + g->nccl.GetErrorString(rc ? rc : rc2));
    if (rank == 0) {   // rank 0's own records
        CK(cudaMemcpyAsync(d_all_chunks, d_chunks, cb, cudaMemcpyDeviceToDevice, g->side), "copy own chunks");
        CK(cudaMemcpyAsync(d_all_masks, d_mask, mb, cudaMemcpyDeviceToDevice, g->side), "copy own masks");
    }
    CK(cudaEventRecord(g->ev_done[buffer], g->side), "record");
    return CB200_OK;
}

int cb200_gather_chunks_wait(cb200_ctx* c, int buffer)
{
    if (!c || buffer < 0 || buffer > 1) return fail(CB200_ERR_ARG, "bad arguments");
    if (!c->gather || !c->gather->ev_done[buffer]) return CB200_OK;   // nothing was ever sent from this buffer
    CK(cudaStreamWaitEvent(c->stream, c->gather->ev_done[buffer], 0), "wait gather");
    return CB200_OK;
}

}  // extern "C"
