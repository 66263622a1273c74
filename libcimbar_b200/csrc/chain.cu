// chain.cu -- the CC_FIT colour-correction state carried across the ranks of a multi-GPU decode.
//
// Under CB200_FLAG_CC_FIT a frame without a usable fountain header decodes with the CCM of the frame before it (k_ccm_carry):
// the only state that crosses frames.  When a batch is cut into contiguous stripes, one per rank (rank-major order = batch
// order), the CCM entering rank r's stripe is the last fit among the stripes of ranks 0 .. r-1 of the same step, or -- when none
// of them fit -- the matrix rank 0 entered the step with (the global exit of the previous step).  That is a prefix "last valid"
// over one value per rank, so a rank only waits for the other ranks' k_ccm_fit, never for their decode.
//
// A region in rank 0's HBM, mapped by the other ranks through CUDA IPC, holds per epoch parity and rank one Slot:
//   publish (after k_ccm_fit)  : the stripe's last fit (had_fit = 1), or "no fit" -- rank 0 then writes the matrix it entered
//                                the step with, so that every rank finds the fallback in slot 0; epoch with st.release.sys
//   link    (before k_ccm_carry): ld.acquire.sys of the epochs of ranks < r, entry matrix -> the context's chain entry, which the
//                                carry takes as its device initial (CcmArg.per_frame)
//   settle  (after the decode) : all ranks' slots of the step -> the global exit into d_carry (every rank then holds the same
//                                CCM), then this rank's read acknowledgement
// The slots are double-buffered by epoch parity: the publish of step s waits until every rank has acknowledged the last step that
// used the same parity.  Every wait is bounded; a timeout records the rank that did not arrive (cb200_ccm_chain_status).
#include "ctx.cuh"

#include <cstdio>
#include <cstring>

namespace cb200 {

namespace {

constexpr int kMaxRanks = 32;
constexpr unsigned long long kTimeoutNs = 30ull * 1000000000ull;

struct Slot {
    float m[9];
    uint32_t epoch;
    uint8_t active, had_fit, pad[2];
    uint32_t pad2[5];
};
static_assert(sizeof(Slot) == 64, "slot size");

struct Region {
    Slot slot[2][kMaxRanks];      // [epoch parity][rank]
    uint32_t ack[kMaxRanks];      // last epoch whose slots rank r has finished reading
    uint32_t error;               // 0, or 1 + the rank a wait gave up on
};

__device__ __forceinline__ uint32_t ld_acquire(const uint32_t* p)
{
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release(uint32_t* p, uint32_t v)
{
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// spins (bounded, with back-off) until *p has reached epoch; a timeout records `rank` in the region's error word
__device__ void wait_epoch(const uint32_t* p, uint32_t epoch, int rank, uint32_t* error)
{
    unsigned long long t0;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
    while ((int32_t)(ld_acquire(p) - epoch) < 0) {
        unsigned long long t1;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
        if (t1 - t0 > kTimeoutNs) { atomicCAS(error, 0u, 1u + (uint32_t)rank); return; }
        __nanosleep(500);
    }
}

// this stripe's exit state: its last fit, or "no fit" (rank 0: the matrix it entered the step with)
__global__ void __launch_bounds__(256)
k_chain_publish(Region* reg, int rank, int nranks, uint32_t epoch, uint32_t reuse_epoch, int n, const float* __restrict__ fit,
                const uint8_t* __restrict__ valid, const CcmArg own)
{
    __shared__ int last[256];
    const int t = threadIdx.x;
    // the slot of this parity is free once every rank has read what it held (the last step with the same parity)
    if (reuse_epoch && t < nranks) wait_epoch(&reg->ack[t], reuse_epoch, t, &reg->error);
    int l = -1;
    for (int f = t; f < n; f += 256) if (valid[f]) l = f;
    last[t] = l;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (t < o && last[t + o] > last[t]) last[t] = last[t + o];
        __syncthreads();
    }
    if (t != 0) return;
    __threadfence();
    Slot* s = &reg->slot[epoch & 1][rank];
    const int f = last[0];
    if (f >= 0) {
        for (int i = 0; i < 9; ++i) s->m[i] = fit[(size_t)f * 9 + i];
        s->active = 1; s->had_fit = 1;
    } else {
        for (int i = 0; i < 9; ++i) s->m[i] = own.per_frame ? own.per_frame[i] : own.m[i];
        s->active = own.per_frame ? own.per_frame_active[0] : (uint8_t)(own.active != 0);
        s->had_fit = 0;
    }
    __threadfence_system();
    st_release(&s->epoch, epoch);
}

// lane q waits for slot q of `epoch` (q < upto), reads whether it fit; returns in `pick` the highest rank < upto whose stripe
// fit (slot 0 when none did: rank 0's slot then holds the matrix it entered the step with)
__device__ void pick_slot(Region* reg, int upto, uint32_t epoch, int* pick)
{
    __shared__ int fitted[kMaxRanks];
    const int q = threadIdx.x;
    fitted[q] = 0;
    if (q < upto) {
        const Slot* s = &reg->slot[epoch & 1][q];
        wait_epoch(&s->epoch, epoch, q, &reg->error);
        fitted[q] = *(volatile const uint8_t*)&s->had_fit;
    }
    __syncthreads();
    if (q == 0) {
        int p = 0;
        for (int r = upto - 1; r >= 0; --r) if (fitted[r]) { p = r; break; }
        *pick = p;
    }
    __syncthreads();
}

__device__ void copy_slot(const Slot* s, float* dst)
{
    const volatile Slot* v = s;
    for (int i = 0; i < 9; ++i) dst[i] = v->m[i];
    reinterpret_cast<uint8_t*>(dst + 9)[0] = v->active;
}

// the CCM entering this rank's stripe -> entry (9 floats, activity byte at float index 9).  Rank 0 enters with its own matrix
__global__ void __launch_bounds__(kMaxRanks) k_chain_link(Region* reg, int rank, uint32_t epoch, const CcmArg own, float* entry)
{
    __shared__ int pick;
    if (rank == 0) {
        if (threadIdx.x == 0) {
            for (int i = 0; i < 9; ++i) entry[i] = own.per_frame ? own.per_frame[i] : own.m[i];
            reinterpret_cast<uint8_t*>(entry + 9)[0] = own.per_frame ? own.per_frame_active[0] : (uint8_t)(own.active != 0);
        }
        return;
    }
    pick_slot(reg, rank, epoch, &pick);
    if (threadIdx.x == 0) { __threadfence(); copy_slot(&reg->slot[epoch & 1][pick], entry); }
}

// the global exit of the step (the last fit of all stripes, else rank 0's entry) -> carry; then this rank's read acknowledgement
__global__ void __launch_bounds__(kMaxRanks) k_chain_settle(Region* reg, int rank, int nranks, uint32_t epoch, float* carry)
{
    __shared__ int pick;
    pick_slot(reg, nranks, epoch, &pick);
    if (threadIdx.x != 0) return;
    __threadfence();
    copy_slot(&reg->slot[epoch & 1][pick], carry);
    __threadfence_system();
    st_release(&reg->ack[rank], epoch);
}

}  // namespace

struct ChainState {
    Region* reg = nullptr;         // as this process sees it
    bool owner = false;
    int nranks = 0, rank = 0;      // of the region (create / open)
    bool attached = false;
    uint32_t step = 0;             // epoch of the next chained call (0: none set)
    uint32_t last = 0;             // epoch of the last chained call
    uint32_t used[2] = {0, 0};     // last epoch of each parity
    DevBuf<float> d_entry;         // the CCM entering this rank's stripe: 9 floats + activity byte
    cudaEvent_t ev[2] = {nullptr, nullptr};   // around the link kernel of the last chained call (cb200_set_timing on)
    bool timed = false;
};

void chain_destroy(ChainState* s)
{
    if (!s) return;
    for (cudaEvent_t e : s->ev) if (e) cudaEventDestroy(e);
    if (s->reg) { if (s->owner) cudaFree(s->reg); else cudaIpcCloseMemHandle(s->reg); }
    delete s;
}

bool chain_attached(const cb200_ctx* c) { return c && c->chain && c->chain->attached; }

bool chain_linked(const cb200_ctx* c, uint32_t flags)
{
    return c && c->chain && c->chain->attached && (flags & CB200_FLAG_CC_FIT);
}

int check_chain_call(const cb200_ctx* c, uint32_t flags)
{
    if (!chain_linked(c, flags)) return CB200_OK;
    if (!c->chain->step) return fail(CB200_ERR_ARG, "a CC_FIT call on a context linked to a CCM chain needs cb200_ccm_chain_step first");
    return CB200_OK;
}

int check_host_ccm(const cb200_ctx* c)
{
    if (c && c->chain && c->chain->attached)
        return fail(CB200_ERR_ARG, "the context is linked to a CCM chain: its CCM is the chain's, not set or fitted on the host");
    return CB200_OK;
}

int chain_publish_link(cb200_ctx* c, int n, const float* d_fit, const uint8_t* d_valid, const CcmArg& own, CcmArg* entry)
{
    ChainState* s = c->chain;
    const uint32_t e = s->step;
    k_chain_publish<<<1, 256, 0, c->stream>>>(s->reg, s->rank, s->nranks, e, s->used[e & 1], n, d_fit, d_valid, own); count_launch();
    CK(cudaGetLastError(), "chain publish launch");
    if (!entry) return CB200_OK;
    CK(s->d_entry.ensure(12), "cudaMalloc chain entry");
    s->timed = c->timing;
    if (s->timed) {
        for (cudaEvent_t& ev : s->ev) if (!ev) CK(cudaEventCreate(&ev), "cudaEventCreate (chain)");
        CK(cudaEventRecord(s->ev[0], c->stream), "record (chain)");
    }
    k_chain_link<<<1, kMaxRanks, 0, c->stream>>>(s->reg, s->rank, e, own, s->d_entry); count_launch();
    CK(cudaGetLastError(), "chain link launch");
    if (s->timed) CK(cudaEventRecord(s->ev[1], c->stream), "record (chain)");
    memset(entry, 0, sizeof(*entry));
    entry->per_frame = s->d_entry;
    entry->per_frame_active = reinterpret_cast<const uint8_t*>(s->d_entry + 9);
    return CB200_OK;
}

int chain_settle(cb200_ctx* c, float* d_carry)
{
    ChainState* s = c->chain;
    const uint32_t e = s->step;
    k_chain_settle<<<1, kMaxRanks, 0, c->stream>>>(s->reg, s->rank, s->nranks, e, d_carry); count_launch();
    CK(cudaGetLastError(), "chain settle launch");
    s->used[e & 1] = e;
    s->last = e;
    s->step = 0;
    return CB200_OK;
}

}  // namespace cb200

using namespace cb200;

extern "C" {

int cb200_ccm_chain_root_create(cb200_ctx* c, int nranks, uint8_t* handle_out)
{
    if (nranks < 1 || nranks > kMaxRanks) return fail(CB200_ERR_ARG, "nranks out of range (1 .. 32)");
    if (!c || !handle_out) return fail(CB200_ERR_ARG, !c ? "null context" : "null handle");
    if (c->chain) return fail(CB200_ERR_ARG, "the context already has a CCM chain region");
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    ChainState* s = new ChainState();
    void* p = nullptr;
    cudaError_t e = cudaMalloc(&p, sizeof(Region));
    if (e != cudaSuccess) { delete s; return fail_cuda(e, "cudaMalloc ccm chain region"); }
    s->reg = static_cast<Region*>(p); s->owner = true; s->nranks = nranks; s->rank = 0;
    c->chain = s;
    CK(cudaMemset(p, 0, sizeof(Region)), "memset ccm chain region");
    cudaIpcMemHandle_t h;
    CK(cudaIpcGetMemHandle(&h, p), "cudaIpcGetMemHandle");
    memcpy(handle_out, &h, sizeof(h));
    return CB200_OK;
}

int cb200_ccm_chain_peer_open(cb200_ctx* c, int nranks, int rank, const uint8_t* handle)
{
    if (nranks < 2 || nranks > kMaxRanks || rank < 1 || rank >= nranks) return fail(CB200_ERR_ARG, "rank / nranks out of range (a peer: 1 <= rank < nranks <= 32)");
    if (!c || !handle) return fail(CB200_ERR_ARG, !c ? "null context" : "null handle");
    if (c->chain) return fail(CB200_ERR_ARG, "the context already has a CCM chain region");
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, sizeof(h));
    void* p = nullptr;
    CK(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess), "cudaIpcOpenMemHandle (rank 0's ccm chain region)");
    ChainState* s = new ChainState();
    s->reg = static_cast<Region*>(p); s->owner = false; s->nranks = nranks; s->rank = rank;
    c->chain = s;
    return CB200_OK;
}

int cb200_ccm_chain_attach(cb200_ctx* c, int rank, int nranks)
{
    if (nranks < 1 || nranks > kMaxRanks || rank < 0 || rank >= nranks) return fail(CB200_ERR_ARG, "rank / nranks out of range (0 <= rank < nranks <= 32)");
    if (!c) return fail(CB200_ERR_ARG, "null context");
    if (!c->chain) return fail(CB200_ERR_ARG, "no CCM chain region: cb200_ccm_chain_root_create / cb200_ccm_chain_peer_open first");
    if (rank != c->chain->rank || nranks != c->chain->nranks) return fail(CB200_ERR_ARG, "rank / nranks differ from the chain region's");
    c->chain->attached = true;
    return CB200_OK;
}

int cb200_ccm_chain_step(cb200_ctx* c, uint32_t epoch)
{
    if (epoch == 0) return fail(CB200_ERR_ARG, "epoch 0");
    if (!c) return fail(CB200_ERR_ARG, "null context");
    if (!c->chain || !c->chain->attached) return fail(CB200_ERR_ARG, "the context is not linked to a CCM chain");
    if (c->chain->step) return fail(CB200_ERR_ARG, "the step set last has not been decoded yet");
    if ((int32_t)(epoch - c->chain->last) <= 0) return fail(CB200_ERR_ARG, "epochs must increase from step to step");
    c->chain->step = epoch;
    return CB200_OK;
}

int cb200_ccm_chain_link_ms(cb200_ctx* c, float* ms)
{
    if (!c || !ms) return fail(CB200_ERR_ARG, "bad arguments");
    if (!c->chain || !c->chain->timed) return fail(CB200_ERR_ARG, "no timed chained call (cb200_set_timing before the call)");
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    CK(cudaEventSynchronize(c->chain->ev[1]), "sync (chain)");
    CK(cudaEventElapsedTime(ms, c->chain->ev[0], c->chain->ev[1]), "elapsed (chain)");
    return CB200_OK;
}

int cb200_ccm_chain_status(cb200_ctx* c)
{
    if (!c) return fail(CB200_ERR_ARG, "null context");
    if (!c->chain) return fail(CB200_ERR_ARG, "no CCM chain region");
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    CK(cudaStreamSynchronize(c->stream), "sync");
    uint32_t err = 0;
    CK(cudaMemcpy(&err, &c->chain->reg->error, sizeof(err), cudaMemcpyDeviceToHost), "read ccm chain status");
    if (err) { char msg[96]; snprintf(msg, sizeof(msg), "ccm chain: rank %u did not arrive in time", err - 1); return fail(CB200_ERR_CUDA, msg); }
    return CB200_OK;
}

}  // extern "C"
