// history.cu -- the group history of cb200_scan_extract_decode_chunks_grouped_history_dev (include/cb200.h): the final cells, walk
// distances and tags of the pictures of earlier calls that have not yet given a whole frame, kept on the device, so that each new
// batch is grouped against them as if they came first in it.  The rule is combine_core.cuh's (history_*).
//
// Layout.  Two staging regions, used alternately: each holds H + P positions (P: the largest batch so far) of cell bytes, walk
// traces and position statuses, plus H tags and the count h.  A call reads region `cur`: slots [0, H) hold the history (status 1
// for the h pictures, 0 for the empty slots), and the batch's final cells, traces and statuses are copied behind them.  The grouped
// call's k_pair_match and k_assign_groups then run over the H + n positions unchanged, k_history_groups keeps the groups with a
// batch member, the combined call's vote reads the region, and k_history_keep / k_history_copy write the new history into region
// cur ^ 1.  The count h stays on the device: the launches are sized for H + n positions.
#include "ctx.cuh"
#include "combine_core.cuh"

struct cb200_group_history {
    cb200_ctx* ctx = nullptr;
    int H = 0;                       // capacity
    int P = 0;                       // batch positions the regions hold
    int cur = 0;                     // the region the next call reads
    long long call = 0;              // accepted calls since create or reset
    cb200::DevBuf<uint8_t> cells[2];             // (H + P) x num_cells
    cb200::DevBuf<cb200::CellTrace> traces[2];   // (H + P) x num_cells
    cb200::DevBuf<int32_t> status[2];            // H + P
    cb200::DevBuf<int64_t> tags[2];              // H
    cb200::DevBuf<int32_t> count[2];             // 1
    // scratch of a call of n pictures, N = H + n positions: the assignment's group_of (N) and count (1), the table of n slots
    // (n + 1 offsets, N members), each position's group of the call (N), the done flags (n) and the new slots' sources (H)
    cb200::DevBuf<int32_t> work;
};

namespace cb200 {

static size_t work_ints(int H, int n)
{
    const size_t N = (size_t)H + n;
    return N + 1 + ((size_t)n + 1 + N) + N + (size_t)n + (size_t)H;
}

int history_check(const cb200_ctx* c, const cb200_group_history* h)
{
    if (!h) return fail(CB200_ERR_ARG, "null history");
    if (h->ctx != c) return fail(CB200_ERR_ARG, "the history belongs to another context");
    return CB200_OK;
}

int history_positions(const cb200_group_history* h) { return h->H; }

// b grown to `count` elements, keeping its first `keep`
template <class T> static int regrow(cb200_ctx* c, DevBuf<T>& b, size_t count, size_t keep, const char* what)
{
    if (count <= b.capacity()) return CB200_OK;
    DevBuf<T> nb;
    CK(nb.ensure(count), what);
    if (keep) CK(cudaMemcpyAsync(nb.get(), b.get(), keep * sizeof(T), cudaMemcpyDeviceToDevice, c->stream), what);
    b.swap(nb);                      // nb's destructor frees the old buffer: cudaFree waits for the copy
    return CB200_OK;
}

int history_reserve(cb200_ctx* c, cb200_group_history* h, int n)
{
    const size_t cells = (size_t)c->mode.num_cells, H = (size_t)h->H;
    if (n > h->P) {
        const size_t pos = H + (size_t)n;
        for (int r = 0; r < 2; ++r) {
            const size_t keep = r == h->cur ? H : 0;     // the other region's history slots are rewritten before they are read
            int rc;
            if ((rc = regrow(c, h->cells[r], pos * cells, keep * cells, "cudaMalloc history cells")) ||
                (rc = regrow(c, h->traces[r], pos * cells, keep * cells, "cudaMalloc history traces")) ||
                (rc = regrow(c, h->status[r], pos, keep, "cudaMalloc history statuses")))
                return rc;
        }
        h->P = n;
    }
    CK(h->work.ensure(work_ints(h->H, n)), "cudaMalloc history scratch");
    return CB200_OK;
}

// the groups of the assignment over the N positions (its group_of `of`, count, and table: offsets[0 .. N / 2], members) that have a
// batch member, one warp: numbered in their leaders' position order into d_group_of (batch positions only), d_group_count, the table
// of n slots (offsets[0 .. n], members: the groups' positions, in position order; slots past the count empty) and pos_group
__global__ void __launch_bounds__(32) k_history_groups(int N, int first, int n, const int32_t* __restrict__ acount,
                                                       const int32_t* __restrict__ aoffsets, const int32_t* __restrict__ amembers,
                                                       int32_t* __restrict__ group_of, int32_t* __restrict__ count,
                                                       int32_t* __restrict__ offsets, int32_t* __restrict__ members,
                                                       int32_t* __restrict__ pos_group)
{
    const int lane = threadIdx.x;
    const uint32_t below = (1u << lane) - 1u;
    for (int p = lane; p < N; p += 32) pos_group[p] = -1;
    __syncwarp();
    const int m = *acount;
    int groups = 0, placed = 0;
    for (int g0 = 0; g0 < m; g0 += 32) {
        const int g = g0 + lane;
        const int b = g < m ? aoffsets[g] : 0, e = g < m ? aoffsets[g + 1] : 0;
        const bool keep = g < m && combine::has_batch_member(amembers[e - 1], first);
        const uint32_t bal = __ballot_sync(~0u, keep);
        const int s = keep ? e - b : 0;
        int incl = s;
        for (int d = 1; d < 32; d <<= 1) {
            const int v = __shfl_up_sync(~0u, incl, d);
            if (lane >= d) incl += v;
        }
        if (keep) {
            const int ng = groups + __popc(bal & below), at = placed + incl - s;
            offsets[ng] = at;
            for (int j = b; j < e; ++j) {
                members[at + j - b] = amembers[j];
                pos_group[amembers[j]] = ng;
            }
        }
        groups += __popc(bal);
        placed += __shfl_sync(~0u, incl, 31);
    }
    for (int g = groups + lane; g <= n; g += 32) offsets[g] = placed;
    if (lane == 0) *count = groups;
    __syncwarp();
    for (int i = lane; i < n; i += 32) group_of[i] = pos_group[first + i];
}

constexpr int kKeepThreads = 1024;

// the block-wide exclusive prefix sum of one flag per thread, and the total
__device__ int block_rank(bool flag, int* total)
{
    __shared__ int warp_sums[kKeepThreads / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t bal = __ballot_sync(~0u, flag);
    if (lane == 0) warp_sums[warp] = __popc(bal);
    __syncthreads();
    int before = 0, all = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) {
        before += w < warp ? warp_sums[w] : 0;
        all += warp_sums[w];
    }
    __syncthreads();
    *total = all;
    return before + __popc(bal & ((1u << lane) - 1u));
}

// the keep rule of combine_core.cuh over the N positions, one CTA: the done groups from the groups' and the batch's chunk masks
// (done: n ints of scratch), then the kept positions counted and ranked, and the last H of them listed in src[0 .. h'); h' into *kept
__global__ void __launch_bounds__(kKeepThreads) k_history_keep(int N, int first, int H, int chunks_per_frame, const int32_t* __restrict__ status,
                                                               const uint32_t* __restrict__ own, const int32_t* __restrict__ count,
                                                               const uint32_t* __restrict__ gmask, const int32_t* __restrict__ pos_group,
                                                               int32_t* __restrict__ done, int32_t* __restrict__ src, int32_t* __restrict__ kept)
{
    const int m = *count;
    for (int g = threadIdx.x; g < m; g += blockDim.x) done[g] = combine::complete(gmask[g], chunks_per_frame);
    __syncthreads();
    for (int p = first + threadIdx.x; p < N; p += blockDim.x)
        if (pos_group[p] >= 0 && combine::complete(own[p - first], chunks_per_frame)) done[pos_group[p]] = 1;
    __syncthreads();
    auto keeps = [&](int p) {
        if (p >= N) return false;
        const bool own_complete = p >= first && combine::complete(own[p - first], chunks_per_frame);
        return combine::keeps(p, first, status[p], own_complete, pos_group[p] >= 0 && done[pos_group[p]] != 0);
    };
    int total = 0;
    for (int p0 = 0; p0 < N; p0 += blockDim.x) {
        int t;
        block_rank(keeps(p0 + threadIdx.x), &t);
        total += t;
    }
    int base = 0;
    for (int p0 = 0; p0 < N; p0 += blockDim.x) {
        const int p = p0 + threadIdx.x;
        const bool k = keeps(p);
        int t;
        const int r = base + block_rank(k, &t);
        const int s = combine::keep_destination(r, total, H);
        if (k && s >= 0) src[s] = p;
        base += t;
    }
    if (threadIdx.x == 0) *kept = total < H ? total : H;
}

constexpr int kCopyThreads = 256;

// the new history into the other region, one CTA row per slot s < H: slot s < h' (= *kept) takes position src[s]'s cells, traces
// and tag (a batch picture's: call << 32 | batch index), status 1; the other slots status 0.  Cells and traces go 8 bytes at a time
// (num_cells is a multiple of 8)
__global__ void __launch_bounds__(kCopyThreads) k_history_copy(int cells, int first, long long call, const int32_t* __restrict__ src,
                                                               const int32_t* __restrict__ kept, const uint8_t* __restrict__ from_cells,
                                                               const CellTrace* __restrict__ from_traces, const int64_t* __restrict__ from_tags,
                                                               uint8_t* __restrict__ to_cells, CellTrace* __restrict__ to_traces,
                                                               int32_t* __restrict__ to_status, int64_t* __restrict__ to_tags,
                                                               int32_t* __restrict__ to_count)
{
    const int s = blockIdx.y, h = *kept;
    const bool lead = blockIdx.x == 0 && threadIdx.x == 0;
    if (lead) to_status[s] = combine::history_slot_status(s, h);
    if (lead && s == 0) *to_count = h;
    if (s >= h) return;
    const int p = src[s];
    if (lead) to_tags[s] = p < first ? from_tags[p] : (int64_t)((unsigned long long)call << 32 | (unsigned)(p - first));
    const uint64_t* fc = reinterpret_cast<const uint64_t*>(from_cells + (size_t)p * cells);
    uint64_t* tc = reinterpret_cast<uint64_t*>(to_cells + (size_t)s * cells);
    const uint64_t* ft = reinterpret_cast<const uint64_t*>(from_traces + (size_t)p * cells);
    uint64_t* tt = reinterpret_cast<uint64_t*>(to_traces + (size_t)s * cells);
    const int stride = gridDim.x * blockDim.x;
    for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < cells / 8; k += stride) tc[k] = fc[k];
    for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < cells; k += stride) tt[k] = ft[k];
}

// the scratch of a call of n pictures (work_ints)
struct Work {
    int32_t *of, *acount, *table, *pos_group, *done, *src;
    Work(cb200_group_history* h, int n)
    {
        const size_t N = (size_t)h->H + n;
        of = h->work.get();
        acount = of + N;
        table = acount + 1;
        pos_group = table + (size_t)n + 1 + N;
        done = pos_group + N;
        src = done + n;
    }
};

int history_groups(cb200_ctx* c, cb200_group_history* h, int n, const int32_t* d_status, int32_t* d_group_of, int32_t* d_group_count,
                   HistoryStage* st)
{
    const size_t cells = (size_t)c->mode.num_cells, H = (size_t)h->H;
    const int N = h->H + n, r = h->cur;
    CK(cudaMemcpyAsync(h->cells[r].get() + H * cells, c->d_cellvals.get(), (size_t)n * cells, cudaMemcpyDeviceToDevice, c->stream),
       "stage batch cells");
    CK(cudaMemcpyAsync(h->traces[r].get() + H * cells, c->d_traces.get(), (size_t)n * cells * sizeof(CellTrace), cudaMemcpyDeviceToDevice,
                       c->stream), "stage batch traces");
    CK(cudaMemcpyAsync(h->status[r].get() + H, d_status, sizeof(int32_t) * (size_t)n, cudaMemcpyDeviceToDevice, c->stream),
       "stage batch statuses");
    Work w(h, n);
    int rc = find_groups(c, N, h->status[r], w.of, w.acount, nullptr, h->cells[r]);
    if (rc) return rc;
    const int aslots = N / 2;                        // find_groups' table in c->d_groups: offsets[0 .. aslots], then the members
    k_history_groups<<<1, 32, 0, c->stream>>>(N, h->H, n, w.acount, c->d_groups.get(), c->d_groups.get() + aslots + 1, d_group_of,
                                              d_group_count, w.table, w.table + n + 1, w.pos_group);
    count_launch();
    CK(cudaGetLastError(), "history groups launch");
    *st = {h->cells[r].get(), h->traces[r].get(), h->status[r].get(), w.table};
    return CB200_OK;
}

int history_settle(cb200_ctx* c, cb200_group_history* h, int n, const uint32_t* d_chunk_mask, const int32_t* d_group_count,
                   const uint32_t* d_group_mask)
{
    const Mode& md = c->mode;
    const int N = h->H + n, r = h->cur, o = r ^ 1;
    Work w(h, n);
    int32_t* kept = w.acount;                        // the assignment's count: k_history_groups, before this, was its last reader
    k_history_keep<<<1, kKeepThreads, 0, c->stream>>>(N, h->H, h->H, md.chunks_per_frame, h->status[r], d_chunk_mask, d_group_count,
                                                     d_group_mask, w.pos_group, w.done, w.src, kept);
    count_launch();
    CK(cudaGetLastError(), "history keep launch");
    const dim3 grid((unsigned)((md.num_cells + 4 * kCopyThreads - 1) / (4 * kCopyThreads)), (unsigned)h->H);
    k_history_copy<<<grid, kCopyThreads, 0, c->stream>>>(md.num_cells, h->H, h->call, w.src, kept, h->cells[r], h->traces[r], h->tags[r],
                                                         h->cells[o], h->traces[o], h->status[o], h->tags[o], h->count[o]);
    count_launch();
    CK(cudaGetLastError(), "history copy launch");
    h->cur = o;
    ++h->call;
    return CB200_OK;
}

void history_skip(cb200_group_history* h) { ++h->call; }

}  // namespace cb200

using namespace cb200;

extern "C" {

int cb200_group_history_create(cb200_ctx* c, int capacity, cb200_group_history** out)
{
    if (!out) return fail(CB200_ERR_ARG, "null output");
    *out = nullptr;
    if (!c) return fail(CB200_ERR_ARG, "null context");
    if (capacity < 1 || capacity > kMaxHistory)
        return fail(CB200_ERR_ARG, "capacity = " + std::to_string(capacity) + " outside [1, " + std::to_string(kMaxHistory) + "]");
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    cb200_group_history* h = new cb200_group_history;
    h->ctx = c;
    h->H = capacity;
    const size_t cells = (size_t)c->mode.num_cells, H = (size_t)capacity;
    for (int r = 0; r < 2; ++r) {
        cudaError_t e = h->cells[r].ensure(H * cells);
        if (e == cudaSuccess) e = h->traces[r].ensure(H * cells);
        if (e == cudaSuccess) e = h->status[r].ensure(H);
        if (e == cudaSuccess) e = h->tags[r].ensure(H);
        if (e == cudaSuccess) e = h->count[r].ensure(1);
        if (e == cudaSuccess) e = cudaMemsetAsync(h->status[r].get(), 0, sizeof(int32_t) * H, c->stream);
        if (e == cudaSuccess) e = cudaMemsetAsync(h->count[r].get(), 0, sizeof(int32_t), c->stream);
        if (e != cudaSuccess) {
            delete h;
            return fail_cuda(e, "history create");
        }
    }
    *out = h;
    return CB200_OK;
}

int cb200_group_history_reset(cb200_group_history* h)
{
    if (!h) return fail(CB200_ERR_ARG, "null history");
    cb200_ctx* c = h->ctx;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    h->cur = 0;
    h->call = 0;
    CK(cudaMemsetAsync(h->status[0].get(), 0, sizeof(int32_t) * (size_t)h->H, c->stream), "reset history");
    CK(cudaMemsetAsync(h->count[0].get(), 0, sizeof(int32_t), c->stream), "reset history count");
    return CB200_OK;
}

int cb200_group_history_read(cb200_group_history* h, int64_t* tags, int max, int32_t* count)
{
    if (!h) return fail(CB200_ERR_ARG, "null history");
    if (!count) return fail(CB200_ERR_ARG, "null count");
    if (max < 0) return fail(CB200_ERR_ARG, "max = " + std::to_string(max) + " < 0");
    if (max > 0 && !tags) return fail(CB200_ERR_ARG, "null tags with max > 0");
    cb200_ctx* c = h->ctx;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    int32_t k = 0;
    CK(cudaMemcpyAsync(&k, h->count[h->cur].get(), sizeof(int32_t), cudaMemcpyDeviceToHost, c->stream), "D2H history count");
    CK(cudaStreamSynchronize(c->stream), "sync");
    const int take = k < max ? k : max;
    if (take > 0) {
        CK(cudaMemcpyAsync(tags, h->tags[h->cur].get(), sizeof(int64_t) * (size_t)take, cudaMemcpyDeviceToHost, c->stream), "D2H history tags");
        CK(cudaStreamSynchronize(c->stream), "sync");
    }
    *count = k;
    return CB200_OK;
}

int cb200_group_history_destroy(cb200_group_history* h)
{
    if (!h) return fail(CB200_ERR_ARG, "null history");
    cudaSetDevice(h->ctx->device);
    delete h;
    return CB200_OK;
}

}  // extern "C"
