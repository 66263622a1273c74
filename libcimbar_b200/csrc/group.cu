// group.cu -- the groups of cb200_scan_extract_decode_chunks_grouped_dev (and, within each receiver, of the grouped receivers call),
// found on the device from the pictures' final cell bytes and extract statuses by the rule of combine_core.cuh: k_pair_match gives
// the match rows of all pairs (of one receiver's pairs), k_assign_groups the assignment and the group table that scan.cu's
// combine_groups (the combined call's vote and decode) reads.  Its own translation
// unit: the assignment's dynamic shared memory would change the shared-memory lines of scan.cu's kernels
#include "ctx.cuh"
#include "combine_core.cuh"

namespace cb200 {

constexpr int kPairTile = combine::kPairTile;
constexpr int kPairWords = 32;       // packed words (8 cells each) per picture and stage
constexpr int kPairThreads = 256;    // 16 x 16 threads, 4 x 4 pairs each
constexpr int kAssignWarps = 32;     // k_assign_groups: segments assigned at once

// the match rows of n pictures (combine_core.cuh), one CTA per pair of tiles (I, J <= I) of kPairTile positions.  Each stage packs
// kPairWords words of both tiles' symbol nibbles into shared memory (every mode's cell count is a multiple of 8, and so is the row
// pitch of the cell bytes), and each thread counts the differing symbols of its 4 x 4 pairs.  Each word of row i up to column i
// belongs to one tile pair; a diagonal tile also writes bits j >= i, which are never read.
// map: NULL for one receiver (position = batch index, every tile pair, blockIdx.x = I (I + 1) / 2 + J); else the receivers map (the n
// receivers, then the receiver-major order): position p is picture order[p], the CTAs take the `ntiles` pairs of `tiles` (I, J;
// combine::pair_tiles) and a CTA past them (a launch of one CTA for none) returns, and the bits of pairs of two receivers are cleared
__global__ void __launch_bounds__(kPairThreads) k_pair_match(int n, int cells, int symbol_bits, const uint8_t* __restrict__ cellvals,
                                                             const int32_t* __restrict__ status, uint32_t* __restrict__ rows,
                                                             const int32_t* __restrict__ map, const int2* __restrict__ tiles, int ntiles)
{
    __shared__ uint32_t sa[kPairTile][kPairWords + 1], sb[kPairTile][kPairWords + 1];
    __shared__ int32_t pa[kPairTile], pb[kPairTile];         // the tiles' pictures (batch indices), -1 past n
    int I, J;
    if (map) {
        if ((int)blockIdx.x >= ntiles) return;
        I = tiles[blockIdx.x].x;
        J = tiles[blockIdx.x].y;
    } else {
        const long long b = blockIdx.x;                      // = I (I + 1) / 2 + J
        I = (int)((sqrt(8.0 * (double)b + 1.0) - 1.0) / 2.0);
        while ((long long)I * (I + 1) / 2 > b) --I;
        while ((long long)(I + 1) * (I + 2) / 2 <= b) ++I;
        J = (int)(b - (long long)I * (I + 1) / 2);
    }
    const int i0 = I * kPairTile, j0 = J * kPairTile;
    const int t = threadIdx.x, ty = t >> 4, tx = t & 15;
    const int words = cells / 8;
    if (t < 2 * kPairTile) {
        const int p = (t < kPairTile ? i0 : j0 - kPairTile) + t;
        (t < kPairTile ? pa : pb)[t & (kPairTile - 1)] = p >= n ? -1 : map ? map[n + p] : p;
    }
    __syncthreads();
    auto packed = [&](int pic, int k) -> uint32_t {
        if (pic < 0 || k >= words) return 0u;
        return combine::pack_symbols(*reinterpret_cast<const uint64_t*>(cellvals + (size_t)pic * cells + 8 * (size_t)k), symbol_bits);
    };
    int diff[4][4] = {};
    for (int k0 = 0; k0 < words; k0 += kPairWords) {
        for (int e = t; e < kPairTile * kPairWords; e += kPairThreads) {
            const int p = e / kPairWords, k = e % kPairWords;
            sa[p][k] = packed(pa[p], k0 + k);
            sb[p][k] = packed(pb[p], k0 + k);
        }
        __syncthreads();
#pragma unroll 4
        for (int k = 0; k < kPairWords; ++k) {
            uint32_t a[4], w[4];
#pragma unroll
            for (int r = 0; r < 4; ++r) { a[r] = sa[ty + 16 * r][k]; w[r] = sb[tx + 16 * r][k]; }
#pragma unroll
            for (int r = 0; r < 4; ++r)
#pragma unroll
                for (int q = 0; q < 4; ++q) diff[r][q] += combine::differing_symbols(a[r], w[q]);
        }
        __syncthreads();
    }
    // the bits of pair (ty + 16 r, tx + 16 q): a warp holds two rows (lanes 0-15 the even ty, 16-31 the odd one) and, per q, 16
    // columns, so word q / 2 of a row takes one ballot for its low and one for its high half.  Bit 4 r + q of `both`: both pictures
    // take part and have one receiver (always so without a map)
    bool ej[4];
    int32_t rj[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const int j = pb[tx + 16 * q];
        ej[q] = j >= 0 && combine::takes_part(status[j]);
        rj[q] = map && j >= 0 ? map[j] : 0;
    }
    uint32_t both = 0;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        const int i = pa[ty + 16 * r];
        const bool ei = i >= 0 && combine::takes_part(status[i]);
        const int32_t ri = map && i >= 0 ? map[i] : 0;
#pragma unroll
        for (int q = 0; q < 4; ++q) both |= (uint32_t)(ei && ej[q] && ri == rj[q]) << (4 * r + q);
    }
    const int lane = t & 31;
    const size_t W = ((size_t)n + 31) / 32;
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const uint32_t lo = __ballot_sync(~0u, (both >> (4 * r + 2 * h) & 1u) && combine::match(cells - diff[r][2 * h], cells));
            const uint32_t hi = __ballot_sync(~0u, (both >> (4 * r + 2 * h + 1) & 1u) && combine::match(cells - diff[r][2 * h + 1], cells));
            const int i = i0 + ty + 16 * r;
            const size_t w = (size_t)j0 / 32 + h;
            if ((lane & 15) == 0 && i < n && w < W)
                rows[(size_t)i * W + w] = lane == 0 ? (lo & 0xFFFFu) | (hi << 16) : (lo >> 16) | (hi & 0xFFFF0000u);
        }
}

// the assignment of combine_core.cuh over the match rows (indexed by position, as k_pair_match wrote them), one warp per segment
// (combine::assign_segment), up to kAssignWarps at once.  Per position p of a segment [s, e), in order, the lanes search its row 32
// words at a time for the earliest open leader in [s, p) (open_matches; `open` is ceil(n / 32) words of dynamic shared memory, which
// several segments share, so join() then changes it atomically), and lane 0 applies join().  map / starts: NULL for one segment
// [0, n) in batch order (the grouped call); else the receivers map (receivers, then the order) and the segs + 1 segment starts
// (combine::segment_starts).  Then, in one warp, the groups are numbered in their leaders' batch order, their ranges laid out in
// offsets[0 .. slots] (slots past the count get empty ones) and their members placed in batch order: the table combine::group_table
// builds from group_of; with group_receiver, group g's receiver (its leader's) and -1 past the count.  work: each picture's leader,
// then each leader's group size, which becomes its next member's place (batch indices, 2 n ints); with a map, first the same two by
// position (2 n ints more)
__global__ void __launch_bounds__(32 * kAssignWarps) k_assign_groups(int n, int slots, const uint32_t* __restrict__ rows,
                                                                     const int32_t* __restrict__ status, const int32_t* __restrict__ map,
                                                                     const int32_t* __restrict__ starts, int segs,
                                                                     int32_t* __restrict__ group_of, int32_t* __restrict__ count,
                                                                     int32_t* __restrict__ offsets, int32_t* __restrict__ members,
                                                                     int32_t* __restrict__ work, int32_t* __restrict__ group_receiver)
{
    extern __shared__ uint32_t open[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, warps = blockDim.x >> 5;
    const size_t W = ((size_t)n + 31) / 32;
    const int32_t* order = map ? map + n : nullptr;
    int32_t* lead = work;
    int32_t* size = work + n;
    int32_t* plead = map ? work + 2 * (size_t)n : lead;
    int32_t* psize = map ? work + 3 * (size_t)n : size;
    for (size_t w = threadIdx.x; w < W; w += blockDim.x) open[w] = 0;
    __syncthreads();
    for (int seg = warp; seg < segs; seg += warps) {
        const int s = starts ? starts[seg] : 0, e = starts ? starts[seg + 1] : n;
        for (int p = s; p < e; ++p) {
            int j = -1;
            if (combine::takes_part(status[order ? order[p] : p])) {
                j = p;
                const uint32_t* row = rows + (size_t)p * W;
                for (int w0 = s >> 5; w0 <= p >> 5 && j == p; w0 += 32) {
                    const uint32_t x = combine::open_matches(row, open, p, w0 + lane, s);
                    const uint32_t hit = __ballot_sync(~0u, x != 0);
                    if (hit) {
                        const int l = __ffs(hit) - 1;
                        j = 32 * (w0 + l) + __ffs(__shfl_sync(~0u, x, l)) - 1;
                    }
                }
                if (lane == 0) combine::join(p, j, psize, open, segs > 1);
            }
            if (lane == 0) plead[p] = j;
            __syncwarp();
        }
    }
    if (map) {
        __syncthreads();
        for (int p = threadIdx.x; p < n; p += blockDim.x) {
            const int i = order[p];
            lead[i] = plead[p] < 0 ? -1 : order[plead[p]];
            size[i] = psize[p];
        }
    }
    __syncthreads();
    if (warp) return;
    const uint32_t below = (1u << lane) - 1u;
    int groups = 0, placed = 0;
    for (int i0 = 0; i0 < n; i0 += 32) {
        const int i = i0 + lane;
        const bool leads = i < n && lead[i] == i && size[i] >= 2;
        const uint32_t bal = __ballot_sync(~0u, leads);
        const int s = leads ? size[i] : 0;
        int incl = s;
        for (int d = 1; d < 32; d <<= 1) {
            const int v = __shfl_up_sync(~0u, incl, d);
            if (lane >= d) incl += v;
        }
        const int g = groups + __popc(bal & below);
        if (leads) {
            offsets[g] = placed + incl - s;
            size[i] = placed + incl - s;
            if (group_receiver) group_receiver[g] = map[i];
        }
        if (i < n) group_of[i] = leads ? g : -1;
        groups += __popc(bal);
        placed += __shfl_sync(~0u, incl, 31);
    }
    for (int g = groups + lane; g <= slots; g += 32) {
        offsets[g] = placed;
        if (group_receiver && g < slots) group_receiver[g] = -1;
    }
    if (lane == 0) *count = groups;
    __syncwarp();
    for (int i0 = 0; i0 < n; i0 += 32) {
        const int i = i0 + lane;
        const int l = i < n ? lead[i] : -1;
        const int g = l >= 0 ? group_of[l] : -1;             // the leader's number (-1: alone), which this loop writes back unchanged
        const uint32_t peers = __match_any_sync(~0u, g >= 0 ? l : -1 - lane);
        const int at = g >= 0 ? size[l] + __popc(peers & below) : 0;
        __syncwarp();
        if (g >= 0) {
            members[at] = i;
            group_of[i] = g;
            if (lane == 31 - __clz(peers)) size[l] = at + 1;
        }
        __syncwarp();
    }
}

int find_groups(cb200_ctx* c, int n, const int32_t* d_status, int32_t* d_group_of, int32_t* d_group_count, const GroupLists* lists,
                const uint8_t* d_cellvals)
{
    const Mode& md = c->mode;
    const int slots = n / 2;
    const long long tiles = (n + kPairTile - 1) / kPairTile;
    const unsigned grid = lists ? (unsigned)std::max(lists->ntiles, 1) : (unsigned)(tiles * (tiles + 1) / 2);
    k_pair_match<<<grid, kPairThreads, 0, c->stream>>>(n, md.num_cells, md.symbol_bits, d_cellvals ? d_cellvals : c->d_cellvals.get(),
                                                        d_status, c->d_pairs,
                                                        lists ? lists->d_map : nullptr, lists ? lists->d_tiles : nullptr,
                                                        lists ? lists->ntiles : 0);
    count_launch();
    CK(cudaGetLastError(), "pair launch");
    const size_t open_bytes = sizeof(uint32_t) * (((size_t)n + 31) / 32);
    if (open_bytes > 48 * 1024)
        CK(cudaFuncSetAttribute(k_assign_groups, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)open_bytes), "assign smem");
    int32_t* table = c->d_groups;
    const int segs = lists ? lists->segs : 1;
    k_assign_groups<<<1, 32 * std::min(segs, kAssignWarps), open_bytes, c->stream>>>(
        n, slots, c->d_pairs, d_status, lists ? lists->d_map : nullptr, lists ? lists->d_starts : nullptr, segs, d_group_of, d_group_count,
        table, table + slots + 1, table + slots + 1 + n, lists ? lists->d_group_receiver : nullptr);
    count_launch();
    CK(cudaGetLastError(), "assign launch");
    return CB200_OK;
}

}  // namespace cb200
