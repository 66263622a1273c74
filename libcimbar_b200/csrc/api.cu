// api.cu -- the C ABI of libcb200.so (include/cb200.h): context, tables, and the kernel pipelines.
// There is no CPU decode path in this library: every entry point that produces decode results launches the
// sm_90a kernels, and cb200_create fails with CB200_ERR_NODEVICE when no CUDA device is usable.
#include "ctx.cuh"
#include "k1_decode.cuh"
#include "k2_rs.cuh"
#include "render.cuh"
#include "encode.cuh"

#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

using namespace cb200;

namespace {

thread_local std::string g_err;
std::atomic<unsigned long long> g_launches{0};

}  // namespace
namespace cb200 {
int fail(int code, const std::string& msg) { g_err = msg; return code; }
int fail_cuda(cudaError_t e, const char* what)
{
    g_err = std::string(what) + ": " + cudaGetErrorString(e);
    return CB200_ERR_CUDA;
}
}  // namespace cb200
namespace {

// tile dictionary = CimbDecoder::_tileHashes for symbol_bits=4, dark (src/lib/cimb_translator/CimbDecoder.cpp:87-99),
// i.e. average_hash of bitmap/4/00..0f.png; values pinned by src/lib/image_hash/test/averageHashTest.cpp:43-50.
const unsigned long long kTilesH[16] = {
    0xfffefcf8f0e0c080ULL, 0x80c0e0f0f8fcfeffULL, 0xff7f3f1f0f070301ULL, 0x0103070f1f3f7fffULL,
    0x181818ffff181818ULL, 0x66e7e70000e7e766ULL, 0x3c7ee7c3c3e77e3cULL, 0x18183c3c7e7effffULL,
    0xc0f0fcfffffcf0c0ULL, 0xfffcf00000f0fcffULL, 0xff3f0f00000f3fffULL, 0xe7e7e7e7c3c38181ULL,
    0x8181c3c3e7e7e7e7ULL, 0x0000c3e77e3c1800ULL, 0x0c1c387070381c0cULL, 0x1e1e38381c1c7878ULL,
};

unsigned long long brev64(unsigned long long x)
{
    unsigned long long r = 0;
    for (int i = 0; i < 64; ++i) if (x & (1ULL << i)) r |= 1ULL << (63 - i);
    return r;
}

// palettes: getColor4 / getColor8 (color_mode 1) and getColor4_old / getColor8_old (color_mode 0),
// src/lib/cimb_translator/Common.cpp:21-85, selection :122-139
void fill_palette(int num_colors, int color_mode, uint8_t out[8][4])
{
    uint8_t pal[2][8][3];
    static const uint8_t c4[4][3] = {{0, 255, 0}, {0, 255, 255}, {255, 255, 0}, {255, 0, 255}};
    static const uint8_t c4old[4][3] = {{0, 255, 255}, {255, 255, 0}, {255, 0, 255}, {0, 255, 0}};
    static const uint8_t c8[8][3] = {{0, 255, 255}, {255, 255, 0}, {0x7F, 0x7F, 255}, {255, 255, 255}, {0, 255, 0}, {255, 0x9F, 0}, {255, 0, 255}, {255, 65, 65}};
    static const uint8_t c8old[8][3] = {{0, 255, 255}, {0x7F, 0x7F, 255}, {255, 0, 255}, {255, 65, 65}, {255, 0x9F, 0}, {255, 255, 0}, {255, 255, 255}, {0, 255, 0}};
    memset(pal, 0, 48);
    for (int i = 0; i < 8; ++i)
        for (int k = 0; k < 3; ++k) {
            pal[0][i][k] = (num_colors <= 4) ? c4old[i & 3][k] : c8old[i][k];
            pal[1][i][k] = (num_colors <= 4) ? c4[i & 3][k] : c8[i][k];
        }
    for (int i = 0; i < 8; ++i) { for (int k = 0; k < 3; ++k) out[i][k] = pal[color_mode ? 1 : 0][i][k]; out[i][3] = 0; }
}

// cimbar::conf table: src/lib/cimb_translator/GridConf.h:121-189, Config.h:20-43
bool mode_init(Mode& m, int mode_val)
{
    memset(&m, 0, sizeof(m));
    m.mode_val = mode_val;
    m.color_bits = 2; m.symbol_bits = 4; m.ecc_bytes = 30; m.ecc_block = 155;
    m.width = 1024; m.height = 1024; m.cell_offset = 8; m.cells_x = 112; m.cells_y = 112;
    int chunks_scalar = 2;
    switch (mode_val) {
    case 68: break;
    case 4: m.legacy = 1; chunks_scalar = -10; break;
    case 8: m.color_bits = 3; m.legacy = 1; chunks_scalar = -10; break;
    case 66: m.ecc_bytes = 33; m.ecc_block = 168; m.width = 736; m.height = 637; m.cell_offset = 9; m.cells_x = 80; m.cells_y = 69; chunks_scalar = 1; break;
    case 67: m.ecc_bytes = 36; m.ecc_block = 179; m.width = 1024; m.height = 720; m.cell_offset = 9; m.cells_x = 112; m.cells_y = 78; chunks_scalar = 2; break;
    default: return false;
    }
    m.corner = (int)lrint(54.0 / kSpacing);                                   // GridConf.h:32-40
    m.color_mode = m.legacy ? 0 : 1;                                            // Config.h:61-64
    m.num_cells = m.cells_x * m.cells_y - 4 * m.corner * m.corner;              // GridConf.h:42-45
    int bpc = m.color_bits + m.symbol_bits;
    m.cap_all = m.num_cells * bpc / 8;                                          // GridConf.h:47-52
    m.cap_sym = m.legacy ? m.cap_all : m.num_cells * m.symbol_bits / 8;
    m.cap_col = m.legacy ? 0 : m.num_cells * m.color_bits / 8;
    m.msg_len = m.ecc_block - m.ecc_bytes;
    m.nblocks = m.cap_all / m.ecc_block;
    m.nblocks_sym = m.cap_sym / m.ecc_block;
    m.chunks_per_frame = chunks_scalar < 0 ? -chunks_scalar : bpc * chunks_scalar;   // GridConf.h:54-61
    m.chunk_size = m.cap_all * m.msg_len / m.ecc_block / m.chunks_per_frame;    // GridConf.h:63-72
    m.blocks_per_chunk = m.chunk_size / m.msg_len;
    m.data_bytes = m.nblocks * m.msg_len;
    m.top_cells = (m.cells_x - 2 * m.corner) * m.corner;
    m.mid_cells = m.cells_x * (m.cells_y - 2 * m.corner);
    // layout invariants the kernels rely on (true for every 8x8 mode in GridConf.h)
    if (m.cap_sym % m.ecc_block || m.cap_all % m.ecc_block || m.chunk_size % m.msg_len || m.width % 8 || (m.width * 3) % 16) return false;
    if (m.nblocks * m.msg_len != m.chunks_per_frame * m.chunk_size) return false;
    // perfect hash over the little-endian tile words: slot = (L_lo * mul) >> 28 distinct for the 16 tiles (the dictionary
    // is the same in every mode: searched once per process)
    static const uint32_t hash_mul = [] {
        uint32_t x = 0x2545F491u;
        for (int trial = 0; trial < 50000000; ++trial) {
            x ^= x << 13; x ^= x >> 17; x ^= x << 5;
            uint32_t mul = x | 1u, seen = 0;
            bool ok = true;
            for (int t = 0; t < 16 && ok; ++t) {
                uint32_t slot = ((uint32_t)brev64(kTilesH[t]) * mul) >> 28;
                if (seen & (1u << slot)) ok = false;
                seen |= 1u << slot;
            }
            if (ok) return mul;
        }
        return 0u;
    }();
    m.hash_mul = hash_mul;
    fill_palette(1 << m.color_bits, m.color_mode, m.palette);
    for (int i = 0; i < 8; ++i) {
        const int p0 = (int)m.palette[i][0] - (int)m.palette[i][1], p1 = (int)m.palette[i][1] - (int)m.palette[i][2],
                  p2 = (int)m.palette[i][2] - (int)m.palette[i][0];
        m.pal_c[i] = p0 * p0 + p1 * p1 + p2 * p2; m.pal_u[i] = 2 * (p0 - p2); m.pal_w[i] = 2 * (p1 - p2);
    }
    return m.hash_mul != 0;
}

void fill_info(const Mode& m, int max_frames, int sm_count, cb200_info* o)
{
    o->mode_val = m.mode_val; o->image_size_x = m.width; o->image_size_y = m.height; o->frame_bytes = m.width * m.height * 3;
    o->total_cells = m.num_cells; o->symbol_bits = m.symbol_bits; o->color_bits = m.color_bits;
    o->raw_bytes = m.cap_all; o->raw_symbol_bytes = m.cap_sym; o->ecc_bytes = m.ecc_bytes; o->ecc_block_size = m.ecc_block;
    o->rs_blocks = m.nblocks; o->data_bytes = m.data_bytes; o->chunk_size = m.chunk_size; o->chunks_per_frame = m.chunks_per_frame;
    o->legacy_mode = m.legacy; o->max_frames = max_frames; o->sm_count = sm_count;
}

// Interleave::interleave_indices (src/lib/cimb_translator/Interleave.h:8-24)
void interleave_indices(const Mode& m, std::vector<uint16_t>& idx)
{
    unsigned size = (unsigned)m.num_cells, chunks = (unsigned)m.ecc_block, partitions = 2;
    idx.clear();
    unsigned psize = size / partitions;
    for (unsigned part = 0; part < size; part += psize)
        for (unsigned c = 0; c < chunks; ++c)
            for (unsigned i = c; i < psize; i += chunks)
                idx.push_back((uint16_t)(i + part));
}

// neighbour table for the exact walk: AdjacentCellFinder::find (src/lib/cimb_translator/AdjacentCellFinder.cpp:54-105),
// evaluated literally (position comparisons included) over the linear cell positions (CellPositions.cpp:5-50)
void build_adjacency(const Mode& m, std::vector<uint16_t>& adj)
{
    const int n_cells = m.num_cells;
    std::vector<int> xs(n_cells);
    for (int k = 0, i = 0; k < m.cells_y; ++k) {
        int base, ncols, x0;
        cell_row_geom(m, k, base, ncols, x0);
        for (int cc = 0; cc < ncols; ++cc, ++i) xs[i] = x0 + kSpacing * cc;
    }
    const int first_mid = m.top_cells, first_bottom = m.top_cells + m.mid_cells;
    auto margin = [&](int index) { return (index < first_mid) ? 1 : (index < first_bottom ? 0 : 1); };
    auto right = [&](int index) -> int { if (index < 0 || index >= n_cells - 1) return -1; int next = index + 1; return xs[next] < xs[index] ? -1 : next; };
    auto left = [&](int index) -> int { int next = index - 1; if (next < 0) return -1; return xs[next] > xs[index] ? -1 : next; };
    auto bottom = [&](int index) -> int {
        if (index < 0 || index >= n_cells) return -1;
        int inc = m.cells_x; if (margin(index)) inc -= m.corner;
        int next = index + inc; if (margin(next)) next -= m.corner;
        if (next < 0 || next >= n_cells) return -1;
        return xs[next] != xs[index] ? -1 : next;
    };
    auto top = [&](int index) -> int {
        int inc = m.cells_x; if (margin(index)) inc -= m.corner;
        int next = index - inc; if (margin(next)) next += m.corner;
        if (next < 0) return -1;
        return xs[next] != xs[index] ? -1 : next;
    };
    adj.assign((size_t)n_cells * 4, 0);
    for (int i = 0; i < n_cells; ++i) {
        int v[4] = {right(i), left(i), bottom(i), top(i)};
        for (int d = 0; d < 4; ++d) adj[(size_t)i * 4 + d] = v[d] < 0 ? (uint16_t)0xFFFF : (uint16_t)v[d];
    }
}

// the kernels use the (row, column) form of the same relation (cell_neighbour): the two must agree everywhere
bool adjacency_consistent(const Mode& m, const std::vector<uint16_t>& adj)
{
    for (int i = 0; i < m.num_cells; ++i) {
        int k, cc, k2, c2;
        cell_row_col(m, i, k, cc);
        int base, ncols, x0;
        cell_row_geom(m, k, base, ncols, x0);
        if (base + cc != i) return false;
        for (int d = 0; d < 4; ++d) {
            int v = cell_neighbour(m, k, cc, d, k2, c2);
            if ((v < 0 ? 0xFFFF : v) != adj[(size_t)i * 4 + d]) return false;
        }
    }
    return true;
}

}  // namespace

namespace cb200 {
void count_launch(int n) { g_launches.fetch_add((unsigned long long)n, std::memory_order_relaxed); }

int stage_take(cb200_ctx* c, size_t bytes, int* slot, uint8_t** h)
{
    *slot = c->stage_next;
    c->stage_next = (*slot + 1) % cb200_ctx::kStageSlots;
    cb200_ctx::StageSlot& s = c->stage[*slot];
    if (!s.ev) CK(cudaEventCreateWithFlags(&s.ev, cudaEventDisableTiming), "cudaEventCreate upload slot");
    CK(cudaEventSynchronize(s.ev), "sync (upload slot)");      // the slot may only grow once its last copy has run
    CK(s.h.ensure(bytes), "cudaMallocHost upload slot");
    *h = s.h;
    return CB200_OK;
}

int stage_send(cb200_ctx* c, int slot, void* d_dst, size_t bytes, const char* what)
{
    CK(cudaMemcpyAsync(d_dst, c->stage[slot].h, bytes, cudaMemcpyHostToDevice, c->stream), what);
    CK(cudaEventRecord(c->stage[slot].ev, c->stream), "record upload slot");
    return CB200_OK;
}
}  // namespace cb200

namespace {

// CB200_FLAG_SHARPEN_IF_NEEDED is a decision about camera pictures: the entry points that take extracted frames refuse it
int check_frame_flags(uint32_t flags)
{
    if (flags & CB200_FLAG_SHARPEN_IF_NEEDED) return fail(CB200_ERR_ARG, "CB200_FLAG_SHARPEN_IF_NEEDED applies to camera pictures, not to frames");
    return CB200_OK;
}
// the frame entry points with a per-frame selection
int check_selection_args(uint32_t flags, const uint8_t* sharpen)
{
    int rc = check_frame_flags(flags); if (rc) return rc;
    if (flags & CB200_FLAG_SHARPEN) return fail(CB200_ERR_ARG, "CB200_FLAG_SHARPEN with a per-frame sharpen selection");
    if (!sharpen) return fail(CB200_ERR_ARG, "null sharpen selection");
    return CB200_OK;
}

int check_n(const cb200_ctx* c, int n)
{
    if (!c) return fail(CB200_ERR_ARG, "null context");
    if (n < 0 || n > c->max_frames) return fail(CB200_ERR_ARG, "n exceeds the context's max_frames");
    return CB200_OK;
}

// the context's CCM as the colour kernels take it; resolves the matrix a CC_SIMPLE batch left behind
int ccm_resolve(cb200_ctx* c)
{
    if (!c->ccm_pending) return CB200_OK;
    // the copies were enqueued on whatever stream was current then (cb200_set_stream may have changed it since)
    CK(cudaEventSynchronize(c->ccm_ev), "sync (ccm)");
    memcpy(c->ccm, c->h_ccm, sizeof(c->ccm));
    if (c->ccm_pending_flag) c->ccm_active = reinterpret_cast<const uint8_t*>(c->h_ccm + 9)[0] != 0;
    c->ccm_pending = c->ccm_pending_flag = false;
    return CB200_OK;
}
int ccm_arg(cb200_ctx* c, CcmArg& cc)
{
    memset(&cc, 0, sizeof(cc));
    int rc = ccm_resolve(c); if (rc) return rc;
    if (c->ccm_active) { cc.active = 1; memcpy(cc.m, c->ccm, sizeof(cc.m)); }
    return CB200_OK;
}

// the slot -> cell map of this call: Interleave::interleave_indices, or the identity for Decoder(use_ecc, interleave=false)
// (Interleave.h:10-16 with num_chunks == 0)
int idx_for(cb200_ctx* c, uint32_t flags, const uint16_t** out)
{
    *out = c->d_idx;
    if (!(flags & CB200_FLAG_NO_INTERLEAVE)) return CB200_OK;
    if (!c->d_idx_ident) {
        std::vector<uint16_t> id((size_t)c->mode.num_cells);
        for (size_t i = 0; i < id.size(); ++i) id[i] = (uint16_t)i;
        CK(c->d_idx_ident.ensure(id.size()), "cudaMalloc identity map");
        CK(cudaMemcpy(c->d_idx_ident, id.data(), id.size() * sizeof(uint16_t), cudaMemcpyHostToDevice), "upload identity map");
    }
    *out = c->d_idx_ident;
    return CB200_OK;
}

// the colour-correction buffers: the per-frame matrices and fits, and the last frame's matrix on its way to the host
int ccm_buffers(cb200_ctx* c)
{
    CK(c->d_ccm.ensure(9 * (size_t)c->max_frames), "cudaMalloc ccm");
    CK(c->d_carry.ensure(12), "cudaMalloc ccm carry");
    CK(c->h_ccm.ensure(12), "cudaMallocHost ccm");
    if (!c->ccm_ev) CK(cudaEventCreateWithFlags(&c->ccm_ev, cudaEventDisableTiming), "cudaEventCreate ccm");
    CK(c->d_fit.ensure(9 * (size_t)c->max_frames), "cudaMalloc fit");
    CK(c->d_fit_valid.ensure((size_t)c->max_frames), "cudaMalloc fit flags");
    return CB200_OK;
}

// the decoder keeps the CCM of the batch's last frame (CimbDecoder.cpp:82-85): its matrix in d_ccm -- and with d_active (CC_FIT)
// whether that frame had one at all -- goes to d_carry behind the batch (for the next batch enqueued before this one is done) and
// from there to h_ccm (for ccm_resolve)
int ccm_keep_last(cb200_ctx* c, int n, const uint8_t* d_active)
{
    uint8_t* d_flag = reinterpret_cast<uint8_t*>(c->d_carry + 9);
    CK(cudaMemcpyAsync(c->d_carry, c->d_ccm + 9 * (size_t)(n - 1), sizeof(float) * 9, cudaMemcpyDeviceToDevice, c->stream), "copy ccm");
    if (d_active) CK(cudaMemcpyAsync(d_flag, d_active + (n - 1), 1, cudaMemcpyDeviceToDevice, c->stream), "copy ccm flag");
    else CK(cudaMemsetAsync(d_flag, 1, 1, c->stream), "set ccm flag");
    CK(cudaMemcpyAsync(c->h_ccm, c->d_carry, sizeof(float) * 10, cudaMemcpyDeviceToHost, c->stream), "D2H ccm");
    CK(cudaEventRecord(c->ccm_ev, c->stream), "record ccm");
    c->ccm_pending = true; c->ccm_pending_flag = d_active != nullptr;
    if (!d_active) c->ccm_active = true;
    return CB200_OK;
}
// a chained CC_FIT call keeps the step's global exit instead (the same matrix on every rank of the chain): chain_settle writes it
// to d_carry, from there it goes to h_ccm as above
int ccm_keep_chain(cb200_ctx* c)
{
    int rc = chain_settle(c, c->d_carry); if (rc) return rc;
    CK(cudaMemcpyAsync(c->h_ccm, c->d_carry, sizeof(float) * 10, cudaMemcpyDeviceToHost, c->stream), "D2H ccm");
    CK(cudaEventRecord(c->ccm_ev, c->stream), "record ccm");
    c->ccm_pending = c->ccm_pending_flag = true;
    return CB200_OK;
}
// color_correction == 1: one matrix per frame of n frames in d_rgb into d_ccm, computed on the device before the colour pass
// (CimbReader.cpp:124-125); the last one becomes the context's CCM
int ccm_simple(cb200_ctx* c, const uint8_t* d_rgb, int n)
{
    int rc = ccm_buffers(c); if (rc) return rc;
    CK(ccm_simple_launch(c->mode, d_rgb, n, c->d_ccm, c->stream), "ccm launch");
    return ccm_keep_last(c, n, nullptr);
}

// the frame lists of a sharpen selection (cb200_ctx::d_sel): an order-preserving compaction of the n selection bytes in one CTA
// (every thread counts a contiguous segment, a block-wide scan of the counts gives each segment's first slot in both lists), the
// bytes rewritten as 0 / 1, and per list {count, K1 bands, first entry} in sched -- the band count is run_cells' rule for a grid
// of ctas[k] CTAs
__global__ void __launch_bounds__(1024)
k_select(uint8_t* __restrict__ sel, int n, int ctas0, int ctas1, int max_bands, int* __restrict__ sched)
{
    __shared__ int sums[1024];
    uint32_t* list = reinterpret_cast<uint32_t*>(sel);
    uint8_t* sharp = sel + (size_t)n * 4;
    const int t = threadIdx.x;
    const int seg = (n + 1023) / 1024, f0 = t * seg, f1 = min(f0 + seg, n);
    int mine = 0;
    for (int f = f0; f < f1; ++f) mine += sharp[f] != 0;
    sums[t] = mine;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {                  // inclusive scan of the sharpened counts
        const int v = t >= o ? sums[t - o] : 0;
        __syncthreads();
        sums[t] += v;
        __syncthreads();
    }
    const int n1 = sums[1023], n0 = n - n1;
    int at1 = sums[t] - mine, at0 = min(f0, n) - at1;     // sharpened / plain frames before this segment
    for (int f = f0; f < f1; ++f) {
        const bool k = sharp[f] != 0;
        if (k) list[n0 + at1++] = (uint32_t)f; else list[at0++] = (uint32_t)f;
        sharp[f] = k ? 1 : 0;
    }
    if (t < 2) {
        const int nk = t ? n1 : n0, ctas = t ? ctas1 : ctas0;
        int bands = 1;
        if (nk > 0 && nk < ctas) { bands = (ctas + nk - 1) / nk; if (bands > max_bands) bands = max_bands; if (bands < 1) bands = 1; }
        sched[3 * t] = nk; sched[3 * t + 1] = bands; sched[3 * t + 2] = t ? n0 : 0;
    }
}

// K1's persistent grid for one kind of frame (0 = plain, 1 = sharpened)
int k1_grid(const cb200_ctx* c, int k) { return c->sm_count * k1_ctas_per_sm(k == 1); }

// the frame lists of a selection whose n bytes (nonzero = sharpen) are in c->d_sel + 4 n, built there by k_select
int build_selection(cb200_ctx* c, int n)
{
    CK(c->d_sched.ensure(6), "cudaMalloc selection schedule");
    k_select<<<1, 1024, 0, c->stream>>>(c->d_sel, n, k1_grid(c, 0), k1_grid(c, 1), c->mode.cells_y / 4, c->d_sched); count_launch();
    CK(cudaGetLastError(), "selection launch");
    return CB200_OK;
}

// a mixed sharpen selection from the host: its n bytes go up through the context's pinned slots (stage_take), k_select builds the
// batch indices of the plain frames (d_list[0], nl[0] of them) and of the sharpened ones (d_list[1]), both in batch order, and
// one 0 / 1 byte per frame (d_sharp)
int upload_selection(cb200_ctx* c, const uint8_t* sel, int n, const int nl[2], const uint32_t* d_list[2], const uint8_t** d_sharp)
{
    CK(c->d_sel.ensure((size_t)c->max_frames * 5), "cudaMalloc selection");
    int slot;
    uint8_t* h;
    int rc = stage_take(c, (size_t)n, &slot, &h); if (rc) return rc;
    memcpy(h, sel, (size_t)n);
    rc = stage_send(c, slot, c->d_sel + (size_t)n * 4, (size_t)n, "H2D selection"); if (rc) return rc;
    rc = build_selection(c, n); if (rc) return rc;
    d_list[0] = reinterpret_cast<const uint32_t*>(c->d_sel.get());
    d_list[1] = d_list[0] + nl[0];
    *d_sharp = c->d_sel + (size_t)n * 4;
    return CB200_OK;
}

// K1 (+ exact-walk fallback) : frames -> per-cell bytes in ctx->d_cellvals, per-frame flags in ctx->d_flags.
// d_means != nullptr: first pass of a CC_FIT batch -- no colour decisions, the cells' mean colours go to d_means.
// sel: NULL = every frame is preprocessed as CB200_FLAG_SHARPEN says; else n host bytes, nonzero = sharpen that frame (flags
// must not carry CB200_FLAG_SHARPEN then).  A selection of one kind only takes the list-less path of that kind.
// d_sel_bytes (instead of sel): the selection is n bytes at c->d_sel + 4 n on the device; the lists are built there and K1 takes
// their lengths from the device (both kinds are launched, one may be empty)
int run_cells(cb200_ctx* c, const uint8_t* d_rgb, int n, uint32_t flags, const uint8_t* sel, CellTrace* d_trace = nullptr,
              uint32_t* d_means = nullptr, const uint8_t* d_sel_bytes = nullptr)
{
    const Mode& m = c->mode;
    cudaStream_t st = c->stream;
    CcmArg cc;
    if (d_means) {
        memset(&cc, 0, sizeof(cc));
        cc.means = d_means;
    } else if ((flags & CB200_FLAG_CC_SIMPLE) && n > 0) {
        int rcb = ccm_simple(c, d_rgb, n); if (rcb) return rcb;
        memset(&cc, 0, sizeof(cc));
        cc.per_frame = c->d_ccm; cc.active = 1;
    } else {
        int rc = ccm_arg(c, cc); if (rc) return rc;
    }
    bool sharpen = (flags & CB200_FLAG_SHARPEN) != 0;
    const bool exact_only = d_trace != nullptr;   // a cell trace needs the walk itself
    // nl[k] frames of kind k (0 = plain, 1 = sharpened), listed in d_list[k] (NULL: all n frames of the batch)
    int nl[2] = {sharpen ? 0 : n, sharpen ? n : 0};
    const uint32_t* d_list[2] = {nullptr, nullptr};
    const uint8_t* d_sharp = nullptr;
    const int* d_sched = nullptr;
    if (d_sel_bytes) {
        int rc = build_selection(c, n); if (rc) return rc;
        d_list[0] = d_list[1] = reinterpret_cast<const uint32_t*>(c->d_sel.get());
        d_sharp = d_sel_bytes;
        d_sched = c->d_sched;
        nl[0] = nl[1] = 1;                     // launched whatever the device counts are
    } else if (sel) {
        nl[1] = 0;
        for (int f = 0; f < n; ++f) nl[1] += sel[f] != 0;
        nl[0] = n - nl[1];
        sharpen = nl[1] == n;
        if (nl[0] && nl[1]) { int rc = upload_selection(c, sel, n, nl, d_list, &d_sharp); if (rc) return rc; }
    }
    CK(cudaMemsetAsync(c->d_dirty, 0, sizeof(uint32_t) * (size_t)n, st), "memset dirty");
    begin_timed_call(c);
    mark(c);                                   // ev0: before K1
    for (int k = 0; k < 2 && !exact_only; ++k) {
        const int nk = nl[k];
        if (nk == 0) continue;
        // bands: whole frames when there are enough of them to fill the machine, else split frames into bands of cell rows
        // (k_select applies the same rule on the device)
        int ctas = k1_grid(c, k);
        int bands = 1;
        if (nk < ctas) { bands = (ctas + nk - 1) / nk; if (bands > m.cells_y / 4) bands = m.cells_y / 4; if (bands < 1) bands = 1; }
        int units = nk * bands;
        int grid = d_sched || units > ctas ? ctas : units;
        CK(k1_launch(m, d_rgb, d_list[k], nk, bands, grid, k == 1, c->d_cellvals, c->d_dirty, cc, st, d_sched ? d_sched + 3 * k : nullptr),
           "k1 launch");
    }
    mark(c);                                   // ev1: after K1
    // frames K1 flagged (or all of them when exact_only) are re-done by the exact walk on the same preprocessing (sharpen or not)
    CK(flood_launch(m, c->flood, d_rgb, n, (flags & CB200_FLAG_NO_FALLBACK) != 0, exact_only, sharpen, d_sharp,
                    c->d_cellvals, c->d_dirty, c->d_flags, d_trace, cc, st), "flood launch");
    mark(c);                                   // ev2: after K1x
    return CB200_OK;
}

}  // namespace

namespace cb200 {
// init_ccm is only reached from Decoder::do_decode (not the legacy coupled layout) and needs a header from the RS stream
bool ccm_fits(const Mode& m, uint32_t flags) { return (flags & CB200_FLAG_CC_FIT) && !m.legacy && m.ecc_bytes > 0 && m.color_bits > 0; }

int flood_reserve(cb200_ctx* c, int n)
{
    if (flood_workspace_fits(c->flood, n)) return CB200_OK;
    if (!c->plans.empty()) return plan_frozen(c, "exact walk workspace", (size_t)c->flood.entry_cap, (size_t)n);
    CK(flood_workspace_ensure(c->mode, c->flood, n), "cudaMalloc exact walk workspace");
    return CB200_OK;
}

int decode_reserve(cb200_ctx* c, uint32_t flags)
{
    int rc = ccm_buffers(c); if (rc) return rc;
    CK(c->d_means.ensure((size_t)c->max_frames * c->mode.num_cells), "cudaMalloc means");
    CK(c->d_ccm_active.ensure((size_t)c->max_frames), "cudaMalloc ccm flags");
    CK(c->d_sel.ensure((size_t)c->max_frames * 5), "cudaMalloc selection");
    CK(c->d_sched.ensure(6), "cudaMalloc selection schedule");
    const uint16_t* idx;
    return idx_for(c, flags, &idx);
}

int carry_from_host(cb200_ctx* c)
{
    if (c->plans.empty()) return CB200_OK;
    float v[10] = {};
    if (c->ccm_active) memcpy(v, c->ccm, sizeof(c->ccm));
    reinterpret_cast<uint8_t*>(v + 9)[0] = c->ccm_active ? 1 : 0;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    // from pageable memory: the copy is staged before the call returns
    CK(cudaMemcpyAsync(c->d_carry, v, sizeof(v), cudaMemcpyHostToDevice, c->stream), "H2D ccm carry");
    return CB200_OK;
}
}  // namespace cb200

int upload_frames(cb200_ctx* c, const uint8_t* rgb, int n)
{
    const Mode& m = c->mode;
    size_t fb = (size_t)m.width * m.height * 3;
    CK(c->d_rgb.ensure(fb * (size_t)c->max_frames), "cudaMalloc rgb staging");
    CK(cudaMemcpyAsync(c->d_rgb, rgb, fb * (size_t)n, cudaMemcpyHostToDevice, c->stream), "H2D frames");
    return CB200_OK;
}


extern "C" {

const char* cb200_last_error(void) { return g_err.c_str(); }
int cb200_version(void) { return 2; }
unsigned long long cb200_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

int cb200_mode_info(int mode_val, cb200_info* out)
{
    if (!out) return fail(CB200_ERR_ARG, "null out");
    Mode m;
    if (!mode_init(m, mode_val)) return fail(CB200_ERR_MODE, "unsupported mode_val");
    fill_info(m, 0, 0, out);
    return CB200_OK;
}

int cb200_selfcheck(int mode_val)
{
    Mode m;
    if (!mode_init(m, mode_val)) return fail(CB200_ERR_MODE, "unsupported mode_val");
    std::vector<uint16_t> adj;
    build_adjacency(m, adj);
    if (!adjacency_consistent(m, adj)) return fail(CB200_ERR_MODE, "adjacency self-check failed");
    return CB200_OK;
}

int cb200_interleave_indices(int mode_val, uint16_t* idx)
{
    if (!idx) return fail(CB200_ERR_ARG, "null idx");
    Mode m;
    if (!mode_init(m, mode_val)) return fail(CB200_ERR_MODE, "unsupported mode_val");
    std::vector<uint16_t> v;
    interleave_indices(m, v);
    memcpy(idx, v.data(), v.size() * sizeof(uint16_t));
    return CB200_OK;
}

// everything of cb200_create that can fail after the context object exists: the caller destroys `c` on any error
static int create_impl(cb200_ctx* c, int device, int mode_val, int max_frames)
{
    if (!mode_init(c->mode, mode_val)) return fail(CB200_ERR_MODE, "unsupported mode_val");
    const Mode& m = c->mode;
    c->device = device; c->max_frames = max_frames;
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, device), "cudaGetDeviceProperties");
    if (prop.major != 9 || prop.minor != 0) return fail(CB200_ERR_NODEVICE, "libcb200 is built for sm_90a (compute capability 9.0) only");
    c->sm_count = prop.multiProcessorCount;
    CK(cudaStreamCreateWithFlags(&c->own_stream, cudaStreamNonBlocking), "cudaStreamCreate");
    c->stream = c->own_stream;

    // ---- tables
    float adjust[256];
    adjust[0] = 0.0f;
    for (int d = 1; d < 256; ++d) adjust[d] = (float)(255.0 / (double)(float)d);   // CimbDecoder.cpp:185
    unsigned long long tilesL[16];
    for (int t = 0; t < 16; ++t) tilesL[t] = brev64(kTilesH[t]);
    CK(k1_init_tables(adjust, tilesL), "k1 tables");
    CK(render_init_tables(kTilesH), "render tables");
    uint8_t gexp[512], glog[256];
    {   // GF(2^8), primitive polynomial 0x187 (ReedSolomon.h:26; libcorrect field.h:26-62)
        unsigned el = 1; gexp[0] = 1; glog[0] = 0;
        for (unsigned i = 1; i < 512; ++i) {
            el *= 2; if (el > 255) el ^= 0x187u;
            gexp[i] = (uint8_t)el;
            if (i < 256) glog[el] = (uint8_t)i;
        }
    }
    CK(k2_init_tables(gexp, glog), "k2 tables");
    CK(flood_init_tables(adjust, tilesL, m.hash_mul), "flood tables");

    // ---- workspaces
    size_t n = (size_t)max_frames;
    CK(c->d_cellvals.ensure(n * m.num_cells), "cudaMalloc cellvals");
    CK(c->d_dirty.ensure(n), "cudaMalloc dirty");
    CK(c->d_raw.ensure(n * m.cap_all + 16), "cudaMalloc raw");
    CK(c->d_data.ensure(n * m.data_bytes), "cudaMalloc data");
    CK(c->d_ok.ensure(n * m.nblocks), "cudaMalloc ok");
    CK(c->d_mask.ensure(n), "cudaMalloc mask");
    CK(c->d_flags.ensure(n), "cudaMalloc flags");
    std::vector<uint16_t> idx;
    interleave_indices(m, idx);
    CK(c->d_idx.ensure(idx.size()), "cudaMalloc idx");
    CK(cudaMemcpy(c->d_idx, idx.data(), idx.size() * sizeof(uint16_t), cudaMemcpyHostToDevice), "upload idx");
    {
        std::vector<uint16_t> inv(idx.size());
        for (size_t sidx = 0; sidx < idx.size(); ++sidx) inv[idx[sidx]] = (uint16_t)sidx;
        CK(c->d_inv.ensure(inv.size()), "cudaMalloc inv");
        CK(cudaMemcpy(c->d_inv, inv.data(), inv.size() * sizeof(uint16_t), cudaMemcpyHostToDevice), "upload inv");
        // generator polynomial prod_{i=1..parity} (x + alpha^i) (libcorrect reed-solomon.c:5-12, polynomial.c:215-262)
        std::vector<uint8_t> g(1, 1);
        auto mul = [&](uint8_t a, uint8_t b) -> uint8_t { return (a && b) ? gexp[glog[a] + glog[b]] : 0; };
        for (int i = 1; i <= m.ecc_bytes; ++i) {
            uint8_t root = gexp[i % 255];
            std::vector<uint8_t> ng(g.size() + 1, 0);
            for (size_t k = 0; k < g.size(); ++k) { ng[k + 1] ^= g[k]; ng[k] ^= mul(g[k], root); }
            g.swap(ng);
        }
        CK(c->d_gen.ensure(g.size()), "cudaMalloc gen");
        CK(cudaMemcpy(c->d_gen, g.data(), g.size(), cudaMemcpyHostToDevice), "upload gen");
        uint8_t rho[4 * 64];
        k2_remainder_basis(g.data(), m.ecc_bytes, gexp, glog, rho);
        CK(c->d_rho.ensure(sizeof(rho)), "cudaMalloc rho");
        CK(cudaMemcpy(c->d_rho, rho, sizeof(rho), cudaMemcpyHostToDevice), "upload rho");
        CK(encode_init_tables(gexp, glog), "encode tables");
    }
    {
        std::vector<uint16_t> adj;
        build_adjacency(m, adj);
        if (!adjacency_consistent(m, adj)) return fail(CB200_ERR_MODE, "adjacency self-check failed");
        CK(flood_workspace_create(m, c->sm_count, adj.data(), &c->flood), "flood workspace");
    }
    return CB200_OK;
}

int cb200_create(cb200_ctx** out, int device, int mode_val, int max_frames)
{
    if (!out || max_frames < 1) return fail(CB200_ERR_ARG, "bad arguments");
    *out = nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
        return fail(CB200_ERR_NODEVICE, "no CUDA device: libcb200 has no CPU fallback");
    if (device < 0) { CK(cudaGetDevice(&device), "cudaGetDevice"); }
    if (device >= ndev) return fail(CB200_ERR_ARG, "device index out of range");
    CK(cudaSetDevice(device), "cudaSetDevice");
    cb200_ctx* c = new cb200_ctx();
    c->device = device;
    int rc = create_impl(c, device, mode_val, max_frames);
    if (rc != CB200_OK) {            // one cleanup path: whatever was allocated so far is released (cb200_last_error keeps the cause)
        std::string why = cb200_last_error();
        cb200_destroy(c);
        return fail(rc, why);
    }
    *out = c;
    return CB200_OK;
}

int cb200_destroy(cb200_ctx* c)
{
    if (!c) return CB200_OK;
    while (!c->plans.empty()) cb200_camera_plan_destroy(c->plans.back());
    cudaSetDevice(c->device);          // the buffers free themselves in `delete c`, on this device
    for (int k = 0; k < cb200_ctx::kEvSets; ++k) for (int i = 0; i < 8; ++i) if (c->ev[k][i]) cudaEventDestroy(c->ev[k][i]);
    for (const auto& s : c->stage) if (s.ev) cudaEventDestroy(s.ev);
    if (c->ccm_ev) cudaEventDestroy(c->ccm_ev);
    gather_destroy(c->gather);
    chain_destroy(c->chain);
    deskew_destroy(c->deskew); scan_destroy(c->scan); jpeg_destroy(c->jpeg); png_destroy(c->png);
    if (c->own_stream) cudaStreamDestroy(c->own_stream);
    delete c;
    return CB200_OK;
}

int cb200_get_info(const cb200_ctx* c, cb200_info* out)
{
    if (!c || !out) return fail(CB200_ERR_ARG, "null argument");
    fill_info(c->mode, c->max_frames, c->sm_count, out);
    return CB200_OK;
}

int cb200_set_stream(cb200_ctx* c, void* cuda_stream)
{
    if (!c) return fail(CB200_ERR_ARG, "null context");
    c->stream = cuda_stream ? (cudaStream_t)cuda_stream : c->own_stream;
    return CB200_OK;
}

int cb200_sync(cb200_ctx* c)
{
    if (!c) return fail(CB200_ERR_ARG, "null context");
    CK(cudaStreamSynchronize(c->stream), "cudaStreamSynchronize");
    return CB200_OK;
}

int cb200_decode_raw_dev(cb200_ctx* c, const uint8_t* d_rgb, int n, uint32_t flags, uint8_t* d_raw_out, uint8_t* d_frame_flags)
{
    int rc = check_frame_flags(flags); if (rc) return rc;
    rc = check_n(c, n); if (rc) return rc;
    if (n == 0) return CB200_OK;
    if (!d_rgb || !d_raw_out) return fail(CB200_ERR_ARG, "null buffer");
    rc = check_frozen_frames(c, n); if (rc) return rc;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    const uint16_t* idx;
    rc = idx_for(c, flags, &idx); if (rc) return rc;
    rc = run_cells(c, d_rgb, n, flags, nullptr); if (rc) return rc;
    CK(k2_pack_launch(c->mode, c->d_cellvals, idx, n, d_raw_out, c->stream), "pack launch");
    mark(c);                                   // ev3: after pack
    if (d_frame_flags) CK(cudaMemcpyAsync(d_frame_flags, c->d_flags, (size_t)n, cudaMemcpyDeviceToDevice, c->stream), "copy flags");
    return CB200_OK;
}

int cb200_rs_correct_dev(cb200_ctx* c, const uint8_t* d_raw, int n, uint8_t* d_data_out, uint8_t* d_block_ok)
{
    int rc = check_n(c, n); if (rc) return rc;
    if (n == 0) return CB200_OK;
    if (!d_raw || !d_data_out) return fail(CB200_ERR_ARG, "null buffer");
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    uint8_t* ok = d_block_ok ? d_block_ok : c->d_ok;
    CK(k2_rs_launch(c->mode, d_raw, n, d_data_out, ok, c->d_rho, c->sm_count, c->stream), "rs launch");
    return CB200_OK;
}

}  // extern "C"

namespace {
// cb200_decode_chunks_dev with an optional per-frame selection (run_cells: sharpen on the host, or d_sel_bytes on the device).
// enqueue_only: a CCM still on its way from an earlier batch (ccm_keep_last) is not waited for but read
// from c->d_carry on the device -- through k_ccm_carry, so a batch without a fit then takes the fitted-CCM route with no fits
// (mean colours, carry, colour decisions), which decides every colour as K1 would with that matrix or without one
int decode_chunks(cb200_ctx* c, const uint8_t* d_rgb, int n, uint32_t flags, const uint8_t* sharpen, uint8_t* d_chunks,
                  uint32_t* d_chunk_mask, uint8_t* d_frame_flags, const uint8_t* d_sel_bytes = nullptr, bool enqueue_only = false)
{
    int rc = check_n(c, n); if (rc) return rc;
    // a chained CC_FIT call takes part in the step even with no frames: an empty stripe publishes "no fit" and settles
    const bool chained = chain_linked(c, flags);
    if (n == 0 && !chained) return CB200_OK;
    if ((flags & CB200_FLAG_CC_FIT) && (flags & CB200_FLAG_CC_SIMPLE)) return fail(CB200_ERR_ARG, "CC_SIMPLE and CC_FIT are exclusive");
    rc = check_chain_call(c, flags); if (rc) return rc;
    if (n > 0 && (!d_rgb || !d_chunks || !d_chunk_mask)) return fail(CB200_ERR_ARG, "null buffer");
    rc = check_frozen_frames(c, n); if (rc) return rc;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    const Mode& m = c->mode;
    const bool fit = ccm_fits(m, flags);
    // the CCM going into frame 0 is only known on the device -- always so for a camera plan, whose graph replays later
    bool carried = enqueue_only && !(flags & CB200_FLAG_CC_SIMPLE) && c->capturing;
    if (enqueue_only && !(flags & CB200_FLAG_CC_SIMPLE) && c->ccm_pending && !carried) {
        const cudaError_t q = cudaEventQuery(c->ccm_ev);
        if (q == cudaErrorNotReady) carried = true;
        else if (q != cudaSuccess) return fail_cuda(q, "query ccm");
    }
    if (n == 0) {                              // chained, empty stripe
        rc = ccm_buffers(c); if (rc) return rc;
        CcmArg own;
        if (carried) {
            memset(&own, 0, sizeof(own));
            own.per_frame = c->d_carry;
            own.per_frame_active = reinterpret_cast<const uint8_t*>(c->d_carry + 9);
        } else {
            rc = ccm_arg(c, own); if (rc) return rc;
        }
        rc = chain_publish_link(c, 0, nullptr, nullptr, own, nullptr); if (rc) return rc;
        c->ccm_frames = 0;
        return ccm_keep_chain(c);
    }
    const uint16_t* idx;
    rc = idx_for(c, flags, &idx); if (rc) return rc;
    if (!fit && !carried && !chained) {
        rc = run_cells(c, d_rgb, n, flags & ~CB200_FLAG_CC_FIT, sharpen, nullptr, nullptr, d_sel_bytes); if (rc) return rc;
        mark(c);                               // ev3: (no separate pack kernel on this path: the RS kernel gathers from the cell bytes)
        CK(k2_rs_fused_launch(m, c->d_cellvals, idx, n, d_chunks, c->d_ok, c->d_rho, c->sm_count, c->stream), "rs launch");
    } else {
        // color_correction == 2: symbols (+ mean colours) -> RS of the symbol stream -> header -> CCM fit -> colours -> RS of
        // the colour stream (Decoder.h:83-117)
        rc = ccm_buffers(c); if (rc) return rc;
        CK(c->d_means.ensure((size_t)c->max_frames * m.num_cells), "cudaMalloc means");
        CK(c->d_ccm_active.ensure((size_t)c->max_frames), "cudaMalloc ccm flags");
        CcmArg initial;                        // the decoder's CCM going into frame 0
        if (carried) {
            memset(&initial, 0, sizeof(initial));
            initial.per_frame = c->d_carry;
            initial.per_frame_active = reinterpret_cast<const uint8_t*>(c->d_carry + 9);
        } else {
            rc = ccm_arg(c, initial); if (rc) return rc;
        }
        rc = run_cells(c, d_rgb, n, flags & ~(CB200_FLAG_CC_FIT | CB200_FLAG_CC_SIMPLE), sharpen, nullptr, c->d_means, d_sel_bytes); if (rc) return rc;
        mark(c);                               // ev3
        if (fit) {
            CK(k2_rs_fused_launch(m, c->d_cellvals, idx, n, d_chunks, c->d_ok, c->d_rho, c->sm_count, c->stream, 0, m.nblocks_sym), "rs launch (symbols)");
            CK(ccm_fit_launch(m, d_rgb, d_chunks, c->d_ok, idx, n, c->d_fit, c->d_fit_valid, c->stream), "ccm fit");
        } else {
            CK(cudaMemsetAsync(c->d_fit_valid, 0, (size_t)n, c->stream), "memset fit flags");
        }
        // across ranks: this stripe's fits out, the CCM entering the stripe in (from the lower ranks' fits of the same step)
        if (chained) { rc = chain_publish_link(c, n, c->d_fit, c->d_fit_valid, initial, &initial); if (rc) return rc; }
        CK(ccm_carry_launch(n, c->d_fit, c->d_fit_valid, initial, c->d_ccm, c->d_ccm_active, c->stream), "ccm carry");
        CK(ccm_apply_launch(m, c->d_means, n, c->d_ccm, c->d_ccm_active, c->d_cellvals, c->stream), "ccm apply");
        c->ccm_frames = n;
        if (fit) {
            CK(k2_rs_fused_launch(m, c->d_cellvals, idx, n, d_chunks, c->d_ok, c->d_rho, c->sm_count, c->stream, m.nblocks_sym, m.nblocks - m.nblocks_sym),
               "rs launch (colours)");
        } else {
            CK(k2_rs_fused_launch(m, c->d_cellvals, idx, n, d_chunks, c->d_ok, c->d_rho, c->sm_count, c->stream), "rs launch");
        }
        if (chained) { rc = ccm_keep_chain(c); if (rc) return rc; }
        else if (fit) { rc = ccm_keep_last(c, n, c->d_ccm_active); if (rc) return rc; }
    }
    mark(c);                                   // ev4: after RS
    CK(k2_mask_launch(m, c->d_ok, n, d_chunk_mask, c->stream), "mask launch");
    mark(c);                                   // ev5: after chunk mask
    if (d_frame_flags) CK(cudaMemcpyAsync(d_frame_flags, c->d_flags, (size_t)n, cudaMemcpyDeviceToDevice, c->stream), "copy flags");
    return CB200_OK;
}
}  // namespace

extern "C" {

int cb200_decode_chunks_dev(cb200_ctx* c, const uint8_t* d_rgb, int n, uint32_t flags, uint8_t* d_chunks, uint32_t* d_chunk_mask, uint8_t* d_frame_flags)
{
    int rc = check_frame_flags(flags); if (rc) return rc;
    return decode_chunks(c, d_rgb, n, flags, nullptr, d_chunks, d_chunk_mask, d_frame_flags);
}

int cb200_decode_chunks_sharpen_dev(cb200_ctx* c, const uint8_t* d_rgb, int n, uint32_t flags, const uint8_t* sharpen, uint8_t* d_chunks,
                                    uint32_t* d_chunk_mask, uint8_t* d_frame_flags)
{
    int rc = check_selection_args(flags, sharpen); if (rc) return rc;
    return decode_chunks(c, d_rgb, n, flags, sharpen, d_chunks, d_chunk_mask, d_frame_flags);
}

// ---- host-pointer entry points
int cb200_decode_raw(cb200_ctx* c, const uint8_t* rgb, int n, uint32_t flags, uint8_t* raw_out, uint8_t* frame_flags)
{
    int rc = check_frame_flags(flags); if (rc) return rc;
    rc = check_n(c, n); if (rc) return rc;
    if (n == 0) return CB200_OK;
    if (!rgb || !raw_out) return fail(CB200_ERR_ARG, "null buffer");
    rc = check_frozen_frames(c, n); if (rc) return rc;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    rc = upload_frames(c, rgb, n); if (rc) return rc;
    rc = cb200_decode_raw_dev(c, c->d_rgb, n, flags, c->d_raw, nullptr); if (rc) return rc;
    CK(cudaMemcpyAsync(raw_out, c->d_raw, (size_t)n * c->mode.cap_all, cudaMemcpyDeviceToHost, c->stream), "D2H raw");
    if (frame_flags) CK(cudaMemcpyAsync(frame_flags, c->d_flags, (size_t)n, cudaMemcpyDeviceToHost, c->stream), "D2H flags");
    CK(cudaStreamSynchronize(c->stream), "sync");
    return CB200_OK;
}

int cb200_decode(cb200_ctx* c, const uint8_t* rgb, int n, uint32_t flags, uint8_t* data_out, uint8_t* block_ok, uint8_t* frame_flags)
{
    int rc = check_frame_flags(flags); if (rc) return rc;
    rc = check_n(c, n); if (rc) return rc;
    rc = check_chain_call(c, flags); if (rc) return rc;
    if (n == 0) return chain_linked(c, flags) ? decode_chunks(c, nullptr, 0, flags, nullptr, nullptr, nullptr, nullptr) : CB200_OK;
    if (!rgb || !data_out) return fail(CB200_ERR_ARG, "null buffer");
    rc = check_frozen_frames(c, n); if (rc) return rc;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    rc = upload_frames(c, rgb, n); if (rc) return rc;
    rc = cb200_decode_chunks_dev(c, c->d_rgb, n, flags, c->d_data, c->d_mask, nullptr); if (rc) return rc;
    CK(cudaMemcpyAsync(data_out, c->d_data, (size_t)n * c->mode.data_bytes, cudaMemcpyDeviceToHost, c->stream), "D2H data");
    if (block_ok) CK(cudaMemcpyAsync(block_ok, c->d_ok, (size_t)n * c->mode.nblocks, cudaMemcpyDeviceToHost, c->stream), "D2H ok");
    if (frame_flags) CK(cudaMemcpyAsync(frame_flags, c->d_flags, (size_t)n, cudaMemcpyDeviceToHost, c->stream), "D2H flags");
    CK(cudaStreamSynchronize(c->stream), "sync");
    return CB200_OK;
}

}  // extern "C"

namespace {
// the host-pointer fountain entry points: H2D of the frames, then the device-frame path
int decode_fountain_from_host(cb200_ctx* c, const uint8_t* rgb, int n, uint32_t flags, const uint8_t* sharpen, uint8_t* chunks_out,
                              uint32_t* chunk_count, uint32_t* chunk_mask, uint8_t* frame_flags)
{
    int rc = check_n(c, n); if (rc) return rc;
    rc = check_chain_call(c, flags); if (rc) return rc;
    if (n == 0) return chain_linked(c, flags) ? decode_chunks(c, nullptr, 0, flags, nullptr, nullptr, nullptr, nullptr) : CB200_OK;
    if (!rgb || !chunks_out || !chunk_count) return fail(CB200_ERR_ARG, "null buffer");
    rc = check_frozen_frames(c, n); if (rc) return rc;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    rc = upload_frames(c, rgb, n); if (rc) return rc;
    return decode_fountain_to_host(c, c->d_rgb, n, flags, sharpen, chunks_out, chunk_count, chunk_mask, frame_flags);
}
}  // namespace

// frames already on the device (the staging buffer, or the deskew kernel's output), results to host memory
int cb200::decode_fountain_to_host(cb200_ctx* c, const uint8_t* d_rgb, int n, uint32_t flags, const uint8_t* sharpen, uint8_t* chunks_out,
                                   uint32_t* chunk_count, uint32_t* chunk_mask, uint8_t* frame_flags)
{
    int rc = check_n(c, n); if (rc) return rc;
    rc = check_chain_call(c, flags); if (rc) return rc;
    if (n == 0) return chain_linked(c, flags) ? decode_chunks(c, nullptr, 0, flags, nullptr, nullptr, nullptr, nullptr) : CB200_OK;
    if (!d_rgb || !chunks_out || !chunk_count) return fail(CB200_ERR_ARG, "null buffer");
    rc = check_frozen_frames(c, n); if (rc) return rc;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    rc = decode_chunks(c, d_rgb, n, flags, sharpen, c->d_data, c->d_mask, nullptr); if (rc) return rc;
    return fetch_fountain(c, n, nullptr, chunks_out, chunk_count, chunk_mask, frame_flags, nullptr);
}

int cb200::decode_chunks_enqueue(cb200_ctx* c, const uint8_t* d_rgb, int n, uint32_t flags, const uint8_t* d_sharp, uint8_t* d_chunks,
                                 uint32_t* d_chunk_mask, uint8_t* d_frame_flags)
{
    return decode_chunks(c, d_rgb, n, flags, nullptr, d_chunks, d_chunk_mask, d_frame_flags, d_sharp, true);
}

int cb200::fetch_fountain(cb200_ctx* c, int n, const int32_t* d_status, uint8_t* chunks_out, uint32_t* chunk_count, uint32_t* chunk_mask,
                          uint8_t* frame_flags, int32_t* extract_status)
{
    const Mode& m = c->mode;
    CK(c->h_pinned.ensure((size_t)n * m.data_bytes + (size_t)n * sizeof(uint32_t)), "cudaMallocHost");
    uint32_t* h_mask = reinterpret_cast<uint32_t*>(c->h_pinned.get());
    uint8_t* h_data = c->h_pinned + (size_t)n * sizeof(uint32_t);
    CK(cudaMemcpyAsync(h_data, c->d_data, (size_t)n * m.data_bytes, cudaMemcpyDeviceToHost, c->stream), "D2H chunks");
    CK(cudaMemcpyAsync(h_mask, c->d_mask, (size_t)n * sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream), "D2H mask");
    if (frame_flags) CK(cudaMemcpyAsync(frame_flags, c->d_flags, (size_t)n, cudaMemcpyDeviceToHost, c->stream), "D2H flags");
    if (d_status) CK(cudaMemcpyAsync(extract_status, d_status, sizeof(int32_t) * (size_t)n, cudaMemcpyDeviceToHost, c->stream), "D2H status");
    CK(cudaStreamSynchronize(c->stream), "sync");
    // escrow_buffer_writer order: good chunks appended densely (src/lib/encoder/escrow_buffer_writer.h:44-60)
    for (int f = 0; f < n; ++f) {
        uint8_t* dst = chunks_out + (size_t)f * m.data_bytes;
        const uint8_t* src = h_data + (size_t)f * m.data_bytes;
        uint32_t cnt = 0;
        for (int q = 0; q < m.chunks_per_frame; ++q)
            if (h_mask[f] & (1u << q)) { memcpy(dst + (size_t)cnt * m.chunk_size, src + (size_t)q * m.chunk_size, (size_t)m.chunk_size); ++cnt; }
        chunk_count[f] = cnt;
        if (chunk_mask) chunk_mask[f] = h_mask[f];
    }
    return CB200_OK;
}

extern "C" {

int cb200_decode_fountain(cb200_ctx* c, const uint8_t* rgb, int n, uint32_t flags, uint8_t* chunks_out, uint32_t* chunk_count,
                          uint32_t* chunk_mask, uint8_t* frame_flags)
{
    int rc = check_frame_flags(flags); if (rc) return rc;
    return decode_fountain_from_host(c, rgb, n, flags, nullptr, chunks_out, chunk_count, chunk_mask, frame_flags);
}

int cb200_decode_fountain_sharpen(cb200_ctx* c, const uint8_t* rgb, int n, uint32_t flags, const uint8_t* sharpen, uint8_t* chunks_out,
                                  uint32_t* chunk_count, uint32_t* chunk_mask, uint8_t* frame_flags)
{
    int rc = check_selection_args(flags, sharpen); if (rc) return rc;
    return decode_fountain_from_host(c, rgb, n, flags, sharpen, chunks_out, chunk_count, chunk_mask, frame_flags);
}

int cb200_decode_fountain_from_dev(cb200_ctx* c, const uint8_t* d_rgb, int n, uint32_t flags, uint8_t* chunks_out, uint32_t* chunk_count,
                                   uint32_t* chunk_mask, uint8_t* frame_flags)
{
    int rc = check_frame_flags(flags); if (rc) return rc;
    return decode_fountain_to_host(c, d_rgb, n, flags, nullptr, chunks_out, chunk_count, chunk_mask, frame_flags);
}

int cb200_decode_cells(cb200_ctx* c, const uint8_t* rgb, int n, uint32_t flags, uint8_t* cellvals_out, cb200_cell_trace* trace_out)
{
    return cb200_decode_cells_means(c, rgb, n, flags, cellvals_out, trace_out, nullptr);
}

int cb200_decode_cells_means(cb200_ctx* c, const uint8_t* rgb, int n, uint32_t flags, uint8_t* cellvals_out, cb200_cell_trace* trace_out,
                             uint32_t* means_out)
{
    int rc = check_frame_flags(flags); if (rc) return rc;
    rc = check_n(c, n); if (rc) return rc;
    if (n == 0) return CB200_OK;
    if (!rgb || !cellvals_out || !trace_out) return fail(CB200_ERR_ARG, "null buffer");
    static_assert(sizeof(cb200_cell_trace) == sizeof(CellTrace), "trace layout");
    rc = check_frozen_frames(c, n); if (rc) return rc;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    rc = upload_frames(c, rgb, n); if (rc) return rc;
    size_t tb = (size_t)n * c->mode.num_cells * sizeof(CellTrace);
    size_t mb = means_out ? (size_t)n * c->mode.num_cells * sizeof(uint32_t) : 0;
    CK(c->d_scratch.ensure(tb + mb), "cudaMalloc scratch");
    CellTrace* d_trace = reinterpret_cast<CellTrace*>(c->d_scratch.get());
    uint32_t* d_means = means_out ? reinterpret_cast<uint32_t*>(c->d_scratch + tb) : nullptr;
    // with means_out the colours are not decided here (the caller classifies the means later, with whatever CCM its decoder
    // holds by then: CimbReader::read_color after init_ccm); CC_SIMPLE still installs the frame's matrix as the context's CCM
    if (d_means && (flags & CB200_FLAG_CC_SIMPLE)) { rc = ccm_simple(c, c->d_rgb, n); if (rc) return rc; }
    rc = run_cells(c, c->d_rgb, n, flags & ~(CB200_FLAG_NO_FALLBACK | (d_means ? CB200_FLAG_CC_SIMPLE : 0u)), nullptr, d_trace, d_means); if (rc) return rc;
    if (means_out) CK(cudaMemcpyAsync(means_out, d_means, mb, cudaMemcpyDeviceToHost, c->stream), "D2H means");
    CK(cudaMemcpyAsync(cellvals_out, c->d_cellvals, (size_t)n * c->mode.num_cells, cudaMemcpyDeviceToHost, c->stream), "D2H cells");
    CK(cudaMemcpyAsync(trace_out, d_trace, tb, cudaMemcpyDeviceToHost, c->stream), "D2H trace");
    CK(cudaStreamSynchronize(c->stream), "sync");
    return CB200_OK;
}

int cb200_decode_symbols(cb200_ctx* c, const uint16_t* windows, const uint8_t* cooldown, int n, uint8_t* symbol, uint8_t* drift_offset, uint8_t* distance)
{
    if (!c || !windows || !symbol || !drift_offset || !distance || n < 0) return fail(CB200_ERR_ARG, "bad arguments");
    if (n == 0) return CB200_OK;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    size_t wb = (size_t)n * 10 * sizeof(uint16_t);
    CK(c->d_scratch.ensure(wb + 4 * (size_t)n + 64), "cudaMalloc scratch");
    uint8_t* base = c->d_scratch;
    uint16_t* d_win = reinterpret_cast<uint16_t*>(base);
    uint8_t* d_cd = base + wb; uint8_t* d_sym = d_cd + n; uint8_t* d_off = d_sym + n; uint8_t* d_dist = d_off + n;
    CK(cudaMemcpyAsync(d_win, windows, wb, cudaMemcpyHostToDevice, c->stream), "H2D windows");
    if (cooldown) CK(cudaMemcpyAsync(d_cd, cooldown, (size_t)n, cudaMemcpyHostToDevice, c->stream), "H2D cooldown");
    CK(k1_symbols_launch(d_win, cooldown ? d_cd : nullptr, n, d_sym, d_off, d_dist, c->stream), "symbols launch");
    CK(cudaMemcpyAsync(symbol, d_sym, (size_t)n, cudaMemcpyDeviceToHost, c->stream), "D2H");
    CK(cudaMemcpyAsync(drift_offset, d_off, (size_t)n, cudaMemcpyDeviceToHost, c->stream), "D2H");
    CK(cudaMemcpyAsync(distance, d_dist, (size_t)n, cudaMemcpyDeviceToHost, c->stream), "D2H");
    CK(cudaStreamSynchronize(c->stream), "sync");
    return CB200_OK;
}

int cb200_best_colors(cb200_ctx* c, const uint8_t* rgb_means, int n, uint8_t* color)
{
    if (!c || !rgb_means || !color || n < 0) return fail(CB200_ERR_ARG, "bad arguments");
    if (n == 0) return CB200_OK;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    CK(c->d_scratch.ensure(4 * (size_t)n + 64), "cudaMalloc scratch");
    uint8_t* d_in = c->d_scratch; uint8_t* d_out = d_in + 3 * (size_t)n;
    CK(cudaMemcpyAsync(d_in, rgb_means, 3 * (size_t)n, cudaMemcpyHostToDevice, c->stream), "H2D");
    CcmArg cc;
    int rc = ccm_arg(c, cc); if (rc) return rc;
    CK(k1_colors_launch(c->mode, d_in, n, d_out, cc, c->stream), "colors launch");
    CK(cudaMemcpyAsync(color, d_out, (size_t)n, cudaMemcpyDeviceToHost, c->stream), "D2H");
    CK(cudaStreamSynchronize(c->stream), "sync");
    return CB200_OK;
}

int cb200_set_ccm(cb200_ctx* c, const float* m9)
{
    if (!c) return fail(CB200_ERR_ARG, "null context");
    int rc = check_host_ccm(c); if (rc) return rc;
    c->ccm_pending = c->ccm_pending_flag = false;    // an explicit matrix replaces whatever the last batch left
    c->ccm_active = m9 != nullptr;
    if (m9) memcpy(c->ccm, m9, sizeof(c->ccm));
    return carry_from_host(c);
}

int cb200_get_ccm(cb200_ctx* c, float* m9)
{
    if (!c) return fail(CB200_ERR_ARG, "null context");
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    int rc = ccm_resolve(c); if (rc) return rc;
    if (c->ccm_active && m9) memcpy(m9, c->ccm, sizeof(c->ccm));
    return c->ccm_active ? 1 : 0;
}

int cb200_get_frame_ccms(cb200_ctx* c, int n, float* m9n, uint8_t* active)
{
    if (!c || n < 0 || (n > 0 && (!m9n || !active))) return fail(CB200_ERR_ARG, "bad arguments");
    if (n > c->ccm_frames) return fail(CB200_ERR_ARG, "the last CC_FIT call had " + std::to_string(c->ccm_frames) + " frames");
    if (n == 0) return CB200_OK;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    CK(cudaMemcpyAsync(m9n, c->d_ccm, sizeof(float) * 9 * (size_t)n, cudaMemcpyDeviceToHost, c->stream), "D2H frame ccms");
    CK(cudaMemcpyAsync(active, c->d_ccm_active, (size_t)n, cudaMemcpyDeviceToHost, c->stream), "D2H frame ccm flags");
    CK(cudaStreamSynchronize(c->stream), "sync");
    return CB200_OK;
}

int cb200_fit_ccm(cb200_ctx* c, const uint8_t* rgb, const uint8_t* header6, uint32_t radioactive_block_id, uint32_t flags, float* m9_out)
{
    if (!c || !header6) return fail(CB200_ERR_ARG, "bad arguments");
    int rc = check_host_ccm(c); if (rc) return rc;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    const Mode& m = c->mode;
    if (m.color_bits == 0) return 0;
    if (rgb) { rc = upload_frames(c, rgb, 1); if (rc) return rc; }
    else if (!c->d_rgb) return fail(CB200_ERR_ARG, "no frame in the context's staging buffer");
    rc = ccm_buffers(c); if (rc) return rc;
    const uint16_t* idx;
    rc = idx_for(c, flags, &idx); if (rc) return rc;
    GivenHeader g;
    memset(&g, 0, sizeof(g));
    memcpy(g.hdr, header6, 6); g.use = 1; g.radioactive = radioactive_block_id;
    CK(ccm_fit_launch(m, c->d_rgb, nullptr, nullptr, idx, 1, c->d_fit, c->d_fit_valid, c->stream, &g), "ccm fit");
    float fitm[9]; uint8_t valid = 0;
    CK(cudaMemcpyAsync(fitm, c->d_fit, sizeof(fitm), cudaMemcpyDeviceToHost, c->stream), "D2H fit");
    CK(cudaMemcpyAsync(&valid, c->d_fit_valid, 1, cudaMemcpyDeviceToHost, c->stream), "D2H fit flag");
    CK(cudaStreamSynchronize(c->stream), "sync");
    if (!valid) return 0;
    c->ccm_pending = c->ccm_pending_flag = false;
    c->ccm_active = true;
    memcpy(c->ccm, fitm, sizeof(fitm));
    if (m9_out) memcpy(m9_out, fitm, sizeof(fitm));
    rc = carry_from_host(c); if (rc) return rc;
    return 1;
}

int cb200_palette_color(int color_bits, unsigned color_mode, int i, uint8_t* rgb_out)
{
    if (color_bits < 0 || color_bits > 3 || i < 0 || !rgb_out) return fail(CB200_ERR_ARG, "bad arguments");
    uint8_t pal[8][4];
    fill_palette(1 << color_bits, (int)color_mode, pal);
    if (i >= (color_bits >= 3 ? 8 : 4)) return fail(CB200_ERR_ARG, "colour index outside the palette");   // the reference indexes a 4 / 8 entry array
    rgb_out[0] = pal[i][0]; rgb_out[1] = pal[i][1]; rgb_out[2] = pal[i][2];
    return CB200_OK;
}

int cb200_encode_cells_dev(cb200_ctx* c, const uint8_t* d_payload, int n, uint8_t* d_cellvals)
{
    int rc = check_n(c, n); if (rc) return rc;
    if (n == 0) return CB200_OK;
    if (!d_payload || !d_cellvals) return fail(CB200_ERR_ARG, "null buffer");
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    CK(encode_launch(c->mode, c->d_gen, c->d_inv, d_payload, n, c->d_raw, d_cellvals, c->stream), "encode launch");
    return CB200_OK;
}

int cb200_set_timing(cb200_ctx* c, int enable)
{
    if (!c) return fail(CB200_ERR_ARG, "null context");
    if (enable && !c->ev[0][0]) {    // the 512 events are only created for callers that measure
        CK(cudaSetDevice(c->device), "cudaSetDevice");
        for (int k = 0; k < cb200_ctx::kEvSets; ++k) for (int i = 0; i < 8; ++i) CK(cudaEventCreate(&c->ev[k][i]), "cudaEventCreate");
    }
    c->timing = enable != 0;
    c->calls = 0; c->cur = 0;
    for (int k = 0; k < cb200_ctx::kEvSets; ++k) c->ev_count[k] = 0;
    return CB200_OK;
}

int cb200_get_timing(cb200_ctx* c, int calls_back, float* ms, int max_entries, int* n_entries)
{
    if (!c || !ms || !n_entries || calls_back < 0) return fail(CB200_ERR_ARG, "bad argument");
    if (calls_back >= cb200_ctx::kEvSets || calls_back >= c->calls) return fail(CB200_ERR_ARG, "no such timed call");
    CK(cudaStreamSynchronize(c->stream), "sync");
    int set = (int)((c->calls - 1 - calls_back) % cb200_ctx::kEvSets);
    int n = c->ev_count[set] > 0 ? c->ev_count[set] - 1 : 0;
    if (n > max_entries) n = max_entries;
    for (int i = 0; i < n; ++i) CK(cudaEventElapsedTime(&ms[i], c->ev[set][i], c->ev[set][i + 1]), "cudaEventElapsedTime");
    *n_entries = n;
    return CB200_OK;
}

int cb200_render_frames_dev(cb200_ctx* c, const uint8_t* d_cellvals, int n, uint8_t* d_rgb_out)
{
    if (!c || !d_cellvals || !d_rgb_out || n < 0) return fail(CB200_ERR_ARG, "bad arguments");
    if (n == 0) return CB200_OK;
    CK(cudaSetDevice(c->device), "cudaSetDevice");
    CK(render_launch(c->mode, d_cellvals, n, d_rgb_out, c->stream), "render launch");
    return CB200_OK;
}

}  // extern "C"
