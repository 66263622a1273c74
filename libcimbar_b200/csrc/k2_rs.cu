// k2_rs.cu -- K2: de-interleave/bit-pack + Reed-Solomon block correction + fountain-chunk masks, sm_90a.
//
// Replaces (reference file:line relative to /root/reference/):
//   P7/P10 Decoder::do_decode bit packing     src/lib/encoder/Decoder.h:77-117 (:121-161 coupled), Interleave.h:8-36,
//                                              bit_file/bitbuffer.h:62-84 (MSB-first)
//   P11    reed_solomon_stream::write         src/lib/encoder/reed_solomon_stream.h:54-76
//   P12    correct_reed_solomon_decode        src/third_party_lib/libcorrect/src/reed-solomon/decode.c:299-379
//          (GF(2^8) poly 0x187, roots alpha^1..alpha^parity; Berlekamp-Massey decode.c:30-116, Chien :120-143,
//           locations :198-222, Forney :163-194; no syndrome re-check, x/0 = 0, success iff #roots == locator order)
//   P13    aligned_stream chunk acceptance    src/lib/encoder/aligned_stream.h:39-116 (+ reed_solomon_stream.h:109-114)
//
// One warp per RS block.  Syndromes: lane j runs Horner with the constant alpha^(j+1) through exp/log LUTs in shared
// memory; Berlekamp-Massey keeps one locator coefficient per lane-slot in shared memory and updates them lane-parallel
// in libcorrect's exact operation order (its output for uncorrectable blocks depends on that order); Chien search
// evaluates the locator at 8 field elements per lane; Forney evaluates one error value per lane.
#include "cb200_common.cuh"
#include "k2_rs.cuh"
#include <cstring>
#include <cstdint>

namespace cb200 {

constexpr int kMaxParity = 64;

__constant__ uint8_t c_gf_exp[512];
__constant__ uint8_t c_gf_log[256];

// ---------------------------------------------------------------------------------------------- pack
// value of interleave slot s in a given stream: 0 = symbols, 1 = colours, 2 = coupled (colour << symbol_bits | symbol)
__device__ __forceinline__ uint32_t slot_value(const uint8_t* __restrict__ cells, const uint16_t* __restrict__ idx,
                                               uint32_t s, int stream, int symbol_bits)
{
    uint32_t v = cells[idx[s]] & 0x7Fu;
    uint32_t sym_mask = (1u << symbol_bits) - 1u;
    if (stream == 0) return v & sym_mask;
    if (stream == 1) return v >> symbol_bits;
    return v;
}

// byte B of a bit stream made of w-bit slots written MSB-first (bitbuffer::write)
__device__ __forceinline__ uint32_t stream_byte(const uint8_t* __restrict__ cells, const uint16_t* __restrict__ idx,
                                                uint32_t B, int w, int stream, int symbol_bits, uint32_t nslots)
{
    uint32_t bit0 = 8u * B;
    uint32_t s = bit0 / (uint32_t)w;
    uint32_t skip = bit0 - s * (uint32_t)w;
    uint32_t acc = 0, nbits = 0;
    while (nbits < skip + 8u) {
        uint32_t v = (s < nslots) ? slot_value(cells, idx, s, stream, symbol_bits) : 0u;
        acc = (acc << w) | v;
        nbits += (uint32_t)w;
        ++s;
    }
    return (acc >> (nbits - skip - 8u)) & 0xFFu;
}

__global__ void __launch_bounds__(256)
k_pack_raw(const Mode m, const uint8_t* __restrict__ cellvals, const uint16_t* __restrict__ idx, int n_frames,
           uint8_t* __restrict__ raw)
{
    int B = blockIdx.x * blockDim.x + threadIdx.x;
    int f = blockIdx.y;
    if (B >= m.cap_all || f >= n_frames) return;
    const uint8_t* cells = cellvals + (size_t)f * m.num_cells;
    uint32_t v;
    if (m.legacy) v = stream_byte(cells, idx, (uint32_t)B, m.symbol_bits + m.color_bits, 2, m.symbol_bits, (uint32_t)m.num_cells);
    else if (B < m.cap_sym) v = stream_byte(cells, idx, (uint32_t)B, m.symbol_bits, 0, m.symbol_bits, (uint32_t)m.num_cells);
    else v = stream_byte(cells, idx, (uint32_t)(B - m.cap_sym), m.color_bits, 1, m.symbol_bits, (uint32_t)m.num_cells);
    raw[(size_t)f * m.cap_all + B] = (uint8_t)v;
}

// ---------------------------------------------------------------------------------------------- GF(256) helpers
constexpr int kRsWarpsPerCta = 16;
constexpr int kLaDim = 40;               // >= the largest parity (36)
constexpr int kStagePitch = 196;         // bytes per staged block: >= 1 + 179, a multiple of 4, 49 words (rows start in different banks)

template <int T>
struct RsSmem {
    static constexpr bool kSynTable = false;
    static constexpr int GL = 8 * T;     // lanes per block in the remainder stage
    static constexpr int G = 32 / GL;    // blocks a warp takes at a time
    uint8_t exp[512];
    uint8_t log[256];
    struct PerWarp {
        alignas(16) uint8_t stage[G * kStagePitch];   // the block bytes, `lead` zero bytes first so that the length is a multiple of 4
        alignas(4) uint8_t rem[64];                   // remainder of the block being corrected (state words of its lane group)
        alignas(2) uint16_t remlog[kMaxParity];       // per remainder byte: byte | log(byte) << 8
        uint8_t synd[kMaxParity];
        uint8_t loc[kMaxParity + 8];
        uint8_t last[kMaxParity + 8];
        uint8_t omega[kMaxParity];
        uint8_t roots[kMaxParity + 8];
    } w[kRsWarpsPerCta];
    // la[k][j] = log of alpha^((j+1)(k - parity)): the weight of remainder byte k in syndrome j (see k_rs_decode)
    uint8_t la[kLaDim][kLaDim];
    // followed in dynamic shared memory by the four remainder tables: uint32 lt[4][256][GL] (see k_rs_decode)
};

template <class S>
__device__ __forceinline__ uint32_t gf_mul(const S& s, uint32_t a, uint32_t b)
{   // field_mul, libcorrect field.h:92-110
    if (a == 0 || b == 0) return 0;
    return s.exp[(uint32_t)s.log[a] + (uint32_t)s.log[b]];
}
template <class S>
__device__ __forceinline__ uint32_t gf_div(const S& s, uint32_t a, uint32_t b)
{   // field_div, field.h:112-129 (x / 0 == 0)
    if (a == 0 || b == 0) return 0;
    return s.exp[255u + (uint32_t)s.log[a] - (uint32_t)s.log[b]];
}
__device__ __forceinline__ uint32_t lds_u32(uint32_t shared_addr)
{
    uint32_t v;
    asm("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(shared_addr));
    return v;
}
__device__ __forceinline__ uint32_t warp_xor(uint32_t v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v ^= __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// ---------------------------------------------------------------------------------------------- one dirty block
// The whole warp corrects ONE block whose remainder modulo x^pad g is nonzero: enc[0 .. blk) is corrected in place; returns
// false when libcorrect would report failure (root count != locator order).  `holds`: this lane carries state word k of the
// block's remainder in `word`.  S: exp/log/la tables, W: the warp's scratch (rem, remlog, synd, loc, last, omega, roots).
template <int T, class S, class W>
__device__ __forceinline__ bool rs_correct_block(const S& s, W& w, uint8_t* enc, const int md, const int blk, const int pad,
                                                 const bool holds, const uint32_t word, const int k, const int lane)
{
            // ---- syndromes from the remainder: S_j = r'(alpha^(j+1)) alpha^(-(j+1) parity) = sum_k r'[k] alpha^((j+1)(k - parity)),
            // r'[k] = state byte pad + k.  A plain sum (no Horner chain): the terms are independent, log r'[k] is the same for
            // every lane, the weights come from the la table
            __syncwarp();
            if (holds) reinterpret_cast<uint32_t*>(w.rem)[k] = word;
            __syncwarp();
            if constexpr (S::kSynTable) {
                // (parity <= 32) multiplication by the constant c = alpha^((j+1)(i - parity)) is linear over GF(2): r c = XOR over the set
                // bits b of r of c 2^b.  wsyn[i][j] holds those eight products, masks[i] has byte b = 0xFF iff bit b of r'[i] is set
                // (the same for every lane): two 64-bit loads and two AND-XORs per remainder byte, no log/exp chain
                if (lane < md) {
                    const uint32_t rb = w.rem[pad + lane];
                    w.masks[lane] = make_uint2((((rb & 15u) * 0x00204081u) & 0x01010101u) * 0xFFu, (((rb >> 4) * 0x00204081u) & 0x01010101u) * 0xFFu);
                }
                __syncwarp();
                uint32_t ax = 0, ay = 0;
#pragma unroll 6
                for (int i = 0; i < md; ++i) {
                    const uint2 mk = w.masks[i];                                                // broadcast
                    const uint2 tw = s.wsyn[i][lane];
                    ax ^= tw.x & mk.x; ay ^= tw.y & mk.y;
                }
                uint32_t x = ax ^ ay;
                x ^= x >> 16; x ^= x >> 8;
                if (lane < md) w.synd[lane] = (uint8_t)x;
            } else {
            for (int i = lane; i < md; i += 32) { const uint32_t rb = w.rem[pad + i]; w.remlog[i] = (uint16_t)(rb | ((uint32_t)s.log[rb] << 8)); }
            __syncwarp();
#pragma unroll
            for (int q = 0; q < T; ++q) {
                const int j = lane + 32 * q;
                if (j < md) {
                    uint32_t acc = 0;
#pragma unroll 6
                    for (int i = 0; i < md; ++i) {
                        const uint32_t rl = w.remlog[i];                                        // broadcast
                        const uint32_t t = s.exp[(rl >> 8) + (uint32_t)s.la[i][j]];             // index <= 254 + 254
                        acc ^= (rl & 0xFFu) ? t : 0u;
                    }
                    w.synd[j] = (uint8_t)acc;
                }
            }
            }
            __syncwarp();
        // ---- Berlekamp-Massey (decode.c:30-116).  Field arithmetic is exact, so scale = disc / last_disc is applied as one
        //      multiplication (libcorrect writes mul-then-div per coefficient: same element); what must match libcorrect is
        //      the update rule and the order bookkeeping, because they decide the locator it reports for uncorrectable blocks.
        uint32_t numerrors = 0, loc_order = 0, last_order = 0, last_disc = 1, delay = 1;
        if (T == 1) {
            // parity <= 32: coefficient j of the locator / previous locator lives in lane j, syndrome j in lane j (value and log
            // packed in one word so that one shuffle moves both); lloc = log(loc) is refreshed only when loc changes
            uint32_t loc = (lane == 0), last = (lane == 0), lloc = 0;
            const uint32_t syn = (lane < md) ? (uint32_t)w.synd[lane] : 0u;
            const uint32_t spk = syn | ((uint32_t)s.log[syn] << 8);
            for (uint32_t i = 0; i < (uint32_t)md; ++i) {
                // disc = S[i] ^ sum_{j=1..numerrors} loc[j] * S[i-j]; lane 0 contributes loc[0] * S[i] = S[i] (loc[0] stays 1)
                const uint32_t p = __shfl_sync(0xffffffffu, spk, (int)(i - (uint32_t)lane) & 31);
                uint32_t term = 0;
                if ((uint32_t)lane <= numerrors && loc != 0 && (p & 0xFFu) != 0) term = s.exp[lloc + (p >> 8)];
                const uint32_t disc = __reduce_xor_sync(0xffffffffu, term);
                if (disc == 0) { delay++; continue; }
                const uint32_t lscale = 255u + (uint32_t)s.log[disc] - (uint32_t)s.log[last_disc];      // log(disc / last_disc), last_disc != 0
                const uint32_t top = last_order + delay;
                const uint32_t shifted = __shfl_up_sync(0xffffffffu, last, delay);                              // last[j - delay]
                const uint32_t lsc = lscale >= 255u ? lscale - 255u : lscale;                                   // in [0, 254]: exp index stays < 512
                const uint32_t sh = ((uint32_t)lane >= delay && (uint32_t)lane <= top && shifted != 0) ? (uint32_t)s.exp[(uint32_t)s.log[shifted] + lsc] : 0u;
                if (2 * numerrors <= i) {
                    // last <- x^delay * scale * last ; then loc, last <- loc - last, loc   over [0, last_order+delay]
                    if ((uint32_t)lane <= top) { const uint32_t t0 = loc; loc ^= sh; last = t0; }
                    lloc = s.log[loc];
                    const uint32_t tmp = loc_order;
                    loc_order = top; last_order = tmp;
                    numerrors = i + 1 - numerrors;
                    last_disc = disc;
                    delay = 1;
                    continue;
                }
                // no length change: loc[j+delay] ^= scale * last[j]
                loc ^= sh;
                lloc = s.log[loc];
                if (top > loc_order) loc_order = top;
                delay++;
            }
            w.loc[lane] = (uint8_t)loc;
            if (lane < 8) w.loc[32 + lane] = 0;
            __syncwarp();
        } else {
        // coefficients in shared memory, updated lane-parallel (parity > 31 needs more than one coefficient per lane)
        for (int j = lane; j < kMaxParity + 8; j += 32) { w.loc[j] = (j == 0); w.last[j] = (j == 0); }
        __syncwarp();
        for (uint32_t i = 0; i < (uint32_t)md; ++i) {
            uint32_t part = 0;
            for (uint32_t j = 1 + lane; j <= numerrors; j += 32) part ^= gf_mul(s, w.loc[j], w.synd[i - j]);
            uint32_t disc = warp_xor(part) ^ w.synd[i];
            if (disc == 0) { delay++; continue; }
            if (2 * numerrors <= i) {
                // last <- x^delay * (disc/last_disc) * last ; then loc, last <- loc - last, loc   over [0, last_order+delay]
                uint32_t top = last_order + delay;
                uint32_t sh[3], lc[3];
                int q = 0;
                for (uint32_t j = lane; j <= top; j += 32, ++q) {
                    sh[q] = (j < delay) ? 0u : gf_div(s, gf_mul(s, w.last[j - delay], disc), last_disc);
                    lc[q] = w.loc[j];
                }
                __syncwarp();
                q = 0;
                for (uint32_t j = lane; j <= top; j += 32, ++q) {
                    w.loc[j] = (uint8_t)(lc[q] ^ sh[q]);
                    w.last[j] = (uint8_t)lc[q];
                }
                __syncwarp();
                uint32_t tmp = loc_order;
                loc_order = top; last_order = tmp;
                numerrors = i + 1 - numerrors;
                last_disc = disc;
                delay = 1;
                continue;
            }
            // no length change: loc[j+delay] ^= (disc/last_disc) * last[j]
            for (uint32_t j = lane; j <= last_order; j += 32)
                w.loc[j + delay] ^= (uint8_t)gf_div(s, gf_mul(s, w.last[j], disc), last_disc);
            __syncwarp();
            if (last_order + delay > loc_order) loc_order = last_order + delay;
            delay++;
        }
        }
        const uint32_t order = loc_order;

        // ---- Chien search over all field elements in increasing order (decode.c:120-143); element 0 is never a
        //      root (loc[0] == 1); root count must equal the locator order, else the block fails
        uint32_t myroots = 0;   // bit k set: element lane*8+k is a root
        for (int k = 0; k < 8; ++k) {
            uint32_t e = (uint32_t)lane * 8u + (uint32_t)k;
            if (e == 0) continue;
            uint32_t le = s.log[e];
            uint32_t acc = w.loc[order];
            for (int i = (int)order - 1; i >= 0; --i) {
                uint32_t t = acc ? (uint32_t)s.exp[(uint32_t)s.log[acc] + le] : 0u;
                acc = t ^ w.loc[i];
            }
            if (acc == 0) myroots |= 1u << k;
        }
        uint32_t cnt = __popc(myroots);
        uint32_t incl = cnt;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { uint32_t v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
        uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
        if (total != order || order == 0) {   // order==0 cannot happen with nonzero syndromes; guarded for safety
            if (order == 0 && total == 0) {
                // libcorrect would "succeed" with no corrections; unreachable because S != 0 forces order >= 1
            }
            return false;
        }
        {
            uint32_t pos = incl - cnt;
            for (int k = 0; k < 8; ++k) if (myroots & (1u << k)) w.roots[pos++] = (uint8_t)(lane * 8 + k);
        }
        // ---- error evaluator omega = S(x) * loc(x) mod x^md  (decode.c:146-161, polynomial.c:17-31)
        for (int k = lane; k < md; k += 32) {
            uint32_t acc = 0;
            int lim = (int)order < k ? (int)order : k;
            for (int i = 0; i <= lim; ++i) acc ^= gf_mul(s, w.loc[i], w.synd[k - i]);
            w.omega[k] = (uint8_t)acc;
        }
        __syncwarp();
        // ---- Forney (decode.c:163-194) + apply (decode.c:369-372).  libcorrect evaluates omega(X) and loc'(X) by Horner, one root
        //      after the other; field arithmetic is exact, so the same elements come out of the plain sums
        //      omega(X) = sum_i omega[i] X^i and loc'(X) = sum_{i even, i < order} loc[i+1] X^i (polynomial.c:97-111: the formal
        //      derivative keeps the odd coefficients) -- one term per lane, one XOR reduction per root
        for (uint32_t q = 0; q < order; ++q) {
            const uint32_t X = w.roots[q];
            const uint32_t lx = s.log[X];
            uint32_t tn = 0, td = 0;
#pragma unroll
            for (int qq = 0; qq < T; ++qq) {
                const uint32_t i = (uint32_t)lane + 32u * (uint32_t)qq;
                const uint32_t ex = (i * lx) % 255u;                     // log(X^i)
                if (i < (uint32_t)md) { const uint32_t o = w.omega[i]; if (o) tn ^= s.exp[(uint32_t)s.log[o] + ex]; }
                if (i < order && (i & 1u) == 0u) { const uint32_t c = w.loc[i + 1]; if (c) td ^= s.exp[(uint32_t)s.log[c] + ex]; }
            }
            const uint32_t num = __reduce_xor_sync(0xffffffffu, tn), den = __reduce_xor_sync(0xffffffffu, td);
            const uint32_t err = gf_div(s, num, den);      // X^(fcr-1) = 1 for fcr = 1
            const uint32_t inv = s.exp[510u - lx];       // field_div(1, X): log[1] = 255
            const uint32_t location = s.log[inv];        // coefficient index (255 when inv == 1: out of range in libcorrect)
            if (lane == 0 && location >= (uint32_t)md && location < (uint32_t)blk)
                enc[blk - 1 - (int)location] ^= (uint8_t)err;
        }
        __syncwarp();
        return true;
}

// ---------------------------------------------------------------------------------------------- RS decode
// FUSED: the block's bytes are gathered straight from K1's per-cell bytes through the interleave map (P7/P10 bit packing
// folded in); otherwise they are read from a packed raw stream (n_frames * cap_all bytes, symbol stream blocks then colour
// stream blocks).  data_out: n_frames * nblocks * msg_len (zeros for failed blocks, reed_solomon_stream.h:96-107);
// ok: n_frames * nblocks.
//
// The clean-block test and the syndromes do not evaluate the received word c(x) at the parity roots one by one (libcorrect's
// decode.c:12-28: `parity` Horner chains over all n bytes).  All syndromes vanish iff the generator g divides c, so the block is
// first reduced modulo g: a warp takes 32 / GL blocks at a time, the GL = 8 T lanes of a group hold the remainder (4 bytes
// each), and every step consumes FOUR input bytes ("slicing by 4"): with G(x) = x^pad g(x) of degree D = 4 Pw (a whole number
// of words) the state obeys  S' = (S_low << 32) ^ sum_j T_j[byte j of (top word ^ input word)],  T_j[v] = v (x^(D+j) mod G),
// i.e. one word broadcast, one lane shift and four conflict-light 32-byte table rows per four bytes and four blocks -- a
// quarter of the shared-memory traffic of the per-root chains and half the instructions.  The final state is x^pad r' with
// r' = c x^parity mod g: zero iff the block is clean; otherwise the syndromes libcorrect computes are
// S_j = c(a^(j+1)) = r'(a^(j+1)) a^(-(j+1) parity), `parity` short Horner steps over r' instead of n long ones, and the decode
// continues exactly as before (Berlekamp-Massey, Chien, Forney in libcorrect's operation order), one block per warp.
template <int T, bool FUSED>
__global__ void __launch_bounds__(kRsWarpsPerCta * 32, (T == 1 ? 4 : 2))
k_rs_decode(const Mode m, const uint8_t* __restrict__ raw, const uint8_t* __restrict__ cellvals, const uint16_t* __restrict__ idx,
            int n_frames, int b_begin, int b_count, uint8_t* __restrict__ data_out, uint8_t* __restrict__ block_ok,
            const uint8_t* __restrict__ rho)
{   // blocks [b_begin, b_begin + b_count) of every frame (all of them, or the symbol / the colour stream on their own)
    using Smem = RsSmem<T>;
    constexpr int GL = Smem::GL, G = Smem::G;
    extern __shared__ __align__(16) uint8_t rs_smem_raw[];
    Smem& s = *reinterpret_cast<Smem*>(rs_smem_raw);
    uint32_t* lt = reinterpret_cast<uint32_t*>(rs_smem_raw + ((sizeof(Smem) + 127) & ~size_t(127)));
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    for (int i = tid; i < 512; i += blockDim.x) s.exp[i] = c_gf_exp[i];
    for (int i = tid; i < 256; i += blockDim.x) s.log[i] = c_gf_log[i];
    __syncthreads();
    for (int e = tid; e < m.ecc_bytes * kLaDim; e += blockDim.x) {
        const int kk = e / kLaDim, j = e % kLaDim;
        s.la[kk][j] = (uint8_t)((255 - ((j + 1) * (m.ecc_bytes - kk)) % 255) % 255);
    }
    for (int e = tid; e < 4 * 256 * GL; e += blockDim.x) {
        const int j = e / (256 * GL), v = (e / GL) & 255, k = e % GL;
        uint32_t word = 0;
#pragma unroll
        for (int bb = 0; bb < 4; ++bb) word |= gf_mul(s, (uint32_t)v, (uint32_t)rho[j * 64 + 4 * k + bb]) << (8 * bb);
        lt[e] = word;
    }
    __syncthreads();

    const int md = m.ecc_bytes, blk = m.ecc_block, msg_len = m.msg_len;
    const int Pw = (md + 3) >> 2, pad = 4 * Pw - md, lead = (4 - (blk & 3)) & 3, nsteps = (lead + blk) >> 2;
    const long total_blocks = (long)n_frames * b_count;
    const long total_units = (total_blocks + G - 1) / G;
    typename Smem::PerWarp& w = s.w[warp];
    const int grp = lane / GL, k = lane % GL;
    const uint32_t lt_lane = (uint32_t)__cvta_generic_to_shared(lt) + 4u * (uint32_t)k;
    const uint32_t stage_lane = (uint32_t)__cvta_generic_to_shared(w.stage) + (uint32_t)(grp * kStagePitch);

    for (long unit = (long)blockIdx.x * kRsWarpsPerCta + warp; unit < total_units; unit += (long)gridDim.x * kRsWarpsPerCta) {
        __syncwarp();
        // ---- stage the G blocks of this unit
#pragma unroll 1
        for (int g = 0; g < G; ++g) {
            const long gb = unit * G + g;
            uint8_t* st = w.stage + g * kStagePitch;
            if (lane < lead) st[lane] = 0;                    // the `lead` zero bytes in front (never overlap the block bytes)
            if (gb >= total_blocks) { for (int i = lane; i < blk; i += 32) st[lead + i] = 0; continue; }   // an absent block reads as clean
            const int f = (int)(gb / b_count), b = b_begin + (int)(gb - (long)f * b_count);
            uint8_t* enc = st + lead;
            if (FUSED) {
                const uint8_t* cells = cellvals + (size_t)f * m.num_cells;
                const bool fast = !m.legacy && m.symbol_bits == 4 && m.color_bits == 2 && blk <= 160;
                if (fast) {
                    // a block lies entirely in the symbol stream or in the colour stream (cap_sym is a whole number of blocks).
                    // All interleave-map words of the block are loaded first, then all cell bytes: two dependent round trips
                    // to L2 per block instead of two per 32 bytes.
                    const uint32_t B0 = (uint32_t)b * (uint32_t)blk;
                    constexpr int kU = 5;                      // 5 x 32 >= ecc_block (155 in every mode; checked at launch)
                    if ((int)B0 < m.cap_sym) {                 // two 4-bit symbols per byte, MSB first (Decoder.h:91-92)
                        uint32_t sl[kU];
#pragma unroll
                        for (int u = 0; u < kU; ++u) {
                            const int i = lane + 32 * u;
                            sl[u] = i < blk ? *reinterpret_cast<const uint32_t*>(idx + 2u * (B0 + (uint32_t)i)) : 0u;
                        }
                        uint32_t c0[kU], c1[kU];
#pragma unroll
                        for (int u = 0; u < kU; ++u) {
                            const int i = lane + 32 * u;
                            if (i < blk) { c0[u] = cells[sl[u] & 0xFFFFu]; c1[u] = cells[sl[u] >> 16]; } else { c0[u] = c1[u] = 0; }
                        }
#pragma unroll
                        for (int u = 0; u < kU; ++u) {
                            const int i = lane + 32 * u;
                            if (i < blk) enc[i] = (uint8_t)(((c0[u] & 15u) << 4) | (c1[u] & 15u));
                        }
                    } else {                                   // four 2-bit colours per byte (Decoder.h:112-113)
                        uint2 sl[kU];
#pragma unroll
                        for (int u = 0; u < kU; ++u) {
                            const int i = lane + 32 * u;
                            sl[u] = i < blk ? *reinterpret_cast<const uint2*>(idx + 4u * (B0 + (uint32_t)i - (uint32_t)m.cap_sym)) : make_uint2(0u, 0u);
                        }
                        uint32_t c0[kU], c1[kU], c2[kU], c3[kU];
#pragma unroll
                        for (int u = 0; u < kU; ++u) {
                            const int i = lane + 32 * u;
                            if (i < blk) { c0[u] = cells[sl[u].x & 0xFFFFu]; c1[u] = cells[sl[u].x >> 16]; c2[u] = cells[sl[u].y & 0xFFFFu]; c3[u] = cells[sl[u].y >> 16]; }
                            else { c0[u] = c1[u] = c2[u] = c3[u] = 0; }
                        }
#pragma unroll
                        for (int u = 0; u < kU; ++u) {
                            const int i = lane + 32 * u;
                            if (i < blk)
                                enc[i] = (uint8_t)((((c0[u] >> 4) & 3u) << 6) | (((c1[u] >> 4) & 3u) << 4) | (((c2[u] >> 4) & 3u) << 2) | ((c3[u] >> 4) & 3u));
                        }
                    }
                } else {
                    for (int i = lane; i < blk; i += 32) {
                        uint32_t B = (uint32_t)b * (uint32_t)blk + (uint32_t)i, v;
                        if (m.legacy) v = stream_byte(cells, idx, B, m.symbol_bits + m.color_bits, 2, m.symbol_bits, (uint32_t)m.num_cells);
                        else if ((int)B < m.cap_sym) v = stream_byte(cells, idx, B, m.symbol_bits, 0, m.symbol_bits, (uint32_t)m.num_cells);
                        else v = stream_byte(cells, idx, B - (uint32_t)m.cap_sym, m.color_bits, 1, m.symbol_bits, (uint32_t)m.num_cells);
                        enc[i] = (uint8_t)v;
                    }
                }
            } else {
                // symbol-stream blocks are consecutive ecc_block pieces of the first cap_sym bytes, colour blocks of the rest
                // (the two reed_solomon_streams of Decoder.h:100-101 and :115-117); cap_sym is a whole number of blocks
                const uint8_t* enc_g = raw + (size_t)f * m.cap_all + (size_t)b * blk;
                for (int i = lane; i < blk; i += 32) enc[i] = enc_g[i];
            }
        }
        __syncwarp();

        // ---- remainder modulo x^pad g, four bytes per step, the G blocks of the unit side by side
        uint32_t word = 0;
        {
            const int top_src = grp * GL + (Pw - 1);
#pragma unroll 2
            for (int t = 0; t < nsteps; ++t) {
                const uint32_t ew = lds_u32(stage_lane + 4u * (uint32_t)t);     // first byte = highest power
                const uint32_t tw = __shfl_sync(0xffffffffu, word, top_src);
                const uint32_t v = tw ^ __byte_perm(ew, 0u, 0x0123);
                const uint32_t r0 = lds_u32(lt_lane + (((v) & 0xFFu) + 0u) * (4u * GL));
                const uint32_t r1 = lds_u32(lt_lane + (((v >> 8) & 0xFFu) + 256u) * (4u * GL));
                const uint32_t r2 = lds_u32(lt_lane + (((v >> 16) & 0xFFu) + 512u) * (4u * GL));
                const uint32_t r3 = lds_u32(lt_lane + ((v >> 24) + 768u) * (4u * GL));
                uint32_t prev = __shfl_up_sync(0xffffffffu, word, 1, GL);
                if (k == 0) prev = 0;
                word = prev ^ r0 ^ r1 ^ r2 ^ r3;
            }
        }
        const uint32_t dirty = __ballot_sync(0xffffffffu, k < Pw && word != 0u);

#pragma unroll 1
        for (int g = 0; g < G; ++g) {
            const long gb = unit * G + g;
            if (gb >= total_blocks) break;                     // warp-uniform
            const int f = (int)(gb / b_count), b = b_begin + (int)(gb - (long)f * b_count);
            uint8_t* out = data_out + ((size_t)f * m.nblocks + b) * msg_len;
            uint8_t* enc = w.stage + g * kStagePitch + lead;
            if (((dirty >> (g * GL)) & ((1u << GL) - 1u)) == 0u) {   // clean block: copy out (decode.c:337-343)
                for (int i = lane; i < msg_len; i += 32) out[i] = enc[i];
                if (lane == 0) block_ok[(size_t)f * m.nblocks + b] = 1;
                continue;
            }
            __syncwarp();
            const bool good = rs_correct_block<T>(s, w, enc, md, blk, pad, grp == g && k < Pw, word, k, lane);
            __syncwarp();
            if (!good) {
                for (int i = lane; i < msg_len; i += 32) out[i] = 0;
                if (lane == 0) block_ok[(size_t)f * m.nblocks + b] = 0;
                continue;
            }
        for (int i = lane; i < msg_len; i += 32) out[i] = enc[i];
        if (lane == 0) block_ok[(size_t)f * m.nblocks + b] = 1;
        }
    }
}

// ---------------------------------------------------------------------------------------------- RS decode, whole frames per CTA
// The hot configuration (4 symbol + 2 colour bits per cell, 155-byte blocks, parity <= 32, all blocks of every frame: mode B and
// its siblings) does not let every warp chase the interleave map through L2 on its own.  A CTA of 32 warps takes TWO frames
// at a time:
//   1. their per-cell bytes (K1's output, 12,400 B each) arrive in shared memory by cp.async -- issued one step ahead, so
//      the copy overlaps the previous step's corrections;
//   2. all 1024 threads build the de-interleaved, bit-packed RS blocks (P7/P10) in shared memory, one 4-byte word of a staged
//      block per thread and step: the interleave map is read coalesced (it is the same for every frame: L1/L2 hits), the
//      cell bytes come from shared memory;
//   3. one warp per unit of four consecutive blocks: remainder modulo x^pad g (as in k_rs_decode), the rare dirty block is
//      corrected in place by the whole warp, and the unit's four messages -- contiguous in the output -- leave as 32-bit
//      stores.
constexpr int kFrWarps = 32;
constexpr int kFrFrames = 2;
constexpr int kFrBlk = 155, kFrWords = 39, kFrPitch = 160;   // block bytes; words per staged block (1 zero byte + 155); row pitch:
                                                             // 40 words, so the four rows of a unit start 8 banks apart

struct RsFrSmem {
    static constexpr bool kSynTable = true;
    uint8_t exp[512];
    uint8_t log[256];
    struct PerWarp {
        alignas(8) uint2 masks[32];           // per remainder byte: byte b = 0xFF iff its bit b is set (syndromes of a dirty block)
        alignas(4) uint8_t rem[64];
        alignas(2) uint16_t remlog[kMaxParity];
        uint8_t synd[kMaxParity];
        uint8_t loc[kMaxParity + 8];
        uint8_t last[kMaxParity + 8];
        uint8_t omega[kMaxParity];
        uint8_t roots[kMaxParity + 8];
    } w[kFrWarps];
    uint8_t la[kLaDim][kLaDim];
    // wsyn[i][j] byte b = alpha^((j+1)(i - parity)) * 2^b: the weight of bit b of remainder byte i in syndrome j
    alignas(8) uint2 wsyn[32][32];
    // followed in dynamic shared memory by: uint32 lt[4][256][8]; the cell bytes of kFrFrames frames (cell_pitch each);
    // the staged blocks of kFrFrames frames (nblocks rows of kFrPitch bytes each)
};

__device__ __forceinline__ void cp_async16(uint32_t dst_shared, const void* src)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst_shared), "l"(src) : "memory");
}

__global__ void __launch_bounds__(kFrWarps * 32, 2)
k_rs_frames(const Mode m, const uint8_t* __restrict__ cellvals, const uint16_t* __restrict__ idx, int n_frames,
            uint8_t* __restrict__ data_out, uint8_t* __restrict__ block_ok, const uint8_t* __restrict__ rho, int cell_pitch)
{
    constexpr int GL = 8, G = 4;
    extern __shared__ __align__(16) uint8_t rs_smem_raw[];
    RsFrSmem& s = *reinterpret_cast<RsFrSmem*>(rs_smem_raw);
    uint8_t* dyn = rs_smem_raw + ((sizeof(RsFrSmem) + 127) & ~size_t(127));
    uint32_t* lt = reinterpret_cast<uint32_t*>(dyn);
    uint8_t* cellbuf = dyn + sizeof(uint32_t) * 4 * 256 * GL;
    uint8_t* rows = cellbuf + (size_t)kFrFrames * cell_pitch;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int md = m.ecc_bytes, msg_len = m.msg_len, nb = m.nblocks, upf = nb / G;
    const int Pw = (md + 3) >> 2, pad = 4 * Pw - md;
    const int words_per_frame = nb * kFrWords, sym_rows = m.cap_sym / kFrBlk, cell_vecs = m.num_cells >> 4;
    const bool coupled6 = m.legacy != 0;          // (launch condition: symbol_bits + color_bits == 6)
    const int n_groups = (n_frames + kFrFrames - 1) / kFrFrames;
    const uint32_t cellbuf_s = (uint32_t)__cvta_generic_to_shared(cellbuf);

    auto load_cells = [&](int gi) {
        for (int fs = 0; fs < kFrFrames; ++fs) {
            const int f = gi * kFrFrames + fs;
            if (f >= n_frames) break;
            const uint8_t* src = cellvals + (size_t)f * m.num_cells;
            for (int i = tid; i < cell_vecs; i += (int)blockDim.x) cp_async16(cellbuf_s + (uint32_t)(fs * cell_pitch + 16 * i), src + 16 * i);
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
    int gi = blockIdx.x;
    if (gi < n_groups) load_cells(gi);

    for (int i = tid; i < 512; i += blockDim.x) s.exp[i] = c_gf_exp[i];
    for (int i = tid; i < 256; i += blockDim.x) s.log[i] = c_gf_log[i];
    __syncthreads();
    for (int e = tid; e < md * kLaDim; e += blockDim.x) {
        const int kk = e / kLaDim, j = e % kLaDim;
        s.la[kk][j] = (uint8_t)((255 - ((j + 1) * (md - kk)) % 255) % 255);
    }
    for (int e = tid; e < 32 * 32; e += blockDim.x) {
        const int i = e >> 5, j = e & 31;
        uint2 t = make_uint2(0u, 0u);
        if (i < md && j < md) {
            const uint32_t l = (uint32_t)((255 - ((j + 1) * (md - i)) % 255) % 255);
            t.x = (uint32_t)s.exp[l] | ((uint32_t)s.exp[l + 1] << 8) | ((uint32_t)s.exp[l + 2] << 16) | ((uint32_t)s.exp[l + 3] << 24);
            t.y = (uint32_t)s.exp[l + 4] | ((uint32_t)s.exp[l + 5] << 8) | ((uint32_t)s.exp[l + 6] << 16) | ((uint32_t)s.exp[l + 7] << 24);
        }
        s.wsyn[i][j] = t;
    }
    // the four remainder tables interleaved: row (v, j) = T_j[v] (32 bytes) at word (4 v + j) 8, i.e. table j only ever occupies
    // banks 8 j .. 8 j + 7.  In one lookup instruction lane group g reads table i ^ g (the four rows are XORed together, so the
    // order does not matter): four different bank octets, no conflict whatever the four byte values are.
    for (int e = tid; e < 4 * 256 * GL; e += blockDim.x) {
        const int v = e / (4 * GL), j = (e / GL) & 3, kk = e % GL;
        uint32_t word = 0;
#pragma unroll
        for (int bb = 0; bb < 4; ++bb) word |= gf_mul(s, (uint32_t)v, (uint32_t)rho[j * 64 + 4 * kk + bb]) << (8 * bb);
        lt[e] = word;
    }

    RsFrSmem::PerWarp& w = s.w[warp];
    const int grp = lane / GL, k = lane % GL;
    const uint32_t lt_lane = (uint32_t)__cvta_generic_to_shared(lt) + 4u * (uint32_t)k;
    // byte i of __byte_perm(v, 0, vsel) = byte i ^ grp of v; lookup i of this lane goes to table i ^ grp
    const uint32_t vsel = 0x3210u ^ (0x1111u * (uint32_t)grp);
    const uint32_t lt0 = lt_lane + 32u * (uint32_t)(0 ^ grp), lt1 = lt_lane + 32u * (uint32_t)(1 ^ grp);
    const uint32_t lt2 = lt_lane + 32u * (uint32_t)(2 ^ grp), lt3 = lt_lane + 32u * (uint32_t)(3 ^ grp);

    for (; gi < n_groups; gi += gridDim.x) {
        asm volatile("cp.async.wait_all;" ::: "memory");
        __syncthreads();        // this group's cell bytes have landed (and the tables, first time); nobody still reads the rows of the previous group
        const int nf = (n_frames - gi * kFrFrames) < kFrFrames ? (n_frames - gi * kFrFrames) : kFrFrames;

        // ---- P7/P10: staged word q of block r = stream bytes 155 r + 4 q - 1 .. + 2 (byte -1 of a block is the zero in front)
        for (int wi = tid; wi < nf * words_per_frame; wi += (int)blockDim.x) {
            const int fs = wi >= words_per_frame ? 1 : 0;
            const int rem = wi - fs * words_per_frame;
            const int r = rem / kFrWords, q = rem - r * kFrWords;
            const uint8_t* cb = cellbuf + fs * cell_pitch;
            uint32_t b0, b1, b2, b3;
            if (coupled6) {             // legacy modes: ONE stream of 6-bit values colour << 4 | symbol (Decoder.h:121-161), MSB first:
                // stream byte B = bits [8 B, 8 B + 8) of the slot sequence; it always lies inside the two slots s = 8 B / 6, s + 1
                auto byte6 = [&](const int B) -> uint32_t {
                    const uint32_t bit0 = 8u * (uint32_t)B, sl = bit0 / 6u, skip = bit0 - 6u * sl;
                    const uint32_t v0 = cb[idx[sl]] & 63u, v1 = cb[idx[sl + 1]] & 63u;
                    return (((v0 << 6) | v1) >> (4u - skip)) & 0xFFu;
                };
                const int B0 = r * kFrBlk + 4 * q - 1;
                b0 = q ? byte6(B0) : 0u; b1 = byte6(B0 + 1); b2 = byte6(B0 + 2); b3 = byte6(B0 + 3);
            } else if (r < sym_rows) {  // two 4-bit symbols per byte, MSB first (Decoder.h:91-92)
                const uint32_t* ix = reinterpret_cast<const uint32_t*>(idx) + (r * kFrBlk + 4 * q);
                const uint32_t i0 = q ? ix[-1] : ix[0], i1 = ix[0], i2 = ix[1], i3 = ix[2];
                b0 = ((cb[i0 & 0xFFFFu] & 15u) << 4) | (cb[i0 >> 16] & 15u);
                b1 = ((cb[i1 & 0xFFFFu] & 15u) << 4) | (cb[i1 >> 16] & 15u);
                b2 = ((cb[i2 & 0xFFFFu] & 15u) << 4) | (cb[i2 >> 16] & 15u);
                b3 = ((cb[i3 & 0xFFFFu] & 15u) << 4) | (cb[i3 >> 16] & 15u);
            } else {                    // four 2-bit colours per byte (Decoder.h:112-113)
                const uint2* ix = reinterpret_cast<const uint2*>(idx) + ((r - sym_rows) * kFrBlk + 4 * q);
                const uint2 i0 = q ? ix[-1] : ix[0], i1 = ix[0], i2 = ix[1], i3 = ix[2];
                auto pack = [&](const uint2 ii) {
                    return (((uint32_t)cb[ii.x & 0xFFFFu] >> 4) & 3u) << 6 | (((uint32_t)cb[ii.x >> 16] >> 4) & 3u) << 4 |
                           (((uint32_t)cb[ii.y & 0xFFFFu] >> 4) & 3u) << 2 | (((uint32_t)cb[ii.y >> 16] >> 4) & 3u);
                };
                b0 = pack(i0); b1 = pack(i1); b2 = pack(i2); b3 = pack(i3);
            }
            if (q == 0) b0 = 0;
            *reinterpret_cast<uint32_t*>(rows + (size_t)(fs * nb + r) * kFrPitch + 4 * q) = b0 | (b1 << 8) | (b2 << 16) | (b3 << 24);
        }
        __syncthreads();        // the rows are complete; the cell buffer is free again
        if (gi + (int)gridDim.x < n_groups) load_cells(gi + (int)gridDim.x);

        if (warp >= nf * upf) continue;
        const int fs = warp >= upf ? 1 : 0, u = warp - fs * upf, f = gi * kFrFrames + fs;
        uint8_t* urow = rows + (size_t)(fs * nb + G * u) * kFrPitch;

        // ---- remainder modulo x^pad g, four bytes per step, the four blocks of the unit side by side (see k_rs_decode)
        uint32_t word = 0;
        {
            const uint32_t stage_lane = (uint32_t)__cvta_generic_to_shared(urow) + (uint32_t)(grp * kFrPitch);
            const int top_src = grp * GL + (Pw - 1);
#pragma unroll 3
            for (int t = 0; t < kFrWords; ++t) {
                const uint32_t ew = lds_u32(stage_lane + 4u * (uint32_t)t);
                const uint32_t tw = __shfl_sync(0xffffffffu, word, top_src);
                const uint32_t v = __byte_perm(tw ^ __byte_perm(ew, 0u, 0x0123), 0u, vsel);
                const uint32_t r0 = lds_u32(lt0 + ((v) & 0xFFu) * 128u);
                const uint32_t r1 = lds_u32(lt1 + ((v >> 8) & 0xFFu) * 128u);
                const uint32_t r2 = lds_u32(lt2 + ((v >> 16) & 0xFFu) * 128u);
                const uint32_t r3 = lds_u32(lt3 + (v >> 24) * 128u);
                uint32_t prev = __shfl_up_sync(0xffffffffu, word, 1, GL);
                if (k == 0) prev = 0;
                word = prev ^ r0 ^ r1 ^ r2 ^ r3;
            }
        }
        const uint32_t dirty = __ballot_sync(0xffffffffu, k < Pw && word != 0u);
        uint32_t okflags = 0x01010101u;
        if (dirty) {
#pragma unroll 1
            for (int g = 0; g < G; ++g) {
                if (((dirty >> (g * GL)) & ((1u << GL) - 1u)) == 0u) continue;
                uint8_t* enc = urow + g * kFrPitch + 1;
                __syncwarp();
                const bool good = rs_correct_block<1>(s, w, enc, md, kFrBlk, pad, grp == g && k < Pw, word, k, lane);
                __syncwarp();
                if (!good) {        // zeros for a failed block (reed_solomon_stream.h:96-107)
                    for (int i = lane; i < msg_len; i += 32) enc[i] = 0;
                    okflags &= ~(1u << (8 * g));
                }
            }
            __syncwarp();
        }
        // ---- the unit's four messages are contiguous in the output: 4 msg_len bytes, msg_len 32-bit words
        uint32_t* out32 = reinterpret_cast<uint32_t*>(data_out + ((size_t)f * nb + (size_t)(G * u)) * msg_len);
        const uint32_t urow_s = (uint32_t)__cvta_generic_to_shared(urow);
        for (int wq = lane; wq < msg_len; wq += 32) {
            const int B = 4 * wq;
            int g = (B >= msg_len) + (B >= 2 * msg_len) + (B >= 3 * msg_len);
            int i = B - g * msg_len;
            uint32_t val;
            if (i + 4 <= msg_len) {                           // the four bytes lie in one block: two aligned words, one funnel shift
                const uint32_t a = (uint32_t)(g * kFrPitch + 1 + i);
                const uint32_t w0 = lds_u32(urow_s + (a & ~3u)), w1 = lds_u32(urow_s + (a & ~3u) + 4u);   // (w1 stays inside the row: a + 3 <= 125)
                val = __funnelshift_r(w0, w1, 8u * (a & 3u));
            } else {                                          // the three words of a unit that straddle two blocks
                val = 0;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    val |= (uint32_t)urow[g * kFrPitch + 1 + i] << (8 * j);
                    if (++i == msg_len) { i = 0; ++g; }
                }
            }
            out32[wq] = val;
        }
        if (lane == 0) *reinterpret_cast<uint32_t*>(block_ok + (size_t)f * nb + (size_t)(G * u)) = okflags;
    }
}

// ---------------------------------------------------------------------------------------------- chunk masks (P13)
// chunk q is emitted iff all of its RS blocks decoded and the last block of chunk q-1 was not bad: a bad block sets
// aligned_stream::_badChunk, which is only cleared when a later good write crosses a chunk boundary
// (aligned_stream.h:66-73, :97-104); if the bad block is the chunk's last one, _offset wraps to 0 first and the
// flag survives into the next chunk.
__global__ void k_chunk_mask(const Mode m, const uint8_t* __restrict__ block_ok, int n_frames, uint32_t* __restrict__ mask)
{
    int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n_frames) return;
    const uint8_t* ok = block_ok + (size_t)f * m.nblocks;
    uint32_t out = 0;
    bool carry = false;
    for (int q = 0; q < m.chunks_per_frame; ++q) {
        bool all = true;
        for (int k = 0; k < m.blocks_per_chunk; ++k) all = all && (ok[q * m.blocks_per_chunk + k] != 0);
        if (all && !carry) out |= 1u << q;
        carry = ok[q * m.blocks_per_chunk + m.blocks_per_chunk - 1] == 0;
    }
    mask[f] = out;
}

cudaError_t k2_init_tables(const uint8_t* exp512, const uint8_t* log256)
{
    cudaError_t e = cudaMemcpyToSymbol(c_gf_exp, exp512, 512);
    if (e != cudaSuccess) return e;
    return cudaMemcpyToSymbol(c_gf_log, log256, 256);
}

cudaError_t k2_pack_launch(const Mode& m, const uint8_t* d_cellvals, const uint16_t* d_idx, int n_frames, uint8_t* d_raw, cudaStream_t st)
{
    dim3 grid((m.cap_all + 255) / 256, n_frames);
    k_pack_raw<<<grid, 256, 0, st>>>(m, d_cellvals, d_idx, n_frames, d_raw); count_launch();
    return cudaGetLastError();
}

template <int T, bool FUSED>
static cudaError_t rs_launch_t(const Mode& m, const uint8_t* d_raw, const uint8_t* d_cellvals, const uint16_t* d_idx, int n_frames,
                               uint8_t* d_data, uint8_t* d_ok, const uint8_t* d_rho, int sm_count, cudaStream_t st, int b_begin = 0, int b_count = -1)
{
    if (b_count < 0) b_count = m.nblocks;
    if (m.ecc_block + 4 > kStagePitch || m.ecc_bytes > 8 * T * 4 || m.ecc_bytes > kLaDim) return cudaErrorInvalidValue;
    const size_t smem = ((sizeof(RsSmem<T>) + 127) & ~size_t(127)) + sizeof(uint32_t) * 4 * 256 * 8 * T;
    {   // a per-device attribute: set on every launch (a process may hold contexts on several GPUs)
        cudaError_t e = cudaFuncSetAttribute(k_rs_decode<T, FUSED>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
    }
    const int G = 4 / T;
    long total = (long)n_frames * b_count;
    long units = (total + G - 1) / G;
    long ctas = (units + kRsWarpsPerCta - 1) / kRsWarpsPerCta;
    long max_ctas = (long)sm_count * (T == 1 ? 4 : 2);       // persistent: the table build is amortised over many blocks
    if (ctas > max_ctas) ctas = max_ctas;
    if (ctas < 1) ctas = 1;
    k_rs_decode<T, FUSED><<<(int)ctas, kRsWarpsPerCta * 32, smem, st>>>(m, d_raw, d_cellvals, d_idx, n_frames, b_begin, b_count, d_data, d_ok, d_rho); count_launch();
    return cudaGetLastError();
}

cudaError_t k2_rs_launch(const Mode& m, const uint8_t* d_raw, int n_frames, uint8_t* d_data, uint8_t* d_ok, const uint8_t* d_rho, int sm_count, cudaStream_t st)
{
    if (m.ecc_bytes <= 32) return rs_launch_t<1, false>(m, d_raw, nullptr, nullptr, n_frames, d_data, d_ok, d_rho, sm_count, st);
    return rs_launch_t<2, false>(m, d_raw, nullptr, nullptr, n_frames, d_data, d_ok, d_rho, sm_count, st);
}

cudaError_t k2_rs_fused_launch(const Mode& m, const uint8_t* d_cellvals, const uint16_t* d_idx, int n_frames, uint8_t* d_data,
                               uint8_t* d_ok, const uint8_t* d_rho, int sm_count, cudaStream_t st, int b_begin, int b_count)
{
    if (b_count < 0) b_count = m.nblocks;
    const bool whole = b_begin == 0 && b_count == m.nblocks;
    const bool bits_ok = m.symbol_bits == 4 && m.color_bits == 2 && (!m.legacy || (size_t)m.num_cells * 6 == (size_t)m.cap_all * 8);
    if (whole && bits_ok && m.ecc_block == kFrBlk && m.ecc_bytes <= 32 &&
        m.ecc_bytes <= kLaDim && m.nblocks % 4 == 0 && kFrFrames * (m.nblocks / 4) <= kFrWarps && m.num_cells % 16 == 0 &&
        m.cap_sym % kFrBlk == 0 && (m.nblocks * m.msg_len) % 4 == 0 && ((uintptr_t)d_data & 3u) == 0 && n_frames > 0) {
        const int cell_pitch = m.num_cells;
        const size_t smem = ((sizeof(RsFrSmem) + 127) & ~size_t(127)) + sizeof(uint32_t) * 4 * 256 * 8 +
                            (size_t)kFrFrames * cell_pitch + (size_t)kFrFrames * m.nblocks * kFrPitch;
        if (smem <= 113 * 1024) {
            cudaError_t e = cudaFuncSetAttribute(k_rs_frames, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            if (e != cudaSuccess) return e;
            int groups = (n_frames + kFrFrames - 1) / kFrFrames, ctas = groups < 2 * sm_count ? groups : 2 * sm_count;
            // one warp per unit of the two frames a CTA holds (30 for mode B): no warp sits out the correction phase
            k_rs_frames<<<ctas, 32 * kFrFrames * (m.nblocks / 4), smem, st>>>(m, d_cellvals, d_idx, n_frames, d_data, d_ok, d_rho, cell_pitch); count_launch();
            return cudaGetLastError();
        }
    }
    if (m.ecc_bytes <= 32) return rs_launch_t<1, true>(m, nullptr, d_cellvals, d_idx, n_frames, d_data, d_ok, d_rho, sm_count, st, b_begin, b_count);
    return rs_launch_t<2, true>(m, nullptr, d_cellvals, d_idx, n_frames, d_data, d_ok, d_rho, sm_count, st, b_begin, b_count);
}

// rho[j][0 .. D-1] = coefficients (low to high) of x^(D + j) mod G, G = x^pad g, D = 4 ceil(parity / 4); gen = g low to high,
// gen[parity] = 1.  64 bytes per j, zero padded.  (host)
void k2_remainder_basis(const uint8_t* gen, int parity, const uint8_t* gexp512, const uint8_t* glog256, uint8_t* rho_out /* 4 * 64 */)
{
    const int Pw = (parity + 3) / 4, D = 4 * Pw, pad = D - parity;
    uint8_t G[72] = {0};
    for (int k = 0; k <= parity; ++k) G[pad + k] = gen[k];
    auto mul = [&](uint8_t x, uint8_t y) -> uint8_t { return (x && y) ? gexp512[glog256[x] + glog256[y]] : 0; };
    uint8_t r[64] = {0};
    r[0] = 1;                                                  // x^0, multiplied by x step by step
    for (int e = 1; e <= D + 3; ++e) {
        const uint8_t top = r[D - 1];
        for (int k = D - 1; k > 0; --k) r[k] = r[k - 1];
        r[0] = 0;
        if (top) for (int k = 0; k < D; ++k) r[k] ^= mul(top, G[k]);
        if (e >= D) { for (int k = 0; k < 64; ++k) rho_out[(e - D) * 64 + k] = k < D ? r[k] : 0; }
    }
}

cudaError_t k2_mask_launch(const Mode& m, const uint8_t* d_ok, int n_frames, uint32_t* d_mask, cudaStream_t st)
{
    k_chunk_mask<<<(n_frames + 127) / 128, 128, 0, st>>>(m, d_ok, n_frames, d_mask); count_launch();
    return cudaGetLastError();
}

}  // namespace cb200
