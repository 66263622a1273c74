// receivers_core.cuh -- the CCM carry of a batch whose pictures belong to several receivers (include/cb200.h, the _receivers_dev
// calls): each receiver is one reference Decoder, whose CimbDecoder keeps the CCM of its last fit (CimbDecoder.cpp:69-85).  So
// picture f takes the fit of the last picture g <= f of the same receiver that has one, else that receiver's entry state.
//
// The host lists the batch receiver-major (`order`: a stable counting sort of the receiver map, so each receiver's pictures stay in
// batch order and form one segment).  Over that order, "the last position with a fit" and "the last segment start" are both
// running maxima: a position takes the fit at the first one when it is not before the second, else its receiver's entry state.
// k_ccm_carry_receivers (ccm.cu) splits the order into one contiguous range per thread, combines the ranges' maxima with a block
// scan and replays each range from its prefix.  Every function is __host__ __device__ so that tests/cpp/receivers_core_host.cpp
// runs the same rule on the CPU.
#pragma once
#include <stdint.h>
#include <vector>

#include "scan_core.cuh"            // CB_HD

namespace cb200 {
namespace receivers {

// over a range of the order: the last position with a fit (-1: none) and the last segment start (0: none, position 0 starts one)
struct Carry { int fit, start; };

CB_HD Carry combine(Carry a, Carry b) { return {a.fit > b.fit ? a.fit : b.fit, a.start > b.start ? a.start : b.start}; }

// position j of the order opens its receiver's segment / closes it
CB_HD bool opens(const int32_t* of, const int32_t* order, int j) { return j == 0 || of[order[j]] != of[order[j - 1]]; }
CB_HD bool closes(const int32_t* of, const int32_t* order, int n, int j) { return j == n - 1 || of[order[j + 1]] != of[order[j]]; }

// positions [j0, j1) on their own
CB_HD Carry range(const int32_t* of, const int32_t* order, const uint8_t* valid, int j0, int j1)
{
    Carry c = {-1, 0};
    for (int j = j0; j < j1; ++j) {
        if (opens(of, order, j)) c.start = j;
        if (valid[order[j]]) c.fit = j;
    }
    return c;
}

// position j after the positions before it (c: their carry, updated): the picture whose fit picture order[j] is decoded with, or
// -1 for its receiver's entry state
CB_HD int step(const int32_t* of, const int32_t* order, const uint8_t* valid, int j, Carry& c)
{
    if (opens(of, order, j)) c.start = j;
    if (valid[order[j]]) c.fit = j;
    return c.fit >= c.start ? order[c.fit] : -1;
}

// the host side: the stable receiver-major order of n pictures of receivers [0, receivers), every of[i] in range or -1 for an empty
// slot (a detect receivers call's, below), which goes after every other.  (A receiver flags table's refused receivers are emptied
// on the device after the order is built: their runs of -1 stay where their receivers were)
inline void make_order(const int32_t* of, int n, int receivers, int32_t* order)
{
    std::vector<int32_t> first((size_t)receivers + 2, 0);
    auto bucket = [&](int i) { return (size_t)(of[i] < 0 ? receivers : of[i]); };
    for (int i = 0; i < n; ++i) ++first[bucket(i) + 1];
    for (int r = 0; r < receivers; ++r) first[(size_t)r + 1] += first[(size_t)r];
    for (int i = 0; i < n; ++i) order[first[bucket(i)]++] = i;
}

// The host side of a detect receivers call (cb200_detect_scan_extract_decode_chunks_receivers_dev, detect.cu).  Picture i is decoded
// under mode k when bit k of cand[i] is set; P_k: those pictures in batch order.  The modes of one frame geometry (group[k]) share
// one sub-batch U_g, the batch-ordered union of their P_k: it is extracted, deskewed and walked once.  For mode k, a position of U_g
// outside P_k is an empty slot -- receiver -1, after every other position in the order -- as in a receivers plan's map
constexpr int kMaxModes = 5;                 // detect.cu's kDetectModes
struct DetectLists {
    std::vector<int32_t> slots[kMaxModes];   // per geometry: U_g's batch indices
    std::vector<int32_t> map[kMaxModes];     // per mode with P_k nonempty: |U_g| receivers (-1: empty), then the order
    std::vector<int32_t> pos;                // n_modes x n: picture i's position in U_{group[k]} when i is in P_k, else -1
    int count[kMaxModes] = {};               // |P_k|
};
inline void detect_lists(const uint32_t* cand, const int32_t* of, int n, int receivers, int n_modes, const int* group, DetectLists& l)
{
    uint32_t modes_of[kMaxModes] = {};       // per geometry: its modes' bits
    for (int k = 0; k < n_modes; ++k) { modes_of[group[k]] |= 1u << k; l.count[k] = 0; l.map[k].clear(); }
    for (int g = 0; g < kMaxModes; ++g) l.slots[g].clear();
    l.pos.assign((size_t)n_modes * (size_t)n, -1);
    for (int i = 0; i < n; ++i)
        for (int g = 0; g < n_modes; ++g) {
            if (!(cand[i] & modes_of[g])) continue;
            const int at = (int)l.slots[g].size();
            l.slots[g].push_back(i);
            for (int k = 0; k < n_modes; ++k)
                if (group[k] == g && (cand[i] >> k & 1u)) { l.pos[(size_t)k * n + i] = at; ++l.count[k]; }
        }
    for (int k = 0; k < n_modes; ++k) {
        if (!l.count[k]) continue;
        const std::vector<int32_t>& u = l.slots[group[k]];
        const int m = (int)u.size();
        l.map[k].resize(2 * (size_t)m);
        for (int j = 0; j < m; ++j) l.map[k][(size_t)j] = (cand[u[(size_t)j]] >> k & 1u) ? of[u[(size_t)j]] : -1;
        make_order(l.map[k].data(), m, receivers, l.map[k].data() + m);
    }
}

// The device side (a receivers camera plan, whose map is read at replay time, k_receivers_order in ccm.cu): the same order, built
// without a pass over the receivers, and with "empty" slots -- a receiver outside [0, receivers) -- after every other slot.  Slot i
// sorts by key(i) = (receiver, i), an empty slot's receiver counting as 2^32 - 1; the keys are distinct, and the position of slot i
// is its rank, the number of slots with a smaller key.  On the non-empty slots that is make_order's stable counting sort.  Work
// and memory depend on n only: a service may bind 10^6 receivers.
CB_HD bool empty_slot(int32_t r, int receivers) { return r < 0 || r >= receivers; }
// the receiver a kernel reads for a slot: -1 for an empty one, so that the empty slots form one run at the end of the order
CB_HD int32_t slot_receiver(int32_t r, int receivers) { return empty_slot(r, receivers) ? -1 : r; }
CB_HD uint64_t slot_key(int32_t r, int receivers, int i)
{
    return ((uint64_t)(empty_slot(r, receivers) ? 0xFFFFFFFFu : (uint32_t)r) << 32) | (uint32_t)i;
}
// the slots j = j0, j0 + stride, ... < n whose key is below k: one lane's part of a rank
CB_HD int rank_part(const int32_t* of, int n, int receivers, uint64_t k, int j0, int stride)
{
    int below = 0;
    for (int j = j0; j < n; j += stride) below += slot_key(of[j], receivers, j) < k;
    return below;
}

// The device side of a detect receivers call (a detect receivers camera plan, whose candidates and map are read at replay time:
// k_detect_plan_lists in detect.cu).  There are no sub-batches: every geometry works on all n slots, and slot i is picture i.  Slot
// i with candidates cand and receiver r is empty when r lies outside [0, receivers) or cand has no bit below n_modes (higher bits
// are ignored); otherwise mode k decodes it when bit k is set.  plan_slot writes slot i's part of the lists:
//   raw[k n + i]      mode k's receiver of the slot, -1 where k does not decode it (an empty slot of mode k's map);
//   present[g n + i]  1 when some mode of geometry g decodes it, else 0: the geometry's walk skips the slot;
//   at[k n + i]       i when k decodes it, else -1 (detect_lists' pos, with each geometry's sub-batch left in place).
// So compacting raw[k], at[k] over the present slots of group[k] gives detect_lists on the non-empty slots alone
CB_HD uint32_t plan_modes(uint32_t cand, int32_t r, int receivers, int n_modes)
{
    return empty_slot(r, receivers) ? 0u : cand & ((1u << n_modes) - 1u);
}
CB_HD void plan_slot(uint32_t cand, int32_t r, int receivers, int n_modes, const int* group, int n_geoms, int n, int i, int32_t* raw,
                     uint8_t* present, int32_t* at)
{
    const uint32_t modes = plan_modes(cand, r, receivers, n_modes);
    uint32_t geoms = 0;
    for (int k = 0; k < n_modes; ++k) {
        const bool in = (modes >> k & 1u) != 0;
        raw[(size_t)k * n + i] = in ? r : -1;
        at[(size_t)k * n + i] = in ? i : -1;
        if (in) geoms |= 1u << group[k];
    }
    for (int g = 0; g < n_geoms; ++g) present[(size_t)g * n + i] = (uint8_t)(geoms >> g & 1u);
}

// A receiver flags table (cb200_scan_extract_decode_chunks_receivers_flags_dev and its plan): one word per receiver with that
// receiver's own sharpen policy and colour correction, read on the device.  A word is valid when it holds no bit but these four, and
// at most one of each pair (as check_camera_flags requires of a call's flags); a receiver with an invalid word is refused.  Bits
// 0x2 SHARPEN, 0x20 SHARPEN_IF_NEEDED, 0x4 CC_SIMPLE, 0x8 CC_FIT (include/cb200.h)
constexpr uint32_t kWordSharpen = 0x2u, kWordSharpenIfNeeded = 0x20u, kWordCcSimple = 0x4u, kWordCcFit = 0x8u;
constexpr uint32_t kWordBits = kWordSharpen | kWordSharpenIfNeeded | kWordCcSimple | kWordCcFit;
CB_HD bool word_refused(uint32_t w)
{
    return (w & ~kWordBits) != 0 || (w & (kWordSharpen | kWordSharpenIfNeeded)) == (kWordSharpen | kWordSharpenIfNeeded) ||
           (w & (kWordCcSimple | kWordCcFit)) == (kWordCcSimple | kWordCcFit);
}
// a valid word's sharpen decision for a picture whose extract status is st (2: NEEDS_SHARPEN), as the call with those flags makes it
CB_HD bool word_sharpens(uint32_t w, int st) { return (w & kWordSharpen) != 0 || ((w & kWordSharpenIfNeeded) != 0 && st == 2); }
// a valid word whose receiver's CCM passes through the call unchanged (no CC bit, or CC_FIT in a mode that never fits: `fits` false),
// as the call with those flags leaves it; its pictures decode with the receiver's matrix, the identity when it is inactive
CB_HD bool word_passes(uint32_t w, bool fits) { return !(w & kWordCcSimple) && !((w & kWordCcFit) && fits); }

}  // namespace receivers
}  // namespace cb200
