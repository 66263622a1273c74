// combine_core.cuh -- the per-cell vote of cb200_scan_extract_decode_chunks_combined_dev (include/cb200.h): several pictures of one
// frame ("a group") give one frame of cell bytes, which then takes the ordinary de-interleave, Reed-Solomon and chunk-mask rule.
//
// Picture i takes part in group g iff group_of[i] == g and its extract status is 1 or 2.  For each cell the value bits (bits 0-6 of
// the cell byte: symbol | colour << symbol_bits) of the participating pictures are compared and the winner is, in this order:
//   1. the value held by the most pictures;
//   2. among values tied on count, the one whose smallest walk distance (CellTrace::distance) among its pictures is smallest;
//   3. then the value of the earliest picture in batch order.
// One picture gives its own bytes; two give the cell of the lower distance; three or more also outvote a wrong colour, which the
// symbol distance cannot see.  k_combine (scan.cu) runs vote() per (group, cell); tests/cpp/combine_core_host.cpp runs the same
// functions on the CPU.
#pragma once
#include <stdint.h>
#include <algorithm>
#include <vector>

#include "scan_core.cuh"            // CB_HD

namespace cb200 {
namespace combine {

constexpr int kMaxGroup = 16;       // pictures with one group index: the vote loop's bound, larger groups are refused
constexpr uint8_t kValueBits = 0x7F;
constexpr int kPairTile = 64;       // pictures per side of a k_pair_match tile (group.cu)

// the winning value of k participating pictures' value bits v[0 .. k) and walk distances d[0 .. k), both in batch order (k >= 1)
CB_HD uint8_t vote(const uint8_t* v, const uint8_t* d, int k)
{
    uint8_t best = v[0];
    int best_count = 0, best_dist = 256;
    for (int i = 0; i < k; ++i) {
        bool seen = false;
        for (int j = 0; j < i; ++j) seen |= v[j] == v[i];
        if (seen) continue;                  // the value's first picture stands for it: the earliest one, for rule 3
        int count = 0, dist = 256;
        for (int j = 0; j < k; ++j)
            if (v[j] == v[i]) { ++count; dist = d[j] < dist ? d[j] : dist; }
        if (count > best_count || (count == best_count && dist < best_dist)) { best = v[i]; best_count = count; best_dist = dist; }
    }
    return best;
}

// an extract status that takes part in its group
CB_HD bool takes_part(int32_t status) { return status == 1 || status == 2; }

// the host side.  group_error: 0 when group_of[0 .. n) is a valid assignment to m groups; else 1 for an entry outside [-1, m) and 2
// for a group of more than kMaxGroup pictures, with *at = the offending picture: the first one outside, or the one that exceeds the
// cap (whichever comes first in batch order).  Its memory and time are bounded by n, whatever m is (m is checked
// against max_frames only after the context): m is compared with, never used as a size
inline int group_error(const int32_t* group_of, int n, int m, int* at)
{
    int outside = -1;
    for (int i = 0; i < n && outside < 0; ++i)
        if (group_of[i] < -1 || group_of[i] >= m) outside = i;
    std::vector<uint64_t> keys;                  // (group, picture) of the pictures in a group before the first one outside
    for (int i = 0; i < (outside < 0 ? n : outside); ++i)
        if (group_of[i] >= 0) keys.push_back((uint64_t)(uint32_t)group_of[i] << 32 | (uint32_t)i);
    std::sort(keys.begin(), keys.end());
    int over = -1;                               // the earliest picture that is its group's (kMaxGroup + 1)-th
    for (size_t j = kMaxGroup; j < keys.size(); ++j)
        if (keys[j] >> 32 == keys[j - kMaxGroup] >> 32) {
            const int i = (int)(uint32_t)keys[j];
            if (over < 0 || i < over) over = i;
            while (j + 1 < keys.size() && keys[j + 1] >> 32 == keys[j] >> 32) ++j;    // later members of that group come later
        }
    if (over >= 0) { *at = over; return 2; }
    if (outside >= 0) { *at = outside; return 1; }
    return 0;
}

// the group table of a valid assignment: offsets[0 .. m] (CSR: group g's members are members[offsets[g] .. offsets[g + 1])) and the
// members, a stable counting sort of the pictures with group_of >= 0 (each group's pictures in batch order).  members holds
// offsets[m] entries
inline void group_table(const int32_t* group_of, int n, int m, int32_t* offsets, int32_t* members)
{
    for (int g = 0; g <= m; ++g) offsets[g] = 0;
    for (int i = 0; i < n; ++i) if (group_of[i] >= 0) ++offsets[group_of[i] + 1];
    for (int g = 0; g < m; ++g) offsets[g + 1] += offsets[g];
    std::vector<int32_t> next(offsets, offsets + (m > 0 ? m : 0));
    for (int i = 0; i < n; ++i) if (group_of[i] >= 0) members[next[(size_t)group_of[i]]++] = i;
}

// ---- finding the groups (cb200_scan_extract_decode_chunks_grouped_dev): pictures of one frame agree on their cells' symbol bits.
// The colour bits do not take part: a colour cast changes them on a third of the cells of the same frame.
//   match(i, j): both pictures take part (takes_part) and 2 * agree(i, j) >= cells, where agree counts the cells whose symbol bits
//                (value & ((1 << symbol_bits) - 1), from the final cell bytes) are equal.
//   assignment, in batch order: a picture that takes part joins the group of the earliest earlier leader it matches whose group has
//                fewer than kMaxGroup pictures; with none it becomes a leader.  A group is a leader with at least one other picture;
//                groups are numbered in their leaders' batch order, and every other picture gets group -1.
// k_pair_match (scan.cu) packs the symbol bits eight cells to a word (pack_symbols) and counts differing ones (differing_symbols);
// k_assign_groups applies the assignment over its match rows with the same word helpers (open_matches, join) as assign_groups here.

// the number of cells of a and b (cells bytes each) whose symbol bits are equal
CB_HD int agree(const uint8_t* a, const uint8_t* b, int cells, int symbol_bits)
{
    const int mask = (1 << symbol_bits) - 1;
    int same = 0;
    for (int k = 0; k < cells; ++k) same += ((a[k] ^ b[k]) & mask) == 0;
    return same;
}

CB_HD bool match(int agreeing, int cells) { return 2 * agreeing >= cells; }

// the symbol bits (symbol_bits <= 4) of eight cell bytes (little-endian in v) as eight nibbles, cell k at bits 4k
CB_HD uint32_t pack_symbols(uint64_t v, int symbol_bits)
{
    v &= 0x0101010101010101ull * (uint64_t)((1u << symbol_bits) - 1);
    v = (v | (v >> 4)) & 0x00FF00FF00FF00FFull;
    v = (v | (v >> 8)) & 0x0000FFFF0000FFFFull;
    return (uint32_t)(v | (v >> 16));
}

// the number of nibbles in which two packed words differ
CB_HD int differing_symbols(uint32_t a, uint32_t b)
{
    uint32_t x = a ^ b;
    x |= x >> 2;
    x |= x >> 1;
#if defined(__CUDA_ARCH__)
    return __popc(x & 0x11111111u);
#else
    return __builtin_popcount(x & 0x11111111u);
#endif
}

// match rows: row i holds bit j (word j / 32, bit j % 32) set iff match(i, j), for j < i; bits from i on are not read.  open: one bit
// per picture, set while it is a leader whose group has fewer than kMaxGroup pictures.  open_matches: word w of row i's candidates
// j in [from, i) (from: the first picture of i's segment, below)
CB_HD uint32_t open_matches(const uint32_t* row, const uint32_t* open, int i, int w, int from = 0)
{
    if (w > i >> 5 || w < from >> 5) return 0;
    const uint32_t below = w < i >> 5 ? ~0u : (1u << (i & 31)) - 1u;
    const uint32_t above = w > from >> 5 ? ~0u : ~((1u << (from & 31)) - 1u);
    return row[w] & open[w] & below & above;
}

// picture i joins leader j (j == i: i leads a new group); size[] counts each leader's pictures.  shared: on the device, the open bits
// change atomically, because k_assign_groups' warps work on segments that may share a word of `open` (several segments)
CB_HD void join(int i, int j, int32_t* size, uint32_t* open, bool shared = false)
{
#if defined(__CUDA_ARCH__)
    if (shared) {
        if (j == i) { size[i] = 1; atomicOr(&open[i >> 5], 1u << (i & 31)); return; }
        if (++size[j] == kMaxGroup) atomicAnd(&open[j >> 5], ~(1u << (j & 31)));
        return;
    }
#endif
    if (j == i) { size[i] = 1; open[i >> 5] |= 1u << (i & 31); return; }
    if (++size[j] == kMaxGroup) open[j >> 5] &= ~(1u << (j & 31));
}

// ---- receivers (cb200_scan_extract_decode_chunks_grouped_receivers_dev): match(i, j) also requires receiver_of[i] == receiver_of[j].
// The pictures are taken in the receiver-major order (receivers_core.cuh make_order: a stable counting sort of the receiver map), in
// which each receiver's pictures form one segment [s, e) of positions, in batch order.  The match rows are indexed by position, so a
// picture's candidates are the positions [s, p) of its own segment and the rule inside a segment is the one above.  The grouped call is
// the one-receiver case: one segment, the identity order.
//   pair_tiles: the kPairTile-position tile pairs (I, J <= I) of k_pair_match that hold at least one same-receiver pair p > q, each
//               once, in increasing (I, J) order.  Their number is at most sum over segments of (tiles the segment spans)^2: it grows
//               with the sum of n_r^2, and neither it nor the work depends on the number of receivers.
//   segment_starts: the first position of every segment, then n.
//   assign_segment: the assignment over one segment's positions: lead[p] = the position of p's leader (-1: does not take part).
//   number_groups: groups numbered in their leaders' batch order, across the segments (lead and size indexed by batch index here).
inline void pair_tiles(const int32_t* of, const int32_t* order, int n, int tile, std::vector<int32_t>& ij)
{
    std::vector<uint64_t> keys;
    for (int s = 0, e; s < n; s = e) {
        for (e = s + 1; e < n && of[order[e]] == of[order[s]]; ++e) {}
        if (e - s < 2) continue;
        const int t0 = s / tile, t1 = (e - 1) / tile;
        for (int I = t0; I <= t1; ++I)
            for (int J = t0; J <= I; ++J) {
                // a diagonal tile needs two of the segment's positions in it
                if (I == J && std::min(e, (I + 1) * tile) - std::max(s, I * tile) < 2) continue;
                keys.push_back((uint64_t)I << 32 | (uint32_t)J);
            }
    }
    std::sort(keys.begin(), keys.end());
    keys.erase(std::unique(keys.begin(), keys.end()), keys.end());
    ij.resize(2 * keys.size());
    for (size_t k = 0; k < keys.size(); ++k) { ij[2 * k] = (int32_t)(keys[k] >> 32); ij[2 * k + 1] = (int32_t)(uint32_t)keys[k]; }
}

inline void segment_starts(const int32_t* of, const int32_t* order, int n, std::vector<int32_t>& starts)
{
    starts.clear();
    for (int p = 0; p < n; ++p)
        if (p == 0 || of[order[p]] != of[order[p - 1]]) starts.push_back(p);
    starts.push_back(n);
}

// order: NULL for the identity.  k_assign_groups runs the same loop in one warp per segment, searching a row's words 32 at a time
inline void assign_segment(const uint32_t* rows, size_t words, const int32_t* status, const int32_t* order, int s, int e, int32_t* lead,
                           int32_t* size, uint32_t* open)
{
    for (int p = s; p < e; ++p) {
        lead[p] = -1;
        if (!takes_part(status[order ? order[p] : p])) continue;
        int j = p;
        for (int w = s >> 5; w <= p >> 5 && j == p; ++w) {
            const uint32_t x = open_matches(rows + (size_t)p * words, open, p, w, s);
            if (x) j = 32 * w + __builtin_ctz(x);
        }
        join(p, j, size, open);
        lead[p] = j;
    }
}

inline int number_groups(const int32_t* lead, const int32_t* size, int n, int32_t* group_of)
{
    std::vector<int32_t> number((size_t)n, -1);
    int groups = 0;
    for (int i = 0; i < n; ++i)
        if (lead[i] == i && size[i] >= 2) number[(size_t)i] = groups++;
    for (int i = 0; i < n; ++i) group_of[i] = lead[i] < 0 ? -1 : number[(size_t)lead[i]];
    return groups;
}

// the assignment of the rule over n pictures' match rows (`words` words each) and extract statuses: group_of[0 .. n), returns the
// number of groups.  (k_assign_groups searches a row's words in parallel, a warp's lanes over 32 words at a time)
inline int assign_groups(const uint32_t* rows, size_t words, const int32_t* status, int n, int32_t* group_of)
{
    std::vector<uint32_t> open(words ? words : 1, 0u);
    std::vector<int32_t> size((size_t)n, 0), lead((size_t)n, -1);
    assign_segment(rows, words, status, nullptr, 0, n, lead.data(), size.data(), open.data());
    return number_groups(lead.data(), size.data(), n, group_of);
}

// the receivers form: rows indexed by position of the receiver-major order (map: the n receivers, then the order), statuses and
// group_of by batch index.  Each segment is assigned on its own, then the leaders are numbered in batch order.  Returns the count
inline int assign_receivers(const uint32_t* rows, size_t words, const int32_t* status, const int32_t* map, int n, int32_t* group_of)
{
    const int32_t* order = map + n;
    std::vector<int32_t> starts;
    segment_starts(map, order, n, starts);
    std::vector<uint32_t> open(words ? words : 1, 0u);
    std::vector<int32_t> psize((size_t)n, 0), plead((size_t)n, -1), size((size_t)n, 0), lead((size_t)n, -1);
    for (size_t k = 0; k + 1 < starts.size(); ++k)
        assign_segment(rows, words, status, order, starts[k], starts[k + 1], plead.data(), psize.data(), open.data());
    for (int p = 0; p < n; ++p) {
        lead[(size_t)order[p]] = plead[(size_t)p] < 0 ? -1 : order[plead[(size_t)p]];
        size[(size_t)order[p]] = psize[(size_t)p];
    }
    return number_groups(lead.data(), size.data(), n, group_of);
}

// ---- a history (cb200_scan_extract_decode_chunks_grouped_history_dev): the grouped call's rule over a batch that follows the
// undecoded pictures of earlier calls.  The device lays out N = H + n positions: history slot s < H holds the s-th oldest history
// picture when s < h (position status 1: always eligible) and is empty otherwise (status 0: never eligible); batch picture i sits
// at position first = H plus i with its extract status.  The empty slots take part in nothing, so the assignment over the positions
// is the rule's over [0, h) followed by the batch.  Then:
//   groups:   a group of the assignment that has a batch member (its last member, in position order, lies at or after `first`);
//             the others (history pictures only) are not decoded again.  Numbered in their leaders' position order.
//   complete: a record whose chunk mask has all chunks_per_frame bits set (k_chunk_mask sets them all when every block decodes).
//   done:     a group whose record is complete or one of whose batch members' own records is complete.
//   keep:     a position that is eligible, is in no done group and, in the batch, whose own record is not complete; of those the
//             last H stay, oldest first (keep_destination), so the pictures of a decoded frame leave at once and the rest first in,
//             first out.
// history_number and history_keep are the host restatements of k_history_groups and k_history_keep (history.cu), which apply the
// same helpers per position
CB_HD int32_t history_slot_status(int s, int h) { return s < h ? 1 : 0; }

CB_HD uint32_t complete_mask(int chunks_per_frame) { return chunks_per_frame >= 32 ? ~0u : (1u << chunks_per_frame) - 1u; }

CB_HD bool complete(uint32_t mask, int chunks_per_frame) { return mask == complete_mask(chunks_per_frame); }

CB_HD bool has_batch_member(int last_member, int first) { return last_member >= first; }

CB_HD bool keeps(int p, int first, int32_t status, bool own_complete, bool group_done)
{
    return takes_part(status) && !group_done && (p < first || !own_complete);
}

// the slot of the rank-th of `kept` kept positions among the last `capacity` of them, or < 0 when it leaves
CB_HD int keep_destination(int rank, int kept, int capacity) { return rank - (kept > capacity ? kept - capacity : 0); }

// the groups of the call from the assignment over the positions (of[0 .. N), m groups): pos_group[p] = p's group of the call or -1.
// Returns the number of groups
inline int history_number(const int32_t* of, int N, int first, int m, int32_t* pos_group)
{
    std::vector<int32_t> last((size_t)(m > 0 ? m : 0), -1), number((size_t)(m > 0 ? m : 0), -1);
    for (int p = 0; p < N; ++p) if (of[p] >= 0) last[(size_t)of[p]] = p;
    int groups = 0;
    for (int g = 0; g < m; ++g) if (has_batch_member(last[(size_t)g], first)) number[(size_t)g] = groups++;
    for (int p = 0; p < N; ++p) pos_group[p] = of[p] < 0 ? -1 : number[(size_t)of[p]];
    return groups;
}

// the new history: own[i] the batch pictures' chunk masks, gmask[g] the groups' (count groups), status the positions'.  src[s] = the
// position of the new slot s (s < the returned h); the history keeps `capacity` pictures at most
inline int history_keep(const int32_t* status, int N, int first, const uint32_t* own, const int32_t* pos_group, int count,
                        const uint32_t* gmask, int chunks_per_frame, int capacity, int32_t* src)
{
    std::vector<uint8_t> done((size_t)(count > 0 ? count : 0), 0);
    for (int g = 0; g < count; ++g) done[(size_t)g] = complete(gmask[g], chunks_per_frame);
    for (int p = first; p < N; ++p)
        if (pos_group[p] >= 0 && complete(own[p - first], chunks_per_frame)) done[(size_t)pos_group[p]] = 1;
    std::vector<int32_t> kept;
    for (int p = 0; p < N; ++p) {
        const bool own_complete = p >= first && complete(own[p - first], chunks_per_frame);
        if (keeps(p, first, status[p], own_complete, pos_group[p] >= 0 && done[(size_t)pos_group[p]])) kept.push_back(p);
    }
    int h = 0;
    for (int r = 0; r < (int)kept.size(); ++r) {
        const int s = keep_destination(r, (int)kept.size(), capacity);
        if (s >= 0) { src[s] = kept[(size_t)r]; h = s + 1; }
    }
    return h;
}

}  // namespace combine
}  // namespace cb200
