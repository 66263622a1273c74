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

}  // namespace combine
}  // namespace cb200
