// group_history_core_host.cpp -- TEST HARNESS: compiles the history rule of the grouped history call (libcimbar_b200/csrc/combine_core.cuh:
// the position statuses, the assignment over the positions, history_number's "at least one batch member" numbering and history_keep's
// done-group, keep and last-H rule) for the host, so that tests/test_group_history_core_host.py can compare them with
// tests/history_fixtures.history_rule where there is no GPU.  Not part of the product.  Built as a shared library and called through ctypes.
#include "../../libcimbar_b200/csrc/combine_core.cuh"

#include <vector>

using namespace cb200::combine;

extern "C" {

// one call as the device lays it out: H history slots (h of them full), then n batch pictures with their statuses.  rows: the match
// rows over the N = H + n positions (`words` words each).  own: the batch's chunk masks; gmask: the masks of the groups' records in
// slot order (n slots).  Out: group_of (n), pos_group (N), src (H: the new history's positions).  Returns count << 16 | new h
int gh_rule(const uint32_t* rows, int words, int H, int h, const int32_t* batch_status, int n, const uint32_t* own, const uint32_t* gmask,
            int chunks_per_frame, int32_t* group_of, int32_t* pos_group, int32_t* src)
{
    const int N = H + n;
    std::vector<int32_t> status((size_t)N), of((size_t)N);
    for (int p = 0; p < N; ++p) status[(size_t)p] = p < H ? history_slot_status(p, h) : batch_status[p - H];
    const int m = assign_groups(rows, (size_t)words, status.data(), N, of.data());
    const int count = history_number(of.data(), N, H, m, pos_group);
    for (int i = 0; i < n; ++i) group_of[i] = pos_group[H + i];
    const int kept = history_keep(status.data(), N, H, own, pos_group, count, gmask, chunks_per_frame, H, src);
    return count << 16 | kept;
}

int gh_complete(uint32_t mask, int chunks_per_frame) { return complete(mask, chunks_per_frame) ? 1 : 0; }

int gh_destination(int rank, int kept, int capacity) { return keep_destination(rank, kept, capacity); }

}  // extern "C"
