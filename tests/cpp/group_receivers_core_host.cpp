// group_receivers_core_host.cpp -- TEST HARNESS: compiles the receivers form of the grouping rule (libcimbar_b200/csrc/combine_core.cuh:
// pair_tiles, segment_starts, assign_segment and the numbering, over the receiver-major order of receivers_core.cuh) for the host, so
// that tests/test_group_receivers_core_host.py can compare it with a numpy restatement where there is no GPU.  Not part of the
// product.  Built as a shared library and called through ctypes.
#include "../../libcimbar_b200/csrc/combine_core.cuh"
#include "../../libcimbar_b200/csrc/receivers_core.cuh"

#include <string.h>

using namespace cb200;

extern "C" {

// the receiver-major order of n pictures of `receivers` receivers (receivers::make_order), as the grouped receivers call builds it
void grc_order(const int32_t* of, int n, int receivers, int32_t* order) { receivers::make_order(of, n, receivers, order); }

// the tile pairs k_pair_match takes: (I, J) pairs into ij (room for cap pairs); returns their number
int grc_tiles(const int32_t* of, int n, int receivers, int tile, int32_t* ij, int cap)
{
    std::vector<int32_t> order((size_t)n);
    receivers::make_order(of, n, receivers, order.data());
    std::vector<int32_t> out;
    combine::pair_tiles(of, order.data(), n, tile, out);
    const int k = (int)(out.size() / 2);
    memcpy(ij, out.data(), sizeof(int32_t) * 2 * (size_t)(k < cap ? k : cap));
    return k;
}

// the assignment over n match rows indexed by position of the receiver-major order (`words` words each), then the table of `slots`
// slots as the device lays it out (combine::group_table with the slots past the count empty) and each group's receiver (-1 past the
// count).  Returns the group count
int grc_assign(const uint32_t* rows, int words, const int32_t* status, const int32_t* of, int n, int receivers, int slots, int32_t* group_of,
               int32_t* offsets, int32_t* members, int32_t* group_receiver)
{
    std::vector<int32_t> map(2 * (size_t)n);
    memcpy(map.data(), of, sizeof(int32_t) * (size_t)n);
    receivers::make_order(of, n, receivers, map.data() + n);
    const int count = combine::assign_receivers(rows, (size_t)words, status, map.data(), n, group_of);
    combine::group_table(group_of, n, slots, offsets, members);
    for (int g = 0; g < slots; ++g) group_receiver[g] = g < count ? of[members[offsets[g]]] : -1;
    return count;
}

}  // extern "C"
