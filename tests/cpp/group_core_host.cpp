// group_core_host.cpp -- TEST HARNESS: compiles the grouping rule of the grouped camera call (libcimbar_b200/csrc/combine_core.cuh:
// agree, match, the packed-symbol helpers k_pair_match uses and the assignment) for the host, so that tests/test_group_core_host.py
// can compare them with a numpy restatement where there is no GPU.  Not part of the product.  Built as a shared library and called
// through ctypes.
#include "../../libcimbar_b200/csrc/combine_core.cuh"

#include <string.h>

using namespace cb200::combine;

extern "C" {

int gc_agree(const uint8_t* a, const uint8_t* b, int cells, int symbol_bits) { return agree(a, b, cells, symbol_bits); }

// agree as k_pair_match counts it: cells / 8 packed words per picture, cells - the differing symbols (cells a multiple of 8)
int gc_agree_packed(const uint8_t* a, const uint8_t* b, int cells, int symbol_bits)
{
    int diff = 0;
    for (int k = 0; k < cells / 8; ++k) {
        uint64_t va, vb;
        memcpy(&va, a + 8 * k, 8);
        memcpy(&vb, b + 8 * k, 8);
        diff += differing_symbols(pack_symbols(va, symbol_bits), pack_symbols(vb, symbol_bits));
    }
    return cells - diff;
}

int gc_match(int agreeing, int cells) { return match(agreeing, cells) ? 1 : 0; }

// the assignment over n match rows of `words` words, then the table of `slots` slots as the device lays it out (combine::group_table
// with the slots past the count empty): offsets[0 .. slots], members[0 .. offsets[slots]).  Returns the group count
int gc_assign(const uint32_t* rows, int words, const int32_t* status, int n, int slots, int32_t* group_of, int32_t* offsets, int32_t* members)
{
    const int count = assign_groups(rows, (size_t)words, status, n, group_of);
    group_table(group_of, n, slots, offsets, members);
    return count;
}

}  // extern "C"
