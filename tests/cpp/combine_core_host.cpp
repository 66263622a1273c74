// combine_core_host.cpp -- TEST HARNESS: compiles the combined call's vote and group table (libcimbar_b200/csrc/combine_core.cuh)
// for the host, so that tests/test_combine_core_host.py can compare them with a numpy restatement where there is no GPU.  Not part
// of the product.  Built as a shared library and called through ctypes.
#include "../../libcimbar_b200/csrc/combine_core.cuh"

using namespace cb200::combine;

extern "C" {

int cc_max_group() { return kMaxGroup; }

// the vote of every cell of a group, as k_combine runs it: cells x k value bytes and distances (picture-major), one output per cell
void cc_vote(const uint8_t* v, const uint8_t* d, int k, int cells, uint8_t* out)
{
    uint8_t vv[kMaxGroup], dd[kMaxGroup];
    for (int c = 0; c < cells; ++c) {
        for (int j = 0; j < k; ++j) { vv[j] = v[(size_t)j * cells + c] & kValueBits; dd[j] = d[(size_t)j * cells + c]; }
        out[c] = vote(vv, dd, k);
    }
}

int cc_takes_part(int32_t status) { return takes_part(status) ? 1 : 0; }

int cc_group_error(const int32_t* of, int n, int m, int* at) { return group_error(of, n, m, at); }

void cc_group_table(const int32_t* of, int n, int m, int32_t* offsets, int32_t* members) { group_table(of, n, m, offsets, members); }

}  // extern "C"
