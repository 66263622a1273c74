// detect_lists_host.cpp -- TEST HARNESS: runs the host builder of a detect receivers call's lists (libcimbar_b200/csrc/
// receivers_core.cuh: detect_lists, make_order) on the CPU, so that it can be compared with a plain model.  Not part of the product.
//
//   detect_lists_host < in > out
//   in:  int32 n, receivers, n_modes, then n_modes geometry indices, n candidate masks, n receiver indices
//   out: int32, per geometry g < n_modes: |U_g| and U_g; per mode: |P_k|, the map's length and the map; then the n_modes x n positions
#include "../../libcimbar_b200/csrc/receivers_core.cuh"

#include <cstdio>
#include <vector>

using namespace cb200::receivers;

int main()
{
    int32_t head[3];
    if (std::fread(head, sizeof(int32_t), 3, stdin) != 3) return 2;
    const int n = head[0], receivers = head[1], n_modes = head[2];
    if (n_modes < 1 || n_modes > kMaxModes) return 2;
    std::vector<int32_t> group((size_t)n_modes), of((size_t)n);
    std::vector<uint32_t> cand((size_t)n);
    if (std::fread(group.data(), sizeof(int32_t), group.size(), stdin) != group.size() ||
        std::fread(cand.data(), sizeof(uint32_t), cand.size(), stdin) != cand.size() ||
        std::fread(of.data(), sizeof(int32_t), of.size(), stdin) != of.size())
        return 2;
    DetectLists l;
    detect_lists(cand.data(), of.data(), n, receivers, n_modes, group.data(), l);
    std::vector<int32_t> out;
    for (int g = 0; g < n_modes; ++g) {
        out.push_back((int32_t)l.slots[g].size());
        out.insert(out.end(), l.slots[g].begin(), l.slots[g].end());
    }
    for (int k = 0; k < n_modes; ++k) {
        out.push_back(l.count[k]);
        out.push_back((int32_t)l.map[k].size());
        out.insert(out.end(), l.map[k].begin(), l.map[k].end());
    }
    out.insert(out.end(), l.pos.begin(), l.pos.end());
    std::fwrite(out.data(), sizeof(int32_t), out.size(), stdout);
    return 0;
}
