// detect_plan_lists_host.cpp -- TEST HARNESS: runs the per-slot rule of a detect receivers plan's lists (libcimbar_b200/csrc/
// receivers_core.cuh: plan_slot, which k_detect_plan_lists runs on the device) on the CPU, so that it can be compared with the host
// builder of the direct call (detect_lists).  Not part of the product.
//
//   detect_plan_lists_host < in > out
//   in:  int32 n, receivers, n_modes, n_geoms, then n_modes geometry indices, n candidate masks, n receiver indices
//   out: int32 n_modes x n raw receivers, n_modes x n positions; then n_geoms x n present bytes
#include "../../libcimbar_b200/csrc/receivers_core.cuh"

#include <cstdio>
#include <vector>

using namespace cb200::receivers;

int main()
{
    int32_t head[4];
    if (std::fread(head, sizeof(int32_t), 4, stdin) != 4) return 2;
    const int n = head[0], receivers = head[1], n_modes = head[2], n_geoms = head[3];
    if (n_modes < 1 || n_modes > kMaxModes || n_geoms < 1 || n_geoms > n_modes) return 2;
    std::vector<int32_t> group((size_t)n_modes), of((size_t)n);
    std::vector<uint32_t> cand((size_t)n);
    if (std::fread(group.data(), sizeof(int32_t), group.size(), stdin) != group.size() ||
        std::fread(cand.data(), sizeof(uint32_t), cand.size(), stdin) != cand.size() ||
        std::fread(of.data(), sizeof(int32_t), of.size(), stdin) != of.size())
        return 2;
    int g[kMaxModes];
    for (int k = 0; k < n_modes; ++k) g[k] = group[(size_t)k];
    // poisoned outputs: every entry must be written
    std::vector<int32_t> raw((size_t)n_modes * n, 0x5A5A5A5A), at((size_t)n_modes * n, 0x5A5A5A5A);
    std::vector<uint8_t> present((size_t)n_geoms * n, 0xA5);
    for (int i = 0; i < n; ++i) plan_slot(cand[(size_t)i], of[(size_t)i], receivers, n_modes, g, n_geoms, n, i, raw.data(), present.data(), at.data());
    std::fwrite(raw.data(), sizeof(int32_t), raw.size(), stdout);
    std::fwrite(at.data(), sizeof(int32_t), at.size(), stdout);
    std::fwrite(present.data(), 1, present.size(), stdout);
    return 0;
}
