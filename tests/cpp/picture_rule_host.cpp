// picture_rule_host.cpp -- TEST HARNESS: runs the picture descriptor rule (libcimbar_b200/csrc/layout_core.cuh: picture_refused) and
// the per-slot table builder of a plan over device descriptors (plan_slot, which k_plan_pictures runs on the device) on the CPU, so
// that they can be compared with the library's host checks and with pic_table's rules.  Not part of the product.
//
//   picture_rule_host < in > out
//   in:  int32 n, receivers, with_bounds, min_short, max_short, max_long; uint64 standin, blur_base, slot_bytes; then n cb200_picture
//        (40 bytes each) and n int32 receiver indices
//   out: n refused bytes (picture_refused, with the bounds when with_bounds, else without), then per slot plan_slot's PicDesc
//        (56 bytes), int32 group, int32 tiles, uint8 refused (plan_slot needs the bounds: only when with_bounds)
#include "../../libcimbar_b200/csrc/layout_core.cuh"

#include <cstdio>
#include <cstring>
#include <vector>

using namespace cb200;

int main()
{
    int32_t head[6];
    uint64_t addr[3];
    if (std::fread(head, sizeof(int32_t), 6, stdin) != 6 || std::fread(addr, sizeof(uint64_t), 3, stdin) != 3) return 2;
    const int n = head[0], receivers = head[1];
    const bool with_bounds = head[2] != 0;
    const cb200_picture_bounds bounds = {head[3], head[4], head[5]};
    static_assert(sizeof(cb200_picture) == 40 && sizeof(PicDesc) == 56, "the layouts the test writes and reads");
    std::vector<cb200_picture> pics((size_t)n);
    std::vector<int32_t> of((size_t)n);
    if (std::fread(pics.data(), sizeof(cb200_picture), pics.size(), stdin) != pics.size() ||
        std::fread(of.data(), sizeof(int32_t), of.size(), stdin) != of.size())
        return 2;
    for (int i = 0; i < n; ++i) {
        const uint8_t r = layout::picture_refused(pics[(size_t)i], with_bounds ? &bounds : nullptr);
        std::fwrite(&r, 1, 1, stdout);
    }
    if (!with_bounds) return 0;
    for (int i = 0; i < n; ++i) {
        PicDesc d;
        std::memset(&d, 0x5A, sizeof(d));                 // poisoned: every field must be written
        const layout::PlanSlot s = layout::plan_slot(pics.data(), of[(size_t)i] < 0 || of[(size_t)i] >= receivers, bounds, addr[0], addr[1], addr[2], i, d);
        const int32_t gt[2] = {s.group, s.tiles};
        const uint8_t refused = s.refused;
        std::fwrite(&d, sizeof(d), 1, stdout);
        std::fwrite(gt, sizeof(int32_t), 2, stdout);
        std::fwrite(&refused, 1, 1, stdout);
    }
    return 0;
}
