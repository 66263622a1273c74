// receivers_order_host.cpp -- TEST HARNESS: compiles the receivers plan's order rule (libcimbar_b200/csrc/receivers_core.cuh:
// empty_slot, slot_receiver, slot_key, rank_part) for the host and runs it the way k_receivers_order (ccm.cu) does -- each slot's
// rank summed over `parts` interleaved lanes -- so that it can be compared with make_order where there is no GPU.  Not part of the
// product.  Every global operator new is counted: the rule must allocate nothing, however many receivers there are.
//
//   receivers_order_host < in > out
//   in:  int32 n, receivers, parts, then n receiver indices
//   out: int32 n map entries (-1 = empty), n order entries, then the number of allocations the rule made
#include "../../libcimbar_b200/csrc/receivers_core.cuh"

#include <cstdio>
#include <cstdlib>
#include <new>
#include <vector>

using namespace cb200::receivers;

static long g_allocations = 0;

void* operator new(std::size_t bytes)
{
    ++g_allocations;
    if (void* p = std::malloc(bytes ? bytes : 1)) return p;
    throw std::bad_alloc();
}
void operator delete(void* p) noexcept { std::free(p); }
void operator delete(void* p, std::size_t) noexcept { std::free(p); }

static void order_rule(const int32_t* of, int n, int receivers, int parts, int32_t* map, int32_t* order)
{
    for (int i = 0; i < n; ++i) {
        const uint64_t k = slot_key(of[i], receivers, i);
        int rank = 0;
        for (int w = 0; w < parts; ++w) rank += rank_part(of, n, receivers, k, w, parts);
        map[i] = slot_receiver(of[i], receivers);
        order[rank] = i;
    }
}

int main()
{
    int32_t head[3];
    if (std::fread(head, sizeof(int32_t), 3, stdin) != 3) return 2;
    const int n = head[0], receivers = head[1], parts = head[2];
    std::vector<int32_t> of((size_t)n), out(2 * (size_t)n + 1, -7);
    if (std::fread(of.data(), sizeof(int32_t), (size_t)n, stdin) != (size_t)n) return 2;
    const long before = g_allocations;
    order_rule(of.data(), n, receivers, parts, out.data(), out.data() + n);
    out[2 * (size_t)n] = (int32_t)(g_allocations - before);
    std::fwrite(out.data(), sizeof(int32_t), out.size(), stdout);
    return 0;
}
