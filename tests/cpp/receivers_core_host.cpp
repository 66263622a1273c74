// receivers_core_host.cpp -- TEST HARNESS: compiles the segmented CCM carry of a batch of several receivers
// (libcimbar_b200/csrc/receivers_core.cuh) for the host and runs it the way k_ccm_carry_receivers (ccm.cu) does, thread by thread
// and phase by phase, so that it can be compared with a sequential per-receiver carry where there is no GPU.  Not part of the
// product; the product runs the same functions in the kernel.
#include "../../libcimbar_b200/csrc/receivers_core.cuh"

#include <vector>

using namespace cb200::receivers;

// n pictures of receivers of[] (each in [0, receivers)) with fit flags valid[]: src[f] = the picture whose fit picture f is decoded
// with (-1: its receiver's entry state); last[r] = the last picture of receiver r (-1: none), which writes its exit state.  threads:
// the block size of the kernel (1024)
extern "C" void rc_carry(const int32_t* of, const uint8_t* valid, int n, int receivers, int threads, int32_t* src, int32_t* last)
{
    std::vector<int32_t> order((size_t)n);
    make_order(of, n, receivers, order.data());
    const int seg = (n + threads - 1) / threads;
    std::vector<Carry> part((size_t)threads);
    for (int t = 0; t < threads; ++t) {
        const int j0 = t * seg < n ? t * seg : n, j1 = j0 + seg < n ? j0 + seg : n;
        part[(size_t)t] = range(of, order.data(), valid, j0, j1);
    }
    std::vector<Carry> incl(part);                       // the block's inclusive max scan, Hillis-Steele as in the kernel
    for (int o = 1; o < threads; o <<= 1) {
        std::vector<Carry> prev(incl);
        for (int t = o; t < threads; ++t) incl[(size_t)t] = combine(prev[(size_t)t], prev[(size_t)(t - o)]);
    }
    for (int r = 0; r < receivers; ++r) last[r] = -1;
    for (int t = 0; t < threads; ++t) {
        const int j0 = t * seg < n ? t * seg : n, j1 = j0 + seg < n ? j0 + seg : n;
        Carry c = t > 0 ? incl[(size_t)(t - 1)] : Carry{-1, 0};
        for (int j = j0; j < j1; ++j) {
            src[order[(size_t)j]] = step(of, order.data(), valid, j, c);
            if (closes(of, order.data(), n, j)) last[of[order[(size_t)j]]] = order[(size_t)j];
        }
    }
}

extern "C" void rc_order(const int32_t* of, int n, int receivers, int32_t* order) { make_order(of, n, receivers, order); }
