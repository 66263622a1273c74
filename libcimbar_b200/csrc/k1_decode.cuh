// k1_decode.cuh -- host-side entry points of the fused K1 kernel (k1_decode.cu)
#pragma once
#include "cb200_common.cuh"
#include "ccm.cuh"

namespace cb200 {
size_t k1_smem_bytes(bool sharpen);
// resident CTAs per SM the grid is sized for: the kernel's launch bounds, four without sharpen, three with it
int k1_ctas_per_sm(bool sharpen);
cudaError_t k1_init_tables(const float* adjust256, const unsigned long long* tiles_L16);
// d_list: NULL = frames 0 .. n_frames-1 of d_rgb; else n_frames batch indices (device memory) -- results stay batch-indexed.
// d_sched != NULL (device memory, with d_list): the list's length, its band count and its first entry in d_list are read there by
// the kernel (n_frames and bands are then ignored), so a selection built on the device needs no host round trip
cudaError_t k1_launch(const Mode& m, const uint8_t* d_rgb, const uint32_t* d_list, int n_frames, int bands, int grid, bool sharpen,
                      uint8_t* d_cellvals, uint32_t* d_dirty, const CcmArg& cc, cudaStream_t stream, const int* d_sched = nullptr);
cudaError_t k1_symbols_launch(const uint16_t* d_windows, const uint8_t* d_cooldown, int n, uint8_t* d_sym, uint8_t* d_off, uint8_t* d_dist, cudaStream_t st);
cudaError_t k1_colors_launch(const Mode& m, const uint8_t* d_rgb, int n, uint8_t* d_color, const CcmArg& cc, cudaStream_t st);
}  // namespace cb200
