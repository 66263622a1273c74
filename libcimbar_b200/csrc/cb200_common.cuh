// cb200_common.cuh -- shared definitions for the sm_90a decode kernels.
// Geometry mirrors cimbar::conf (reference: src/lib/cimb_translator/GridConf.h:8-190, Config.h:20-175).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace cb200 {

// kernel launches issued by this library in this process (cb200_launch_count): every `<<<>>>` is followed by count_launch()
void count_launch(int n = 1);

// A grow-only buffer of `T` in device memory (pinned host memory with kPinned) that owns its allocation.  ensure() keeps the
// buffer, and what it holds, when it is large enough; otherwise it frees the old memory before it allocates -- cudaFree
// synchronises the device, so no kernel still reads the old buffer, and the peak stays one buffer.
template <typename T, bool kPinned = false>
class Buffer {
public:
    Buffer() = default;
    Buffer(const Buffer&) = delete;
    Buffer& operator=(const Buffer&) = delete;
    ~Buffer() { release(); }
    cudaError_t ensure(size_t count)
    {
        if (count <= cap_) return cudaSuccess;
        release();
        const cudaError_t e = kPinned ? cudaMallocHost((void**)&p_, count * sizeof(T)) : cudaMalloc((void**)&p_, count * sizeof(T));
        if (e == cudaSuccess) cap_ = count; else p_ = nullptr;
        return e;
    }
    void swap(Buffer& o) { T* p = p_; p_ = o.p_; o.p_ = p; const size_t c = cap_; cap_ = o.cap_; o.cap_ = c; }
    T* get() const { return p_; }
    operator T*() const { return p_; }
    size_t capacity() const { return cap_; }   // elements
private:
    void release() { if (p_) { if (kPinned) cudaFreeHost(p_); else cudaFree(p_); } p_ = nullptr; cap_ = 0; }
    T* p_ = nullptr;
    size_t cap_ = 0;
};
template <typename T> using DevBuf = Buffer<T>;
template <typename T> using PinnedBuf = Buffer<T, true>;

constexpr int kMaxCells = 12544;   // 112*112
constexpr int kCellSize = 8;       // Config::cell_size() is constexpr 8 (Config.h:106-110)
constexpr int kSpacing = 9;        // every 8x8 mode uses cell_size+1 (GridConf.h:121-189)

// POD mode description, passed to kernels by value (lives in the kernel parameter bank = constant memory).
struct Mode {
    int mode_val;
    int color_bits, symbol_bits;
    int ecc_bytes, ecc_block;          // RS(ecc_block, ecc_block - ecc_bytes), GridConf.h:128-129
    int width, height;                 // image_size_x/y
    int cell_offset;                   // first cell coordinate (8 or 9)
    int cells_x, cells_y;              // cells_per_col_x/y
    int corner;                        // corner_padding (6): anchor exclusion in cells
    int legacy;                        // coupled 6-bit layout (Decoder.h:121-161)
    int color_mode;                    // 0 = legacy palette, 1 = mode-B palette (Config.h:61-64)
    int num_cells;                     // total_cells
    int cap_sym, cap_col, cap_all;     // capacity(symbol_bits), capacity(color_bits), capacity(all) in bytes
    int msg_len;                       // ecc_block - ecc_bytes
    int nblocks;                       // RS blocks per frame
    int nblocks_sym;                   // RS blocks in the symbol stream (== nblocks when legacy)
    int chunk_size, chunks_per_frame;  // fountain chunk geometry (GridConf.h:54-72)
    int blocks_per_chunk;
    int data_bytes;                    // nblocks * msg_len (7500 for mode B)
    int top_cells;                     // cells in the top (and bottom) marker rows: (cells_x - 2*corner) * corner
    int mid_cells;                     // cells_x * (cells_y - 2*corner)
    uint32_t hash_mul;                 // perfect hash over the tile dictionary: slot = (L_lo * hash_mul) >> 28
    uint8_t palette[8][4];             // decode palette for (num_colors, color_mode): Common.cpp:21-85, :122-139
    // colour distance in closed form (CimbDecoder.cpp:168-200): with p = (pr-pg, pg-pb, pb-pr) of palette entry i and
    // a = (r-g, g-b, b-r) of the cell, |a - p|^2 = |a|^2 + pal_c[i] - (a0 * pal_u[i] + a1 * pal_w[i])  (a2 = -a0-a1)
    int pal_c[8], pal_u[8], pal_w[8];  // |p|^2, 2 (p0 - p2), 2 (p1 - p2)
};

// cell row k (0..cells_y-1): first cell index, number of cells, x of first cell
__host__ __device__ inline void cell_row_geom(const Mode& m, int k, int& base, int& ncols, int& x0)
{
    int narrow = m.cells_x - 2 * m.corner;
    if (k < m.corner) { base = k * narrow; ncols = narrow; x0 = m.cell_offset + kSpacing * m.corner; }
    else if (k < m.cells_y - m.corner) { base = m.top_cells + (k - m.corner) * m.cells_x; ncols = m.cells_x; x0 = m.cell_offset; }
    else { base = m.top_cells + m.mid_cells + (k - (m.cells_y - m.corner)) * narrow; ncols = narrow; x0 = m.cell_offset + kSpacing * m.corner; }
}

// linear cell index -> (cell row k, column c within that row)
__host__ __device__ inline void cell_row_col(const Mode& m, int index, int& k, int& c)
{
    int narrow = m.cells_x - 2 * m.corner;
    if (index < m.top_cells) { k = index / narrow; c = index - k * narrow; }
    else if (index < m.top_cells + m.mid_cells) { int q = index - m.top_cells; k = q / m.cells_x; c = q - k * m.cells_x; k += m.corner; }
    else { int q = index - m.top_cells - m.mid_cells; k = q / narrow; c = q - k * narrow; k += m.cells_y - m.corner; }
}

// AdjacentCellFinder::find in (row, column) arithmetic -- equivalent to the reference's index/position logic
// (src/lib/cimb_translator/AdjacentCellFinder.cpp:54-105; equivalence is asserted against the literal evaluation when a
// context is created).  dir: 0 right, 1 left, 2 bottom, 3 top.  Returns the neighbour's linear index or -1.
__host__ __device__ inline int cell_neighbour(const Mode& m, int k, int c, int dir, int& k2, int& c2)
{
    int base, ncols, x0;
    cell_row_geom(m, k, base, ncols, x0);
    k2 = k; c2 = c;
    if (dir == 0) { if (c + 1 >= ncols) return -1; c2 = c + 1; return base + c2; }
    if (dir == 1) { if (c == 0) return -1; c2 = c - 1; return base + c2; }
    k2 = (dir == 2) ? k + 1 : k - 1;
    if (k2 < 0 || k2 >= m.cells_y) return -1;
    // two quirks of the reference's index arithmetic, kept because the walk order depends on them: in the marker rows the
    // row stride is cells_x - corner, so from the second-to-last top row the last `corner` cells step INTO the first mid row
    // (and symmetrically upwards from the second bottom row), fail the x comparison, and report no neighbour
    // (AdjacentCellFinder.cpp:79-105)
    if (dir == 2 && k == m.corner - 2 && c >= ncols - m.corner) return -1;
    if (dir == 3 && k == m.cells_y - m.corner + 1 && c < m.corner) return -1;
    int base2, ncols2, x02;
    cell_row_geom(m, k2, base2, ncols2, x02);
    c2 = c + (x0 - x02) / kSpacing;          // same x in the neighbouring row (rows next to the anchors are narrower)
    if (c2 < 0 || c2 >= ncols2) return -1;
    return base2 + c2;
}

// per-cell result byte written by K1/K1x
constexpr uint8_t kCellDirty = 0x80;   // centre hash did not win -> frame needs the exact flood walk

// frame flags
constexpr uint8_t kFrameFallback = 0x01;   // exact flood-walk kernel was used for this frame
constexpr uint8_t kFrameDirtyK1 = 0x02;    // (internal) K1 saw a cell whose centre hash did not win

}  // namespace cb200
