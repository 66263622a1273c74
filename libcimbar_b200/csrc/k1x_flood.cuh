// k1x_flood.cuh -- host-side entry points of the exact flood-walk kernel (k1x_flood.cu)
#pragma once
#include "cb200_common.cuh"
#include "ccm.cuh"
#include <cstring>
#include <cstdlib>
#include <vector>

namespace cb200 {

// per-cell record of the exact walk (== what CimbReader::read returns step by step, CimbReader.cpp:139-162)
struct CellTrace {
    uint16_t order;        // position in the flood-walk order
    int16_t x, y;          // drift-adjusted cell position (PositionData x, y)
    uint8_t drift_offset;  // winning hash id 0..8 (4 = centre)
    uint8_t distance;      // best Hamming distance
};

struct FloodWorkspace {
    int sm_count = 0;
    int slots = 0;             // walking warps resident at once (one frame each)
    int heap_smem = 0;         // heap entries per walk kept in shared memory (odd)
    size_t walk_smem = 0;      // dynamic shared memory of one walking warp
    int heap_smem_few = 0; size_t walk_smem_few = 0; int few_frames = 0;   // batches of at most few_frames listed frames: the whole heap in shared memory
    size_t spill_cap = 0;      // heap spill entries per slot
    int serial_above = 0;      // heap sizes above this use the one-level-per-step pop (65536; tests lower it)
    DevBuf<uint32_t> spill;    // [slots][spill_cap]
    DevBuf<uint8_t> prio;      // [slots][kMaxCells] per-cell priority bytes of the walk in that slot
    DevBuf<uint16_t> cinfo;    // [num_cells][16] update candidates in push order (0xFFFF = none)
    DevBuf<uint32_t> list, counters;   // work list; counters[0] = listed frames, [1 + c] = chunk c's work counter
    int max_entries = 0;       // upper bound of entry_cap (one chunk); larger work lists are processed chunk by chunk
    int entry_cap = 0; DevBuf<uint16_t> raster; DevBuf<uint32_t> result;  // per listed frame of a chunk: 1-bit raster in 16x16 tiles, per-cell x | y<<11 | sym<<22
};

cudaError_t flood_init_tables(const float* adjust256, const unsigned long long* tiles_L16, uint32_t hash_mul);
// adj_host: [num_cells][4] = AdjacentCellFinder::find for every cell (built by the caller from the cell geometry)
cudaError_t flood_workspace_create(const Mode& m, int sm_count, const uint16_t* adj_host, FloodWorkspace* ws);
// the per-batch buffers for n_frames frames (flood_launch grows them itself; fits: no growth needed)
cudaError_t flood_workspace_ensure(const Mode& m, FloodWorkspace& ws, int n_frames);
bool flood_workspace_fits(const FloodWorkspace& ws, int n_frames);
// writes d_flags[f] for every frame: 0 = K1 result stands, CB200_FRAME_FALLBACK = re-decoded here,
// CB200_FRAME_INEXACT = needed but skipped (no_fallback).  list_all: every frame is walked (for d_trace), the flags stay as the
// dirty bits decide -- a frame K1 did not flag gets the cells K1 gave it (DESIGN.md §3, "Exactness").  d_sharpen_of: NULL = every frame is preprocessed as `sharpen` says;
// else one byte per frame of the batch (device memory, nonzero = sharpen) and `sharpen` is ignored.
// keep != NULL: the walk's per-cell records (x | y << 11 | sym << 22) of all n_frames listed frames stay there, in list order
// (n_frames x num_cells words), instead of one chunk at a time in the workspace.  d_present != NULL: one device byte per frame, and
// a frame whose byte is 0 is neither walked nor flagged (its K1 cells stand)
cudaError_t flood_launch(const Mode& m, FloodWorkspace& ws, const uint8_t* d_rgb, int n_frames, bool no_fallback,
                         bool force_all, bool list_all, bool sharpen, const uint8_t* d_sharpen_of, uint8_t* d_cellvals, const uint32_t* d_dirty,
                         uint8_t* d_flags, CellTrace* d_trace, const CcmArg& cc, cudaStream_t st, uint32_t* keep = nullptr,
                         const uint8_t* d_present = nullptr);
// the colour pass of a walk that flood_launch ran on `walked` with `keep` = kept, for another mode of the same frame geometry: the
// frames it listed get their colours (or, with cc.means, their mean colours) at the walk's positions and its symbols in d_cellvals
cudaError_t flood_colour_launch(const Mode& m, const FloodWorkspace& walked, const uint8_t* d_rgb, int n_frames, const uint32_t* kept,
                                uint8_t* d_cellvals, const CcmArg& cc, cudaStream_t st);

}  // namespace cb200
