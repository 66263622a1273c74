// layout_core_host.cpp -- TEST HARNESS: compiles the per-layout pixel fetch of the camera kernels (libcimbar_b200/csrc/layout_core.cuh:
// the gray k_scan_blur4 takes, by bytes and on its word path, and the tap pairs k_deskew takes) for the host, so that it can be
// compared with numpy where there is no GPU.  Not part of the product; the product runs the same functions in CUDA kernels.
#include "../../libcimbar_b200/csrc/layout_core.cuh"

#include <stddef.h>

using namespace cb200::layout;

// the gray of every pixel of a w x h picture at `base`, as k_scan_blur4 computes it: the word path on the quads x .. x + 3 inside the
// row when `words` is set, the byte fetch elsewhere
extern "C" void lc_gray(const uint8_t* base, int w, int h, int64_t pitch, int64_t plane, int layout, int words, uint8_t* out)
{
    for (int y = 0; y < h; ++y) {
        const uint8_t* row = base + (size_t)y * (size_t)pitch;
        for (int x = 0; x < w; x += 4) {
            if (words && x + 3 < w) {
                const uint32_t g4 = gray4_words(row, x, (uint64_t)plane, layout);
                for (int k = 0; k < 4; ++k) out[(size_t)y * w + x + k] = (uint8_t)(g4 >> (8 * k));
            } else {
                for (int k = 0; k < 4 && x + k < w; ++k) out[(size_t)y * w + x + k] = (uint8_t)gray_at(row, x + k, (uint64_t)plane, layout);
            }
        }
    }
}

// k_deskew's tap pairs: for each (c, y) of cy, pixels c and c + 1 of row y as R G B R G B (out: n x 6)
extern "C" void lc_taps(const uint8_t* base, int w, int h, int64_t pitch, int64_t plane, int layout, const int* cy, int n, uint8_t* out)
{
    const int cpp = channels(layout);
    const uint8_t* end = base + (size_t)(h - 1) * (size_t)pitch + (size_t)w * (size_t)cpp;
    for (int i = 0; i < n; ++i) {
        const int c = cy[2 * i], y = cy[2 * i + 1];
        uint32_t lo, hi;
        tap_pair(base + (size_t)y * (size_t)pitch + (size_t)c * (size_t)cpp, (uint64_t)plane, layout, end, lo, hi);
        for (int k = 0; k < 4; ++k) out[6 * i + k] = (uint8_t)(lo >> (8 * k));
        out[6 * i + 4] = (uint8_t)hi;
        out[6 * i + 5] = (uint8_t)(hi >> 8);
    }
}

// cb200_picture as the C compiler lays it out: size, then the offsets of data, w, h, row_pitch, plane_pitch, layout
extern "C" void lc_picture_abi(int64_t* out)
{
    out[0] = sizeof(cb200_picture);
    out[1] = offsetof(cb200_picture, data); out[2] = offsetof(cb200_picture, w); out[3] = offsetof(cb200_picture, h);
    out[4] = offsetof(cb200_picture, row_pitch); out[5] = offsetof(cb200_picture, plane_pitch); out[6] = offsetof(cb200_picture, layout);
}
