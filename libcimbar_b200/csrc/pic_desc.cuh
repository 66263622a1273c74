// pic_desc.cuh -- one camera picture of a batch as the extractor kernels (scan.cu, deskew.cu) read it.  The host builds the table
// per call, for uniform batches too: picture i of a packed batch starts at byte 3 * sum_{j<i} w_j h_j of the buffer (layout RGB, row
// pitch 3 w), its blurred gray at sum_{j<i} w_j h_j.  A plan over device descriptors builds it on the device (layout_core.cuh:
// plan_slot).  Plain data, so that the host tests compile it too
#pragma once
#include <stdint.h>

namespace cb200 {

struct PicDesc {
    uint64_t src;        // device address of the picture's pixel (0, 0) (of its R plane when planar): layout_core.cuh reads it
    uint64_t blur;       // byte offset of its blurred gray picture in the scan's buffer (k_scan_blur4 / k_scan_anchors)
    int w, h;
    int words;           // k_scan_blur4's word path: w % 4 == 0, the source's base and pitches and the blurred base 4-byte aligned
    int tile0;           // first tile of the picture in the blur launch of its radius
    uint64_t pitch;      // bytes from one row to the next
    uint64_t plane;      // bytes from one plane to the next (CB200_LAYOUT_RGB_PLANAR)
    int layout;          // CB200_LAYOUT_*
};

}  // namespace cb200
