// The per-picture extract decisions of the camera path (libcimbar_b200/csrc/extract_core.cuh, what k_extract runs) compiled for the
// host, for tests/test_extract_core_host.py.  Built with g++ -ffp-contract=off like scan_core_host.cpp.
#include "../../libcimbar_b200/csrc/extract_core.cuh"

using namespace cb200;

extern "C" {

// extract_picture of one scanned picture: anchors = 4 x (x, xmax, y, ymax); returns the status, fills corners (8 floats: the anchor
// centres, or the output points for a status <= 0), fwd and inv (9 doubles each)
int ec_extract(const int* anchors, int count, int overflow, int width, int height, float* corners, double* fwd, double* inv)
{
    scan::Anchor a[4];
    for (int k = 0; k < 4; ++k) a[k] = scan::mk(anchors[4 * k], anchors[4 * k + 1], anchors[4 * k + 2], anchors[4 * k + 3]);
    const int st = extract::extract_picture(a, count, overflow != 0, width, height, fwd, inv);
    if (st > 0) for (int k = 0; k < 4; ++k) { corners[2 * k] = (float)scan::xavg(a[k]); corners[2 * k + 1] = (float)scan::yavg(a[k]); }
    else extract::output_points(width, height, corners);
    return st;
}

int ec_transform(const float* src, const float* dst, double* m9) { return extract::perspective_transform(src, dst, m9) ? 1 : 0; }

int ec_invert(const double* m9, double* inv) { return extract::invert3(m9, inv) ? 1 : 0; }

int ec_granular(const float* xy, int width, int height) { return extract::is_granular_scale(xy, width, height) ? 1 : 0; }

}  // extern "C"
