// extract_core.cuh -- the per-picture decisions of Extractor::extract and the perspective arithmetic of the deskew, written once
// for the host (cb200_perspective_transform, deskew_run, tests/cpp/extract_core_host.cpp) and the device (k_extract in scan.cu).
// Every double operation goes through scan_core.cuh's dmul / dadd / dsub / ddiv, so nvcc cannot contract it into an FMA and the
// device results are bit-identical to the host's and to cv2's.
//
// Replaces (reference file:line relative to /root/reference/):
//   Extractor::extract          src/lib/extractor/Extractor.h:30-46: fewer than four anchors -> FAILURE, Corners = the anchor
//                               centres (Corners.h:13-16), NEEDS_SHARPEN unless Corners::is_granular_scale (Corners.h:57-75)
//   Deskewer::deskew            src/lib/extractor/Deskewer.h:27-39: the output points with padding 0
//   cv::getPerspectiveTransform modules/imgproc/src/imgwarp.cpp: an 8x8 system solved by hal::LU64f
//                               (modules/core/src/matrix_decomp.cpp, LUImpl<double>: partial pivoting, d = -1/pivot, row updates,
//                               back substitution)
//   cv::invert (3x3, DECOMP_LU) modules/core/src/lapack.cpp: det3 + adjugate
#pragma once
#include <float.h>
#include <math.h>

#include "scan_core.cuh"

namespace cb200 {
namespace extract {

using scan::dadd;
using scan::ddiv;
using scan::dmul;
using scan::dsub;

#if defined(__CUDA_ARCH__)
CB_HD float fmul(float a, float b) { return __fmul_rn(a, b); }
#else
CB_HD float fmul(float a, float b) { return a * b; }
#endif

constexpr float kAnchor = 30.0f;        // Config::anchor_size() (Config.h)

// where Deskewer::deskew sends the four anchor centres (tl, tr, bl, br): (anchor, anchor) ... (W - anchor, H - anchor).  A picture
// that fails extraction is deskewed with these as its corners too (its decode is discarded)
CB_HD void output_points(int width, int height, float* xy)
{
    const float w = (float)width - kAnchor, h = (float)height - kAnchor;
    xy[0] = kAnchor; xy[1] = kAnchor; xy[2] = w; xy[3] = kAnchor; xy[4] = kAnchor; xy[5] = h; xy[6] = w; xy[7] = h;
}

// Corners::is_granular_scale: every side of the quadrilateral (tl-tr, tr-br, br-bl, bl-tl) spans more than the frame in x or in y.
// T = int for the anchor centres of a scan, float for corners a caller supplies
template <class T>
CB_HD bool is_granular_scale(const T* xy, int width, int height)
{
    const int pairs[4][2] = {{0, 1}, {1, 3}, {3, 2}, {2, 0}};
    bool granular = true;
    for (int k = 0; k < 4; ++k) {
        const int p = pairs[k][0], q = pairs[k][1];
        const T dx = xy[2 * p] - xy[2 * q], dy = xy[2 * p + 1] - xy[2 * q + 1];
        granular = granular && ((dx < 0 ? -dx : dx) > (T)width || (dy < 0 ? -dy : dy) > (T)height);
    }
    return granular;
}

// hal::LU64f for an m x m system (m <= 8) with one right-hand side; false = singular (cv::solve leaves zeros)
CB_HD bool lu_solve(double* A, int m, double* b)
{
    const double eps = DBL_EPSILON * 100;
    for (int i = 0; i < m; ++i) {
        int k = i;
        for (int j = i + 1; j < m; ++j) if (fabs(A[j * m + i]) > fabs(A[k * m + i])) k = j;
        if (fabs(A[k * m + i]) < eps) return false;
        if (k != i) {
            for (int j = i; j < m; ++j) { const double t = A[i * m + j]; A[i * m + j] = A[k * m + j]; A[k * m + j] = t; }
            const double t = b[i]; b[i] = b[k]; b[k] = t;
        }
        const double d = ddiv(-1., A[i * m + i]);
        for (int j = i + 1; j < m; ++j) {
            const double alpha = dmul(A[j * m + i], d);
            for (int c = i + 1; c < m; ++c) A[j * m + c] = dadd(A[j * m + c], dmul(alpha, A[i * m + c]));
            b[j] = dadd(b[j], dmul(alpha, b[i]));
        }
    }
    for (int i = m - 1; i >= 0; --i) {
        double s = b[i];
        for (int c = i + 1; c < m; ++c) s = dsub(s, dmul(A[i * m + c], b[c]));
        b[i] = ddiv(s, A[i * m + i]);
    }
    return true;
}

// cv::invert of a 3x3 double matrix; false = determinant 0
CB_HD bool invert3(const double* S, double* t)
{
#define SD(r, c) S[(r) * 3 + (c)]
#define CF(a, b, c, d) dsub(dmul(SD a, SD b), dmul(SD c, SD d))
    double d = dadd(dsub(dmul(SD(0, 0), CF((1, 1), (2, 2), (1, 2), (2, 1))), dmul(SD(0, 1), CF((1, 0), (2, 2), (1, 2), (2, 0)))),
                    dmul(SD(0, 2), CF((1, 0), (2, 1), (1, 1), (2, 0))));
    if (d == 0.) return false;
    d = ddiv(1., d);
    t[0] = dmul(CF((1, 1), (2, 2), (1, 2), (2, 1)), d);
    t[1] = dmul(CF((0, 2), (2, 1), (0, 1), (2, 2)), d);
    t[2] = dmul(CF((0, 1), (1, 2), (0, 2), (1, 1)), d);
    t[3] = dmul(CF((1, 2), (2, 0), (1, 0), (2, 2)), d);
    t[4] = dmul(CF((0, 0), (2, 2), (0, 2), (2, 0)), d);
    t[5] = dmul(CF((0, 2), (1, 0), (0, 0), (1, 2)), d);
    t[6] = dmul(CF((1, 0), (2, 1), (1, 1), (2, 0)), d);
    t[7] = dmul(CF((0, 1), (2, 0), (0, 0), (2, 1)), d);
    t[8] = dmul(CF((0, 0), (1, 1), (0, 1), (1, 0)), d);
#undef CF
#undef SD
    return true;
}

// cv::getPerspectiveTransform(src, dst) into m9 (row-major, m9[8] = 1): c00 xi + c01 yi + c02 - ui (c20 xi + c21 yi) = ui, ...
// false for a degenerate quadrilateral: m9 = 0 ... 0, 1 then (what cv::solve leaves)
CB_HD bool perspective_transform(const float* src_xy, const float* dst_xy, double* m9)
{
    double a[8][8], b[8];
    for (int i = 0; i < 4; ++i) {
        // the points are cv::Point2f: the four products are single-precision products, as in OpenCV's source
        const float sx = src_xy[2 * i], sy = src_xy[2 * i + 1], dx = dst_xy[2 * i], dy = dst_xy[2 * i + 1];
        a[i][0] = a[i + 4][3] = sx;
        a[i][1] = a[i + 4][4] = sy;
        a[i][2] = a[i + 4][5] = 1;
        a[i][3] = a[i][4] = a[i][5] = a[i + 4][0] = a[i + 4][1] = a[i + 4][2] = 0;
        a[i][6] = fmul(-sx, dx);
        a[i][7] = fmul(-sy, dx);
        a[i + 4][6] = fmul(-sx, dy);
        a[i + 4][7] = fmul(-sy, dy);
        b[i] = dx;
        b[i + 4] = dy;
    }
    const bool ok = lu_solve(&a[0][0], 8, b);
    for (int i = 0; i < 8; ++i) m9[i] = ok ? b[i] : 0.;
    m9[8] = 1.;
    return ok;
}

// Extractor::extract for one scanned picture, as the batched camera path decides it: anchors = the scan's four (tl, tr, bl, br),
// count = how many it found, overflow = the scan ran out of list capacity.  Returns the status (-1 overflow, 0 FAILURE, 1 SUCCESS,
// 2 NEEDS_SHARPEN); fwd = getPerspectiveTransform(corners, output points), inv = its inverse (what warpPerspective maps with).
// Overflow, fewer than four anchors and a degenerate quadrilateral get the output points as corners (status -1 / 0 / 0).  The
// inverse of a non-degenerate quadrilateral's transform always exists; a determinant that rounds to exactly 0 is a FAILURE too
CB_HD int extract_picture(const scan::Anchor* anchors, int count, bool overflow, int width, int height, double* fwd, double* inv)
{
    float outp[8], corners[8];
    output_points(width, height, outp);
    int status = overflow ? -1 : (count < 4 ? 0 : 1);
    if (status == 1) {
        int xy[8];
        for (int k = 0; k < 4; ++k) {
            xy[2 * k] = scan::xavg(anchors[k]); xy[2 * k + 1] = scan::yavg(anchors[k]);
            corners[2 * k] = (float)xy[2 * k]; corners[2 * k + 1] = (float)xy[2 * k + 1];
        }
        status = is_granular_scale(xy, width, height) ? 1 : 2;
        if (!perspective_transform(corners, outp, fwd) || !invert3(fwd, inv)) status = 0;
    }
    if (status <= 0) {
        perspective_transform(outp, outp, fwd);
        invert3(fwd, inv);
    }
    return status;
}

}  // namespace extract
}  // namespace cb200
