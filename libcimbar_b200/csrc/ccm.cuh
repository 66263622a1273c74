// ccm.cuh -- colour correction matrix (CCM): the float side path of the colour decode, sm_90a.
//
// Reference (file:line relative to /root/reference/):
//   color_correction::transform            src/lib/chromatic_adaptation/color_correction.h:64-68  (cv::Matx<float,3,3> * vec)
//   CimbDecoder::get_best_color            src/lib/cimb_translator/CimbDecoder.cpp:168-200 (transform, then the usual scaling)
//   fix_single_color                       src/lib/cimb_translator/CimbDecoder.cpp:27-36
//   color_correction::get_adaptation_matrix  color_correction.h:12-24, von Kries matrix adaptation_transform.h:22-33
//   calculateWhite / simpleColorCorrection   src/lib/cimb_translator/CimbReader.cpp:55-93  (color_correction == 1)
// Everything is float32 in the reference's operation order; the intrinsics keep nvcc from contracting a*b+c into FMAs,
// which the reference's x86-64 build does not have.  Pinned by the matrix string and colours of the reference's own tests
// (tests/golden/manifest.json: adaptation_golden, ccm_goldens).
#pragma once
#include "cb200_common.cuh"

namespace cb200 {

// which CCM a launch uses: per_frame != nullptr -> matrix of frame f at per_frame + 9 f (color_correction == 1),
// else the context's matrix m (CimbDecoder::update_color_correction) when active
struct CcmArg {
    const float* per_frame;          // [n][9] or nullptr
    const uint8_t* per_frame_active; // with per_frame: [n] 1 = use the matrix, 0 = no CCM for that frame (nullptr = all active)
    uint32_t* means;                 // != nullptr: do not classify, store r | g << 8 | b << 16 per cell (color_correction == 2, first pass)
    float m[9];
    int active;
};

// cv::Matx product element: s = 0; s += a_k * b_k (k ascending), every operation rounded to float
__device__ __forceinline__ float dot3_rn(float a0, float a1, float a2, float b0, float b1, float b2)
{
    return __fadd_rn(__fadd_rn(__fmul_rn(a0, b0), __fmul_rn(a1, b1)), __fmul_rn(a2, b2));
}

__device__ __forceinline__ uint32_t fix_single_color_rn(float c, float adjust, float down)
{   // c -= down; c *= adjustUp; if (c > (245 - down)) c = 255; if (c < 0) c = 0; (uchar)c
    c = __fmul_rn(__fsub_rn(c, down), adjust);
    if (c > __fsub_rn(245.0f, down)) c = 255.0f;
    if (c < 0.0f) c = 0.0f;
    return __float2uint_rz(c);
}

// get_best_color with an active CCM; ri, gi, bi = Cell::mean_rgb of the inner 6x6 (integers); ccm = 9 floats, row-major
template <int NC>
__device__ __forceinline__ uint32_t best_color_ccm(const float* ccm, const Mode& m, uint32_t ri, uint32_t gi, uint32_t bi)
{
    const float r0 = (float)ri, g0 = (float)gi, b0 = (float)bi;
    const float r = dot3_rn(ccm[0], ccm[1], ccm[2], r0, g0, b0);
    const float g = dot3_rn(ccm[3], ccm[4], ccm[5], r0, g0, b0);
    const float b = dot3_rn(ccm[6], ccm[7], ccm[8], r0, g0, b0);
    const float mx = fmaxf(fmaxf(r, g), fmaxf(b, 1.0f));
    float mn = fminf(fminf(r, g), fminf(b, 48.0f));
    if (mn >= mx) mn = 0.0f;
    // float adjust = 255.0 / (max - min): a double division rounded to float in the reference.  For a float divisor d that
    // is the correctly rounded SINGLE quotient: the double quotient could only mis-round if it sat exactly on a float
    // midpoint M (25 significant bits) without being equal to it, i.e. 0 < |M d - 255| <= 2^-45; but M d is a multiple of
    // 2^-41 (25 x 24 significant bits, M d ~ 255), so the product is either 255 exactly or at least 2^-41 away.
    const float adjust = __fdiv_rn(255.0f, __fsub_rn(mx, mn));
    const int cr = (int)fix_single_color_rn(r, adjust, mn), cg = (int)fix_single_color_rn(g, adjust, mn), cb = (int)fix_single_color_rn(b, adjust, mn);
    const int a0 = cr - cg, a1 = cg - cb;
    uint32_t best = 0;
    int best_d = 0x7fffffff;
    const int nc = NC > 0 ? NC : (1 << m.color_bits);
#pragma unroll
    for (int i = 0; i < (NC > 0 ? NC : 8); ++i) {
        if (i >= nc) break;
        const int d = m.pal_c[i] - (a0 * m.pal_u[i] + a1 * m.pal_w[i]);      // see Mode::pal_c
        if (d < best_d) { best_d = d; best = (uint32_t)i; }
    }
    return best;
}

cudaError_t ccm_simple_launch(const Mode& m, const uint8_t* d_rgb, int n_frames, float* d_ccm, cudaStream_t st);
// color_correction == 2, after the symbol stream's RS pass: per frame the header the aligned_stream callbacks leave behind,
// the colours it predicts, the fit (fit[f], valid[f]); then the carry (a frame without a fit keeps its predecessor's CCM,
// frame 0 the context's) into used[f] / used_active[f]; then the colour decision of every cell from the stored means
// given != nullptr (single frame): the header is not derived from the RS output but handed in by the caller
// (CimbReader::init_ccm on a host that ran CimbReader::update_metadata itself); d_data / d_ok are then unused
struct GivenHeader { uint8_t hdr[6]; uint8_t use; uint8_t pad; uint32_t radioactive; };
cudaError_t ccm_fit_launch(const Mode& m, const uint8_t* d_rgb, const uint8_t* d_data, const uint8_t* d_ok, const uint16_t* d_idx,
                           int n_frames, float* d_fit, uint8_t* d_valid, cudaStream_t st, const GivenHeader* given = nullptr);
cudaError_t ccm_carry_launch(int n_frames, const float* d_fit, const uint8_t* d_valid, const CcmArg& initial, float* d_used,
                             uint8_t* d_used_active, cudaStream_t st);
cudaError_t ccm_apply_launch(const Mode& m, const uint32_t* d_means, int n_frames, const float* d_used, const uint8_t* d_used_active,
                             uint8_t* d_cellvals, cudaStream_t st);

}  // namespace cb200
