// The JPEG decode of the camera path (libcimbar_b200/csrc/jpeg_core.cuh: what jpeg.cu's kernels run) compiled for the host, for
// tests/test_jpeg_core_host.py: the same parse, upload layout, segment decoder, IDCT and colour functions, in the kernels' order.
#include "../../libcimbar_b200/csrc/jpeg_core.cuh"

#include <algorithm>

using namespace cb200::jpeg;

extern "C" {

// w, h of the output (after orientation): 0, or 1 with the refusal reason in why
int jc_info(const uint8_t* file, uint64_t size, int* wh, char* why, int why_cap)
{
    Parsed p;
    const std::string r = parse(file, size, p);
    if (!r.empty()) { snprintf(why, (size_t)why_cap, "%s", r.c_str()); return 1; }
    wh[0] = p.pic.ow; wh[1] = p.pic.oh;
    return 0;
}

// the RGB8 picture into rgb (cap bytes): 0, -2 for corrupt data, 1 refused (why), 2 too small a buffer.  *wide: the blocks whose
// IDCT leaves the range where libjpeg-turbo's C and SIMD IDCTs agree (idct_islow), where cv2's bytes depend on its build
int jc_decode_wide(const uint8_t* file, uint64_t size, uint8_t* rgb, uint64_t cap, int* wh, char* why, int why_cap, int* wide)
{
    *wide = 0;
    std::vector<Parsed> ps(1);
    const std::string r = parse(file, size, ps[0]);
    if (!r.empty()) { snprintf(why, (size_t)why_cap, "%s", r.c_str()); return 1; }
    const Layout L = layout(ps, &size);
    if (L.rgb > cap) return 2;
    std::vector<uint8_t> blob(L.bytes);
    pack(ps, &file, &size, L, blob.data());
    const Pic* pics = reinterpret_cast<const Pic*>(blob.data() + L.pics);
    const Scan* scans = reinterpret_cast<const Scan*>(blob.data() + L.scans);
    const Seg* segs = reinterpret_cast<const Seg*>(blob.data() + L.segs);
    const Huff* huffs = reinterpret_cast<const Huff*>(blob.data() + L.huffs);
    const uint16_t* quant = reinterpret_cast<const uint16_t*>(blob.data() + L.quant);
    std::vector<int16_t> coef(L.coef, 0);
    std::vector<uint8_t> planes(L.planes);
    bool bad = pics[0].bad != 0;
    // unstuffing, then the rounds: the parallel decode with k_jpeg_decode's 512 threads, AC refinement in order
    const uint8_t* raw = blob.data() + L.data;
    std::vector<uint8_t> u(L.bytes - L.data);
    std::vector<uint32_t> ulen(L.round0.back());
    for (uint32_t g = 0; g < L.round0.back(); ++g) {
        uint32_t m = 0;
        for (uint64_t i = segs[g].begin; i < segs[g].end; ++i)
            if (kept(raw, i, segs[g].begin)) u[segs[g].begin + m++] = raw[i];
        ulen[g] = m;
    }
    std::vector<uint64_t> masks(4 * (L.coef / 64));
    for (size_t s = 0; s + 1 < L.round0.size(); ++s)
        for (uint32_t g = L.round0[s]; g < L.round0[s + 1]; ++g) {
            const Scan& sc = scans[segs[g].scan];
            const Pic& P = pics[sc.pic];
            const uint8_t* d = u.data() + segs[g].begin;
            if (sc.kind != kAcRefine) {
                if (!decode_segment_sync(512, d, ulen[g], P, sc, segs[g], huffs, coef.data())) bad = true;
                continue;
            }
            const uint32_t nb = segment_blocks(sc, segs[g]);
            for (uint32_t k = 0; k < nb; ++k) {
                const uint64_t o = block_offset(P, sc, segs[g], k);
                refine_prep(coef.data() + o, sc.ss, sc.se, masks.data() + 4 * (o / 64));
            }
            if (!decode_refine(d, ulen[g], P, sc, segs[g], huffs[sc.ac[0]], masks.data())) bad = true;
            for (uint32_t k = 0; k < nb; ++k) {
                const uint64_t o = block_offset(P, sc, segs[g], k);
                refine_apply(coef.data() + o, sc.al, masks.data() + 4 * (o / 64));
            }
        }
    const Pic& P = pics[0];
    wh[0] = P.ow; wh[1] = P.oh;
    if (bad) return -2;
    for (int c = 0; c < P.ncomp; ++c) {
        const Comp& C = P.comp[c];
        for (int by = 0; by < C.bh; ++by)
            for (int bx = 0; bx < C.bw; ++bx) {
                int w = 0;
                idct_islow(coef.data() + C.coef + ((size_t)by * C.bw + bx) * 64, quant + C.quant,
                           planes.data() + C.plane + (size_t)by * 8 * C.bw * 8 + (size_t)bx * 8, (size_t)C.bw * 8, &w);
                *wide += w;
            }
    }
    for (int y = 0; y < P.oh; ++y)
        for (int x = 0; x < P.ow; ++x) pixel_rgb(planes.data(), P, x, y, rgb + P.out + 3 * ((size_t)y * P.ow + x));
    return 0;
}

int jc_decode(const uint8_t* file, uint64_t size, uint8_t* rgb, uint64_t cap, int* wh, char* why, int why_cap)
{
    int wide;
    return jc_decode_wide(file, size, rgb, cap, wh, why, why_cap, &wide);
}

}  // extern "C"
