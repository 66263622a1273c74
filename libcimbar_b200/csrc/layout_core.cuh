// layout_core.cuh -- where the bytes of a camera picture's pixel lie in each layout the camera calls take (include/cb200.h,
// cb200_picture): packed RGB, BGR, RGBA and BGRA rows with any row pitch, and three planes R, G, B.  The two places that read
// pictures use it: k_scan_blur4 (scan.cu) takes the gray of a pixel, or of four pixels at once on its word path, and k_deskew
// (deskew.cu) takes the RGB of a pair of horizontal bilinear taps.  Every function is __host__ __device__ so that
// tests/cpp/layout_core_host.cpp runs the same code on the CPU against numpy.
//
// cvtColor's BGR2RGB, RGBA2RGB and BGRA2RGB only permute channels or drop alpha, and a pitch or a planar split only moves bytes,
// so a picture in any layout gives exactly what its packed RGB copy gives: the gray below is cvtColor(RGB2GRAY)'s
// (9798 R + 19235 G + 3735 B + 2^14) >> 15 whichever byte R, G and B come from.
#pragma once
#include <stdint.h>
#include <string.h>

#include "../../include/cb200.h"
#include "pic_desc.cuh"
#include "scan_core.cuh"            // CB_HD

namespace cb200 {
namespace layout {

CB_HD bool known(int layout) { return layout >= CB200_LAYOUT_RGB && layout <= CB200_LAYOUT_RGB_PLANAR; }
// bytes of one pixel inside a row (a plane's, for the planar layout)
CB_HD int channels(int layout) { return layout == CB200_LAYOUT_RGB_PLANAR ? 1 : ((layout == CB200_LAYOUT_RGBA || layout == CB200_LAYOUT_BGRA) ? 4 : 3); }
CB_HD bool blue_first(int layout) { return layout == CB200_LAYOUT_BGR || layout == CB200_LAYOUT_BGRA; }

// the byte instructions of the word paths (IDP.2A, PRMT, SHF) and an aligned word load through the read-only path, with their host
// restatements
#if defined(__CUDA_ARCH__)
CB_HD uint32_t dp2a_lo(uint32_t a, uint32_t b, uint32_t c) { return __dp2a_lo(a, b, c); }
CB_HD uint32_t dp2a_hi(uint32_t a, uint32_t b, uint32_t c) { return __dp2a_hi(a, b, c); }
CB_HD uint32_t prmt(uint32_t x, uint32_t y, uint32_t s) { return __byte_perm(x, y, s); }
CB_HD uint32_t shr64(uint32_t lo, uint32_t hi, uint32_t sh) { return __funnelshift_r(lo, hi, sh); }
CB_HD uint32_t ldw(const uint8_t* p) { return __ldg(reinterpret_cast<const uint32_t*>(p)); }
#else
CB_HD uint32_t dp2a_lo(uint32_t a, uint32_t b, uint32_t c) { return (a & 0xFFFFu) * (b & 0xFFu) + (a >> 16) * ((b >> 8) & 0xFFu) + c; }
CB_HD uint32_t dp2a_hi(uint32_t a, uint32_t b, uint32_t c) { return (a & 0xFFFFu) * ((b >> 16) & 0xFFu) + (a >> 16) * (b >> 24) + c; }
CB_HD uint32_t prmt(uint32_t x, uint32_t y, uint32_t s)
{
    const uint64_t v = ((uint64_t)y << 32) | x;
    uint32_t r = 0;
    for (int i = 0; i < 4; ++i) r |= (uint32_t)((v >> (8 * ((s >> (4 * i)) & 7u))) & 0xFFu) << (8 * i);
    return r;
}
CB_HD uint32_t shr64(uint32_t lo, uint32_t hi, uint32_t sh) { return (uint32_t)((((uint64_t)hi << 32) | lo) >> (sh & 31u)); }
CB_HD uint32_t ldw(const uint8_t* p) { uint32_t v; memcpy(&v, p, 4); return v; }
#endif
CB_HD uint32_t ldb(const uint8_t* p) { return *p; }

CB_HD uint32_t gray(uint32_t r, uint32_t g, uint32_t b) { return (9798u * r + 19235u * g + 3735u * b + 16384u) >> 15; }

// Where the bytes of pixel x of a row lie, in every layout: R at row + step x + r, G at + g, B at + b.  Branch-free, so the byte
// fetch costs a kernel few registers.  32-bit channel offsets: a picture spans less than 4 GB (the calls refuse larger ones)
struct Fetch { uint32_t step, r, g, b; };

CB_HD Fetch fetch_of(int layout, uint64_t plane)
{
    if (layout == CB200_LAYOUT_RGB_PLANAR) return Fetch{1u, 0u, (uint32_t)plane, 2u * (uint32_t)plane};
    const bool bf = blue_first(layout);
    return Fetch{(uint32_t)channels(layout), bf ? 2u : 0u, 1u, bf ? 0u : 2u};
}

// the R, G, B bytes of pixel x of a row (row = the picture's first byte + y * row pitch)
CB_HD void rgb_px(const uint8_t* row, int x, const Fetch& f, uint32_t& r, uint32_t& g, uint32_t& b)
{
    const uint8_t* p = row + (size_t)f.step * (size_t)x;
    r = ldb(p + f.r); g = ldb(p + f.g); b = ldb(p + f.b);
}

CB_HD uint32_t gray_px(const uint8_t* row, int x, const Fetch& f)
{
    uint32_t r, g, b;
    rgb_px(row, x, f, r, g, b);
    return gray(r, g, b);
}

// the same from the layout and the plane pitch
CB_HD void rgb_at(const uint8_t* row, int x, uint64_t plane, int layout, uint32_t& r, uint32_t& g, uint32_t& b)
{
    rgb_px(row, x, fetch_of(layout, plane), r, g, b);
}

CB_HD uint32_t gray_at(const uint8_t* row, int x, uint64_t plane, int layout) { return gray_px(row, x, fetch_of(layout, plane)); }

// the word path: the gray of pixels x .. x + 3 as the bytes of one word, for a row whose pixel x starts on a 4-byte boundary in
// every plane (x % 4 == 0, base, row pitch and plane pitch multiples of 4).  Each gray is (19596 R + 38470 G + 7470 B + 2^15) >> 16
// (== the 15-bit form), byte 2 of an IDP.2A sum: packed 3-byte pixels come as three words with the coefficients permuted to the
// channel order, 4-byte pixels as one word each, planes as one word per plane
CB_HD uint32_t gray4_words(const uint8_t* row, int x, uint64_t plane, int layout)
{
    const bool bf = blue_first(layout);
    const uint32_t k0 = bf ? 7470u : 19596u, k2 = bf ? 19596u : 7470u;          // the coefficients of a pixel's bytes 0 and 2
    uint32_t n0, n1, n2, n3;
    if (layout == CB200_LAYOUT_RGB_PLANAR) {
        const uint32_t r4 = ldw(row + x), g4 = ldw(row + plane + x), b4 = ldw(row + 2 * plane + x);
        const uint32_t rg01 = prmt(r4, g4, 0x5140), rg23 = prmt(r4, g4, 0x7362);   // R0 G0 R1 G1 | R2 G2 R3 G3
        const uint32_t cRG = 19596u | (38470u << 16), cB0 = 7470u, c0B = 7470u << 16;
        n0 = dp2a_lo(cB0, b4, dp2a_lo(cRG, rg01, 32768u));
        n1 = dp2a_lo(c0B, b4, dp2a_hi(cRG, rg01, 32768u));
        n2 = dp2a_hi(cB0, b4, dp2a_lo(cRG, rg23, 32768u));
        n3 = dp2a_hi(c0B, b4, dp2a_hi(cRG, rg23, 32768u));
    } else if (channels(layout) == 4) {
        const uint8_t* p = row + 4 * (size_t)x;
        const uint32_t q0 = ldw(p), q1 = ldw(p + 4), q2 = ldw(p + 8), q3 = ldw(p + 12);   // c0 c1 c2 alpha, one pixel each
        const uint32_t c01 = k0 | (38470u << 16), c2 = k2;
        n0 = dp2a_hi(c2, q0, dp2a_lo(c01, q0, 32768u));
        n1 = dp2a_hi(c2, q1, dp2a_lo(c01, q1, 32768u));
        n2 = dp2a_hi(c2, q2, dp2a_lo(c01, q2, 32768u));
        n3 = dp2a_hi(c2, q3, dp2a_lo(c01, q3, 32768u));
    } else {
        const uint8_t* p = row + 3 * (size_t)x;
        const uint32_t q0 = ldw(p), q1 = ldw(p + 4), q2 = ldw(p + 8);          // a0 b0 c0 a1 | b1 c1 a2 b2 | c2 a3 b3 c3
        const uint32_t cAB = k0 | (38470u << 16), cC0 = k2, c0A = k0 << 16, cBC = 38470u | (k2 << 16);
        n0 = dp2a_lo(cAB, q0, 32768u); n0 = dp2a_hi(cC0, q0, n0);
        n1 = dp2a_hi(c0A, q0, 32768u); n1 = dp2a_lo(cBC, q1, n1);
        n2 = dp2a_hi(cAB, q1, 32768u); n2 = dp2a_lo(cC0, q2, n2);
        n3 = dp2a_lo(c0A, q2, 32768u); n3 = dp2a_hi(cBC, q2, n3);
    }
    return prmt(prmt(n0, n1, 0x0062), prmt(n2, n3, 0x6200), 0x7610);
}

// k_deskew's taps: the `nb` bytes from p as lo = bytes 0..3, hi = bytes 4.. (the rest unspecified), fetched as aligned words and
// realigned by a funnel shift; `end` = one past the last byte that may be read (the picture's plane), the last few by bytes
CB_HD void load_bytes(const uint8_t* p, const uint8_t* end, uint32_t nb, uint32_t& lo, uint32_t& hi)
{
    const uint32_t a = (uint32_t)(reinterpret_cast<uintptr_t>(p) & 3u);
    const uint8_t* base = p - a;
    if (base + 12 <= end) {
        const uint32_t w0 = ldw(base), w1 = ldw(base + 4);
        const uint32_t w2 = (a + nb > 8u) ? ldw(base + 8) : 0u;
        lo = shr64(w0, w1, 8u * a);
        hi = shr64(w1, w2, 8u * a);
    } else {
        lo = ldb(p) | (nb > 1 ? ldb(p + 1) << 8 : 0u) | (nb > 2 ? ldb(p + 2) << 16 : 0u) | (nb > 3 ? ldb(p + 3) << 24 : 0u);
        hi = (nb > 4 ? ldb(p + 4) : 0u) | (nb > 5 ? ldb(p + 5) << 8 : 0u) | (nb > 6 ? ldb(p + 6) << 16 : 0u) | (nb > 7 ? ldb(p + 7) << 24 : 0u);
    }
}

// The pair of source pixels (c, c + 1) of one row as k_deskew reads packed RGB: lo = R_c G_c B_c R_c+1, hi = G_c+1 B_c+1 (upper half
// unspecified).  An interleaved layout loads its 2 x channels bytes from pixel c with load_bytes and reorders them (pair_rgb); the
// planar layout loads two bytes from each plane (planar_pair; p = pixel c of the R plane, end = the R plane's end)
CB_HD void pair_rgb(int layout, uint32_t& lo, uint32_t& hi)
{
    const uint32_t l = lo;
    switch (layout) {
    case CB200_LAYOUT_BGR: lo = prmt(l, hi, 0x5012); hi = prmt(l, hi, 0x0034); break;
    case CB200_LAYOUT_RGBA: lo = prmt(l, hi, 0x4210); hi = prmt(l, hi, 0x0065); break;
    case CB200_LAYOUT_BGRA: lo = prmt(l, hi, 0x6012); hi = prmt(l, hi, 0x0045); break;
    default: break;
    }
}

CB_HD void planar_pair(const uint8_t* p, uint64_t plane, const uint8_t* end, uint32_t& lo, uint32_t& hi)
{
    uint32_t r, g, b, u;
    load_bytes(p, end, 2, r, u);
    load_bytes(p + plane, end + plane, 2, g, u);
    load_bytes(p + 2 * plane, end + 2 * plane, 2, b, u);
    lo = prmt(prmt(r, g, 0x1040), b, 0x3410);
    hi = prmt(g, b, 0x0051);
}

CB_HD void tap_pair(const uint8_t* p, uint64_t plane, int layout, const uint8_t* end, uint32_t& lo, uint32_t& hi)
{
    if (layout == CB200_LAYOUT_RGB_PLANAR) { planar_pair(p, plane, end, lo, hi); return; }
    load_bytes(p, end, (uint32_t)channels(layout) * 2u, lo, hi);
    pair_rgb(layout, lo, hi);
}

// The scan's Gaussian radius for a w x h picture (Scanner.h:93-103, :155-157): the kernel unit is the power of two above
// 0.002 x the short side, plus one, at least 3 taps.  Short sides 60 .. 1499 give 3 taps, 1500 .. 2499 give 5, 2500 .. 4499 give 9
CB_HD int blur_radius(int w, int h)
{
    unsigned v = (unsigned)((w < h ? w : h) * 0.002);
    v--;
    v |= v >> 1; v |= v >> 2; v |= v >> 4; v |= v >> 8; v |= v >> 16;
    unsigned unit = v + 2;
    if (unit < 3u) unit = 3u;
    return (int)(unit / 2);
}

// The rule every camera call applies to a picture descriptor (scan.cu: picture_batch, check_picture_sizes and check_spans print
// why, in that order): true when the calls refuse it -- a null data pointer, an unknown layout, a negative pitch, a short side below
// 60 or a Gaussian beyond 9 taps (4500 pixels or more), a row pitch below w x channels, overlapping planes, a span of 4 GB or more.
// With bounds (a plan that reads its descriptors from device memory) it also refuses a short side outside [min_short, max_short]
// and a long side above max_long.  The pitch rules come before any product that could overflow: a row pitch of 4 GB or more is
// refused whatever the rest says
CB_HD bool picture_refused(const cb200_picture& p, const cb200_picture_bounds* bounds)
{
    if (!p.data || !known(p.layout) || p.row_pitch < 0 || p.plane_pitch < 0) return true;
    const int s = p.w < p.h ? p.w : p.h, l = p.w < p.h ? p.h : p.w;
    if (s < 60 || blur_radius(p.w, p.h) > 4) return true;
    if (bounds && (s < bounds->min_short || s > bounds->max_short || l > bounds->max_long)) return true;
    const int64_t lim = (int64_t)1 << 32, row = (int64_t)p.w * channels(p.layout);
    const bool planar = p.layout == CB200_LAYOUT_RGB_PLANAR;
    if (p.row_pitch < row || p.row_pitch >= lim || (planar && p.plane_pitch >= lim)) return true;
    if (planar && p.plane_pitch < (int64_t)p.h * p.row_pitch) return true;
    return (planar ? 2 * p.plane_pitch : 0) + (int64_t)(p.h - 1) * p.row_pitch + row >= lim;
}

constexpr int kBlurTileW = 128, kBlurTileH = 32;          // k_scan_blur4's tile

CB_HD int64_t blur_tiles(int w, int h) { return (((int64_t)w + kBlurTileW - 1) / kBlurTileW) * (((int64_t)h + kBlurTileH - 1) / kBlurTileH); }
// the blur radii 1, 2, 4 (3, 5, 9 taps) as the plan's radius groups 0, 1, 2
CB_HD int radius_group(int R) { return R == 1 ? 0 : (R == 2 ? 1 : 2); }

// Slot i of a plan over device descriptors (k_plan_pictures, scan.cu), everything but its tile0: the descriptor table entry, its blur
// radius group and tile count.  An empty slot (its receiver out of range, or in a detect plan no candidate mode: the caller decides)
// does not read its descriptor; it and a refused slot
// get the plan's stand-in -- a black min_short x min_short RGB picture of pitch 0 at `standin`, which fails extraction.  The blurred
// picture of slot i sits at i x slot_bytes (a multiple of 4) in the scan's buffer at blur_base; the word path is pic_table's rule
struct PlanSlot { int group, tiles; bool refused; };
CB_HD PlanSlot plan_slot(const cb200_picture* pics, bool empty, const cb200_picture_bounds& bounds, uint64_t standin, uint64_t blur_base,
                         uint64_t slot_bytes, int i, PicDesc& d)
{
    cb200_picture p;
    bool refused = false;
    if (!empty) { p = pics[i]; refused = picture_refused(p, &bounds); }
    if (empty || refused) p = cb200_picture{reinterpret_cast<const uint8_t*>(standin), bounds.min_short, bounds.min_short, 0, 0, CB200_LAYOUT_RGB};
    const bool planar = p.layout == CB200_LAYOUT_RGB_PLANAR;
    d.src = reinterpret_cast<uint64_t>(p.data); d.blur = (uint64_t)i * slot_bytes; d.w = p.w; d.h = p.h;
    d.pitch = (uint64_t)p.row_pitch; d.plane = planar ? (uint64_t)p.plane_pitch : 0; d.layout = p.layout;
    d.words = (p.w % 4 == 0) && (d.src % 4 == 0) && (d.pitch % 4 == 0) && (d.plane % 4 == 0) && ((blur_base + d.blur) % 4 == 0);
    d.tile0 = 0;
    return PlanSlot{radius_group(blur_radius(p.w, p.h)), (int)blur_tiles(p.w, p.h), refused && !empty};   // < 2^31: the bounds
}

}  // namespace layout
}  // namespace cb200
