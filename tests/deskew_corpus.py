"""The deskew's arithmetic contract as a float64 numpy model, and a generated corpus of transforms that reaches its edges.  Test
infrastructure only (no GPU).

warp_model restates what libcimbar_b200/csrc/deskew.cu says k_deskew computes -- cv::warpPerspective(INTER_LINEAR, BORDER_CONSTANT
0) with OpenCV's own arithmetic: the forward transform inverted by cv::invert (det3 + adjugate), OpenCV's block origin bx,
W = 32 / w, cvRound (ties to even), the clamp to int and saturate_cast<short>, 5-bit fractions, the fixed-point bilinear blend
(sum + 512) >> 10 and taps outside the source as 0.  Every operation is one IEEE double operation (numpy and Python floats never
contract into an FMA), as in the kernel.

cases(W, H) gives the corpus for one output geometry: each case carries a premise, a predicate on the model's statistics that
says the case reaches the edge it is there for (a pixel with w == 0, an exact tie, a saturated coordinate, a clamped tap pair...),
so a corpus that drifted away from its edges fails rather than passing quietly."""
from dataclasses import dataclass
from functools import lru_cache
from typing import Callable

import cv2
import numpy as np

INT_MIN, INT_MAX = -2147483648.0, 2147483647.0
GEOMETRIES = [(1024, 1024), (1024, 720), (736, 637)]        # modes 68 (B), 67 (Bm), 66 (Bu): (W, H)
MODE_OF = {(1024, 1024): 68, (1024, 720): 67, (736, 637): 66}
FAMILIES = ["quad", "turn", "tie", "tiny", "large", "horizon", "scale", "scan"]


def invert3(M):
    """cv::invert of a 3x3 double matrix (DECOMP_LU: det3 + adjugate), or None when the determinant is 0"""
    S = [float(v) for v in np.asarray(M, np.float64).reshape(9)]

    def cf(a, b, c, d):
        return S[a] * S[b] - S[c] * S[d]

    d = S[0] * cf(4, 8, 5, 7) - S[1] * cf(3, 8, 5, 6) + S[2] * cf(3, 7, 4, 6)
    if d == 0.0:
        return None
    d = 1.0 / d
    return np.array([cf(4, 8, 5, 7) * d, cf(2, 7, 1, 8) * d, cf(1, 5, 2, 4) * d,
                     cf(5, 6, 3, 8) * d, cf(0, 8, 2, 6) * d, cf(2, 3, 0, 5) * d,
                     cf(3, 7, 4, 6) * d, cf(1, 6, 0, 7) * d, cf(0, 4, 1, 3) * d])


def _round(v, half_away):
    """cvRound (to nearest, ties to even); half_away: ties away from zero instead (a deliberate slip, for the mutation check)"""
    if not half_away:
        return np.rint(v)
    t = np.trunc(v)
    return np.where(np.abs(v - t) >= 0.5, t + np.sign(v), t)


def warp_model(src_rgb, M, W, H, half_away=False, stats=False):
    """cv2.warpPerspective(src_rgb, M, (W, H), flags=INTER_LINEAR) as deskew.cu states it: an (H, W, 3) uint8 frame, and with
    stats=True also a dict of what the transform did (see the keys below)"""
    src = np.ascontiguousarray(src_rgb, np.uint8)
    h, w = src.shape[:2]
    inv = invert3(M)
    if inv is None:
        raise ValueError("singular perspective transform")
    m0, m1, m2, m3, m4, m5, m6, m7, m8 = (float(v) for v in inv)
    bh0 = min(16, H)
    bw0 = min(1024 // bh0, W)
    xi = np.arange(W)
    bx = (xi // bw0 * bw0).astype(np.float64)
    x1 = (xi - xi // bw0 * bw0).astype(np.float64)
    y = np.arange(H, dtype=np.float64)[:, None]
    X0 = (m0 * bx + m1 * y) + m2
    Y0 = (m3 * bx + m4 * y) + m5
    W0 = (m6 * bx + m7 * y) + m8
    Wv = W0 + m6 * x1
    nz = Wv != 0
    Wr = np.where(nz, 32.0 / np.where(nz, Wv, 1.0), 0.0)
    fX0 = (X0 + m0 * x1) * Wr
    fY0 = (Y0 + m3 * x1) * Wr
    # std::max((double)INT_MIN, std::min((double)INT_MAX, v)), with std::min / std::max's own comparisons
    fX = np.where(fX0 < INT_MAX, fX0, INT_MAX)
    fX = np.where(INT_MIN < fX, fX, INT_MIN)
    fY = np.where(fY0 < INT_MAX, fY0, INT_MAX)
    fY = np.where(INT_MIN < fY, fY, INT_MIN)
    X = _round(fX, half_away).astype(np.int64)
    Y = _round(fY, half_away).astype(np.int64)
    sx0, sy0 = X >> 5, Y >> 5
    sx, sy = np.clip(sx0, -32768, 32767), np.clip(sy0, -32768, 32767)        # saturate_cast<short>
    ax, ay = X & 31, Y & 31
    x0in, x1in = (sx >= 0) & (sx < w), (sx + 1 >= 0) & (sx + 1 < w)
    y0in, y1in = (sy >= 0) & (sy < h), (sy + 1 >= 0) & (sy + 1 < h)
    acc = np.full((H, W, 3), 512, np.int64)
    for wx, wy, dx, dy, inx, iny in ((32 - ax, 32 - ay, 0, 0, x0in, y0in), (ax, 32 - ay, 1, 0, x1in, y0in),
                                     (32 - ax, ay, 0, 1, x0in, y1in), (ax, ay, 1, 1, x1in, y1in)):
        tap = src[np.clip(sy + dy, 0, h - 1), np.clip(sx + dx, 0, w - 1)].astype(np.int64)
        acc += np.where(inx & iny, wx * wy, 0)[..., None] * tap
    out = (acc >> 10).astype(np.uint8)
    if not stats:
        return out
    rows = y0in | y1in
    even, away = _round(fX, False), _round(fX, True)
    wrap_x = (sx0 + 32768) % 65536 - 32768                                      # what a plain (short) cast would keep
    st = {
        "w_zero": int((~nz).sum()),                                             # pixels with w == 0 exactly
        "horizon": bool((Wv > 0).any() and (Wv < 0).any()),                     # the line w = 0 crosses the frame
        "int_clamped": int(((fX0 != fX) | (fY0 != fY)).sum()),                  # fX or fY beyond the int range
        "short_saturated": int(((sx0 != sx) | (sy0 != sy)).sum()),              # X >> 5 or Y >> 5 beyond the short range
        # saturated pixels whose 16-bit wrap would have landed on a source pixel: a truncating cast would read there
        "wrap_inside": int(((sx0 != sx) & (wrap_x >= 0) & (wrap_x < w) & y0in).sum()),
        "tie_moves": int(((even != away) | (_round(fY, False) != _round(fY, True))).sum()),   # ties where even != away
        "left_live": int(((sx == -1) & (ax > 0) & rows).sum()),                 # pair clamped left, its tap x1 = 0 weighted
        "right_live": int(((sx == w - 1) & rows).sum()),                        # pair clamped right, its tap x0 = w - 1 weighted
        "decreasing": bool((np.diff(sx, axis=1) < 0).any() or (np.diff(sy, axis=1) < 0).any()),
        # the largest step in the source between neighbouring pixels, along the rows (sx) and down the columns (sy)
        "max_step": int(max(np.abs(np.diff(sx, axis=1)).max(initial=0), np.abs(np.diff(sy, axis=0)).max(initial=0))),
        "inside": int((x0in & y0in).sum()),                                     # pixels whose top-left tap is in the source
    }
    return out, st


@dataclass
class Case:
    name: str
    family: str
    src: np.ndarray                     # (h, w, 3) uint8 RGB
    M: np.ndarray                       # forward 3x3 float64, as cv2.warpPerspective takes it
    premise: str
    holds: Callable[[dict], bool]


def output_points(W, H):
    """where Deskewer::deskew sends the four anchor centres (tl, tr, bl, br)"""
    return np.float32([[30, 30], [W - 30, 30], [30, H - 30], [W - 30, H - 30]])


@lru_cache(maxsize=None)
def noise(w, h, seed):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)


@lru_cache(maxsize=None)
def _scanned():
    """the sample photographs in which the scan oracle finds four anchors, with the corners Extractor::extract takes from them"""
    from oracle_lib import load_sample
    from scan_oracle_lib import ScanOracle
    so = ScanOracle()
    out = []
    for name in ("6bit/4_30_f0_627.jpg", "6bit/4_30_f2_734.jpg", "6bit/4_30_f1_360.jpg", "b/ex2434.jpg", "b/ex380.jpg"):
        pic = load_sample(name)
        anchors, _ = so.scan(pic)
        if anchors is not None and len(anchors) == 4:
            out.append((name, pic, np.float32(so.corners(anchors)).reshape(4, 2)))
    return out


def camera_quad(rng, w, h, integer):
    base = np.float32([[0.12 * w, 0.1 * h], [0.9 * w, 0.14 * h], [0.08 * w, 0.88 * h], [0.93 * w, 0.9 * h]])
    q = base + rng.uniform(-0.06, 0.06, (4, 2)).astype(np.float32) * np.float32([w, h])
    return np.round(q).astype(np.float32) if integer else q


def _affine(a, b, c, d, e, f):
    return np.array([[a, b, c], [d, e, f], [0.0, 0.0, 1.0]])


@lru_cache(maxsize=None)
def cases(W, H):
    """the corpus for frames of W x H (a list of Case; cached, do not modify)"""
    outp = output_points(W, H)
    rng = np.random.default_rng(2024)
    out = []

    def add(name, family, src, M, premise, holds):
        out.append(Case(name, family, src, np.asarray(M, np.float64), premise, holds))

    mostly_inside = ("most pixels sample the source", lambda s: s["inside"] > 0.5 * W * H)
    # camera-like quads: float corners and integer ones (the reference's anchor centres are integer points)
    src = noise(1300, 1000, 1)
    for k in range(4):
        for integer in (False, True):
            q = camera_quad(rng, 1300, 1000, integer)
            add(f"quad{k}{' int' if integer else ''}", "quad", src, cv2.getPerspectiveTransform(q, outp), *mostly_inside)
    # quarter and half turns and a mirror: the source coordinates fall along a thread's four pixels
    src = noise(900, 700, 2)
    q = camera_quad(rng, 900, 700, True)
    tl, tr, bl, br = q
    for name, perm in (("rot90", [bl, tl, br, tr]), ("rot180", [br, bl, tr, tl]), ("rot270", [tr, br, tl, bl]), ("mirror", [tr, tl, br, bl])):
        add(name, "turn", src, cv2.getPerspectiveTransform(np.float32(perm), outp),
            "a source coordinate decreases along the row", lambda s: s["decreasing"] and s["inside"] > 0.5 * W * H)
    # translations by odd multiples of 1/64 pixel: fX or fY is exactly k + 0.5 and cvRound's ties to even decide
    src = noise(W + 8, H + 8, 3)
    for tx, ty in ((3 / 64, -5 / 64), (1 / 64, 7 / 64), (-9 / 64, 3 / 64)):
        add(f"shift {round(tx * 64)}/64 {round(ty * 64)}/64", "tie", src, _affine(1, 0, tx, 0, 1, ty),
            "some tie rounds differently to even than away from zero", lambda s: s["tie_moves"] > 0)
    add("scale 1/2, shift 1/128 -3/128", "tie", noise(2 * W + 4, 2 * H + 4, 4), _affine(0.5, 0, 1 / 128, 0, 0.5, -3 / 128),
        "some tie rounds differently to even than away from zero", lambda s: s["tie_moves"] > 0)
    # tiny sources: every tap pair is clamped at some edge (2 wide: c = 0 = w - 2 throughout)
    for w, h in ((2, 2), (3, 2), (2, 5), (7, 3)):
        rect = np.float32([[-0.6, -0.7], [w - 0.4, -0.7], [-0.6, h - 0.3], [w - 0.4, h - 0.3]])
        add(f"tiny {w}x{h}", "tiny", noise(w, h, 10 + w * 10 + h), cv2.getPerspectiveTransform(rect, outp),
            "pairs clamped left and right are both weighted", lambda s: s["left_live"] > 0 and s["right_live"] > 0)
    # strong minification from large pictures
    for w, h in ((4000, 3000), (2000, 4400)):
        add(f"large {w}x{h}", "large", noise(w, h, 5), cv2.getPerspectiveTransform(camera_quad(rng, w, h, False), outp),
            "neighbouring pixels are 3 or more source pixels apart", lambda s: s["max_step"] >= 3 and s["inside"] > 0.5 * W * H)
    # the horizon inside the frame; power-of-two entries whose inverse has w == 0 exactly on a column of 64-pixel block origins
    src = noise(1200, 1100, 6)
    add("horizon w == 0", "horizon", src, np.array([[1, 0, 0], [0, 1, 0], [1 / 512, 1 / 1024, 1]]),
        "w == 0 exactly on some pixel", lambda s: s["w_zero"] > 0 and s["horizon"])
    add("horizon tilted", "horizon", src, np.array([[0.9, 0.05, 20], [-0.03, 1.1, 10], [1 / 700.3, -1 / 1900.7, 1]]),
        "the line w = 0 crosses the frame", lambda s: s["horizon"])
    # tiny forward scales: coordinates past the short range (1e-4) and past the int range (1e-7)
    src = noise(640, 480, 7)
    add("scale 1e-4", "scale", src, _affine(1e-4, 0, 0, 0, 1e-4, 0),
        "X >> 5 saturates where a 16-bit wrap would land in the source", lambda s: s["wrap_inside"] > 0)
    add("scale -1e-4, 1e-4", "scale", src, _affine(-1e-4, 0, 0, 0, 1e-4, 0),
        "X >> 5 saturates", lambda s: s["short_saturated"] > 0)
    add("scale 1e-7", "scale", src, _affine(1e-7, 0, 0, 0, 1e-7, 0),
        "fX leaves the int range", lambda s: s["int_clamped"] > 0)
    # the scan oracle's corners on the sample photographs: the transforms the camera path makes
    for name, pic, corners in _scanned():
        add(f"scan {name}", "scan", pic, cv2.getPerspectiveTransform(corners, outp), *mostly_inside)
    return out


def cv2_warp(src_rgb, M, W, H):
    return cv2.warpPerspective(src_rgb, np.asarray(M, np.float64), (W, H), flags=cv2.INTER_LINEAR)


def first_mismatch(got, want, src_rgb, M):
    """a failure message: how many bytes differ, and the first bad pixel with the kernel's, cv2's and the model's values"""
    bad = np.argwhere((got != want).any(axis=2))
    if not len(bad):
        return "equal"
    y, x = (int(v) for v in bad[0])
    H, W = want.shape[:2]
    model = warp_model(src_rgb, M, W, H)
    return (f"{int((got != want).sum())} bytes in {len(bad)} pixels differ; first ({x}, {y}): kernel {got[y, x].tolist()}, "
            f"cv2 {want[y, x].tolist()}, model {model[y, x].tolist()}")
