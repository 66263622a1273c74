"""A seeded corpus for the colour-correction side path, and the plain cv2 / numpy references it is checked against.

References (nothing here calls the oracle's or the kernels' arithmetic):
- cv2_fit: color_correction::get_moore_penrose_lsm verbatim, cv2.invert(DECOMP_SVD) then cv2.gemm in float32.  For a 3 x N
  matrix with N <= 9 both stay on OpenCV's own Jacobi SVD and gemm (tests/test_ccm_contract.py pins cv2_fit to the reference's
  printed matrices first, so a cv2 that routes them elsewhere fails there).
- von_kries: get_adaptation_matrix<von_kries>(white, (255, 255, 255)) in float32, in cv::Matx's product order (s = 0;
  s += a(i, k) * b(k, j)) with Matx::inv's closed-form 3 x 3 inverse.
- best_color: CimbDecoder::get_best_color under a CCM, vectorised: Matx * vector, std::max({r, g, b, 1}) and std::min({r, g, b,
  48}) as max_element / min_element with first-wins `<` (so a NaN in r wins both, a NaN in g or b is skipped), 255.0 / (max - min)
  as a double division rounded to float, fix_single_color's clamps, the (uchar) cast as x86-64 gcc compiles it (cvttss2si to
  int32, low byte: NaN and out-of-range values give 0) and color_diff with first-wins `<` over the palette.

Cases (seeded; the whole corpus is generated in a few seconds of one core):
- fit_cases(): N x 3 `actual` / `desired` pairs, N = 5..9, desired rows from the palettes of every colour mode, the last row the
  white (255, 255, 255).  Families: camera-like tints with noise, grey (rank 1), near-grey, one or two channels constant near 0 or
  near 255, all rows equal, black with the white floor of 1, and rows of 0 and 255 only.  Each case carries a premise on
  cv2.SVDecomp's singular values W that says which edge of the back-substitution it reaches: the threshold is ΣW * 2^-51 in
  OpenCV's float SVBkSb ((float)(DBL_EPSILON * 2)), and the "band" (2^-51 ΣW, 2 FLT_EPSILON ΣW] is where a restatement with
  FLT_EPSILON's factor drops a singular value that OpenCV inverts.
- simple_whites(): whites for CC_SIMPLE, including anchor whites (multiples of 1/16) whose von Kries denominator T . white is
  exactly 0.0f in float, so the matrix holds inf and NaN.
- classifier_matrices(): every fitted matrix of the corpus, the CC_SIMPLE matrices of those whites, and hand-made ones (0, +-I,
  1e-30 I, 1e30 I, denormals, a single inf, NaN in row 0 only, NaN in row 2 only)."""
import ctypes as C
import functools

import cv2
import numpy as np

F32 = np.float32
FLT_EPS = float(np.finfo(np.float32).eps)
FLT_MIN = float(np.finfo(np.float32).tiny)
CV_EPS = float(F32(2 * np.finfo(np.float64).eps))          # SVBkSb's (float)(DBL_EPSILON * 2) = 2^-51
FLT_FACTOR = float(F32(2 * FLT_EPS))                        # the factor that drops a singular value in the band
T_VON_KRIES = np.array([0.4002400, 0.7076000, -0.0808100, -0.2263000, 1.1653200, 0.0457000, 0.0, 0.0, 0.9182200], F32)

# (num_colors, color_mode) of every colour palette a decoder uses: legacy modes 4 / 8 use colour mode 0, the 8x8 modes 66-68 mode 1
PALETTE_KEYS = [(4, 0), (8, 0), (4, 1), (8, 1)]


@functools.lru_cache(maxsize=None)
def palette(num_colors, color_mode):
    """CimbDecoder::get_color of every index (the palettes are data: the oracle's table, Common.cpp)"""
    from oracle_lib import Oracle
    lib = Oracle().lib
    out = np.zeros((num_colors, 3), np.uint8)
    for i in range(num_colors):
        lib.cbo_palette(i, num_colors, color_mode, out[i].ctypes.data_as(C.POINTER(C.c_uint8)))
    return out


# ------------------------------------------------------------------------------------------------ references
def cv2_fit(actual, desired):
    """get_moore_penrose_lsm: x = desired^T, y = actual^T, z = invert(y, DECOMP_SVD), x * z (float32 3 x 3)"""
    y = np.ascontiguousarray(np.asarray(actual, F32).T)
    x = np.ascontiguousarray(np.asarray(desired, F32).T)
    _, z = cv2.invert(y, flags=cv2.DECOMP_SVD)
    return cv2.gemm(x, z, 1, None, 0).astype(F32)


def singular_values(actual):
    """cv2.SVDecomp's W of y = actual^T (float32, descending)"""
    w, _, _ = cv2.SVDecomp(np.ascontiguousarray(np.asarray(actual, F32).T))
    return w.reshape(-1).astype(F32)


def _matx_mul(a, b):
    out = np.zeros(9, F32)
    for i in range(3):
        for j in range(3):
            s = F32(0)
            for k in range(3):
                s = F32(s + F32(a[3 * i + k] * b[3 * k + j]))
            out[3 * i + j] = s
    return out


def _matx_inv(a):
    """cv::Matx<float, 3, 3>::inv(): determinant in float, d = 1 / d, cofactors * d; zeros when singular"""
    a = np.asarray(a, F32)
    mm = lambda x, y, z, w: F32(F32(x * y) - F32(z * w))
    d = F32(F32(F32(a[0] * mm(a[4], a[8], a[7], a[5])) - F32(a[1] * mm(a[3], a[8], a[6], a[5]))) + F32(a[2] * mm(a[3], a[7], a[6], a[4])))
    if d == 0:
        return np.zeros(9, F32)
    d = F32(F32(1) / d)
    cof = [mm(a[4], a[8], a[5], a[7]), mm(a[2], a[7], a[1], a[8]), mm(a[1], a[5], a[2], a[4]),
           mm(a[5], a[6], a[3], a[8]), mm(a[0], a[8], a[2], a[6]), mm(a[2], a[3], a[0], a[5]),
           mm(a[3], a[7], a[4], a[6]), mm(a[1], a[6], a[0], a[7]), mm(a[0], a[4], a[1], a[3])]
    return np.array([F32(c * d) for c in cof], F32)


def von_kries(white, desired=(255.0, 255.0, 255.0)):
    """get_adaptation_matrix<von_kries>(white, desired): T.inv() * diag((T desired) / (T white)) * T, 9 floats row-major"""
    T = T_VON_KRIES
    w, dd = np.asarray(white, F32), np.asarray(desired, F32)
    with np.errstate(all="ignore"):
        d = np.zeros(9, F32)
        for i in range(3):
            m1 = m2 = F32(0)
            for k in range(3):
                m1 = F32(m1 + F32(T[3 * i + k] * w[k]))
                m2 = F32(m2 + F32(T[3 * i + k] * dd[k]))
            d[4 * i] = F32(m2 / m1)
        return _matx_mul(_matx_mul(_matx_inv(T), d), T)


def von_kries_denominators(white):
    """T . white per row, in Matx's order (a row whose value is exactly 0 makes the matrix non-finite)"""
    T, w = T_VON_KRIES, np.asarray(white, F32)
    out = []
    for i in range(3):
        s = F32(0)
        for k in range(3):
            s = F32(s + F32(T[3 * i + k] * w[k]))
        out.append(s)
    return np.array(out, F32)


def _uchar(c):
    """(uchar) of a float as x86-64 gcc compiles it: cvttss2si to int32 (NaN and |c| >= 2^31 give 0x80000000), low byte"""
    ok = np.isfinite(c) & (np.abs(c) < 2.0 ** 31)
    return np.where(ok, np.trunc(np.where(ok, c, 0)).astype(np.int64) & 0xFF, 0).astype(np.int64)


def best_color(ccm, means, num_colors, color_mode, pal=None):
    """CimbDecoder::get_best_color(r, g, b) with the CCM active, for every row of means ((n, 3) integers) -> (n,) uint8"""
    m = np.asarray(ccm, F32).reshape(9)
    x = np.asarray(means).astype(F32)
    pal = palette(num_colors, color_mode).astype(np.int64) if pal is None else pal
    with np.errstate(all="ignore"):
        ch = []
        for i in range(3):
            s = np.zeros(len(x), F32)
            for k in range(3):
                s = (s + m[3 * i + k] * x[:, k]).astype(F32)
            ch.append(s)
        r, g, b = ch
        one, floor = F32(1.0), F32(48.0)
        mx = r.copy()
        for v in (g, b):
            mx = np.where(mx < v, v, mx)
        mx = np.where(mx < one, one, mx)
        mn = r.copy()
        for v in (g, b):
            mn = np.where(v < mn, v, mn)
        mn = np.where(floor < mn, floor, mn)
        mn = np.where(mn >= mx, F32(0), mn).astype(F32)
        adjust = (255.0 / (mx - mn).astype(F32).astype(np.float64)).astype(F32)
        cols = []
        for c in (r, g, b):
            c = ((c - mn).astype(F32) * adjust).astype(F32)
            c = np.where(c > (F32(245) - mn).astype(F32), F32(255), c)
            c = np.where(c < 0, F32(0), c)
            cols.append(_uchar(c))
    a = np.stack([cols[0] - cols[1], cols[1] - cols[2], cols[2] - cols[0]], 1)
    p = np.stack([pal[:, 0] - pal[:, 1], pal[:, 1] - pal[:, 2], pal[:, 2] - pal[:, 0]], 1)
    d = ((a[:, None, :] - p[None, :, :]) ** 2).sum(2)
    return d.argmin(1).astype(np.uint8)                     # argmin: the first minimum, as `distance < best_distance`


# ------------------------------------------------------------------------------------------------ fit cases
class FitCase:
    def __init__(self, name, family, actual, desired, premises):
        self.name, self.family, self.premises = name, family, premises
        self.actual, self.desired = np.asarray(actual, F32), np.asarray(desired, F32)

    @property
    def rows(self):
        return len(self.actual)

    @property
    def premise(self):
        return " and ".join(PREMISES[k][0] for k in self.premises)

    def holds(self):
        w = singular_values(self.actual)
        return all(PREMISES[k][1](w) for k in self.premises)


def _band(w):
    s = float(w.astype(np.float64).sum())
    return any(CV_EPS * s < float(v) <= FLT_FACTOR * s for v in w)


def _full(w):
    return float(w.min()) > FLT_FACTOR * float(w.astype(np.float64).sum())


def _dropped(w):
    return float(w.min()) <= CV_EPS * float(w.astype(np.float64).sum())


def _tiny(w):
    return float(w.min()) <= FLT_MIN


PREMISES = {
    "full": ("every W > 2 FLT_EPSILON ΣW: full rank, both factors invert all three", _full),
    "band": ("some W lies in (2^-51 ΣW, 2 FLT_EPSILON ΣW]: OpenCV inverts it, the FLT_EPSILON factor drops it", _band),
    "dropped": ("the smallest W <= 2^-51 ΣW: OpenCV drops it too", _dropped),
    "tiny": ("some W <= FLT_MIN (OpenCV's random-vector branch; the threshold >= 2^-51 |white| is far above FLT_MIN)", _tiny),
}
# what every case of a family reaches; the mixed families' share of each edge is checked by the contract test
FAMILY_PREMISES = {"tint": ("full",), "grey": ("band", "tiny"), "equal_rows": ("dropped", "tiny")}
FAMILIES = ["tint", "grey", "near_grey", "low_channels", "high_channels", "equal_rows", "black", "binary"]


def _desired(rng, n_rows):
    """n_rows - 1 distinct palette colours of a palette that has that many, then the white row"""
    keys = [k for k in PALETTE_KEYS if k[0] >= n_rows - 1]
    nc, cm = keys[rng.integers(len(keys))]
    pal = palette(nc, cm)
    pick = rng.permutation(nc)[: n_rows - 1]
    return np.concatenate([pal[pick].astype(F32), np.full((1, 3), 255, F32)]), (nc, cm)


def _white(rng, lo=1.0, hi=255.0):
    return np.round(rng.uniform(lo, hi, 3) * 16) / 16           # calculateWhite: a mean of 16 pixels, floor 1


def fit_cases(seed=0, per_family=48):
    rng = np.random.default_rng(seed)
    out = []
    for family in FAMILIES:
        for i in range(per_family):
            n = 5 + i % 5
            desired, key = _desired(rng, n)
            k = n - 1
            if family == "tint":
                gain, off = rng.uniform(0.4, 1.1, 3), rng.uniform(0, 40, 3)
                act = np.clip(np.floor(desired[:k] * gain + off + rng.normal(0, 6, (k, 3))), 0, 255)
                white = np.clip(np.round((255 * gain + off + rng.normal(0, 4, 3)) * 16) / 16, 1, 255)
            elif family == "grey":
                v = rng.integers(0, 256, k)
                act = np.repeat(v[:, None], 3, 1).astype(F32)
                white = np.full(3, float(max(1, rng.integers(0, 256))) if i % 3 else np.round(rng.uniform(1, 255) * 16) / 16)
            elif family == "near_grey":
                v = rng.integers(1, 255, k)
                act = np.repeat(v[:, None], 3, 1).astype(np.int64)
                r, c = rng.integers(k), rng.integers(3)
                act[r, c] += rng.choice([-1, 1])
                white = np.full(3, float(rng.integers(1, 256)))
            elif family in ("low_channels", "high_channels"):
                act = rng.integers(0, 256, (k, 3)).astype(np.int64)
                white = _white(rng)
                chans = rng.permutation(3)[: 1 + i % 2]
                for c in chans:
                    if family == "low_channels":
                        act[:, c] = rng.integers(0, 3, k) if i % 4 >= 2 else rng.integers(0, 3)
                        white[c] = 1.0 if i % 4 < 2 else white[c]
                    else:
                        act[:, c] = rng.integers(250, 256, k) if i % 4 >= 2 else rng.integers(250, 256)
                        white[c] = float(act[0, c]) if i % 4 < 2 else white[c]
            elif family == "equal_rows":
                row = rng.integers(0, 256, 3)
                act = np.repeat(row[None], k, 0)
                white = row.astype(np.float64).clip(1) if i % 2 else _white(rng)
            elif family == "black":
                act = np.zeros((k, 3)) if i % 2 == 0 else rng.integers(0, 2, (k, 3))
                white = np.ones(3)
            else:                                                   # binary
                act = rng.choice([0, 255], (k, 3))
                white = rng.choice([1.0, 255.0], 3) if i % 2 else np.full(3, 255.0)
            actual = np.concatenate([np.asarray(act, F32), np.asarray(white, F32)[None]])
            out.append(FitCase(f"{family}-{i}-n{n}-c{key[0]}m{key[1]}", family, actual, desired, FAMILY_PREMISES.get(family, ())))
    return out


def premise_counts(cases):
    """how many cases reach each premise (a case can reach several)"""
    counts = {k: 0 for k in PREMISES}
    for c in cases:
        w = singular_values(c.actual)
        for k in counts:
            counts[k] += bool(PREMISES[k][1](w))
    return counts


# ------------------------------------------------------------------------------------------------ CC_SIMPLE whites
def zero_denominator_whites(limit=24, seed=0):
    """anchor whites (multiples of 1/16 in [1, 255]) with T . white == 0.0f exactly in some row: a vectorised search over
    rows 0 and 1 (row 2 is 0.91822 w_b > 0), a fixed sample of what it finds"""
    T = T_VON_KRIES
    grid = (np.arange(16, 255 * 16 + 1) / 16).astype(F32)      # the 4065 possible means of one channel
    found = set()
    for row in (0, 1):
        t0, t1, t2 = T[3 * row: 3 * row + 3]
        a = (t0 * grid).astype(F32)                              # s = ((0 + t0 r) + t1 g) + t2 b == 0 exactly
        for b in grid[::5]:                                      # <=> fl(t0 r + fl(t1 g)) == -fl(t2 b)
            c = F32(t2 * b)
            g0 = np.rint((-c - a.astype(np.float64)) / float(t1) * 16)
            for off in (-1, 0, 1):
                gi = g0 + off
                ok = (gi >= 16) & (gi <= 255 * 16)
                g = (np.where(ok, gi, 16) / 16).astype(F32)
                s = ((a + (t1 * g).astype(F32)).astype(F32) + c).astype(F32)
                for h in np.nonzero(ok & (s == 0))[0]:
                    found.add((row, float(grid[h]), float(g[h]), float(b)))
    found = sorted(found)
    rng = np.random.default_rng(seed)
    pick = rng.permutation(len(found))[:limit] if len(found) > limit else np.arange(len(found))
    out = [found[i] for i in sorted(pick)]
    for row, r, g, b in out:
        assert von_kries_denominators((r, g, b))[row] == 0, (row, r, g, b)
    return out


def simple_whites():
    """(name, white, premise) for CC_SIMPLE: the floor, 255, single-channel whites and zero-denominator whites"""
    out = [("floor", (1.0, 1.0, 1.0), "finite"), ("full", (255.0, 255.0, 255.0), "finite"),
           ("red", (255.0, 1.0, 1.0), "finite"), ("green", (1.0, 255.0, 1.0), "finite"), ("blue", (1.0, 1.0, 255.0), "finite"),
           ("mid", (128.5625, 64.0625, 200.9375), "finite"),
           ("zero-row1-issue", (13.0, 1.25, 32.5), "zero"), ("zero-row0-issue", (1.6875, 19.9375, 182.9375), "zero")]
    for row, r, g, b in zero_denominator_whites():
        out.append((f"zero-row{row}-{r}-{g}-{b}", (r, g, b), "zero"))
    return out


# ------------------------------------------------------------------------------------------------ classifier matrices
def hand_matrices():
    I = np.eye(3, dtype=F32).reshape(9)
    den = np.full(9, F32(1e-40), F32)
    one_inf = I.copy(); one_inf[4] = np.inf
    nan0 = I.copy(); nan0[0:3] = np.nan
    nan2 = I.copy(); nan2[6:9] = np.nan
    nan0_one = I.copy(); nan0_one[1] = np.nan
    return [("zero", np.zeros(9, F32)), ("identity", I), ("minus-identity", -I), ("1e-30 I", (I * F32(1e-30)).astype(F32)),
            ("1e30 I", (I * F32(1e30)).astype(F32)), ("denormals", den), ("denormal-diag", (I * F32(1e-42)).astype(F32)),
            ("single-inf", one_inf), ("nan-row0", nan0), ("nan-row2", nan2), ("nan-entry01", nan0_one)]


def classifier_matrices(fits=None):
    """(name, 9 floats) for the colour decision: the fits of the corpus (cv2's), the CC_SIMPLE matrices and the hand-made ones"""
    out = list(hand_matrices())
    for name, white, _ in simple_whites():
        out.append((f"simple-{name}", von_kries(white)))
    for c in (fit_cases() if fits is None else fits):
        out.append((f"fit-{c.name}", cv2_fit(c.actual, c.desired).reshape(9)))
    return out


# ------------------------------------------------------------------------------------------------ painted CC_FIT frames
class Painted:
    """a frame painted for CimbReader::init_ccm under a given header: `actual` / `desired` are the rows the paint was designed to
    give (colours in reverse order of first appearance, white last), None when fewer than four colours appear"""

    def __init__(self, mode_val, frame, hdr, radioactive, actual, desired, name):
        self.mode_val, self.frame, self.hdr, self.radioactive = mode_val, frame, hdr, radioactive
        self.actual, self.desired, self.name = actual, desired, name


@functools.lru_cache(maxsize=None)
def _header_layout(mode_val):
    from oracle_lib import Oracle
    ora = Oracle()
    m = ora.mode(mode_val)
    xs, ys = np.zeros(m.total_cells, np.int32), np.zeros(m.total_cells, np.int32)
    ora.lib.cbo_cell_positions(C.byref(m), 0, xs.ctypes.data_as(C.POINTER(C.c_int)), ys.ctypes.data_as(C.POINTER(C.c_int)))
    idx = np.zeros(m.total_cells, np.uint32)
    ora.lib.cbo_interleave_indices(m.total_cells, m.interleave_blocks, m.interleave_partitions, idx.ctypes.data_as(C.POINTER(C.c_uint)))
    cb = m.color_bits
    end = ora.capacity(m, cb) * 8 // cb
    interval = ora.capacity(m, m.symbol_bits + cb) * 8 // m.chunks_per_frame // cb
    return m, xs, ys, idx, list(range(0, end, interval)), 48 // cb


def header_values(mode_val, hdr, radioactive):
    """(chunk start, cell index in the header, expected colour) of every header cell init_ccm reads, in its order"""
    m, _, _, _, starts, hlen = _header_layout(mode_val)
    h, cb, out = bytearray(bytes(hdr)), m.color_bits, []
    for start in starts:
        for i in range(hlen):
            v = 0
            for k in range(cb):
                bit = i * cb + k
                v = (v << 1) | ((h[bit >> 3] >> (7 - (bit & 7))) & 1)
            out.append((start, i, v))
        nxt = ((h[4] << 8) | h[5]) + 1
        if nxt == radioactive:
            nxt += 1
        h[4], h[5] = (nxt >> 8) & 0xFF, nxt & 0xFF
    return out


def search_headers(mode_val, seed=0, tries=4000):
    """headers (6 bytes, radioactive id) that reach every row count the mode allows: {rows: (hdr, radioactive)}; rows 0 stands
    for fewer than four colours (no fit).  Headers are drawn from small alphabets of colour values, so few colours are reachable"""
    m = _header_layout(mode_val)[0]
    cb = m.color_bits
    rng = np.random.default_rng(seed)
    found = {}
    for t in range(tries):
        alphabet = rng.permutation(1 << cb)[: 1 + t % (1 << cb)]
        vals = rng.choice(alphabet, 48 // cb + 1)
        bits = "".join(format(int(v), f"0{cb}b") for v in vals)[:48]
        hdr = bytes(int(bits[8 * k: 8 * k + 8], 2) for k in range(6))
        if not any(hdr[:4]):
            continue
        bid = (hdr[4] << 8) | hdr[5]
        radioactive = (bid + 1 + t % 3) & 0xFFFF if t % 2 else 0xFFFFFFFF
        n = len({v for _, _, v in header_values(mode_val, hdr, radioactive)})
        rows = n + 1 if n >= 4 else 0
        found.setdefault(rows, (hdr, radioactive))
    return found


def _inner(rng, mean, uniform):
    """6 x 6 pixels of one channel whose integer mean (sum / 36) is `mean`"""
    px = np.full(36, mean, np.int64)
    if not uniform:
        d = min(mean, 255 - mean, 9)
        px[0::2] += d
        px[1::2] -= d
        extra = min(35, 255 - (mean - d))
        px[1] += rng.integers(0, extra + 1)
    return px.reshape(6, 6)


def paint_fit_frame(mode_val, hdr, radioactive, targets, white16, rng, name=""):
    """noise, then every header cell init_ccm reads holds targets[expected colour] (some cells with non-uniform inner pixels,
    cell means spread by +-1 around the target with the per-colour integer average still the target, junk in the outer ring),
    then the three anchor patches: patch 0 per channel sums to white16 (white = white16 / 16, white16 >= 16), the others less"""
    m, xs, ys, idx, _, _ = _header_layout(mode_val)
    W, H = m.image_size_x, m.image_size_y
    frame = rng.integers(0, 256, (H, W, 3)).astype(np.uint8)
    cells = header_values(mode_val, hdr, radioactive)
    seen, order = {}, []
    for start, i, v in cells:
        if v not in seen:
            seen[v] = 0
            order.append(v)
    count = {v: 0 for v in seen}
    for _, _, v in cells:
        count[v] += 1
    for start, i, v in cells:
        j = seen[v]
        seen[v] += 1
        cell = int(idx[start + i])
        x, y = int(xs[cell]), int(ys[cell])
        t = np.asarray(targets[v], np.int64)
        spread = 0 if j == count[v] - 1 and count[v] % 2 else (1 if j % 2 == 0 else -1)     # the spreads of a colour sum to 0
        e = np.where((t >= 1) & (t <= 254), spread, 0)
        frame[y:y + 8, x:x + 8] = rng.integers(0, 256, (8, 8, 3))
        for c in range(3):
            frame[y + 1:y + 7, x + 1:x + 7, c] = _inner(rng, int(t[c] + e[c]), uniform=j % 3 == 0)
    tl, right, bottom = 28, W - 32, H - 32
    for k, (ax, ay) in enumerate(((tl, tl), (tl, bottom), (right, tl))):
        for c in range(3):
            s = int(white16[c]) if k == 0 else int(rng.integers(0, int(white16[c]) + 1))
            px = np.full(16, s // 16, np.int64)
            px[: s % 16] += 1
            frame[ay:ay + 4, ax:ax + 4, c] = rng.permutation(px).reshape(4, 4)
    if len(order) < 4:
        return Painted(mode_val, frame, hdr, radioactive, None, None, name)
    pal = palette(1 << m.color_bits, m.color_mode)
    rows = order[::-1]
    actual = np.array([targets[v] for v in rows] + [np.asarray(white16, np.float64) / 16], F32)
    desired = np.array([pal[v] for v in rows] + [(255, 255, 255)], F32)
    return Painted(mode_val, frame, hdr, radioactive, actual, desired, name)


COLOUR_MODES = [4, 8, 66, 67, 68]


def painted_frames(mode_val, seed=0):
    """for every row count the header search reaches: a camera-like tinted frame and a grey one (the rank-1 edge), plus a frame
    with one channel black and one saturated"""
    m = _header_layout(mode_val)[0]
    pal = palette(1 << m.color_bits, m.color_mode).astype(np.int64)
    rng = np.random.default_rng(seed + mode_val)
    out = []
    for rows, (hdr, radioactive) in sorted(search_headers(mode_val, seed).items()):
        gain, off = rng.uniform(0.45, 1.0, 3), rng.uniform(5, 40, 3)
        tint = {v: tuple(int(x) for x in np.clip(pal[v] * gain + off + rng.integers(-5, 6, 3), 0, 255)) for v in range(len(pal))}
        grey = {v: (g, g, g) for v, g in enumerate(rng.integers(10, 250, len(pal)).tolist())}
        flat = {v: (int(rng.integers(0, 256)), 0, 255) for v in range(len(pal))}
        w_tint = tuple(int(x) for x in np.clip((255 * gain + off) * 16, 16, 4080))
        g16 = int(rng.integers(16, 4081))
        for kind, targets, white16 in (("tint", tint, w_tint), ("grey", grey, (g16, g16, g16)), ("flat", flat, (4080, 16, 4080))):
            out.append(paint_fit_frame(mode_val, hdr, radioactive, targets, white16, rng, f"m{mode_val}-rows{rows}-{kind}"))
    return out
