"""PNG files for the device decoder's tests (test infrastructure only): the golden frames and a generated matrix.

The matrix has three parts:
  - cv2.imencode at compression 0-9 x every IMWRITE_PNG_STRATEGY on a crop of a cimbar frame and of a photograph, and 1-, 3- and
    4-channel pictures at 8 and 16 bit;
  - files written here with Python's zlib for what cv2 cannot write: palettes at 1/2/4/8 bit with and without tRNS, grey at 1/2/4
    bit, grey + alpha, all five filter types forced row by row, IDAT chunks of 1 byte, widths 1 and 7, a 61-row strip, the sizes
    60 and 4499, and gAMA / sRGB / iCCP / bKGD / eXIf chunks;
  - a fixed-Huffman stream written token by token, for matches of distance 1 and 32 768 and of length 258 (zlib never emits a
    distance above 32 506).
Every file is named; `premise()` lists the block types, filter types, colour types and bit depths the matrix covers."""
import glob
import os
import struct
import zlib

import cv2
import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SIG = b"\x89PNG\r\n\x1a\n"
CHANNELS = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}
STRATEGIES = {"default": cv2.IMWRITE_PNG_STRATEGY_DEFAULT, "filtered": cv2.IMWRITE_PNG_STRATEGY_FILTERED,
              "huffman": cv2.IMWRITE_PNG_STRATEGY_HUFFMAN_ONLY, "rle": cv2.IMWRITE_PNG_STRATEGY_RLE,
              "fixed": cv2.IMWRITE_PNG_STRATEGY_FIXED}


def golden_files():
    """[(name, bytes)] of every PNG frame under tests/golden/ (mycell.png, a 10 x 10 cell, is not a frame)"""
    return [(os.path.basename(f), open(f, "rb").read()) for f in sorted(glob.glob(os.path.join(GOLDEN, "*.png")))
            if not f.endswith("mycell.png")]


def chunk(kind, body):
    return struct.pack(">I", len(body)) + kind + body + struct.pack(">I", zlib.crc32(kind + body))


def ihdr(w, h, ct, bd, interlace=0):
    return chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, bd, ct, 0, 0, interlace))


def stride(w, ct, bd):
    return (w * CHANNELS[ct] * bd + 7) // 8


def paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
    return a if pa <= pb and pa <= pc else (b if pb <= pc else c)


def filter_rows(raw, ct, bd, filters):
    """raw: (h, stride) unfiltered bytes; filters: one type per row -> the filtered scanlines"""
    bpp = max(1, CHANNELS[ct] * bd // 8)
    raw = np.asarray(raw, np.uint8)
    out = bytearray()
    prev = bytes(raw.shape[1])
    for y in range(raw.shape[0]):
        cur, f = bytes(raw[y]), filters[y]
        row = bytearray(len(cur))
        for x in range(len(cur)):
            a = cur[x - bpp] if x >= bpp else 0
            b = prev[x]
            c = prev[x - bpp] if x >= bpp else 0
            pred = (0, a, b, (a + b) // 2, paeth(a, b, c))[f]
            row[x] = (cur[x] - pred) & 0xFF
        out += bytes([f]) + row
        prev = cur
    return bytes(out)


def pack_bits(vals, bd):
    """(h, w*channels) samples of bd bits -> (h, stride) bytes, big-endian, MSB first"""
    vals = np.asarray(vals)
    if bd == 16:
        return vals.astype(">u2").view(np.uint8).reshape(vals.shape[0], -1)
    if bd == 8:
        return vals.astype(np.uint8)
    per = 8 // bd
    h, n = vals.shape
    padded = np.zeros((h, (n + per - 1) // per * per), np.uint8)
    padded[:, :n] = vals
    out = np.zeros((h, padded.shape[1] // per), np.uint8)
    for k in range(per):
        out |= (padded[:, k::per] << (8 - bd * (k + 1))).astype(np.uint8)
    return out


def png(w, h, ct, bd, samples, filters=None, level=9, before=(), after_plte=(), palette=None, idat_size=None, zdata=None):
    """a PNG of samples (h, w * channels) at depth bd; filters: per-row types (default all None); before / after_plte: extra
    (kind, body) chunks after IHDR / after PLTE; idat_size: bytes per IDAT chunk (default one chunk); zdata: the zlib stream as is"""
    raw = pack_bits(samples, bd)
    assert raw.shape == (h, stride(w, ct, bd))
    if zdata is None:
        zdata = zlib.compress(filter_rows(raw, ct, bd, filters or [0] * h), level)
    out = SIG + ihdr(w, h, ct, bd)
    for k, b in before:
        out += chunk(k, b)
    if palette is not None:
        out += chunk(b"PLTE", bytes(np.asarray(palette, np.uint8).reshape(-1)))
    for k, b in after_plte:
        out += chunk(k, b)
    step = idat_size or max(1, len(zdata))
    for i in range(0, len(zdata), step):
        out += chunk(b"IDAT", zdata[i:i + step])
    return out + chunk(b"IEND", b"")


# ---- a fixed-Huffman deflate writer, token by token --------------------------------------------------------------------------

LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEN_EXTRA = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145,
             8193, 12289, 16385, 24577]
DIST_EXTRA = [0, 0, 0, 0] + [k // 2 for k in range(2, 28)]


class BitWriter:
    def __init__(self):
        self.out, self.acc, self.n = bytearray(), 0, 0

    def bits(self, v, n):                # n bits of v, LSB first
        self.acc |= v << self.n
        self.n += n
        while self.n >= 8:
            self.out.append(self.acc & 0xFF)
            self.acc >>= 8
            self.n -= 8

    def code(self, c, n):                # a Huffman code, MSB first
        self.bits(int(format(c, "0%db" % n)[::-1], 2), n)

    def done(self):
        if self.n:
            self.out.append(self.acc & 0xFF)
        return bytes(self.out)


def fixed_sym(bw, s):
    if s < 144:
        bw.code(0x30 + s, 8)
    elif s < 256:
        bw.code(0x190 + s - 144, 9)
    elif s < 280:
        bw.code(s - 256, 7)
    else:
        bw.code(0xC0 + s - 280, 8)


def fixed_stream(tokens, data):
    """a zlib stream of one final fixed-Huffman block: tokens are ints (literals) or (length, distance); data checks them"""
    bw = BitWriter()
    bw.bits(1, 1)
    bw.bits(1, 2)
    out = bytearray()
    for t in tokens:
        if isinstance(t, int):
            fixed_sym(bw, t)
            out.append(t)
            continue
        ln, d = t
        i = max(k for k in range(29) if LEN_BASE[k] <= ln)
        fixed_sym(bw, 257 + i)
        bw.bits(ln - LEN_BASE[i], LEN_EXTRA[i])
        j = max(k for k in range(30) if DIST_BASE[k] <= d)
        bw.code(j, 5)
        bw.bits(d - DIST_BASE[j], DIST_EXTRA[j])
        for _ in range(ln):
            out.append(out[-d])
    fixed_sym(bw, 256)
    assert bytes(out) == data
    return b"\x78\x01" + bw.done() + struct.pack(">I", zlib.adler32(data))


def long_matches():
    """grey 8-bit, 255 x 160: rows 128.. repeat rows 0.. (distance 32 768 = 128 rows of 256 bytes), matched by length-258 tokens,
    and a run of one value matched at distance 1"""
    rng = np.random.default_rng(11)
    w, h = 255, 160
    rows = rng.integers(0, 256, (h, w), dtype=np.uint8)
    rows[5, 10:200] = 77                                  # a run: one literal, then distance-1 matches
    rows[128:] = rows[:32]
    data = filter_rows(rows, 0, 8, [0] * h)
    tokens, i = [], 0
    while i < len(data):
        if i >= 32768 and len(data) - i >= 3:
            ln = min(258, len(data) - i)
            tokens.append((ln, 32768))
            i += ln
        elif 5 * 256 + 12 <= i < 5 * 256 + 201:
            ln = 5 * 256 + 201 - i
            tokens.append((ln, 1))
            i += ln
        else:
            tokens.append(data[i])
            i += 1
    return png(w, h, 0, 8, rows, zdata=fixed_stream(tokens, data))


# ---- the matrix ------------------------------------------------------------------------------------------------------------

def _frame():
    return cv2.imread(os.path.join(GOLDEN, "b__tr_1.png"), cv2.IMREAD_COLOR)


def _photo():
    return cv2.imread(os.path.join(GOLDEN, "6bit__4_30_802.jpg"), cv2.IMREAD_COLOR)


def encoded():
    """cv2.imencode: compression 0-9 x every strategy on a frame crop and a photograph crop; 1/3/4 channels at 8 and 16 bit"""
    out = []
    crops = {"frame": np.ascontiguousarray(_frame()[100:100 + 141, 200:200 + 173]),
             "photo": np.ascontiguousarray(_photo()[37:37 + 123, 51:51 + 157])}
    for cname, img in crops.items():
        for lvl in range(10):
            for sname, s in STRATEGIES.items():
                ok, buf = cv2.imencode(".png", img, [cv2.IMWRITE_PNG_COMPRESSION, lvl, cv2.IMWRITE_PNG_STRATEGY, s])
                assert ok
                out.append(("cv2_%s_c%d_%s" % (cname, lvl, sname), buf.tobytes()))
    rng = np.random.default_rng(3)
    base = crops["photo"][:64, :96]
    for ch in (1, 3, 4):
        img8 = cv2.cvtColor(base, cv2.COLOR_BGR2GRAY) if ch == 1 else (base if ch == 3 else cv2.cvtColor(base, cv2.COLOR_BGR2BGRA))
        if ch == 4:
            img8[..., 3] = rng.integers(0, 256, img8.shape[:2], dtype=np.uint8)
        img16 = np.clip(img8.astype(np.int32) * 256 + rng.integers(0, 65536, img8.shape), 0, 65535).astype(np.uint16)
        for bd, img in ((8, img8), (16, img16)):
            ok, buf = cv2.imencode(".png", img)
            assert ok
            out.append(("cv2_ch%d_%dbit" % (ch, bd), buf.tobytes()))
    return out


def crafted():
    """files written here: [(name, bytes)]"""
    rng = np.random.default_rng(7)
    out = []
    w, h = 75, 64
    for bd in (1, 2, 4, 8):
        n = 1 << bd
        pal = rng.integers(0, 256, (n, 3))
        idx = rng.integers(0, n, (h, w))
        for trns in (False, True):
            extra = [(b"tRNS", bytes(rng.integers(0, 256, n).astype(np.uint8)))] if trns else []
            out.append(("palette_%dbit%s" % (bd, "_trns" if trns else ""),
                        png(w, h, 3, bd, idx, palette=pal, after_plte=extra, filters=[y % 5 for y in range(h)])))
    for bd in (1, 2, 4):
        out.append(("grey_%dbit" % bd, png(w, h, 0, bd, rng.integers(0, 1 << bd, (h, w)), filters=[y % 5 for y in range(h)])))
    out.append(("grey_8bit_trns", png(w, h, 0, 8, rng.integers(0, 256, (h, w)), before=[(b"tRNS", b"\x00\x10")])))
    out.append(("rgb_8bit_trns", png(w, h, 2, 8, rng.integers(0, 256, (h, 3 * w)), before=[(b"tRNS", b"\x00\x10\x00\x20\x00\x30")])))
    for bd in (8, 16):
        out.append(("grey_alpha_%dbit" % bd, png(w, h, 4, bd, rng.integers(0, 1 << bd, (h, 2 * w)), filters=[y % 5 for y in range(h)])))
    photo = cv2.cvtColor(_photo()[:h, :w], cv2.COLOR_BGR2RGB)
    for f in range(5):
        out.append(("rgb_filter%d" % f, png(w, h, 2, 8, photo.reshape(h, -1), filters=[f] * h)))
    out.append(("rgb_filters_mixed", png(w, h, 2, 8, photo.reshape(h, -1), filters=[(y * 3) % 5 for y in range(h)])))
    rgba16 = rng.integers(0, 65536, (h, 4 * w))
    out.append(("rgba_16bit_filters", png(w, h, 6, 16, rgba16, filters=[y % 5 for y in range(h)])))
    out.append(("rgb_16bit_filters", png(w, h, 2, 16, rgba16[:, :3 * w], filters=[(y + 2) % 5 for y in range(h)])))
    out.append(("grey_16bit_filters", png(w, h, 0, 16, rgba16[:, :w], filters=[(y + 1) % 5 for y in range(h)])))
    out.append(("idat_1byte", png(w, h, 2, 8, photo.reshape(h, -1), filters=[y % 5 for y in range(h)], idat_size=1)))
    out.append(("idat_7bytes_stored", png(w, h, 2, 8, photo.reshape(h, -1), level=0, idat_size=7)))
    out.append(("long_matches", long_matches()))
    for wd in (1, 7):
        out.append(("width_%d" % wd, png(wd, 90, 2, 8, rng.integers(0, 256, (90, 3 * wd)), filters=[y % 5 for y in range(90)])))
    strip = cv2.cvtColor(_frame()[:61, :997], cv2.COLOR_BGR2RGB)
    out.append(("strip_997x61", png(997, 61, 2, 8, strip.reshape(61, -1), filters=[y % 5 for y in range(61)], level=6)))
    out.append(("size_60x60", png(60, 60, 2, 8, rng.integers(0, 256, (60, 180)), filters=[y % 5 for y in range(60)])))
    wide = np.tile(np.arange(4499, dtype=np.int64) % 251, (60, 1))
    out.append(("size_4499x60", png(4499, 60, 0, 8, wide, filters=[y % 5 for y in range(60)])))
    out.append(("size_60x4499", png(60, 4499, 0, 8, wide.T % 256, filters=[y % 5 for y in range(4499)])))
    img = photo.reshape(h, -1)
    icc = zlib.compress(b"\x00" * 128)
    out.append(("gama_srgb_iccp_bkgd", png(w, h, 2, 8, img, before=[(b"gAMA", struct.pack(">I", 100000)), (b"sRGB", b"\x00"),
                                                                   (b"iCCP", b"icc\x00\x00" + icc), (b"bKGD", b"\x00\xff\x00\x00\x00\xff")])))
    out.append(("gama_low", png(w, h, 2, 8, img, before=[(b"gAMA", struct.pack(">I", 20000))])))
    out.append(("grey_alpha_bkgd", png(w, h, 4, 8, rng.integers(0, 256, (h, 2 * w)), before=[(b"bKGD", b"\x00\x80")])))
    for k in (1, 3, 6, 8):
        out.append(("exif_orientation_%d" % k, png(w, h, 2, 8, img, before=[(b"eXIf", exif(k))])))
    return out


def exif(orientation):
    """a big-endian TIFF header with one IFD entry: Orientation"""
    return b"MM\x00\x2a" + struct.pack(">I", 8) + struct.pack(">H", 1) + struct.pack(">HHIHH", 0x0112, 3, 1, orientation, 0) + b"\x00" * 4


def matrix():
    """[(name, bytes)]: cv2-written and crafted files"""
    return encoded() + crafted()


def cv2_rgb(data):
    """what cv2.imread(IMREAD_COLOR) + cvtColor(BGR2RGB) gives for these file bytes, or None"""
    if not data:
        return None
    try:
        img = cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_COLOR)
    except cv2.error:                     # OpenCV's own size checks raise instead of returning None
        return None
    return None if img is None else np.ascontiguousarray(cv2.cvtColor(img, cv2.COLOR_BGR2RGB))


def walk(data):
    """[(kind, body)] of a well-formed file's chunks"""
    out, i = [], 8
    while i + 8 <= len(data):
        n = struct.unpack(">I", data[i:i + 4])[0]
        out.append((data[i + 4:i + 8], data[i + 8:i + 8 + n]))
        i += 12 + n
    return out


def premise(files):
    """what the files cover: {'blocks': deflate block types, 'filters': filter types, 'colour': (colour type, depth) pairs}"""
    blocks, filters, colour = set(), set(), set()
    for _, data in files:
        ch = walk(data)
        w, h, bd, ct, _, _, _ = struct.unpack(">IIBBBBB", ch[0][1])
        colour.add((ct, bd))
        z = b"".join(b for k, b in ch if k == b"IDAT")
        blocks |= block_types(z)
        raw = zlib.decompress(z)
        st = stride(w, ct, bd)
        filters |= {raw[y * (st + 1)] for y in range(h)}
    return {"blocks": blocks, "filters": filters, "colour": colour}


def block_types(z):
    """the deflate block types of a zlib stream (a small inflater that only walks the block structure)"""
    pos = [16]                            # bit position, past the zlib header

    def bits(n):
        v = 0
        for k in range(n):
            v |= ((z[pos[0] >> 3] >> (pos[0] & 7)) & 1) << k
            pos[0] += 1
        return v

    def table(lengths):
        codes, bl = {}, {}
        for ln in lengths:
            if ln:
                bl[ln] = bl.get(ln, 0) + 1
        nxt, code = {}, 0
        for b in range(1, 16):
            code = (code + bl.get(b - 1, 0)) << 1
            nxt[b] = code
        for s, ln in enumerate(lengths):
            if ln:
                codes[(ln, nxt[ln])] = s
                nxt[ln] += 1
        return codes

    def sym(t):
        code, ln = 0, 0
        while True:
            code = (code << 1) | bits(1)
            ln += 1
            if (ln, code) in t:
                return t[(ln, code)]

    fixed_l = table([8] * 144 + [9] * 112 + [7] * 24 + [8] * 8)
    fixed_d = table([5] * 30)
    seen = set()
    while True:
        final, kind = bits(1), bits(2)
        seen.add(kind)
        if kind == 0:
            pos[0] = (pos[0] + 7) & ~7
            n = z[pos[0] >> 3] | z[(pos[0] >> 3) + 1] << 8
            pos[0] += 32 + 8 * n
        else:
            if kind == 1:
                lt, dt = fixed_l, fixed_d
            else:
                hl, hd, hc = bits(5) + 257, bits(5) + 1, bits(4) + 4
                order = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
                cl = [0] * 19
                for k in range(hc):
                    cl[order[k]] = bits(3)
                ct = table(cl)
                lens = []
                while len(lens) < hl + hd:
                    s = sym(ct)
                    if s < 16:
                        lens.append(s)
                    elif s == 16:
                        lens += [lens[-1]] * (3 + bits(2))
                    elif s == 17:
                        lens += [0] * (3 + bits(3))
                    else:
                        lens += [0] * (11 + bits(7))
                lt, dt = table(lens[:hl]), table(lens[hl:])
            while True:
                s = sym(lt)
                if s == 256:
                    break
                if s > 256:
                    bits(LEN_EXTRA[s - 257])
                    bits(DIST_EXTRA[sym(dt)])
        if final:
            return seen


def with_matches(w, h, cinfo, matches, seed=0, idat_size=None):
    """grey 8-bit w x h of random rows (filter None) in one fixed-Huffman block, with the given (position, distance, length)
    matches in the filtered stream, and the zlib header's window set to 2^(8 + cinfo) -- for zlib's window rule as libpng drives it"""
    rng = np.random.default_rng(seed)
    rowlen = w + 1
    data = bytearray(rng.integers(0, 256, h * rowlen, dtype=np.uint8).tobytes())
    for r in range(h):
        data[r * rowlen] = 0
    for p, d, ln in matches:
        for k in range(ln):
            data[p + k] = data[p - d + k]
    assert all(data[r * rowlen] == 0 for r in range(h)), "a match changes a filter byte"
    tokens, i, at = [], 0, {p: (ln, d) for p, d, ln in matches}
    while i < len(data):
        if i in at:
            tokens.append(at[i])
            i += at[i][0]
        else:
            tokens.append(data[i])
            i += 1
    z = fixed_stream(tokens, bytes(data))
    cmf = cinfo << 4 | 8
    z = bytes([cmf, (31 - (cmf << 8) % 31) % 31]) + z[2:]
    rows = np.frombuffer(bytes(data), np.uint8).reshape(h, rowlen)[:, 1:]
    return png(w, h, 0, 8, rows, zdata=z, idat_size=idat_size)
