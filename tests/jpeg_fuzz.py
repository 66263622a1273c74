"""A generated JPEG corpus for the device decoder's tests (test infrastructure only), deterministic from fixed seeds and written
only with cv2, PIL and numpy.

What depends on a file's size and content is the risky part of the decoder: the self-synchronising Huffman decode (512
subsequences per restart segment, sync rounds, prefix sums of blocks and DC predictions), EOB runs taken whole, the AC refinement
pass, the extents of non-interleaved scans, and upsampling at the picture edges.  So the corpus varies:
  - sizes: 1-17 on each side (every MCU edge of every sampling) and 60-76 (the same edges at sizes the device calls accept),
    31-33 / 63-65 / 127-129, 60 and 61, odd sizes around 1000, and 3000 x 2000 / 4000 x 3000 pictures;
  - contents: uniform noise (long codes, AC categories up to 10), 8 x 8 black and white blocks (DC category 11 at quality 100),
    flat colour, smooth gradients, black and white crops of a golden cimbar frame, crops and resizes of a golden photograph,
    near-saturated colours (clamping in YCbCr -> RGB), and flat pictures with sparse dots (long EOB runs between short codes);
  - cv2 settings: quality 1 / 10 / 50 / 90 / 100, luma and chroma quality apart, progressive, optimised tables, sampling
    4:4:4 / 4:2:2 / 4:4:0 / 4:2:0 and grey, restart interval 0 / 1 / 2 / 7 / 4096 MCUs (every combination of sampling,
    progressive and restart interval at least once);
  - PIL files (a second libjpeg front end): its subsampling, progressive, optimize and custom qtables, and EXIF orientations 5-8
    (transposes) on pictures with odd, unequal sides.
Every file is named after how it was made.  `walk()` is a marker walk that gives a file's frame, restart interval and entropy-coded
segments; `mutations()` damages corpus files (bit flips, truncation, a lost stuffing byte, two restart segments swapped)."""
import io

import cv2
import numpy as np

from jpeg_matrix import GOLDEN, SAMPLING

RST_LARGE = 4096
RESTARTS = (0, 1, 2, 7, RST_LARGE)
QUALITIES = (1, 10, 50, 90, 100)
KINDS = ("noise", "blocks", "flat", "gradient", "binary", "photo", "saturated", "sparse")
SEED = 20261017


class _Sources:
    def __init__(self):
        self.photo = cv2.imread(GOLDEN + "/6bit__4_30_802.jpg", cv2.IMREAD_COLOR)
        frame = cv2.imread(GOLDEN + "/b__tr_0.png", cv2.IMREAD_GRAYSCALE)
        self.frame = np.where(frame >= 128, 255, 0).astype(np.uint8)


def _crop_or_resize(src, h, w, rng, interp):
    H, W = src.shape[:2]
    if h <= H and w <= W:
        y, x = int(rng.integers(0, H - h + 1)), int(rng.integers(0, W - w + 1))
        return np.ascontiguousarray(src[y:y + h, x:x + w])
    return cv2.resize(src, (w, h), interpolation=interp)


def content(kind, h, w, rng, src):
    """an h x w BGR picture of one kind"""
    if kind == "noise":
        return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    if kind == "blocks":
        cells = rng.integers(0, 2, ((h + 7) // 8, (w + 7) // 8), dtype=np.uint8) * 255
        return np.repeat(np.repeat(cells, 8, 0), 8, 1)[:h, :w, None].repeat(3, 2)
    if kind == "flat":
        return np.full((h, w, 3), rng.integers(0, 256, 3), np.uint8)
    if kind == "gradient":
        y, x = np.mgrid[0:h, 0:w].astype(np.float64)
        fx, fy = x / max(w - 1, 1), y / max(h - 1, 1)
        return np.stack([255 * fx, 255 * fy, 127.5 * (fx + 1 - fy)], -1).round().astype(np.uint8)
    if kind == "binary":
        return _crop_or_resize(src.frame, h, w, rng, cv2.INTER_NEAREST)[:, :, None].repeat(3, 2)
    if kind == "photo":
        return _crop_or_resize(src.photo, h, w, rng, cv2.INTER_AREA if h * w < src.photo.shape[0] * src.photo.shape[1] else cv2.INTER_CUBIC)
    if kind == "saturated":                                   # pure and near-pure colours in 4 x 4 patches
        palette = np.array([[0, 0, 255], [0, 255, 0], [255, 0, 0], [255, 255, 0], [255, 0, 255], [0, 255, 255], [0, 0, 0],
                            [255, 255, 255]], np.int16)
        idx = rng.integers(0, len(palette), ((h + 3) // 4, (w + 3) // 4))
        img = np.repeat(np.repeat(palette[idx], 4, 0), 4, 1)[:h, :w]
        jitter = rng.integers(0, 4, (h, w, 3))
        return np.where(img > 127, img - jitter, img + jitter).astype(np.uint8)
    if kind == "sparse":                                      # flat, with one dot per ~400 pixels
        img = np.full((h, w, 3), rng.integers(0, 256, 3), np.uint8)
        n = max(1, h * w // 400)
        img[rng.integers(0, h, n), rng.integers(0, w, n)] = rng.integers(0, 256, (n, 3), dtype=np.uint8)
        return img
    raise ValueError(kind)


def cv2_file(img, q=90, prog=0, opt=0, samp="420", rst=0, luma=None, chroma=None):
    """cv2.imencode's JPEG file of a BGR picture (grey: samp 'grey', the picture converted first)"""
    params = [cv2.IMWRITE_JPEG_QUALITY, q, cv2.IMWRITE_JPEG_PROGRESSIVE, prog, cv2.IMWRITE_JPEG_OPTIMIZE, opt,
              cv2.IMWRITE_JPEG_RST_INTERVAL, rst]
    if samp == "grey":
        img = cv2.cvtColor(img, cv2.COLOR_BGR2GRAY)
    else:
        params += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, SAMPLING[samp]]
    if luma is not None:
        params += [cv2.IMWRITE_JPEG_LUMA_QUALITY, luma, cv2.IMWRITE_JPEG_CHROMA_QUALITY, chroma]
    ok, buf = cv2.imencode(".jpg", img, params)
    assert ok
    return buf.tobytes()


def cv2_name(kind, h, w, q=90, prog=0, opt=0, samp="420", rst=0, luma=None, chroma=None):
    qs = "q%d" % q if luma is None else "luma%d_chroma%d" % (luma, chroma)
    return "cv2_%s_%s_%dx%d_%s_%s_opt%d_rst%d" % ("prog" if prog else "base", samp, w, h, kind, qs, opt, rst)


def pil_file(img, orientation=None, **kw):
    from PIL import Image
    pic = Image.fromarray(cv2.cvtColor(img, cv2.COLOR_BGR2RGB))
    b = io.BytesIO()
    if orientation is not None:
        exif = Image.Exif()
        exif[0x0112] = orientation
        kw["exif"] = exif.tobytes()
    pic.save(b, "JPEG", **kw)
    return b.getvalue()


# custom quantisation tables (natural order) for PIL: all ones, a steep ramp, and random entries
def _qtables(rng):
    ramp = [min(255, 1 + 4 * (r + c)) for r in range(8) for c in range(8)]
    return {"ones": [[1] * 64, [1] * 64], "ramp": [ramp, ramp[::-1]],
            "random": [rng.integers(1, 256, 64).tolist(), rng.integers(1, 256, 64).tolist()]}


def corpus():
    """[(name, bytes)] of the whole corpus, deterministic"""
    rng = np.random.default_rng(SEED)
    src = _Sources()
    out = []
    samplings = list(SAMPLING)

    def add(kind, h, w, **kw):
        out.append((cv2_name(kind, h, w, **kw), cv2_file(content(kind, h, w, rng, src), **kw)))

    def pick(seq, i):
        return seq[i % len(seq)]

    def size(rst):                                            # intervals of 1 or 2 MCUs on smaller pictures: fewer segments
        hi = 100 if rst in (1, 2) else 200
        return int(rng.integers(60, hi)), int(rng.integers(60, hi))

    # 1-17 and 60-76 on each side: every width with every sampling, heights a permutation of the same range; settings rotate,
    # except that pictures up to 4 pixels wide are noise at quality 50 and up (chroma that differs between neighbours, where the
    # choice of upsampler shows)
    for base in (0, 59):
        for si, samp in enumerate(samplings + ["grey"]):
            for i in range(17):
                w, h = base + 1 + i, base + 1 + (5 * i + 3 * si) % 17
                k = i + 3 * si
                kind, q = (pick(KINDS, k), pick(QUALITIES, k)) if w > 4 else ("noise", pick(QUALITIES[2:], k))
                add(kind, h, w, q=q, prog=k & 1, opt=(k >> 1) & 1, samp=samp, rst=pick(RESTARTS, k))
    # 31-33, 63-65, 127-129 and 60 / 61
    around = (31, 32, 33, 63, 64, 65, 127, 128, 129)
    for si, samp in enumerate(samplings):
        for i, w in enumerate(around):
            k = i + 2 * si
            add(pick(KINDS, k + 1), pick(around, 4 * i + si), w, q=pick(QUALITIES, k + 2), prog=(k >> 1) & 1, opt=k & 1, samp=samp,
                rst=pick(RESTARTS, k + 1))
    for i, (w, h) in enumerate([(60, 60), (61, 60), (60, 61), (61, 61)]):
        add(pick(KINDS, 5 + i), h, w, q=90, prog=i & 1, samp=pick(samplings, i), rst=pick(RESTARTS, i))
    # every sampling x progressive x restart interval
    for samp in samplings + ["grey"]:
        for prog in (0, 1):
            for ri, rst in enumerate(RESTARTS):
                h, w = size(rst)
                add(pick(KINDS, ri + prog), h, w, q=pick(QUALITIES, ri + 2 * prog + 1), prog=prog, opt=ri & 1, samp=samp, rst=rst)
    # every quality on every kind, and luma / chroma quality apart
    for ki, kind in enumerate(KINDS):
        for qi, q in enumerate(QUALITIES):
            rst = pick(RESTARTS, ki + 2 * qi)
            h, w = size(rst)
            add(kind, h, w, q=q, prog=(ki + qi) & 1, opt=qi & 1, samp=pick(samplings, ki + qi), rst=rst)
    for i, (luma, chroma) in enumerate([(90, 10), (10, 90), (100, 1), (1, 100)]):
        add(pick(("photo", "saturated", "noise", "gradient"), i), 97 + i, 131, q=75, luma=luma, chroma=chroma, prog=i & 1,
            samp=pick(samplings, i + 1), rst=pick(RESTARTS, i))
    # segments of a few bytes (flat, one MCU per interval) and single-segment files over 64 KB
    for samp in samplings:
        add("flat", 64, 96, q=50, samp=samp, rst=1)
        add("noise", 333, 301, q=90, samp=samp, rst=0)
    # odd sizes around 1000
    for i, (w, h) in enumerate([(999, 1001), (1003, 997), (1001, 1001), (997, 999)]):
        add(pick(("photo", "noise", "binary", "gradient"), i), h, w, q=pick((90, 100, 75, 50), i), prog=i & 1, opt=1,
            samp=pick(samplings, i + 3), rst=pick((0, RST_LARGE, 64, 0), i))
    # large pictures: segments of tens of KB, one whole-file segment of megabytes, long EOB runs in progressive AC scans
    add("photo", 2000, 3000, q=90, samp="420", rst=RST_LARGE)
    add("photo", 2000, 3000, q=95, prog=1, samp="444", rst=RST_LARGE)
    add("photo", 3000, 4000, q=90, samp="422", rst=0)
    add("flat", 2000, 3000, q=75, prog=1, samp="420", rst=0)
    add("sparse", 3000, 4000, q=50, prog=1, opt=1, samp="420", rst=0)
    # PIL: subsampling x progressive x optimize, custom tables, EXIF orientations 5-8 on odd unequal sides
    for sub in (0, 1, 2):
        for prog in (False, True):
            for opt in (False, True):
                kind = pick(("photo", "saturated", "noise", "gradient"), sub + 2 * prog)
                h, w = int(rng.integers(20, 150)), int(rng.integers(20, 150))
                out.append(("pil_sub%d_prog%d_opt%d_%dx%d_%s_q85" % (sub, prog, opt, w, h, kind),
                            pil_file(content(kind, h, w, rng, src), quality=85, subsampling=sub, progressive=prog, optimize=opt)))
    for ti, (tname, tables) in enumerate(_qtables(rng).items()):
        for sub in (0, 2):
            h, w = 71 + ti, 89 + 2 * ti
            out.append(("pil_sub%d_%dx%d_photo_qtables_%s" % (sub, w, h, tname),
                        pil_file(content("photo", h, w, rng, src), subsampling=sub, qtables=tables, progressive=sub == 2)))
    for o in (5, 6, 7, 8):
        for (w, h), sub in (((67, 61), 2), ((13, 7), 1)):
            out.append(("pil_exif%d_sub%d_%dx%d_photo" % (o, sub, w, h),
                        pil_file(content("photo", h, w, rng, src), orientation=o, quality=90, subsampling=sub)))
    return out


def walk(data):
    """the marker walk of one file (SOI ... SOS, RSTn, EOI): {'size': (w, h) of the frame, 'sampling': '444' / '422' / '440' / '420' / 'grey', 'progressive',
    'restart' (the last DRI's interval), 'segments': [(begin, end)] byte ranges of every scan's entropy-coded data split at RSTn,
    FF 00 stuffing included, 'scans': [[segment indices]] per scan}"""
    assert data[:2] == b"\xff\xd8"
    info = {"size": None, "sampling": None, "progressive": False, "restart": 0, "segments": [], "scans": []}
    pos = 2
    while True:
        assert data[pos] == 0xFF, pos
        while data[pos] == 0xFF:
            pos += 1
        m = data[pos]
        pos += 1
        if m == 0xD9:
            return info
        n = int.from_bytes(data[pos:pos + 2], "big")
        body = data[pos + 2:pos + n]
        pos += n
        if m in (0xC0, 0xC1, 0xC2):
            info["progressive"] = m == 0xC2
            info["size"] = (int.from_bytes(body[3:5], "big"), int.from_bytes(body[1:3], "big"))
            hv = (body[7] >> 4, body[7] & 15)
            info["sampling"] = "grey" if body[5] == 1 else {(1, 1): "444", (2, 1): "422", (1, 2): "440", (2, 2): "420"}[hv]
        elif m == 0xDD:
            info["restart"] = int.from_bytes(body[:2], "big")
        elif m == 0xDA:
            scan, begin = [], pos
            while True:
                i = data.index(b"\xff", pos)
                if data[i + 1] == 0x00:
                    pos = i + 2
                    continue
                scan.append(len(info["segments"]))
                info["segments"].append((begin, i))
                if 0xD0 <= data[i + 1] <= 0xD7:
                    pos = begin = i + 2
                    continue
                pos = i
                break
            info["scans"].append(scan)


def segment_lengths(data):
    return [e - b for b, e in walk(data)["segments"]]


def restart_class(interval):
    """the corpus's restart interval buckets: 0, 1, 2, 7 and 'large'"""
    return interval if interval in (0, 1, 2, 7) else "large"


def _mutate(name, data, how, rng):
    info = walk(data)
    segs = info["segments"]
    if how == "flip":
        b, e = segs[int(rng.choice([k for k, (b, e) in enumerate(segs) if e > b]))]
        i = int(rng.integers(b, e))
        bit = int(rng.integers(0, 8))
        return "%s~flip%d.%d" % (name, i, bit), data[:i] + bytes([data[i] ^ (1 << bit)]) + data[i + 1:]
    if how == "truncate":
        i = int(rng.integers(segs[0][0], len(data)))
        return "%s~truncate%d" % (name, i), data[:i]
    if how == "unstuff":
        stuffed = [b + k + 1 for b, e in segs for k in range(e - b - 1) if data[b + k] == 0xFF and data[b + k + 1] == 0x00]
        i = stuffed[int(rng.integers(0, len(stuffed)))]
        return "%s~unstuff%d" % (name, i), data[:i] + data[i + 1:]
    if how == "swap":
        scan = [s for s in info["scans"] if len(s) >= 2][0]
        a, b = sorted(rng.choice(scan, 2, replace=False).tolist())
        (a0, a1), (b0, b1) = segs[a], segs[b]
        return "%s~swap%d.%d" % (name, a, b), data[:a0] + data[b0:b1] + data[a1:b0] + data[a0:a1] + data[b1:]
    raise ValueError(how)


def mutations(files, n=200, max_bytes=200_000, max_segments=100, seed=SEED + 1):
    """n damaged copies of corpus files, a quarter each of: one bit flipped in an entropy-coded segment, the file truncated after
    its first SOS, one FF 00 stuffing byte removed, two restart segments of one scan swapped.  The files damaged are those of at
    most max_bytes and max_segments (quick under the sanitizers) that the device calls accept (short side 60 or more).
    [(name, bytes)]"""
    rng = np.random.default_rng(seed)
    small = [(nm, d) for nm, d in files
             if len(d) <= max_bytes and len(walk(d)["segments"]) <= max_segments and min(walk(d)["size"]) >= 60]
    can = {"flip": small, "truncate": small,
           "unstuff": [(nm, d) for nm, d in small if any(d[b:e].count(b"\xff\x00") for b, e in walk(d)["segments"])],
           "swap": [(nm, d) for nm, d in small if any(len(s) >= 2 for s in walk(d)["scans"])]}
    out = []
    for k in range(n):
        how = ("flip", "truncate", "unstuff", "swap")[k % 4]
        name, data = can[how][int(rng.integers(0, len(can[how])))]
        out.append(_mutate(name, data, how, rng))
    return out


def orphaned_ff(files, max_bytes=50_000):
    """every byte value after an orphaned FF: for one file of each sampling x progressive (of at most max_bytes, at sizes the device
    calls accept), the first FF 00 stuffing pair of its first scan and the last one of its last scan get each of the 256 values in
    place of their 00 (00 itself gives the file back).  [(name, bytes)]"""
    out, seen = [], set()
    for name, data in files:
        info = walk(data)
        key = (info["sampling"], info["progressive"])
        if key in seen or len(data) > max_bytes or min(info["size"]) < 60:
            continue
        pairs = [[i for b, e in (info["segments"][k] for k in scan) for i in range(b, e - 1) if data[i:i + 2] == b"\xff\x00"]
                 for scan in (info["scans"][0], info["scans"][-1])]
        if not pairs[0] or not pairs[1] or pairs[0][0] == pairs[1][-1]:
            continue
        sites = [pairs[0][0] + 1, pairs[1][-1] + 1]
        seen.add(key)
        for i in sites:
            out += [("%s~ff%d=%02x" % (name, i, v), data[:i] + bytes([v]) + data[i + 1:]) for v in range(256)]
    return out
