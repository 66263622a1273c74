"""JPEG files for the device decoder's tests (test infrastructure only): the golden photographs and a generated matrix.

The matrix is written by cv2.imencode from a crop of a golden photograph whose sizes are not multiples of any MCU: baseline and
progressive x 4:4:4 / 4:2:2 / 4:4:0 / 4:2:0 x quality 50 and 95 x optimised Huffman tables on and off x restart interval 0 and 1 MCU
row; then grey files, a crop of 61 rows, and PIL-written 4:2:0 files carrying each EXIF orientation 1-8."""
import glob
import io
import os

import cv2
import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SAMPLING = {"444": 0x111111, "422": 0x211111, "440": 0x121111, "420": 0x221111}


def golden_files():
    """[(name, bytes)] of every JPEG under tests/golden/"""
    return [(os.path.basename(f), open(f, "rb").read()) for f in sorted(glob.glob(os.path.join(GOLDEN, "*.jpg")))]


def photo_files(prefix):
    """the golden camera photographs of one mode ('6bit' or 'b'), in glob order"""
    return [(n, d) for n, d in golden_files() if n.startswith(prefix + "__")]


def _base():
    return cv2.imread(os.path.join(GOLDEN, "6bit__4_30_802.jpg"), cv2.IMREAD_COLOR)


def matrix():
    """[(name, bytes)]"""
    base = _base()
    crop = np.ascontiguousarray(base[37:37 + 301, 51:51 + 403])
    out = []
    for prog in (0, 1):
        for sname, samp in SAMPLING.items():
            for q in (50, 95):
                for opt in (0, 1):
                    for rst in (0, 1):
                        ok, buf = cv2.imencode(".jpg", crop, [cv2.IMWRITE_JPEG_QUALITY, q, cv2.IMWRITE_JPEG_PROGRESSIVE, prog,
                                                              cv2.IMWRITE_JPEG_OPTIMIZE, opt, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, samp,
                                                              cv2.IMWRITE_JPEG_RST_INTERVAL, rst])
                        assert ok
                        out.append(("%s_%s_q%d_opt%d_rst%d" % ("prog" if prog else "base", sname, q, opt, rst), buf.tobytes()))
    grey = cv2.cvtColor(crop, cv2.COLOR_BGR2GRAY)
    for prog in (0, 1):
        ok, buf = cv2.imencode(".jpg", grey, [cv2.IMWRITE_JPEG_QUALITY, 90, cv2.IMWRITE_JPEG_PROGRESSIVE, prog])
        out.append(("grey_prog%d" % prog, buf.tobytes()))
    ok, buf = cv2.imencode(".jpg", np.ascontiguousarray(base[:61, :997]), [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, SAMPLING["420"]])
    out.append(("strip_61x997_420", buf.tobytes()))
    from PIL import Image
    pil = Image.fromarray(cv2.cvtColor(np.ascontiguousarray(base[100:100 + 173, 200:200 + 259]), cv2.COLOR_BGR2RGB))
    for k in range(1, 9):
        exif = Image.Exif()
        exif[0x0112] = k
        b = io.BytesIO()
        pil.save(b, "JPEG", quality=90, exif=exif.tobytes())
        out.append(("exif_orientation_%d" % k, b.getvalue()))
    return out


def cv2_rgb(data):
    """what cv2.imread + cvtColor(BGR2RGB) gives for these file bytes"""
    img = cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_COLOR)
    return np.ascontiguousarray(cv2.cvtColor(img, cv2.COLOR_BGR2RGB))
