"""CPU-side checks of the JPEG entry points (cb200_jpeg_info, cb200_jpeg_decode_dev, cb200_jpeg_scan_extract_decode_chunks_dev): a
file outside the supported set, a bad size or a null pointer is refused with CB200_ERR_ARG before any CUDA call, and the message
names the picture.  The context is NULL here, so a call whose files are all good fails on the context instead."""
import ctypes as C
import io

import cv2
import numpy as np
import pytest

import libcimbar_b200 as cb
from libcimbar_b200 import build as cbbuild
from cpu_support import PHOTO


@pytest.fixture(scope="module", autouse=True)
def built():
    cbbuild.build()


def lib():
    return cb.load_library()


def encode(img, **kw):
    params = []
    for k, v in kw.items():
        params += [getattr(cv2, "IMWRITE_JPEG_" + k.upper()), v]
    ok, buf = cv2.imencode(".jpg", img, params)
    assert ok
    return buf.tobytes()


IMG = np.random.default_rng(5).integers(0, 256, (120, 160, 3), dtype=np.uint8)


def cmyk():
    from PIL import Image
    b = io.BytesIO()
    Image.fromarray(IMG).convert("CMYK").save(b, "JPEG")
    return b.getvalue()


def sof_patched(data, marker):
    """the file with its frame marker replaced (arithmetic, lossless, ...)"""
    i = data.index(b"\xff\xc0")
    return data[:i + 1] + bytes([marker]) + data[i + 2:]


def twelve_bit(data):
    i = data.index(b"\xff\xc0")
    return data[:i + 4] + b"\x0c" + data[i + 5:]


def adobe(data, transform):
    seg = b"Adobe" + b"\x00\x64\x00\x00\x00\x00" + bytes([transform])
    app14 = b"\xff\xee" + (len(seg) + 2).to_bytes(2, "big") + seg
    j = data.index(b"\xff\xe0")
    n = int.from_bytes(data[j + 2:j + 4], "big")
    return data[:2] + app14 + data[j + 2 + n:]          # the JFIF APP0 out, an Adobe APP14 in


BASE = encode(IMG, quality=90)
REFUSED = [
    ("4:1:1", encode(IMG, sampling_factor=0x411111), "4:4:4, 4:2:2, 4:4:0 and 4:2:0"),
    ("cmyk", None, "CMYK"),
    ("arithmetic", sof_patched(BASE, 0xC9), "arithmetic"),
    ("lossless", sof_patched(BASE, 0xC3), "lossless"),
    ("12-bit", twelve_bit(BASE), "12-bit"),
    ("adobe transform 0", adobe(BASE, 0), "Adobe"),
    ("adobe transform 2", adobe(BASE, 2), "Adobe"),
    ("truncated header", BASE[:40], "truncated"),
    ("not a JPEG", b"\x89PNG\r\n\x1a\n" + bytes(100), "not a JPEG"),
    ("empty", b"", "not a JPEG"),
    ("too small", encode(np.zeros((59, 400, 3), np.uint8)), "smaller than 60"),
    ("too large", encode(np.zeros((4500, 4600, 3), np.uint8), quality=10), "4500"),
]


def calls(files, sizes=None, n=None, flags=0):
    """each JPEG entry point with these files (NULL context); yields (name, rc)"""
    L = lib()
    n = len(files) if n is None else n
    ptrs = None if files is None else (C.c_char_p * max(len(files), 1))(*files)
    if sizes is None and files is not None:
        sizes = (C.c_uint64 * max(len(files), 1))(*[len(f) if f is not None else 0 for f in files])
    buf = np.zeros(64, np.uint8)
    yield "decode_dev", L.cb200_jpeg_decode_dev(None, ptrs, sizes, n, buf.ctypes.data, buf.ctypes.data)
    yield "camera_dev", L.cb200_jpeg_scan_extract_decode_chunks_dev(None, ptrs, sizes, n, flags, buf.ctypes.data, buf.ctypes.data,
                                                                    None, buf.ctypes.data)


def last_error():
    return lib().cb200_last_error().decode()


@pytest.mark.parametrize("what,data,reason", REFUSED, ids=[r[0] for r in REFUSED])
def test_refused_files_name_the_picture(what, data, reason):
    data = cmyk() if data is None else data
    for name, rc in calls([PHOTO, data, PHOTO]):
        assert rc == -1, name
        msg = last_error()
        assert "picture 1" in msg and reason in msg, (name, msg)
    w, h = C.c_int32(), C.c_int32()
    assert lib().cb200_jpeg_info(data, len(data), C.byref(w), C.byref(h)) == -1
    assert reason in last_error()
    with pytest.raises(cb.Cb200Error, match=reason):
        cb.jpeg_info(data)


def test_good_files_fail_only_on_the_context():
    for name, rc in calls([PHOTO, BASE]):
        assert rc == -1 and "null context" in last_error(), name


def test_null_pointers():
    for name, rc in calls(None, n=1):
        assert rc == -1 and "null files" in last_error(), name
    files = (C.c_char_p * 1)(PHOTO)
    L = lib()
    buf = np.zeros(64, np.uint8)
    assert L.cb200_jpeg_decode_dev(None, files, None, 1, buf.ctypes.data, None) == -1 and "null sizes" in last_error()
    for name, rc in calls([PHOTO, None]):
        assert rc == -1 and "picture 1 is a null pointer" in last_error(), name
    for name, rc in calls([PHOTO], n=-1):
        assert rc == -1 and "n < 0" in last_error(), name
    w = C.c_int32()
    assert L.cb200_jpeg_info(None, 10, C.byref(w), C.byref(w)) == -1
    assert L.cb200_jpeg_info(PHOTO, len(PHOTO), None, C.byref(w)) == -1


def test_camera_flags_checked_before_cuda():
    for name, rc in calls([PHOTO], flags=cb.FLAG_CC_FIT | cb.FLAG_CC_SIMPLE):
        if name == "camera_dev":
            assert rc == -1 and "exclusive" in last_error()
