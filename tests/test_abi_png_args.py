"""CPU-side checks of the PNG entry points (cb200_png_info, cb200_png_decode_dev, cb200_png_scan_extract_decode_chunks_dev): a file
outside the supported set, a bad size or a null pointer is refused with CB200_ERR_ARG before any CUDA call, and the message names the
picture and the reason.  The context is NULL here, so a call whose files are all good fails on the context instead.

The crafted corruptions are checked against cv2 as well: where cv2 returns None, the file is refused here or fails on the device
(the host build of the device functions, tests/cpp/png_core_host.cpp, reports -2); where cv2 decodes it, it is decoded to cv2's
bytes or refused."""
import ctypes as C
import os
import struct
import subprocess
import zlib

import numpy as np
import pytest

import libcimbar_b200 as cb
from libcimbar_b200 import build as cbbuild
import png_matrix as pm
from png_matrix import SIG, chunk, cv2_rgb, exif, filter_rows, golden_files, png, walk

ROOT = os.path.dirname(os.path.abspath(os.path.dirname(__file__)))


@pytest.fixture(scope="module", autouse=True)
def built():
    cbbuild.build()


def lib():
    return cb.load_library()


FRAME = dict(golden_files())["b__tr_0.png"]
RNG = np.random.default_rng(1)
W, H = 70, 64
IMG = RNG.integers(0, 256, (H, 3 * W)) // 16 * 16
BASE = png(W, H, 2, 8, IMG, filters=[y % 5 for y in range(H)])
CH = walk(BASE)
Z = b"".join(b for k, b in CH if k == b"IDAT")
RAW = zlib.decompress(Z)
IHDR = CH[0][1]
PAL = RNG.integers(0, 256, (16, 3))
IDX = RNG.integers(0, 16, (H, W))
P4 = png(W, H, 3, 4, IDX, palette=PAL)
PC = walk(P4)


def build(chs):
    return SIG + b"".join(chunk(k, b) for k, b in chs)


def with_z(z, idat=None):
    step = idat or len(z)
    return build([CH[0]] + [(b"IDAT", z[i:i + step]) for i in range(0, len(z), step)] + [(b"IEND", b"")])


def bad_crc(data, kind, which=0):
    i, seen = 8, 0
    while i < len(data):
        n = struct.unpack(">I", data[i:i + 4])[0]
        if data[i + 4:i + 8] == kind:
            if seen == which:
                j = i + 8 + n
                return data[:j] + bytes([data[j] ^ 1]) + data[j + 1:]
            seen += 1
        i += 12 + n
    raise KeyError(kind)


def fixed_far():
    """a fixed block whose first match reaches 3 bytes before the output"""
    from png_matrix import BitWriter, fixed_sym
    bw = BitWriter()
    bw.bits(1, 1)
    bw.bits(1, 2)
    fixed_sym(bw, RAW[0])
    fixed_sym(bw, 257)
    bw.code(3, 5)
    for b in RAW[4:]:
        fixed_sym(bw, b)
    fixed_sym(bw, 256)
    return b"\x78\x01" + bw.done() + b"\x00" * 4


def incomplete_lengths():
    from png_matrix import BitWriter
    bw = BitWriter()
    for v, n in ((1, 1), (2, 2), (0, 5), (0, 5), (0, 4), (1, 3), (0, 3), (0, 3), (0, 3)):
        bw.bits(v, n)
    return b"\x78\x01" + bw.done() + bytes(100)


def stored(h, row, bad_adler, idat=None, lead=False):
    """a grey file of one stored block (after an empty one with `lead`) with (optionally) a wrong Adler-32: whether libpng fails it
    depends on where the check value falls against its 8 KB reads and its chunks (png_core.cuh stream_end_ok)"""
    rows = np.random.default_rng(h * row).integers(0, 256, (h, row - 1))
    raw = filter_rows(rows, 0, 8, [0] * h)
    z = b"\x78\x01" + (b"\x00\x00\x00\xff\xff" if lead else b"") + b"\x01" + struct.pack("<HH", len(raw), ~len(raw) & 0xFFFF) + raw
    z += struct.pack(">I", zlib.adler32(raw) ^ bad_adler)
    return png(row - 1, h, 0, 8, rows, zdata=z, idat_size=idat)


def header_only(w, h, bd=1):
    """a grey file of w x h zero pixels without building the samples (for sizes too large to build)"""
    z = zlib.compress(bytes(h * (1 + (w * bd + 7) // 8)), 9)
    return SIG + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, bd, 0, 0, 0, 0)) + chunk(b"IDAT", z) + chunk(b"IEND", b"")


def window_cinfo(cinfo):
    """a 200 x 80 RGB8 picture whose rows 40.. repeat rows 0.., compressed with a 32 KB window (matches 40 rows back), its zlib
    header rewritten to a window of 2^(8 + cinfo) bytes"""
    rows = np.random.default_rng(9).integers(0, 256, (80, 600))
    rows[40:] = rows[:40]
    co = zlib.compressobj(9, zlib.DEFLATED, 15)
    z = co.compress(filter_rows(rows, 2, 8, [0] * 80)) + co.flush()
    cmf = cinfo << 4 | 8
    return png(200, 80, 2, 8, rows, zdata=bytes([cmf, (31 - (cmf << 8) % 31) % 31]) + z[2:])


def tail_after_rows(same_chunk):
    """the rows in a non-final block ending in a sync flush, then a block of type 3, in the same IDAT chunk or a later one"""
    co = zlib.compressobj(9)
    z = co.compress(RAW) + co.flush(zlib.Z_FULL_FLUSH)
    return build([CH[0]] + ([(b"IDAT", z + b"\x07")] if same_chunk else [(b"IDAT", z), (b"IDAT", b"\x07")]) + [(b"IEND", b"")])


REFUSED = [
    ("bad signature", b"\x89PNG\r\n\x1a\x0b" + BASE[8:], "bad signature"),
    ("empty", b"", "bad signature"),
    ("IHDR CRC", bad_crc(BASE, b"IHDR"), "bad CRC in IHDR"),
    ("no IHDR", build(CH[1:]), "IHDR is not the first chunk"),
    ("IHDR twice", build([CH[0]] + CH), "second IHDR"),
    ("IHDR not first", build([(b"gAMA", struct.pack(">I", 45455))] + CH), "IHDR is not the first chunk"),
    ("IHDR of 12 bytes", build([(b"IHDR", IHDR[:12])] + CH[1:]), "IHDR chunk of 12 bytes"),
    ("IHDR RGB at 4 bit", build([(b"IHDR", IHDR[:8] + b"\x04" + IHDR[9:])] + CH[1:]), "colour type 2 at bit depth 4"),
    ("IHDR colour type 5", build([(b"IHDR", IHDR[:9] + b"\x05" + IHDR[10:])] + CH[1:]), "colour type 5"),
    ("IHDR compression 1", build([(b"IHDR", IHDR[:10] + b"\x01" + IHDR[11:])] + CH[1:]), "compression method"),
    ("IHDR width 0", build([(b"IHDR", b"\x00" * 4 + IHDR[4:])] + CH[1:]), "invalid size"),
    ("palette without PLTE", build([PC[0]] + PC[2:]), "colour type 3 without a PLTE"),
    ("PLTE CRC", bad_crc(P4, b"PLTE"), "bad CRC in PLTE"),
    ("PLTE twice", build(PC[:2] + [PC[1]] + PC[2:]), "second PLTE"),
    ("unknown critical chunk", build([CH[0], (b"ABCD", b"xx")] + CH[1:]), "unknown critical chunk ABCD"),
    ("Adam7", build([(b"IHDR", IHDR[:12] + b"\x01")] + CH[1:]), "Adam7"),
    ("APNG", build([CH[0], (b"acTL", struct.pack(">II", 1, 0))] + CH[1:]), "APNG"),
    ("zlib header check", with_z(bytes([Z[0], Z[1] ^ 1]) + Z[2:]), "invalid zlib header"),
    ("zlib method 9", with_z(bytes([0x79, 0xDA]) + Z[2:]), "invalid zlib header"),
    ("zlib window 64 KB", with_z(bytes([0x88, (31 - 0x8800 % 31) % 31]) + Z[2:]), "invalid zlib header"),
    ("preset dictionary", with_z(b"\x78\x20\x00\x00\x00\x01" + Z[2:]), "preset dictionary"),
    ("truncated header", BASE[:20], "truncated"),
    ("truncated in IDAT", BASE[:len(BASE) // 2], "truncated"),
    ("no IEND", BASE[:-12], "no IEND"),
    ("IDATs not consecutive", (lambda cs: build([cs[0], cs[1], (b"tEXt", b"a\x00b")] + cs[2:]))(walk(with_z(Z, 100))), "not consecutive"),
    ("no IDAT", build([CH[0], CH[-1]]), "no IDAT"),
    ("two eXIf", build([CH[0], (b"eXIf", exif(6)), (b"eXIf", exif(1))] + CH[1:]), "more than one eXIf"),
    ("too small", png(59, 400, 0, 8, np.zeros((400, 59))), "smaller than 60"),
    ("too large", png(4500, 4600, 0, 1, np.zeros((4600, 4500)), level=1), "4500"),
    ("height above 1000000", header_only(60, 1000001), "above 1000000"),
    ("width above 1000000", header_only(1000001, 60), "above 1000000"),
    ("more than 2^30 pixels", SIG + chunk(b"IHDR", struct.pack(">IIBBBBB", 40000, 30000, 1, 0, 0, 0, 0)) + chunk(b"IDAT", b"\x78\x01")
     + chunk(b"IEND", b""), "OpenCV's limit"),
]

CORRUPT = [                                      # found on the device: status -2
    ("IDAT CRC", bad_crc(BASE, b"IDAT")),
    ("IDAT CRC, first of many", bad_crc(with_z(Z, 100), b"IDAT", 0)),
    ("IDAT CRC, last of many", bad_crc(with_z(Z, 100), b"IDAT", len(Z) // 100)),
    ("Adler-32 in the last read", with_z(Z[:-1] + bytes([Z[-1] ^ 1]))),
    ("stream without its Adler-32", with_z(Z[:-4])),
    ("block type 3", with_z(Z[:2] + bytes([Z[2] | 0x06]) + Z[3:])),
    ("stored LEN / NLEN", with_z(b"\x78\x01\x01" + struct.pack("<HH", len(RAW), (~len(RAW) + 1) & 0xFFFF) + RAW + b"\x00" * 4)),
    ("filter type 5", with_z(zlib.compress(bytes([5]) + RAW[1:]))),
    ("filter type 5 in the last row", with_z(zlib.compress(RAW[:(H - 1) * (3 * W + 1)] + b"\x05" + RAW[(H - 1) * (3 * W + 1) + 1:]))),
    ("stream short of the rows", with_z(zlib.compress(RAW[:-10]))),
    ("distance before the output", with_z(fixed_far())),
    ("incomplete code lengths", with_z(incomplete_lengths())),
    ("stored, Adler-32 in the same read", stored(5, 1636, 1)),
    ("stored, Adler-32 in the same 100-byte chunk", stored(1, 95, 1, idat=100)),
    ("stored 60 rows, Adler-32 in the same read", stored(60, 819, 1)),
    ("stored 60 rows, Adler-32 in the same chunk", stored(60, 61, 1, idat=3671)),
    ("window 2^11 under matches 24 040 back", window_cinfo(3)),
    ("window 2^14 under matches 24 040 back", window_cinfo(6)),
    ("window: a match one byte past the limit", pm.with_matches(99, 60, 0, [(1050, 307, 10)])),
    ("window: a match running into a row past the window", pm.with_matches(99, 60, 0, [(1095, 300, 10)])),
    ("window: a match past the limit after a refill", pm.with_matches(99, 120, 0, [(2847, 303, 5)], idat_size=1000)),
    ("a corrupt block right after the rows, same read", tail_after_rows(True)),
]

ACCEPTED = [                                     # cv2 decodes these: so must the device, byte for byte
    ("Adler-32 in a later read", with_z(Z[:-1] + bytes([Z[-1] ^ 1]), 1)),
    ("Adler-32 in its own chunk", with_z(Z[:-4] + bytes([Z[-4] ^ 1]) + Z[-3:], len(Z) - 4)),
    ("stored, Adler-32 past an 8 KB read", stored(5, 1637, 1)),
    ("stored, Adler-32 in the next 100-byte chunk", stored(1, 92, 1, idat=100)),
    ("stored 60 rows, Adler-32 past an 8 KB read", stored(60, 819, 1, lead=True)),
    ("stored 60 rows, Adler-32 in the next chunk", stored(60, 61, 1, idat=3667)),
    ("window 2^15 under matches 24 040 back", window_cinfo(7)),
    ("window: a match at the limit", pm.with_matches(99, 60, 0, [(1050, 306, 10)])),
    ("window: a 512-byte window holds the next row's part", pm.with_matches(99, 60, 1, [(1095, 300, 10)])),
    ("window: a match at the limit after a refill", pm.with_matches(99, 120, 0, [(2847, 261, 5)], idat_size=1000)),
    ("more data than the rows", with_z(zlib.compress(RAW + bytes(500)))),
    ("bytes after the stream", with_z(Z + b"garbage!")),
    ("ancillary CRC", bad_crc(build([CH[0], (b"gAMA", struct.pack(">I", 45455))] + CH[1:]), b"gAMA")),
    ("IEND CRC", bad_crc(BASE, b"IEND")),
    ("empty IDAT chunks", build([CH[0], (b"IDAT", b"")] + CH[1:-1] + [(b"IDAT", b""), CH[-1]])),
    ("PLTE in an RGB file, bad size and CRC", bad_crc(build([CH[0], (b"PLTE", bytes(range(47)))] + CH[1:]), b"PLTE")),
    ("eXIf after IDAT", build(CH[:-1] + [(b"eXIf", exif(6))] + CH[-1:])),
    ("eXIf little-endian", build([CH[0], (b"eXIf", b"II\x2a\x00" + struct.pack("<IH", 8, 1) + struct.pack("<HHIHH", 0x0112, 3, 1, 8, 0)
                                                     + b"\x00" * 4)] + CH[1:])),
    ("eXIf with a bad CRC", bad_crc(build([CH[0], (b"eXIf", exif(6))] + CH[1:]), b"eXIf")),
    ("eXIf garbage", build([CH[0], (b"eXIf", b"garbage")] + CH[1:])),
    ("palette index past PLTE", png(W, H, 3, 4, IDX, palette=PAL[:4])),
    ("tRNS before PLTE", build([PC[0], (b"tRNS", bytes(4)), PC[1]] + PC[2:])),
    ("trailing bytes", BASE + b"garbage"),
]


@pytest.fixture(scope="module")
def core(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("png_core") / "png_core_host.so")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-shared", "-fPIC", "-o", so, os.path.join(ROOT, "tests", "cpp", "png_core_host.cpp")])
    L = C.CDLL(so)
    L.pc_decode.argtypes = [C.c_char_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_char_p, C.c_int]
    return L


def host_decode(core, data):
    out = np.zeros(3 * 200 * 8200, np.uint8)
    wh = np.zeros(2, np.int32)
    why = C.create_string_buffer(256)
    rc = core.pc_decode(data, len(data), out.ctypes.data, out.size, wh.ctypes.data, why, 256)
    return rc, (out[:3 * wh[0] * wh[1]].reshape(wh[1], wh[0], 3) if rc == 0 else None)


def calls(files, sizes=None, n=None, flags=0):
    """each PNG entry point with these files (NULL context); yields (name, rc)"""
    L = lib()
    n = len(files) if n is None else n
    ptrs = None if files is None else (C.c_char_p * max(len(files), 1))(*files)
    if sizes is None and files is not None:
        sizes = (C.c_uint64 * max(len(files), 1))(*[len(f) if f is not None else 0 for f in files])
    buf = np.zeros(64, np.uint8)
    yield "decode_dev", L.cb200_png_decode_dev(None, ptrs, sizes, n, buf.ctypes.data, buf.ctypes.data)
    yield "camera_dev", L.cb200_png_scan_extract_decode_chunks_dev(None, ptrs, sizes, n, flags, buf.ctypes.data, buf.ctypes.data,
                                                                   None, buf.ctypes.data)


def last_error():
    return lib().cb200_last_error().decode()


@pytest.mark.parametrize("what,data,reason", REFUSED, ids=[r[0] for r in REFUSED])
def test_refused_files_name_the_picture(what, data, reason):
    for name, rc in calls([FRAME, data, FRAME]):
        assert rc == -1, name
        msg = last_error()
        assert "picture 1" in msg and reason in msg, (name, msg)
    w, h = C.c_int32(), C.c_int32()
    assert lib().cb200_png_info(data, len(data), C.byref(w), C.byref(h)) == -1
    assert reason in last_error()
    with pytest.raises(cb.Cb200Error, match=reason):
        cb.png_info(data)


@pytest.mark.parametrize("what,data", CORRUPT, ids=[c[0] for c in CORRUPT])
def test_corrupt_files_fail_where_cv2_fails(core, what, data):
    assert cv2_rgb(data) is None                                     # premise: cv2 rejects the file
    rc, _ = host_decode(core, data)
    assert rc == -2, rc


@pytest.mark.parametrize("what,data", ACCEPTED, ids=[a[0] for a in ACCEPTED])
def test_files_cv2_accepts_decode_to_its_bytes(core, what, data):
    want = cv2_rgb(data)
    assert want is not None                                          # premise: cv2 decodes the file
    rc, got = host_decode(core, data)
    assert rc == 0 and np.array_equal(got, want), rc


def test_corrupt_data_after_the_rows_in_a_later_read_is_minus_2():
    """the documented deviation: libpng only warns about corrupt data it reads after the last row in a later zlib call (cv2
    decodes the file), and the device reports it -2; in the same read as the last row both fail the file (CORRUPT above)"""
    data = tail_after_rows(False)
    assert cv2_rgb(data) is not None


def test_corrupt_data_after_the_rows_in_a_later_read_decodes_to_minus_2(core):
    rc, _ = host_decode(core, tail_after_rows(False))
    assert rc == -2


def test_refused_files_are_not_decoded_by_cv2_or_listed():
    """every refusal above is either a file cv2 rejects too or one of the deliberate ones (APNG, repeated eXIf, sizes)"""
    deliberate = {"APNG", "two eXIf", "too small", "too large"}
    for what, data, _ in REFUSED:
        if what not in deliberate:
            assert cv2_rgb(data) is None, what


def test_good_files_fail_only_on_the_context():
    for name, rc in calls([FRAME, BASE]):
        assert rc == -1 and "null context" in last_error(), name


def test_null_pointers():
    for name, rc in calls(None, n=1):
        assert rc == -1 and "null files" in last_error(), name
    files = (C.c_char_p * 1)(FRAME)
    L = lib()
    buf = np.zeros(64, np.uint8)
    assert L.cb200_png_decode_dev(None, files, None, 1, buf.ctypes.data, None) == -1 and "null sizes" in last_error()
    for name, rc in calls([FRAME, None]):
        assert rc == -1 and "picture 1 is a null pointer" in last_error(), name
    for name, rc in calls([FRAME], n=-1):
        assert rc == -1 and "n < 0" in last_error(), name
    w = C.c_int32()
    assert L.cb200_png_info(None, 10, C.byref(w), C.byref(w)) == -1
    assert L.cb200_png_info(FRAME, len(FRAME), None, C.byref(w)) == -1


def test_camera_flags_checked_before_cuda():
    for name, rc in calls([FRAME], flags=cb.FLAG_CC_FIT | cb.FLAG_CC_SIMPLE):
        if name == "camera_dev":
            assert rc == -1 and "exclusive" in last_error()
