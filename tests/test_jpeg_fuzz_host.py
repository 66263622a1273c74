"""The device JPEG decoder's functions (jpeg_core.cuh, compiled for the host as in test_jpeg_core_host.py) on the generated corpus
of tests/jpeg_fuzz.py: every file decodes to exactly cv2.imread + cvtColor(BGR2RGB) and cb200_jpeg_info gives cv2's size (or
refuses a picture below the camera path's 60 pixels); pictures up to 8 pixels wide upsample as libjpeg-turbo's jinit_upsampler
chooses; and damaged files, decoded under AddressSanitizer and UndefinedBehaviorSanitizer, are reported as corrupt or decode to
exactly what cv2 gives for the same bytes -- except for pictures with blocks whose IDCT leaves the range where libjpeg-turbo's C and
SIMD IDCTs agree (jpeg_core.cuh idct_islow), where cv2's bytes depend on how it was built."""
import collections
import ctypes as C
import os
import struct
import subprocess

import cv2
import numpy as np
import pytest

import libcimbar_b200 as cb
from libcimbar_b200 import build as cbbuild
from jpeg_fuzz import RESTARTS, corpus, mutations, orphaned_ff, restart_class, walk
from jpeg_matrix import SAMPLING, cv2_rgb
from test_jpeg_core_host import core, decode  # noqa: F401  (the host build as a fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FILES = corpus()
IDS = [n for n, _ in FILES]


def test_premise_the_corpus_covers_what_it_claims():
    assert len(set(IDS)) == len(IDS) and 200 <= len(FILES) <= 500
    info = {n: walk(d) for n, d in FILES}
    combos = {(i["sampling"], i["progressive"], restart_class(i["restart"])) for i in info.values()}
    assert combos >= {(s, p, restart_class(r)) for s in list(SAMPLING) + ["grey"] for p in (False, True) for r in RESTARTS}
    lengths = [e - b for i in info.values() for b, e in i["segments"]]
    assert min(lengths) < 8
    assert any(len(i["segments"]) == 1 and i["segments"][0][1] - i["segments"][0][0] > 65536 for i in info.values())
    for samp in list(SAMPLING) + ["grey"]:
        sizes = [i["size"] for i in info.values() if i["sampling"] == samp]
        for lo in (1, 60):
            want = set(range(lo, lo + 17))
            assert want <= {w for w, _ in sizes} and want <= {h for _, h in sizes}, (samp, lo)
    assert {3000 * 2000, 4000 * 3000} <= {w * h for w, h in (i["size"] for i in info.values())}
    for o in (5, 6, 7, 8):                                    # transposed by cv2, on odd unequal sides
        for n, d in FILES:
            if n.startswith("pil_exif%d_" % o):
                w, h = info[n]["size"]
                assert w % 2 and h % 2 and w != h and cv2_rgb(d).shape[:2] == (w, h), n


@pytest.mark.parametrize("name,data", FILES, ids=IDS)
def test_decodes_like_cv2(core, name, data):  # noqa: F811
    rc, why, wh, out, want = decode(core, data)
    assert rc == 0, why
    h, w = want.shape[:2]
    assert (wh[0], wh[1]) == (w, h)
    got = out[:want.size].reshape(want.shape)
    assert np.array_equal(got, want), (name, int(np.count_nonzero(got != want)))


@pytest.mark.parametrize("name,data", FILES, ids=IDS)
def test_info_agrees_with_cv2(name, data):
    cbbuild.build()
    h, w = cv2_rgb(data).shape[:2]
    if min(w, h) >= 60:
        assert cb.jpeg_info(data) == (w, h)
    else:
        with pytest.raises(cb.Cb200Error, match="smaller than 60"):
            cb.jpeg_info(data)


# libjpeg-turbo's jinit_upsampler filters a component downsampled horizontally (4:2:2, 4:2:0) only when its downsampled_width is
# above 2, so pictures up to 4 pixels wide are upsampled by replication; 4:4:0 is always filtered
@pytest.mark.parametrize("prog", [0, 1], ids=["base", "prog"])
@pytest.mark.parametrize("h", list(range(1, 10)) + [40])
@pytest.mark.parametrize("w", range(1, 9))
@pytest.mark.parametrize("samp", list(SAMPLING))
def test_narrow_pictures_upsample_like_cv2(core, samp, w, h, prog):  # noqa: F811
    img = np.random.default_rng([w, h, prog, SAMPLING[samp]]).integers(0, 256, (h, w, 3), dtype=np.uint8)
    ok, buf = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, 90, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, SAMPLING[samp],
                                         cv2.IMWRITE_JPEG_PROGRESSIVE, prog])
    assert ok
    rc, why, _, out, want = decode(core, buf.tobytes())
    assert rc == 0, why
    assert np.array_equal(out[:want.size].reshape(want.shape), want)


def run_sanitized(tmp_path, files):
    """[(rc, wide, rgb or None)] of tests/cpp/jpeg_fuzz_host.cpp built with -fsanitize=address,undefined (any finding aborts it)"""
    exe = str(tmp_path / "jpeg_fuzz_host")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
                           "-fno-omit-frame-pointer", "-o", exe, os.path.join(ROOT, "tests", "cpp", "jpeg_fuzz_host.cpp")])
    blob = b"".join(struct.pack("<Q", len(d)) + d for d in files)
    r = subprocess.run([exe], input=blob, capture_output=True)
    assert r.returncode == 0 and not r.stderr, r.stderr.decode(errors="replace")[-4000:]
    res, at = [], 0
    for _ in files:
        rc, w, h, wide = struct.unpack_from("<iiii", r.stdout, at)
        at += 16
        rgb = None
        if rc == 0:
            rgb = np.frombuffer(r.stdout, np.uint8, 3 * w * h, at).reshape(h, w, 3)
            at += 3 * w * h
        res.append((rc, wide, rgb))
    assert at == len(r.stdout)
    return res


def test_damaged_files_are_reported_or_decode_like_cv2(tmp_path):
    """a damaged file is reported as corrupt (-2), or, if it still parses completely, it is decoded as libjpeg-turbo decodes it
    (unless an IDCT block leaves the range where libjpeg-turbo's own IDCTs agree)"""
    damaged = mutations(FILES)
    seen = collections.Counter()
    original = dict(FILES)
    changed = wide_pictures = 0
    for (name, data), (rc, wide, rgb) in zip(damaged, run_sanitized(tmp_path, [d for _, d in damaged])):
        seen[(name.split("~")[1].rstrip("0123456789."), rc)] += 1
        assert rc in (0, -2), (name, rc)
        wide_pictures += rc == 0 and wide > 0
        if rc == 0 and wide == 0:
            want = cv2_rgb(data)
            assert rgb.shape == want.shape and np.array_equal(rgb, want), name
            changed += not np.array_equal(want, cv2_rgb(original[name.split("~")[0]]))
    assert wide_pictures <= len(damaged) // 20, wide_pictures
    # premise: every kind of damage is there, and both verdicts, with pictures that differ from the undamaged file's
    assert {k for k, _ in seen} == {"flip", "truncate", "unstuff", "swap"} and {rc for _, rc in seen} == {0, -2}, seen
    assert changed >= 10, changed


def decode_wide(core, data):  # noqa: F811  (the fixture's library)
    """(rc, wide, rgb or None) of the host build's jc_decode_wide"""
    core.jc_decode_wide.argtypes = [C.c_char_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_char_p, C.c_int, C.c_void_p]
    wh = np.zeros(2, np.int32)
    why = C.create_string_buffer(256)
    assert core.jc_info(data, len(data), wh.ctypes.data, why, 256) == 0, why.value
    out = np.zeros(3 * int(wh[0]) * int(wh[1]), np.uint8)
    wide = np.zeros(1, np.int32)
    rc = core.jc_decode_wide(data, len(data), out.ctypes.data, out.size, wh.ctypes.data, why, 256, wide.ctypes.data)
    return rc, int(wide[0]), out.reshape(wh[1], wh[0], 3) if rc == 0 else None


def test_every_byte_after_an_orphaned_ff_is_corrupt_data(core):  # noqa: F811
    """whatever false marker a lost stuffing byte makes (each of the 256 values after the FF, in the first and the last scan of a
    file of each sampling x progressive), the file is accepted by cb200_jpeg_info and decodes to status -2, or to cv2's picture"""
    cbbuild.build()
    files = orphaned_ff(FILES)
    assert len(files) == 2 * 256 * 2 * 5
    seen = collections.Counter()
    for name, data in files:
        cb.jpeg_info(data)
        rc, wide, rgb = decode_wide(core, data)
        seen[rc] += 1
        assert rc in (0, -2), (name, rc)
        if rc == 0 and wide == 0:
            assert np.array_equal(rgb, cv2_rgb(data)), name
    assert seen[-2] >= len(files) * 9 // 10, seen
