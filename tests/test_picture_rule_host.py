"""The picture descriptor rule of a receivers plan over device descriptors (libcimbar_b200/csrc/layout_core.cuh: picture_refused, run
on the device by k_plan_pictures) compiled for the CPU, against the library's own host checks (picture_batch, check_picture_sizes and
check_spans behind cb200_scan_extract_decode_chunks_pictures_dev, called with a NULL context: a descriptor they accept reaches the
context check).  On 100 000 random descriptors and on every boundary: short side 59 / 60 / 4499 / 4500, a row pitch of w x channels
- 1, planes that overlap by one byte, spans of 2^32 - 1 and 2^32 bytes, negative and huge pitches, null data, unknown layouts.  With
bounds the rule also refuses a short side outside [min_short, max_short] and a long side above max_long.

The per-slot table builder (plan_slot) is checked against pic_table's rules on the slots it accepts: source, pitches and layout
from the descriptor, the blurred picture at slot x slot_bytes, the radius group and tile count of the picture's size and the word
flag from the actual alignments; empty slots (descriptor not read) and refused ones get the plan's stand-in picture."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import libcimbar_b200 as cb
from libcimbar_b200 import build as cbbuild

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIM = 2 ** 32


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    cbbuild.build()
    out = str(tmp_path_factory.mktemp("picture_rule") / "picture_rule_host")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-o", out, os.path.join(ROOT, "tests", "cpp", "picture_rule_host.cpp")])
    return out


PIC = np.dtype([("data", "<u8"), ("w", "<i4"), ("h", "<i4"), ("row", "<i8"), ("plane", "<i8"), ("layout", "<i4"), ("pad", "<i4")])
DESC = np.dtype([("src", "<u8"), ("blur", "<u8"), ("w", "<i4"), ("h", "<i4"), ("words", "<i4"), ("tile0", "<i4"), ("pitch", "<u8"),
                 ("plane", "<u8"), ("layout", "<i4"), ("pad", "<i4"), ("group", "<i4"), ("tiles", "<i4"), ("refused", "u1")], align=False)
CH = {0: 3, 1: 3, 2: 4, 3: 4, 4: 1}
STANDIN, BLUR_BASE = 0x7F0000001000, 0x7E0000000000


def run(exe, pics, of=None, bounds=None, slot_bytes=0, receivers=1):
    n = len(pics)
    of = np.zeros(n, np.int32) if of is None else np.asarray(of, np.int64).astype(np.int32)
    b = (0, 0, 0) if bounds is None else bounds
    data = np.array([n, receivers, bounds is not None, *b], np.int32).tobytes() + np.array([STANDIN, BLUR_BASE, slot_bytes], np.uint64).tobytes()
    out = subprocess.run([exe], input=data + pics.tobytes() + of.tobytes(), stdout=subprocess.PIPE, check=True).stdout
    refused = np.frombuffer(out[:n], np.uint8).astype(bool)
    table = np.frombuffer(out[n:], DESC) if bounds is not None else None
    return refused, table


def host_accepts(pics):
    """the library's host checks, one descriptor at a time"""
    lib = cb.load_library()
    one = (cb.Picture * 1)()
    got = np.zeros(len(pics), bool)
    for i, p in enumerate(pics):
        one[0] = cb.Picture(int(p["data"]) or None, int(p["w"]), int(p["h"]), int(p["row"]), int(p["plane"]), int(p["layout"]))
        rc = lib.cb200_scan_extract_decode_chunks_pictures_dev(None, C.cast(one, C.c_void_p), 1, 0, None, None, None, None)
        msg = lib.cb200_last_error().decode()
        assert rc == -1
        got[i] = msg == "null context"
        assert got[i] or "picture 0" in msg, msg
    return got


def pictures(rows):
    a = np.zeros(len(rows), PIC)
    for i, r in enumerate(rows):
        a[i] = (*r, 0)
    return a


def random_pictures(rng, n):
    lay = rng.choice([0, 1, 2, 3, 4, 4, -1, 5, 9], n)
    short = rng.choice([rng.integers(1, 5000), 59, 60, 61, 1499, 1500, 2499, 2500, 4499, 4500], n)
    w = np.where(rng.random(n) < 0.5, short, short + rng.integers(0, 3000, n))
    h = np.where(rng.random(n) < 0.5, short, short + rng.integers(0, 3000, n))
    w, h = np.where(rng.random(n) < 0.5, (w, h), (h, w))
    ch = np.array([CH.get(int(v), 3) for v in lay])
    row = w.astype(np.int64) * ch + rng.choice([-1, 0, 0, 0, 1, 3, 64, 2 ** 31], n)
    row = np.where(rng.random(n) < 0.02, -row, row)
    row = np.where(rng.random(n) < 0.01, rng.integers(LIM - 10, LIM + 10, n), row)
    plane = h.astype(np.int64) * row + rng.choice([-1, 0, 0, 1, 4096, -4096], n)
    plane = np.where(rng.random(n) < 0.02, -np.abs(plane) - 1, plane)
    plane = np.where(rng.random(n) < 0.01, rng.integers(LIM - 10, LIM + 10, n), plane)
    data = np.where(rng.random(n) < 0.02, 0, rng.integers(1, 2 ** 47, n))
    a = np.zeros(n, PIC)
    a["data"], a["w"], a["h"], a["row"], a["plane"], a["layout"] = data, w, h, row, plane, lay
    return a


def test_random_descriptors_agree_with_the_host_checks(exe):
    rng = np.random.default_rng(2026)
    pics = random_pictures(rng, 100_000)
    got, _ = run(exe, pics)
    want = ~host_accepts(pics)
    assert np.array_equal(got, want), np.flatnonzero(got != want)[:10]
    assert 0.2 < want.mean() < 0.9                       # premise: both verdicts are common


def boundary_pictures():
    rows = []
    for s in (59, 60, 61, 1499, 1500, 2499, 2500, 4499, 4500):
        for w, h in ((s, s), (s, 4 * s + 1), (3 * s, s)):
            rows.append((0x1000, w, h, 3 * w, 0, 0))
    for lay in range(5):
        c, w, h = CH[lay], 641, 480
        rows += [(0x1000, w, h, w * c - 1, h * w * c, lay), (0x1000, w, h, w * c, h * w * c, lay), (0x1000, w, h, w * c + 1, h * (w * c + 1), lay)]
        rows += [(0x1000, w, h, -1, 0, lay), (0x1000, w, h, w * c, -1, lay), (0, w, h, w * c, h * w * c, lay)]
    for pp in (-1, 0, 1):                                  # planes overlapping by one byte, touching, apart
        rows.append((0x1000, 640, 480, 700, 480 * 700 + pp, 4))
    # spans: (h - 1) row pitch + w channels (+ 2 plane pitches) = 2^32 - 1 and 2^32
    for extra in (-1, 0):
        w, h = 1000, 1000
        rows.append((0x1000, w, h, (LIM + extra - 3 * w) // (h - 1), 0, 0))
        rows.append((0x1000, w, 2, LIM + extra - 3 * w, 0, 0))
        rows.append((0x1000, w, 2, LIM - 1 - 3 * w, 0, 2))
        pr = 1024
        rows.append((0x1000, pr, 100, pr, (LIM + extra - 99 * pr - pr) // 2, 4))
        rows.append((0x1000, pr, 100, pr, (LIM + extra - 99 * pr - pr + 1) // 2, 4))
    rows += [(0x1000, 640, 480, LIM, 0, 0), (0x1000, 640, 480, LIM - 1, 0, 0), (0x1000, 640, 480, 1920, LIM, 4),
             (0x1000, 640, 480, 1920, LIM, 0), (0x1000, 640, 480, 2 ** 62, 0, 4), (0x1000, 640, 480, 1920, 2 ** 62, 4)]
    rows += [(0x1000, 640, 480, 1920, 0, -1), (0x1000, 640, 480, 1920, 0, 5), (0x1000, -640, 480, 1920, 0, 0), (0x1000, 640, 0, 1920, 0, 0)]
    return pictures(rows)


def test_boundaries_agree_with_the_host_checks(exe):
    pics = boundary_pictures()
    got, _ = run(exe, pics)
    want = ~host_accepts(pics)
    assert np.array_equal(got, want), [(tuple(pics[i])[:6], got[i]) for i in np.flatnonzero(got != want)]
    short = np.minimum(pics["w"], pics["h"])
    good = (pics["data"] != 0) & (pics["layout"] == 0) & (pics["row"] == 3 * pics["w"].astype(np.int64)) & (pics["h"] * pics["row"] < 2 ** 31)
    assert got[good & (short == 59)].all() and got[good & (short == 4500)].all()
    assert not got[good & ((short == 60) | (short == 4499))].any()


def test_bounds(exe):
    rng = np.random.default_rng(7)
    pics = random_pictures(rng, 20_000)
    plain, _ = run(exe, pics)
    for bounds in ((60, 4499, 8000), (720, 1080, 1920), (1500, 2499, 2499), (500, 500, 500), (2500, 4499, 4499)):
        got, _ = run(exe, pics, bounds=bounds, slot_bytes=16)
        s, l = np.minimum(pics["w"], pics["h"]), np.maximum(pics["w"], pics["h"])
        outside = (s < bounds[0]) | (s > bounds[1]) | (l > bounds[2])
        assert np.array_equal(got, plain | outside), bounds
    # the bounds' edges
    edge = pictures([(0x1000, w, h, 3 * w, 0, 0) for w, h in ((719, 1000), (720, 1000), (1080, 1920), (1081, 1920), (1080, 1921),
                                                               (1920, 1080), (1921, 1080), (1920, 720), (1920, 719))])
    got, _ = run(exe, edge, bounds=(720, 1080, 1920), slot_bytes=16)
    assert got.tolist() == [True, False, False, True, True, False, True, False, True]


def blur_radius(w, h):
    v = int(min(w, h) * 0.002) - 1 & 0xFFFFFFFF
    for sh in (1, 2, 4, 8, 16):
        v |= v >> sh
    unit = (v + 2) & 0xFFFFFFFF
    return max(unit, 3) // 2


def test_plan_slot_table(exe):
    rng = np.random.default_rng(11)
    n, receivers = 3000, 50
    bounds = (60, 2600, 3000)
    slot = (bounds[1] * bounds[2] + 3) & ~3
    pics = random_pictures(rng, n)
    pics["data"] = np.where(rng.random(n) < 0.5, pics["data"] & ~np.uint64(3), pics["data"])
    of = rng.integers(-3, receivers + 3, n)
    refused, table = run(exe, pics, of, bounds=bounds, slot_bytes=slot, receivers=receivers)
    empty = (of < 0) | (of >= receivers)
    assert np.array_equal(table["refused"].astype(bool), refused & ~empty)
    take = ~empty & ~refused
    assert take.sum() > 100 and (refused & ~empty).sum() > 100
    eff_w = np.where(take, pics["w"], bounds[0])
    eff_h = np.where(take, pics["h"], bounds[0])
    assert np.array_equal(table["w"], eff_w) and np.array_equal(table["h"], eff_h)
    assert np.array_equal(table["src"], np.where(take, pics["data"], STANDIN))
    planar = pics["layout"] == 4
    assert np.array_equal(table["pitch"], np.where(take, pics["row"], 0).astype(np.uint64))
    assert np.array_equal(table["plane"], np.where(take & planar, pics["plane"], 0).astype(np.uint64))
    assert np.array_equal(table["layout"], np.where(take, pics["layout"], 0))
    assert np.array_equal(table["blur"], np.arange(n, dtype=np.uint64) * np.uint64(slot))
    # pic_table's word path: w % 4, the source, the pitches and the blurred base all 4-byte aligned
    words = (eff_w % 4 == 0) & (table["src"] % 4 == 0) & (table["pitch"] % 4 == 0) & (table["plane"] % 4 == 0) & \
            ((np.uint64(BLUR_BASE) + table["blur"]) % 4 == 0)
    assert np.array_equal(table["words"] != 0, words) and words.any() and (~words).any()
    group = np.array([{1: 0, 2: 1, 4: 2}[blur_radius(w, h)] for w, h in zip(eff_w, eff_h)])
    tiles = ((eff_w.astype(np.int64) + 127) // 128) * ((eff_h.astype(np.int64) + 31) // 32)
    assert np.array_equal(table["group"], group) and set(group[take]) == {0, 1, 2}
    assert np.array_equal(table["tiles"], tiles)
