"""The camera path's per-picture extract decisions (libcimbar_b200/csrc/extract_core.cuh: what k_extract runs on the device, and what
cb200_perspective_transform and the deskew use on the host) compiled for the host: status, corners and the granular rule against the
oracle's Corners, the transform against cb200_perspective_transform and cv2.getPerspectiveTransform, the inverse against cv2.invert --
bit for bit.  The GPU test (tests/test_gpu_camera_dev.py) compares the device's transforms with the same references."""
import ctypes as C

import cv2
import numpy as np
import pytest

import libcimbar_b200 as cb
from libcimbar_b200 import build as cbbuild
from ragged_samples import GLOB, sample
from scan_oracle_lib import ScanOracle
from host_harness import build_harness

SO = ScanOracle()
MODES = [(1024, 1024), (1024, 720), (736, 637)]
AN = 30


@pytest.fixture(scope="module")
def core(tmp_path_factory):
    cbbuild.build()
    lib = build_harness(tmp_path_factory, "extract_core_host", "-ffp-contract=off")
    vp = C.c_void_p
    lib.ec_extract.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp]
    lib.ec_transform.argtypes = [vp, vp, vp]
    lib.ec_invert.argtypes = [vp, vp]
    lib.ec_granular.argtypes = [vp, C.c_int, C.c_int]
    return lib


def outp(w, h):
    return np.array([AN, AN, w - AN, AN, AN, h - AN, w - AN, h - AN], np.float32)


def extract(core, anchors, count, overflow, w, h):
    a = np.zeros((4, 4), np.int32)
    if anchors:
        a[:len(anchors)] = anchors
    corners, fwd, inv = np.zeros(8, np.float32), np.zeros(9, np.float64), np.zeros(9, np.float64)
    st = core.ec_extract(a.ctypes.data, count, int(overflow), w, h, corners.ctypes.data, fwd.ctypes.data, inv.ctypes.data)
    return st, corners, fwd.reshape(3, 3), inv.reshape(3, 3)


def check_transform(core, src, dst):
    """the header's transform == cb200_perspective_transform == cv2 (when solvable); its inverse == cv2.invert"""
    m9 = np.zeros(9, np.float64)
    ok = core.ec_transform(src.ctypes.data, dst.ctypes.data, m9.ctypes.data)
    m9 = m9.reshape(3, 3)
    if ok:
        assert np.array_equal(m9, cb.perspective_transform(src, dst))
        assert np.array_equal(m9, cv2.getPerspectiveTransform(src.reshape(4, 2), dst.reshape(4, 2)))
        inv = np.zeros(9, np.float64)
        assert core.ec_invert(m9.ctypes.data, inv.ctypes.data) == 1
        assert np.array_equal(inv.reshape(3, 3), cv2.invert(m9)[1])
    else:
        with pytest.raises(cb.Cb200Error):
            cb.perspective_transform(src, dst)
        assert np.array_equal(m9, np.diag([0., 0., 1.]))
    return ok, m9


def check_picture(core, anchors, w, h):
    """extract_picture of a four-anchor scan against the oracle's Corners and granular rule and the transforms"""
    st, corners, fwd, inv = extract(core, anchors, 4, False, w, h)
    xy = SO.corners(anchors)
    want = 1 if SO.is_granular_scale(xy, w, h) else 2
    ok, m9 = check_transform(core, np.array(xy, np.float32), outp(w, h))
    assert core.ec_granular(np.array(xy, np.float32).ctypes.data, w, h) == (want == 1)
    if ok:
        assert st == want and corners.tolist() == [float(v) for v in xy]
        assert np.array_equal(fwd, m9) and np.array_equal(inv, cv2.invert(m9)[1])
    else:
        assert st == 0
    return st


def test_every_scan_of_the_sample_directory(core):
    seen = set()
    for s in GLOB:
        anchors, _ = SO.scan(sample(s))
        assert anchors is not None and len(anchors) == 4, s
        for w, h in MODES:
            seen.add(check_picture(core, anchors, w, h))
    assert seen == {1, 2}


def test_random_quadrilaterals(core):
    rng = np.random.default_rng(2024)
    for trial in range(10000):
        w, h = MODES[trial % 3]
        c = rng.integers(0, 4000, 2)
        pts = c + rng.integers(-1500, 1500, (4, 2))
        anchors = [(int(x) - 5, int(x) + 5 + trial % 2, int(y) - 6, int(y) + 6) for x, y in pts]
        check_picture(core, anchors, w, h)


def test_crafted_cases(core):
    w, h = 1024, 1024
    ident_fwd = check_transform(core, outp(w, h), outp(w, h))[1]
    ident_inv = cv2.invert(ident_fwd)[1]

    def failed(st, corners, fwd, inv, want):
        assert st == want and np.array_equal(corners, outp(w, h))
        assert np.array_equal(fwd, ident_fwd) and np.array_equal(inv, ident_inv)

    # three collinear anchors (and the fourth off the line) and coincident anchors: a degenerate quadrilateral is a FAILURE
    for anchors in ([(90, 110, 90, 110), (490, 510, 90, 110), (890, 910, 90, 110), (490, 510, 890, 910)],
                    [(90, 110, 90, 110), (90, 110, 90, 110), (890, 910, 890, 910), (890, 910, 890, 910)],
                    [(100, 100, 100, 100)] * 4):
        st, corners, fwd, inv = extract(core, anchors, 4, False, w, h)
        xy = np.array(SO.corners(anchors), np.float32)
        ok, _ = check_transform(core, xy, outp(w, h))
        if not ok:
            failed(st, corners, fwd, inv, 0)
    st = extract(core, [(100, 100, 100, 100)] * 4, 4, False, w, h)
    failed(*st, 0)
    good = [(90, 110, 90, 110), (1890, 1910, 80, 120), (100, 120, 1900, 1920), (1880, 1900, 1890, 1910)]
    # counts 0 .. 3 and the overflow status
    for count in range(4):
        failed(*extract(core, good[:count], count, False, w, h), 0)
    failed(*extract(core, good, 4, True, w, h), -1)
    assert extract(core, good, 4, False, w, h)[0] == 1
