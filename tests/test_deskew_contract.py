"""The arithmetic contract deskew.cu states for k_deskew, checked against OpenCV itself on the CPU: deskew_corpus.warp_model (the
contract restated in float64 numpy) equals cv2.warpPerspective(INTER_LINEAR) on every case of the corpus in every frame geometry, and
every case reaches the edge it is there for.  So the GPU corpus (tests/test_gpu_deskew_corpus.py) tests the kernel at those edges,
and an OpenCV whose warp changed its arithmetic fails here, without a GPU.  The model's half-away-from-zero rounding is a planted
slip: the tie family must catch it."""
import cv2
import numpy as np
import pytest

import deskew_corpus as dc

GEOMETRY_IDS = [f"{w}x{h}" for w, h in dc.GEOMETRIES]


@pytest.mark.parametrize("family", dc.FAMILIES)
@pytest.mark.parametrize("geometry", dc.GEOMETRIES, ids=GEOMETRY_IDS)
def test_model_equals_cv2_and_reaches_its_edge(geometry, family):
    W, H = geometry
    cases = [c for c in dc.cases(W, H) if c.family == family]
    assert len(cases) >= (3 if family == "scan" else 2)
    for c in cases:
        got, st = dc.warp_model(c.src, c.M, W, H, stats=True)
        want = dc.cv2_warp(c.src, c.M, W, H)
        assert np.array_equal(got, want), (c.name, int((got != want).sum()))
        assert c.holds(st), f"{c.name}: the premise '{c.premise}' does not hold: {st}"


@pytest.mark.parametrize("geometry", dc.GEOMETRIES, ids=GEOMETRY_IDS)
def test_half_away_rounding_fails_the_tie_family(geometry):
    W, H = geometry
    for c in (c for c in dc.cases(W, H) if c.family == "tie"):
        slipped = dc.warp_model(c.src, c.M, W, H, half_away=True)
        assert not np.array_equal(slipped, dc.cv2_warp(c.src, c.M, W, H)), c.name


def test_invert3_is_cv2_invert():
    """the inverse the model (and deskew_run) maps with is cv::invert's, bit for bit"""
    for c in dc.cases(*dc.GEOMETRIES[0]):
        ok, want = cv2.invert(c.M, flags=cv2.DECOMP_LU)
        assert ok != 0 and np.array_equal(dc.invert3(c.M), want.reshape(9)), c.name
    assert dc.invert3(np.array([[1.0, 2, 3], [2, 4, 6], [0, 0, 1]])) is None
