"""The extractor's deskew (SURVEY 8f-2): cv::getPerspectiveTransform + cv::warpPerspective(INTER_LINEAR) restated on the host /
on the device (libcimbar_b200/csrc/deskew.cu), pinned against OpenCV itself -- the reference calls exactly these two functions
(src/lib/extractor/Deskewer.h:25-40), and python's cv2 is the same library."""
import numpy as np
import pytest

import libcimbar_b200 as cb
from oracle_lib import Oracle, load_sample
from cpu_support import camera_view

ORA = Oracle()


def test_perspective_transform_matches_cv2_bit_for_bit():
    import cv2
    rng = np.random.default_rng(1)
    for _ in range(300):
        src = (rng.random((4, 2)) * 1600 + np.array([[0, 0], [300, 0], [0, 300], [300, 300]])).astype(np.float32)
        src = np.round(src).astype(np.float32) if rng.random() < 0.5 else src      # Corners are integer points in the reference
        dst = np.float32([[30, 30], [994, 30], [30, 994], [994, 994]])
        want = cv2.getPerspectiveTransform(src, dst)
        got = cb.perspective_transform(src, dst)
        assert np.array_equal(got, want), (src, got - want)


@pytest.mark.gpu
def test_deskew_matches_cv2_warp_perspective_bit_for_bit():
    import cv2
    frame = load_sample("b/ex2434.jpg")
    ctx = cb.Context(68, max_frames=2)
    for quad, size in (([[210, 130], [1480, 190], [160, 1350], [1530, 1290]], (1700, 1500)),
                       ([[40, 60], [900, 20], [80, 860], [940, 930]], (1000, 960)),          # downscale and parts outside the source
                       ([[-40, -30], [1100, 10], [5, 1090], [1060, 1130]], (1024, 1024))):
        cam = camera_view(frame, quad, size)
        corners = np.float32([[q[0] + 30 * (1 if i % 2 == 0 else -1) * 0 for q in [quad[i]]][0] for i in range(4)])
        corners = np.float32(quad)
        dst = np.float32([[30, 30], [994, 30], [30, 994], [994, 994]])
        M = cv2.getPerspectiveTransform(corners, dst)
        want = cv2.warpPerspective(cam, M, (1024, 1024), flags=cv2.INTER_LINEAR)
        got = ctx.deskew(cam, M)[0]
        assert np.array_equal(got, want), (quad, int((got != want).sum()))
    ctx.close()


@pytest.mark.gpu
def test_extract_decode_equals_deskew_then_decode():
    """camera image + anchor centres -> chunks in one call; the same chunks as OpenCV's deskew followed by the plain decode
    (and as the oracle decoding the cv2-deskewed frame)"""
    import cv2
    m = ORA.mode(68)
    rng = np.random.default_rng(3)
    payload = rng.integers(0, 256, 7500, dtype=np.uint8)
    frame = ORA.render_frame(m, ORA.payload_to_cells(m, payload))
    # where the anchor centres (30, 30) ... (994, 994) of the frame land in the camera picture
    quad_full = np.float32([[260, 180], [1500, 230], [230, 1400], [1540, 1350]])
    cam = camera_view(frame, quad_full, (1800, 1600))
    Mf = cv2.getPerspectiveTransform(np.float32([[0, 0], [1024, 0], [0, 1024], [1024, 1024]]), quad_full)
    anchors = cv2.perspectiveTransform(np.float32([[[30, 30], [994, 30], [30, 994], [994, 994]]]), Mf)[0]
    anchors = np.round(anchors).astype(np.float32)                     # Anchor centres are integer points (Corners.h)
    dst = np.float32([[30, 30], [994, 30], [30, 994], [994, 994]])
    M = cv2.getPerspectiveTransform(anchors, dst)
    deskewed = cv2.warpPerspective(cam, M, (1024, 1024), flags=cv2.INTER_LINEAR)
    ctx = cb.Context(68, max_frames=2)
    chunks, count, mask, ff = ctx.extract_decode_fountain(np.stack([cam, cam]), np.stack([anchors, anchors]))
    c2, n2, m2, f2 = ctx.decode_fountain(deskewed)
    assert count[0] == n2[0] and mask[0] == m2[0] and np.array_equal(chunks[0], c2[0]) and np.array_equal(chunks[1], c2[0])
    good, ochunks, omask = ORA.decode_fountain(m, deskewed)
    assert mask[0] == omask and count[0] * m.chunk_size == good and np.array_equal(chunks[0][:count[0]], ochunks[:count[0]])
    assert count[0] >= 10                                             # the resampled frame still decodes (RS absorbs the blur)
    ctx.close()
