"""The batches of the multi-process CCM-chain tests (tests/test_gpu_ccm_chain.py, tests/ccm_chain_worker.py), built the same way in
every process.  Test infrastructure only.  Each function returns (list of step batches, pictures per rank); rank r decodes the
contiguous stripe libcimbar_b200.dist.stripe(len(batch), r, per) of every step."""
import os

import cv2
import numpy as np

from ragged_samples import GLOB, sample

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


# a colour cast strong enough that a frame decodes its colours right only with a CCM fitted under the same cast: frames, camera
CAST_FRAMES = (1.0, 1.0, 0.3)
CAST_CAMERA = (0.4, 0.7, 1.0)


def crafted(gains):
    """the fountain frames of crafted_rs.cc_pool (mode B) rendered under a colour cast: frames 0, 1, 3, 4 fit their own
    matrix (frame 1 only after RS correction, frame 3 from its second chunk); frame 2 has no header, so it decodes its colours with
    whatever CCM it is handed, and under these casts its colour blocks and colour-stream chunks come out differently with the
    matrix of a fitted frame than without one"""
    from crafted_rs import ORA, cc_pool, raw_to_cells
    g, _, raw, _ = cc_pool(68)
    out = []
    for r in raw:
        f = ORA.render_frame(g.m, raw_to_cells(g, r)).astype(np.float32)
        out.append(np.clip(np.rint(f * np.asarray(gains, np.float32)), 0, 255).astype(np.uint8))
    return out


def frame_steps(world):
    """three steps of crafted frames, three per rank: fitted and unfitted frames on both sides of every stripe boundary, stripes
    without any fit, and a short third step whose last rank has no frames"""
    fr = crafted(CAST_FRAMES)
    per = 3
    pattern1 = [0, 2, 1, 2, 2, 3, 2, 4, 2]               # ranks 1 and 2 open with unfitted frames after a fit
    pattern2 = [2, 2, 2, 1, 2, 2, 2, 2, 2]               # rank 0 has no fit (enters with step 1's exit), rank 2 none either
    pattern3 = [2, 3, 2, 2, 2, 4]                         # short
    steps = [pattern1[:per * world], pattern2[:per * world], pattern3[:per * (world - 1) - 1]]
    return [np.stack([fr[i] for i in p]) for p in steps], per


def pad(rgb, top, bottom, left, right):
    return cv2.copyMakeBorder(rgb, top, bottom, left, right, cv2.BORDER_CONSTANT, value=(0, 0, 0))


def with_anchors(frame):
    """a crafted frame as a camera picture: the four anchor squares of a real encoder frame pasted into its corners (they lie
    outside every cell's threshold support)"""
    from oracle_lib import load_sample
    tr, c = load_sample("b/tr_0.png"), 62
    f = frame.copy()
    for ys in (slice(0, c), slice(1024 - c, 1024)):
        for xs in (slice(0, c), slice(1024 - c, 1024)):
            f[ys, xs] = tr[ys, xs]
    return f


def camera_pictures():
    """mode-B camera pictures: the two mode-B photographs (zero-padded and upscaled variants among them), a noise picture, and crafted
    frames under CAST_CAMERA as pictures -- two that fit (0, 4) and the headerless one (2), which sits first in the second and the
    third stripe of four, right after a stripe whose last fit is a crafted frame's"""
    from oracle_lib import load_sample
    a, b = load_sample("b/ex2434.jpg"), load_sample("b/ex380.jpg")
    noise = np.random.default_rng(53).integers(0, 256, (800, 1000, 3), dtype=np.uint8)
    c0, _, c2, _, c4 = [with_anchors(f) for f in crafted(CAST_CAMERA)]
    return [a, c0, noise, c2, c2, pad(b, 200, 160, 240, 300), c4, c2, c2, cv2.resize(a, None, fx=1.3, fy=1.3), c0, c2]


def camera_steps(world):
    """three steps of camera pictures, four per rank: the batch in order, the batch rotated by four, and a short batch whose last
    rank has none"""
    pics = camera_pictures()
    per = 4
    full = per * world
    steps = [pics[:full], (pics[4:] + pics[:4])[:full], pics[:per * (world - 1) - 2]]
    return steps, per


def legacy_pictures():
    """the 4C sample photographs and padded and noise pictures (mode 4C is a legacy mode: it never fits a CCM)"""
    pics = [sample(s) for s in GLOB]
    pics.append(pad(sample("6bit/4_30_f0_627.jpg"), 120, 150, 100, 160))
    pics.append(np.random.default_rng(47).integers(0, 256, (900, 1200, 3), dtype=np.uint8))
    pics.append(pad(sample("6bit/4_30_f1_360.jpg"), 90, 70, 200, 140))
    pics.append(sample("6bit/4_30_f2_734.jpg"))
    return pics


def legacy_steps(world):
    pics = legacy_pictures()
    per = 4
    full = per * world
    return [pics[:full], (pics[::-1] + pics)[:full], pics[3:3 + per * (world - 1) - 2]], per


def jpeg_files():
    """mode-B JPEG files: the two photographs and crafted pictures under CAST_CAMERA encoded by cv2 at quality 100"""
    def read(name):
        with open(os.path.join(GOLDEN, name), "rb") as fh:
            return fh.read()

    def enc(rgb):
        ok, buf = cv2.imencode(".jpg", cv2.cvtColor(rgb, cv2.COLOR_RGB2BGR), [cv2.IMWRITE_JPEG_QUALITY, 100])
        assert ok
        return buf.tobytes()
    c0, _, c2, _, c4 = [enc(with_anchors(f)) for f in crafted(CAST_CAMERA)]
    return [read("b__ex2434.jpg"), c2, c0, c2, read("b__ex380.jpg"), c4, c2]


def jpeg_steps(world):
    """one step of the seven JPEG files, three per rank (three ranks: the last stripe short): each later stripe opens with the
    headerless picture, right after a fitted crafted picture"""
    return [jpeg_files()], 3
