"""The reference's samples/6bit/*.jpg in glob order, as the ragged-batch tests use them.  Test infrastructure only.

Six of the eight photographs are in golden/manifest.json; 4_30_802.jpg and 4_30_f0_177_ccm.jpg are recorded in
golden/ragged_samples.json (file, shape, SHA-256 of the decoded RGB).  4_30_f0_big.jpg (3052 x 2704, 2.9 MB) is too large to keep in
the repository: its place in the batch goes to a 2.8x upscale of 4_30_f1_360.jpg (3584 x 2688), which like it is portrait, takes the
9-tap blur, scans as SUCCESS and decodes."""
import hashlib
import json
import os

import cv2
import numpy as np

from oracle_lib import load_sample

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
BIG = "6bit/4_30_f1_360.jpg x2.8"
GLOB = ["6bit/4_30_802.jpg", "6bit/4_30_f0_177_ccm.jpg", "6bit/4_30_f0_627.jpg", "6bit/4_30_f0_627_extract.jpg",
        BIG, "6bit/4_30_f1_360.jpg", "6bit/4_30_f2_246.jpg", "6bit/4_30_f2_734.jpg"]
_cache = {}


def extra_manifest():
    with open(os.path.join(GOLDEN, "ragged_samples.json")) as f:
        return json.load(f)


def sample(name):
    """a photograph of GLOB (imread + BGR2RGB, as the reference's tests load them)"""
    if name not in _cache:
        extra = extra_manifest()
        if name == BIG:
            _cache[name] = cv2.resize(sample("6bit/4_30_f1_360.jpg"), None, fx=2.8, fy=2.8)
        elif name in extra:
            ent = extra[name]
            img = cv2.imread(os.path.join(GOLDEN, ent["file"]), cv2.IMREAD_COLOR)
            rgb = np.ascontiguousarray(cv2.cvtColor(img, cv2.COLOR_BGR2RGB))
            assert list(rgb.shape) == ent["shape"] and hashlib.sha256(rgb.tobytes()).hexdigest() == ent["rgb_sha256"], name
            _cache[name] = rgb
        else:
            _cache[name] = load_sample(name)
    return _cache[name]
