"""Inputs and reporting shared by the feature bench scripts (`python -m libcimbar_b200.<name>_bench`): the picture pools they time,
the card a number was measured on, and the CUDA-event timing loop of the JPEG and PNG benches."""
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GLOB = ["4_30_802", "4_30_f0_177_ccm", "4_30_f0_627", "4_30_f0_627_extract", None, "4_30_f1_360", "4_30_f2_246", "4_30_f2_734"]


def load_pictures():
    import cv2

    def load(name):
        img = cv2.imread(os.path.join(ROOT, "tests", "golden", "6bit__%s.jpg" % name), cv2.IMREAD_COLOR)
        return np.ascontiguousarray(cv2.cvtColor(img, cv2.COLOR_BGR2RGB))
    return [load(n) if n else cv2.resize(load("4_30_f1_360"), None, fx=2.8, fy=2.8) for n in GLOB]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in q.split(",")]
        return name, power
    except Exception as e:          # the numbers are reported without it, never estimated
        return "unknown (%s)" % e, "unknown"


def photographs():
    import cv2
    out = []
    for name in ("b__ex2434.jpg", "b__ex380.jpg"):
        img = cv2.imread(os.path.join(ROOT, "tests", "golden", name), cv2.IMREAD_COLOR)
        out.append(np.ascontiguousarray(cv2.cvtColor(img, cv2.COLOR_BGR2RGB)))
    return out


def entry_states(D):
    """distinct active matrices: a mild cast that differs per receiver"""
    out = []
    for r in range(D):
        g = 1.0 + 0.002 * (r % 50)
        out.append(np.diag([g, 1.0, 2.0 - g]).astype(np.float32))
    return out


MODES = [66, 68, 67, 4]


def candidates(mix, D):
    """per receiver: its candidate bits"""
    auto = (1 << len(MODES)) - 1
    locked = [1 << MODES.index(68 if r % 2 == 0 else 4) for r in range(D)]
    if mix == "auto":
        return [auto] * D
    if mix == "locked":
        return locked
    return [auto if r % 10 == 0 else locked[r] for r in range(D)]


def timed(fn, rounds, stream):
    """best and all of `rounds` runs of fn, CUDA events on the context's stream around it (host work inside the call included)"""
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms = []
    for _ in range(rounds):
        torch.cuda.synchronize()
        e0.record(stream)
        fn()
        e1.record(stream)
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return min(ms), ms
