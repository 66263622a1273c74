"""The word rules of a receiver flags table (libcimbar_b200/csrc/receivers_core.cuh), compiled for the host, against a restatement of
the contract in include/cb200.h: a word is refused when it holds a bit other than SHARPEN, SHARPEN_IF_NEEDED, CC_SIMPLE and CC_FIT, or
both bits of one pair; a valid word sharpens a picture as the call with those flags does (SHARPEN always, SHARPEN_IF_NEEDED at
extract status 2); and it keeps its receiver's CCM unchanged without a CC bit, or with CC_FIT in a mode that never fits.  All 64
values of the six flag bits, and 100 000 random 32-bit words."""
import ctypes as C

import numpy as np
import pytest

import libcimbar_b200 as cb
from host_harness import build_harness

PER_RECEIVER = cb.FLAG_SHARPEN | cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_SIMPLE | cb.FLAG_CC_FIT


@pytest.fixture(scope="module")
def core(tmp_path_factory):
    lib = build_harness(tmp_path_factory, "receiver_flags_host")
    lib.rf_rules.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    return lib


def restated(w):
    refused = (w & ~PER_RECEIVER) != 0 or (w & cb.FLAG_SHARPEN and w & cb.FLAG_SHARPEN_IF_NEEDED) or \
        (w & cb.FLAG_CC_SIMPLE and w & cb.FLAG_CC_FIT)
    sharpen2 = bool(w & (cb.FLAG_SHARPEN | cb.FLAG_SHARPEN_IF_NEEDED))
    sharpen1 = bool(w & cb.FLAG_SHARPEN)
    passes_fit = not (w & (cb.FLAG_CC_SIMPLE | cb.FLAG_CC_FIT))
    passes_nofit = not (w & cb.FLAG_CC_SIMPLE)
    return int(bool(refused)) | sharpen2 << 1 | sharpen1 << 2 | passes_fit << 3 | passes_nofit << 4


def run(core, words):
    words = np.ascontiguousarray(words, np.uint32)
    out = np.zeros(len(words), np.uint8)
    core.rf_rules(words.ctypes.data, len(words), out.ctypes.data)
    return out


def test_every_value_of_the_six_flag_bits(core):
    bits = [cb.FLAG_NO_FALLBACK, cb.FLAG_SHARPEN, cb.FLAG_CC_SIMPLE, cb.FLAG_CC_FIT, cb.FLAG_NO_INTERLEAVE, cb.FLAG_SHARPEN_IF_NEEDED]
    assert sorted(bits) == [1 << k for k in range(6)]
    words = np.arange(64, dtype=np.uint32)
    got = run(core, words)
    assert [int(v) for v in got] == [restated(int(w)) for w in words]
    valid = [int(w) for w in words if not got[w] & 1]
    # exactly the nine combinations {none, SHARPEN, SHARPEN_IF_NEEDED} x {none, CC_SIMPLE, CC_FIT} are valid
    assert len(valid) == 9 and all(w & ~PER_RECEIVER == 0 for w in valid)


def test_random_words(core):
    rng = np.random.default_rng(11)
    words = rng.integers(0, 2 ** 32, 100_000, dtype=np.uint64).astype(np.uint32)
    words[:64] = np.arange(64, dtype=np.uint32) | np.uint32(0x80000000)          # a high bit on every flag combination
    got = run(core, words)
    assert [int(v) for v in got] == [restated(int(w)) for w in words]
    assert got[:64].min() & 1
