"""CPU-side checks of the CCM chain (cb200_ccm_chain_*, csrc/chain.cu): argument errors -- null pointers, rank / nranks out of range,
rank >= nranks -- come before any CUDA call; the context is NULL here, so a call whose ranges are good fails on the context.  The refused
mixes (cb200_set_ccm / cb200_fit_ccm on a linked context, a CC_FIT call without a step, a step on a context that is not linked) need a
real context and are checked on the GPU (tests/test_gpu_ccm_chain.py::test_launch_counts_and_refused_mixes): there they return while
a sleeping kernel still holds the context's stream and launch nothing, so they neither wait for the device nor enqueue work.

The prefix rule the chain computes on the device is checked here against the sequential rule of k_ccm_carry (a frame without a fit
keeps the matrix of the frame before it; the oracle's in-order CC_FIT decode): for any cut of the stream into contiguous stripes, the
matrix entering stripe r is the last fit of stripes 0 .. r-1, else the matrix the stream entered with."""
import numpy as np
import pytest

import libcimbar_b200 as cb
from libcimbar_b200 import build as cbbuild
from libcimbar_b200.dist import stripe
from cpu_support import err, lib


@pytest.fixture(scope="module", autouse=True)
def built():
    cbbuild.build()


H = np.zeros(64, np.uint8)


def test_root_create_arguments():
    for nranks in (0, -1, 33):
        err(lib().cb200_ccm_chain_root_create(None, nranks, H.ctypes.data), b"nranks out of range")
    err(lib().cb200_ccm_chain_root_create(None, 2, H.ctypes.data), b"null context")


def test_peer_open_arguments():
    for nranks, rank in ((2, 2), (3, 5), (2, 0), (1, 0), (33, 1), (4, -1)):
        err(lib().cb200_ccm_chain_peer_open(None, nranks, rank, H.ctypes.data), b"out of range")
    err(lib().cb200_ccm_chain_peer_open(None, 2, 1, H.ctypes.data), b"null context")


def test_attach_arguments():
    for rank, nranks in ((2, 2), (3, 2), (-1, 2), (0, 0), (0, 33)):
        err(lib().cb200_ccm_chain_attach(None, rank, nranks), b"out of range")
    err(lib().cb200_ccm_chain_attach(None, 1, 2), b"null context")


def test_step_and_status_arguments():
    err(lib().cb200_ccm_chain_step(None, 0), b"epoch 0")
    err(lib().cb200_ccm_chain_step(None, 1), b"null context")
    err(lib().cb200_ccm_chain_status(None), b"null context")


def test_stripes_cover_the_batch_in_order():
    for n in range(0, 20):
        for world in (1, 2, 3, 5):
            for per in (1, 3, 4, 7):
                got = [stripe(n, r, per) for r in range(world)]
                covered = [i for a, b in got for i in range(a, b)]
                assert covered == list(range(min(n, world * per))), (n, world, per)
                assert all(b - a <= per for a, b in got)


# ------------------------------------------------------------------------------------------------ the prefix rule
def sequential(fits, initial):
    """k_ccm_carry over the whole stream: the matrix every frame decodes with, and the one after the last frame"""
    cur, used = initial, []
    for f in fits:
        if f is not None:
            cur = f
        used.append(cur)
    return used, cur


def chained(fits, initial, bounds):
    """the chain: each stripe publishes its last fit (or none); stripe r enters with the last fit of stripes < r, else `initial`;
    each stripe then runs the sequential rule on its own frames; the step's exit is the last fit of all stripes, else `initial`"""
    published = []
    for a, b in bounds:
        last = [f for f in fits[a:b] if f is not None]
        published.append(last[-1] if last else None)
    used = []
    for r, (a, b) in enumerate(bounds):
        entry = next((p for p in reversed(published[:r]) if p is not None), initial)
        u, _ = sequential(fits[a:b], entry)
        used += u
    exit_ = next((p for p in reversed(published) if p is not None), initial)
    return used, exit_


@pytest.mark.parametrize("seed", range(8))
def test_prefix_rule_equals_the_sequential_carry(seed):
    rng = np.random.default_rng(seed)
    no_fit_stripes = empty_stripes = 0
    for trial in range(300):
        world = int(rng.integers(1, 9))
        per = int(rng.integers(1, 6))
        n = int(rng.integers(0, world * per + 1))                     # short batches: the last stripes short or empty
        p_fit = float(rng.choice([0.0, 0.1, 0.5, 0.9]))
        fits = [int(rng.integers(1, 1 << 30)) if rng.random() < p_fit else None for _ in range(n)]
        bounds = [stripe(n, r, per) for r in range(world)]
        # several steps: each step enters with the previous step's exit, on every rank alike
        state_seq = state_chain = None if rng.random() < 0.5 else -1
        for step in range(3):
            want_used, state_seq = sequential(fits, state_seq)
            got_used, state_chain = chained(fits, state_chain, bounds)
            assert got_used == want_used and state_chain == state_seq, (seed, trial, step)
            fits = fits[::-1]
        no_fit_stripes += sum(1 for a, b in bounds if b > a and all(f is None for f in fits[a:b]))
        empty_stripes += sum(1 for a, b in bounds if b == a)
    assert no_fit_stripes > 50 and empty_stripes > 50                 # premise: both kinds of stripe were exercised
