"""The auto mode for receivers (cb200_detect_scan_extract_decode_chunks_receivers_dev): each picture is decoded under its candidate
modes, each mode with its own table of receiver states.  The expected result is always what a service gets without the call: for
every mode k, one cb200_scan_extract_decode_chunks_receivers_dev on a fresh context of that mode over P_k (the pictures with
candidate bit k, in batch order) with mode k's table; then the detect call's selection over those results, in numpy.
  - exactness under every flag combination of the detect tests, for one mode, two modes of one geometry and all three geometries,
    with random candidate masks and receiver maps over two calls (the states carry);
  - n_modes = 1 with every bit is the receivers call bit for bit; candidates = NULL with one receiver is the detect call;
  - the session flow (auto, lock on d_mode, locked) matches the per-mode calls; a batch locked to one geometry deskews and walks
    once, auto pictures are walked by every geometry; receivers without pictures keep their entries byte for byte;
  - a picture that fails extraction gets -1 and its first candidate's status."""
import numpy as np
import pytest

from gpu_support import cb  # noqa: F401  (fixtures)
from gpu_support import FLAGS, Out, RECV, camera_call, close, contexts, detect, entry_states, exact_pictures, layouts, run

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pool(cb):
    """mixed mode-B / 4C photographs, rendered 66 and 67 frames with pasted anchors and a noise picture, in mixed layouts"""
    pics = exact_pictures(cb)
    ts, orders = layouts(pics)
    return ts, orders


def per_mode(cb, refs, ts, orders, of, tables, cand, flags):
    """the direct receivers call of every mode k over P_k with table k (updated in place): (P_k, chunks, masks, statuses)"""
    of = np.asarray(of, np.int32)
    out = []
    for k, (ref, table) in enumerate(zip(refs, tables)):
        idx = np.flatnonzero(np.asarray(cand, np.uint32) >> np.uint32(k) & np.uint32(1))
        if not len(idx):
            out.append((idx, None, None, None))
            continue
        chunks, mask, status, _, _ = camera_call(cb, ref, [ts[i] for i in idx], [orders[i] for i in idx], flags, of[idx], table)
        out.append((idx, chunks, mask.view(np.uint32), status))
    return out


def check_selected(ctxs, got, want):
    """the detect call's selection in numpy over the per-mode results"""
    chunks, mask, status, mode, mode_masks = got
    K = len(ctxs)
    for i in range(len(mode)):
        at = {k: int(np.searchsorted(want[k][0], i)) for k in range(K) if i in set(want[k][0].tolist())}
        masks = [int(want[k][2][at[k]]) if k in at else 0 for k in range(K)]
        assert mode_masks[i].tolist() == masks, i
        first = next((k for k in range(K) if k in at and masks[k]), -1)
        assert mode[i] == first, i
        k = first if first >= 0 else min(at)
        assert status[i] == want[k][3][at[k]], i
        if first < 0:
            assert mask[i] == 0 and not chunks[i].any(), i
            continue
        db = ctxs[first].info.data_bytes
        assert mask[i] == masks[first], i
        assert np.array_equal(chunks[i, :db], want[first][1][at[first]]), i
        assert not chunks[i, db:].any(), i


def same_tables(a, b):
    import torch
    return all(torch.equal(x, y) for x, y in zip(a, b))


# ------------------------------------------------------------------------------------------------ exactness
SETS = {"one-mode": [68], "one-geometry": [68, 4], "three-geometries": RECV}


@pytest.mark.parametrize("modes", list(SETS))
@pytest.mark.parametrize("sflag,ccflag", FLAGS)
def test_each_mode_equals_its_receivers_call(cb, pool, modes, sflag, ccflag):
    modes = SETS[modes]
    flags = (getattr(cb, "FLAG_" + sflag) if sflag else 0) | (getattr(cb, "FLAG_" + ccflag) if ccflag else 0)
    ts, orders = pool
    n, K, R = len(ts), len(modes), 5
    rng = np.random.default_rng(len(modes) * 100 + flags)
    ctxs = contexts(cb, modes, n)
    refs = [cb.Context(m, max_frames=n) for m in modes]
    try:
        entries = entry_states(R, flags + K)
        states = [cb.receiver_states(entries) for _ in modes]
        tables = [s.clone() for s in states]
        decoded = 0
        for call in range(2):                                   # two calls: every table carries from the first into the second
            perm = rng.permutation(n) if call else np.arange(n)
            bts, bord = [ts[i] for i in perm], [orders[i] for i in perm]
            of = rng.integers(0, R - 1, n).astype(np.int32)     # receiver R - 1 never has a picture
            cand = rng.integers(1, 1 << K, n).astype(np.uint32)
            got = run(cb, ctxs, bts, bord, of, states, cand, flags)
            want = per_mode(cb, refs, bts, bord, of, tables, cand, flags)
            check_selected(ctxs, got, want)
            assert same_tables(states, tables)
            decoded += int((got[3] >= 0).sum())
        assert decoded > 0                                      # premise: pictures decode
        for s in states:                                        # the receiver without pictures, byte for byte
            assert np.array_equal(s.cpu().numpy().reshape(R, 10)[R - 1], cb.receiver_states(entries).cpu().numpy().reshape(R, 10)[R - 1])
        for c in ctxs:
            assert c.get_ccm() is None                          # no context's own CCM is read or changed
    finally:
        close(ctxs, refs)


# ------------------------------------------------------------------------------------------------ degenerate cases
@pytest.mark.parametrize("mode", [68, 4])
@pytest.mark.parametrize("flags", ["", "CC_SIMPLE", "SHARPEN_IF_NEEDED|CC_FIT", "SHARPEN|CC_FIT"])
def test_one_mode_is_the_receivers_call(cb, pool, mode, flags):
    import torch
    flags = sum(getattr(cb, "FLAG_" + f) for f in flags.split("|") if f)
    ts, orders = pool
    n = len(ts)
    of = np.array([i % 3 for i in range(n)], np.int32)
    entries = entry_states(3, 7)
    ctx, ref = contexts(cb, [mode], n)[0], cb.Context(mode, max_frames=n)
    try:
        states, table = cb.receiver_states(entries), cb.receiver_states(entries)
        torch.cuda.synchronize()
        before = cb.launch_count()
        chunks, mask, status, ff, _ = camera_call(cb, ref, ts, orders, flags, of, table)
        direct = cb.launch_count() - before
        before = cb.launch_count()
        got = run(cb, [ctx], ts, orders, of, [states], np.ones(n, np.uint32), flags)
        assert cb.launch_count() - before == direct + 1        # the receivers call's launches, then the selection
        assert np.array_equal(got[0], chunks) and np.array_equal(got[1], mask.view(np.uint32)) and np.array_equal(got[2], status)
        assert np.array_equal(got[3], np.where(mask != 0, 0, -1)) and np.array_equal(got[4][:, 0], mask.view(np.uint32))
        assert torch.equal(states, table)
        assert (mask != 0).any()
    finally:
        close([ctx, ref])


@pytest.mark.parametrize("flags", ["SHARPEN_IF_NEEDED", "SHARPEN_IF_NEEDED|CC_FIT", "SHARPEN|CC_SIMPLE"])
def test_null_candidates_and_one_receiver_is_the_detect_call(cb, pool, flags):
    """every picture under every mode for one receiver whose entry state is each context's CCM: the detect call's outputs, and each
    table ends at its context's CCM"""
    flags = sum(getattr(cb, "FLAG_" + f) for f in flags.split("|"))
    ts, orders = pool
    pics = exact_pictures(cb)                                   # the pool's pictures, packed RGB for the detect call
    n = len(pics)
    entry = entry_states(2, 11)[1]
    ctxs, dets = contexts(cb, RECV, n), contexts(cb, RECV, n)
    try:
        for c in dets:
            c.set_ccm(entry)
        states = [cb.receiver_states([entry]) for _ in RECV]
        want = detect(cb, dets, pics, flags)
        got = run(cb, ctxs, ts, orders, np.zeros(n, np.int32), states, None, flags)
        for a, b, what in zip(got, want, ["chunks", "mask", "status", "mode", "mode masks"]):
            assert np.array_equal(a, b), what
        for c, s in zip(dets, states):
            st = cb.read_receiver_states(s)[0]
            m = c.get_ccm()
            assert (st is None) == (m is None) and (m is None or np.array_equal(st, m)), c.info.mode_val
        assert (got[3] >= 0).any() and (got[3] < 0).any()
    finally:
        close(ctxs, dets)


# ------------------------------------------------------------------------------------------------ premises
def kernels(cb, fn, names):
    """how many kernels whose name contains each of `names` fn() launches (torch.profiler)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    evs = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    return {k: sum(k in e for e in evs) for k in names}


def test_session_flow_locks_on_the_detected_mode(cb, pool):
    """auto batch, each receiver locked to the mode its first decoded picture gave, then a locked batch: each matches the per-mode
    calls; the locked batch walks one geometry per locked mode's geometry only, the auto batch all three"""
    ts, orders = pool
    n, R = len(ts), 4
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    of = np.array([i % R for i in range(n)], np.int32)
    ctxs = contexts(cb, RECV, n)
    refs = [cb.Context(m, max_frames=n) for m in RECV]
    try:
        entries = entry_states(R, 21)
        states = [cb.receiver_states(entries) for _ in RECV]
        tables = [s.clone() for s in states]
        auto = np.full(n, (1 << len(RECV)) - 1, np.uint32)
        got = run(cb, ctxs, ts, orders, of, states, auto, flags)
        check_selected(ctxs, got, per_mode(cb, refs, ts, orders, of, tables, auto, flags))
        assert same_tables(states, tables)
        lock = {}
        for i in range(n):
            if got[3][i] >= 0 and of[i] not in lock:
                lock[int(of[i])] = int(got[3][i])
        assert len(lock) >= 2                                       # premise: sessions lock
        locked = np.array([1 << lock[r] if r in lock else auto[0] for r in of], np.uint32)
        got = run(cb, ctxs, ts, orders, of, states, locked, flags)
        check_selected(ctxs, got, per_mode(cb, refs, ts, orders, of, tables, locked, flags))
        assert same_tables(states, tables)
        # walks and deskews: the auto pictures are walked by every geometry, a batch locked to 68 by one
        out = Out(ctxs, n)
        for _ in range(2):
            out.call(cb, ctxs, ts, orders, of, states, auto, flags)
        ctxs[0].sync()
        names = ["k_flood_walk", "k_deskew", "k_extract"]
        c = kernels(cb, lambda: (out.call(cb, ctxs, ts, orders, of, states, auto, flags), ctxs[0].sync()), names)
        assert c == {"k_flood_walk": 3, "k_deskew": 3, "k_extract": 4}, c
        only68 = np.full(n, 1 << RECV.index(68), np.uint32)
        c = kernels(cb, lambda: (out.call(cb, ctxs, ts, orders, of, states, only68, flags), ctxs[0].sync()), names)
        assert c == {"k_flood_walk": 1, "k_deskew": 1, "k_extract": 1}, c
        b_and_4c = np.full(n, (1 << RECV.index(68)) | (1 << RECV.index(4)), np.uint32)
        c = kernels(cb, lambda: (out.call(cb, ctxs, ts, orders, of, states, b_and_4c, flags), ctxs[0].sync()), names)
        assert c == {"k_flood_walk": 1, "k_deskew": 1, "k_extract": 2}, c
    finally:
        close(ctxs, refs)


def test_untouched_receivers_and_failed_pictures(cb, pool):
    """mode k's receivers without a picture in P_k keep their entries byte for byte (poisoned entries included); the noise picture
    gets mode -1 and the status under its first candidate"""
    import torch
    ts, orders = pool
    n, K, R = len(ts), len(RECV), 6
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    ctxs = contexts(cb, RECV, n)
    try:
        of = np.array([i % 3 for i in range(n)], np.int32)       # receivers 3 .. 5 have no picture
        cand = np.array([(1 << (i % K)) | (1 << ((i + 2) % K)) for i in range(n)], np.uint32)
        states = [cb.receiver_states(entry_states(R, 30 + k)) for k in range(K)]
        for s in states:
            s.view(torch.int32).reshape(-1, 10)[4] = torch.tensor([0x7FC00001] * 9 + [0xDEAD], dtype=torch.int32, device="cuda")
        before = [s.clone() for s in states]
        got = run(cb, ctxs, ts, orders, of, states, cand, flags)
        for k in range(K):
            have = {int(of[i]) for i in range(n) if cand[i] >> k & 1}
            rows, was = states[k].reshape(R, 10), before[k].reshape(R, 10)
            for r in range(R):
                if r not in have:
                    assert torch.equal(rows[r], was[r]), (k, r)
        refs = [cb.Context(m, max_frames=n) for m in RECV]
        try:
            want = per_mode(cb, refs, ts, orders, of, [b.clone() for b in before], cand, flags)
        finally:
            close(refs)
        failed = [i for i in range(n) if all(want[k][3][np.searchsorted(want[k][0], i)] <= 0 for k in range(K) if cand[i] >> k & 1)]
        assert failed                                            # premise: the noise picture fails extraction
        for i in failed:
            first = next(k for k in range(K) if cand[i] >> k & 1)
            assert got[3][i] == -1 and got[1][i] == 0, i
            assert got[2][i] == want[first][3][np.searchsorted(want[first][0], i)], i
    finally:
        close(ctxs)
