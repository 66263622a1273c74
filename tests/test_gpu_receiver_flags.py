"""Receiver flags tables (cb200_scan_extract_decode_chunks_receivers_flags_dev, cb200_camera_plan_create_receivers_pictures_flags_dev):
each receiver's sharpen policy and colour correction come from its own word in device memory.  The expected result is the existing
receivers call (cb200_scan_extract_decode_chunks_receivers_dev) on a second context with its own state table, made once per flag
word on the pictures of the receivers with that word, in batch order: records, masks, frame flags, statuses, transforms, frame CCMs
and states, bit for bit.  A receiver with an invalid word gets EXTRACT_REFUSED, mask 0 and a zeroed record, and its state is not
touched.  A uniform table is the existing call with those flags: the fitted-CCM route the table takes decides every colour as K1
does with the receiver's matrix, with or without one."""
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from gpu_support import cb, entries, frames  # noqa: E402,F401  (fixtures)
from gpu_support import Out, RECV, bounds_of, contexts, direct, exact_pictures, fresh, graph_kernel_nodes, pool, rendered  # noqa: E402

MODES = [68, 67, 66, 4]


def mode_pool(cb, mode):
    """photographs and pictures of the mode: the mode-B and 4C pools; for 66 and 67 the rendered frames of the mode (padded, and
    upscaled with a tilt) among the detect tests' mixed pictures, most of which that geometry cannot extract"""
    return pool(mode) if mode in (68, 4) else rendered(cb, mode) + exact_pictures(cb)

S, SN, CS, CF = 0x2, 0x20, 0x4, 0x8
VALID = [s | c for s in (0, S, SN) for c in (0, CS, CF)]       # every valid word
INVALID = [S | SN, CS | CF, 0x1, 0x10, 0x100 | CF, 0x80000000]


def table(words):
    import torch
    return torch.tensor(np.asarray(words, np.int64).astype(np.uint32).view(np.int32), dtype=torch.int32, device="cuda")


def grouped(cb, ref, ts, orders, of, words, ref_states):
    """the existing receivers call once per valid word on its receivers' pictures: records, masks, statuses, frame flags, transforms,
    frame CCMs of the accepted pictures (NaN-filled elsewhere), and which pictures are refused"""
    n = len(ts)
    out = [np.zeros((n, ref.info.data_bytes), np.uint8), np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros(n, np.uint8),
           np.full((n, 3, 3), np.nan), np.full((n, 3, 3), np.nan, np.float32)]
    of = np.asarray(of, np.int64)
    inside = of >= 0
    w = np.array([words[r] if r >= 0 else 0 for r in of], np.int64)
    refused = inside & ~np.isin(w, VALID)
    for word in VALID:
        take = np.flatnonzero(inside & (w == word))
        if len(take) == 0:
            continue
        recs, tf, ccms = direct(cb, ref, [ts[i] for i in take], [orders[i] for i in take], of[take], ref_states, word)
        for k in range(4):
            out[k][take] = recs[k]
        out[4][take] = tf
        out[5][take] = ccms.reshape(len(take), 3, 3)
    return out, refused


def check(cb, got, tf, ccms, want, refused, of):
    of = np.asarray(of, np.int64)
    ok = (of >= 0) & ~refused
    for k in range(4):
        assert np.array_equal(got[k][ok], want[k][ok]), k
    assert np.array_equal(tf[ok], want[4][ok])
    assert np.array_equal(ccms.reshape(-1, 3, 3)[ok], want[5][ok], equal_nan=True)
    assert (got[1][refused] == 0).all() and (got[2][refused] == cb.EXTRACT_REFUSED).all() and (got[0][refused] == 0).all()
    empty = of < 0
    assert (got[1][empty] == 0).all() and (got[2][empty] == cb.EXTRACT_EMPTY).all()


def call(cb, ctx, ts, orders, of, states, words):
    import torch
    n = len(ts)
    chunks = torch.full((n, ctx.info.data_bytes), 0xA5, dtype=torch.uint8, device="cuda")
    mask = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    status = torch.full((n,), 7, dtype=torch.int32, device="cuda")
    ff = torch.full((n,), 0xEE, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    ctx.scan_extract_decode_chunks_receivers_dev(ts, np.asarray(of, np.int32), states, chunks.data_ptr(), mask.data_ptr(), status.data_ptr(),
                                                 ff.data_ptr(), order=orders, receiver_flags=words)
    ctx.sync()
    return [t.cpu().numpy() for t in (chunks, mask, status, ff)], ctx.camera_transforms(n), ctx.frame_ccms(n)


@pytest.mark.parametrize("mode", MODES)
def test_mixed_words_equal_one_existing_call_per_word(cb, entries, mode):
    """every valid word and two invalid ones in each batch, receivers interleaved, three batches back to back; a guard receiver that
    never has a picture.  The context's own CCM is neither read nor changed"""
    import torch
    p = mode_pool(cb, mode)
    receivers = len(VALID) + 3
    words = VALID + [S | SN, 0x100, 0]                       # the last receiver (word 0) never has a picture
    ents = [entries[i % 4] for i in range(receivers)]
    ctx, ref = cb.Context(mode, max_frames=24), cb.Context(mode, max_frames=24)
    states, ref_states = cb.receiver_states(ents), cb.receiver_states(ents)
    before = states.clone()
    d_words = table(words)
    own = np.array([[1.25, 0.0, 0.0], [0.0, 0.75, 0.0], [0.0, 0.0, 1.5]], np.float32)
    ctx.set_ccm(own)
    rng = np.random.default_rng(mode)
    for batch in range(3):
        n = 16 + 4 * batch
        pick = rng.integers(0, len(p), n)
        ts, orders = fresh([p[i] for i in pick], rng)
        of = np.concatenate([np.arange(receivers - 1), rng.integers(0, receivers - 1, n - (receivers - 1))])
        rng.shuffle(of)
        got, tf, ccms = call(cb, ctx, ts, orders, of, states, d_words)
        want, refused = grouped(cb, ref, ts, orders, of, words, ref_states)
        assert refused.any() and (~refused).any()
        check(cb, got, tf, ccms, want, refused, of)
        assert torch.equal(states, ref_states)
    raw, raw0 = states.view(torch.int32).reshape(-1, 10), before.view(torch.int32).reshape(-1, 10)
    for r in (len(VALID), len(VALID) + 1, len(VALID) + 2):   # refused and absent receivers: untouched
        assert torch.equal(raw[r], raw0[r])
    assert np.array_equal(ctx.get_ccm(), own)
    ctx.close()
    ref.close()


@pytest.mark.parametrize("word", VALID)
@pytest.mark.parametrize("mode", MODES)
def test_uniform_table_is_the_existing_call(cb, entries, mode, word):
    """every receiver with the same word: the existing call with those flags on the whole batch, two batches back to back"""
    import torch
    p = mode_pool(cb, mode)
    receivers = 4
    ctx, ref = cb.Context(mode, max_frames=12), cb.Context(mode, max_frames=12)
    states, ref_states = cb.receiver_states(entries[:receivers]), cb.receiver_states(entries[:receivers])
    rng = np.random.default_rng(word + 7 * mode)
    for _ in range(2):
        n = 12
        ts, orders = fresh([p[i] for i in rng.integers(0, len(p), n)], rng)
        of = rng.integers(0, receivers, n)
        got, tf, ccms = call(cb, ctx, ts, orders, of, states, table([word] * receivers))
        recs, wtf, wccms = direct(cb, ref, ts, orders, of, ref_states, word)
        for k in range(4):
            assert np.array_equal(got[k], recs[k]), k
        assert np.array_equal(tf, wtf) and np.array_equal(ccms, wccms, equal_nan=True)
        assert torch.equal(states, ref_states)
    ctx.close()
    ref.close()


def test_bad_words_and_flags_refused_on_a_context(cb, entries):
    import torch
    ctx = cb.Context(68, max_frames=4)
    states = cb.receiver_states(entries[:2])
    t = torch.zeros((1200, 1600, 3), dtype=torch.uint8, device="cuda")
    buf = torch.zeros(16, dtype=torch.int32, device="cuda")
    with pytest.raises(cb.Cb200Error, match="per-receiver bit"):
        ctx.scan_extract_decode_chunks_receivers_dev([t], np.zeros(1, np.int32), states, buf.data_ptr(), buf.data_ptr(), buf.data_ptr(),
                                                     flags=cb.FLAG_CC_FIT, receiver_flags=table([0, 0]))
    with pytest.raises(cb.Cb200Error, match="receiver_flags"):
        ctx.scan_extract_decode_chunks_receivers_dev([t], np.zeros(1, np.int32), states, buf.data_ptr(), buf.data_ptr(), buf.data_ptr(),
                                                     receiver_flags=table([0, 0, 0]))
    ctx.close()


def test_plan_over_launches_equals_direct_and_grouped_calls(cb, entries):
    """a plan over device descriptors with a flags table: the table, the map and the descriptors change between launches; every
    launch equals the direct flags call and the grouped existing calls; a launch is one graph launch, and the plan runs inside an outer
    torch graph"""
    import torch
    mode = 68
    p = pool(mode)
    n, receivers = 12, 8
    bounds = bounds_of(p)
    ents = [entries[i % 4] for i in range(receivers)]
    ctx, dref, ref = (cb.Context(mode, max_frames=n) for _ in range(3))
    states, dstates, ref_states = (cb.receiver_states(ents) for _ in range(3))
    d_pics = torch.zeros((n, 40), dtype=torch.uint8, device="cuda")
    of_t = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    words_t = table([0] * receivers)
    chunks = torch.full((n, ctx.info.data_bytes), 0xA5, dtype=torch.uint8, device="cuda")
    mask = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    status = torch.full((n,), 7, dtype=torch.int32, device="cuda")
    ff = torch.full((n,), 0xEE, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    plan = ctx.receivers_camera_plan_pictures_dev(d_pics, bounds, of_t, states, chunks.data_ptr(), mask.data_ptr(), status.data_ptr(),
                                                  ff.data_ptr(), receiver_flags=words_t)
    rng = np.random.default_rng(5)
    keep = []
    outer = None
    for k in range(5):
        ts, orders = fresh([p[i] for i in rng.integers(0, len(p), n)], rng)
        keep.append(ts)
        of = rng.integers(0, receivers, n)
        if k >= 2:
            of[rng.choice(n, 2, replace=False)] = -1
        words = [VALID[int(i)] for i in rng.integers(0, len(VALID), receivers)]
        words[int(rng.integers(receivers))] = INVALID[k % len(INVALID)]
        d_pics.copy_(torch.from_numpy(np.ascontiguousarray(cb.picture_descriptors(ts, orders))))
        of_t.copy_(torch.from_numpy(of.astype(np.int32)))
        words_t.copy_(table(words))
        torch.cuda.synchronize()
        if k < 4:
            before = cb.launch_count()
            plan.launch()
            assert cb.launch_count() - before == graph_kernel_nodes(plan.graph)
        else:                                                # replayed from an outer torch graph
            s = torch.cuda.Stream()
            ctx.set_stream(s.cuda_stream)
            outer = torch.cuda.CUDAGraph()
            with torch.cuda.graph(outer, stream=s):
                plan.launch()
            ctx.set_stream(None)
            outer.replay()
        ctx.sync()
        torch.cuda.synchronize()
        got = [t.cpu().numpy() for t in (chunks, mask, status, ff)]
        take = np.flatnonzero(of >= 0)
        dgot, dtf, dccms = call(cb, dref, [ts[i] for i in take], [orders[i] for i in take], of[take], dstates, table(words))
        for j in range(4):
            assert np.array_equal(got[j][take], dgot[j]), (k, j)
        if k < 4:
            assert np.array_equal(ctx.camera_transforms(n)[take], dtf)
            assert np.array_equal(ctx.frame_ccms(n)[take], dccms, equal_nan=True)
        want, refused = grouped(cb, ref, [ts[i] for i in take], [orders[i] for i in take], of[take], words, ref_states)
        check(cb, dgot, dtf, dccms, want, refused, of[take])
        assert (got[1][of < 0] == 0).all() and (got[2][of < 0] == cb.EXTRACT_EMPTY).all()
        assert torch.equal(states, dstates) and torch.equal(states, ref_states)
    plan.close()
    for c in (ctx, dref, ref):
        c.close()


# ------------------------------------------------------------------------------------------------ the detect forms
def detect_grouped(cb, refs, ts, orders, of, cand, words, tables):
    """one existing detect receivers call per valid word on its receivers' pictures, scattered back: chunks, masks, statuses, modes,
    mode masks; and which pictures are refused"""
    n, K = len(ts), len(refs)
    slot = max(c.info.data_bytes for c in refs)
    out = [np.zeros((n, slot), np.uint8), np.zeros(n, np.uint32), np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros((n, K), np.uint32)]
    of = np.asarray(of, np.int64)
    w = np.array([words[r] for r in of], np.int64)
    for word in VALID:
        take = np.flatnonzero(w == word)
        if len(take) == 0:
            continue
        got = run_detect(cb, refs, [ts[i] for i in take], [orders[i] for i in take], of[take], tables, np.asarray(cand)[take], word, None)
        for k in range(5):
            out[k][take] = got[k]
    return out, ~np.isin(w, VALID)


def run_detect(cb, ctxs, ts, orders, of, tables, cand, flags, words):
    import torch
    out = Out(ctxs, len(ts))
    torch.cuda.synchronize()
    cb.detect_scan_extract_decode_chunks_receivers_dev(ctxs, ts, np.asarray(of, np.int32), tables, out.chunks.data_ptr(), out.mask.data_ptr(),
                                                       out.status.data_ptr(), out.mode.data_ptr(), candidates=cand,
                                                       d_mode_masks=out.mode_masks.data_ptr(), flags=flags, order=orders,
                                                       receiver_flags=words)
    ctxs[0].sync()
    return out.host()


def check_detect(cb, got, want, refused, inside=None):
    ok = ~refused if inside is None else inside & ~refused
    for k in range(5):
        assert np.array_equal(got[k][ok], want[k][ok]), k
    assert (got[1][refused] == 0).all() and (got[2][refused] == cb.EXTRACT_REFUSED).all() and (got[3][refused] == -1).all()
    assert not got[0][refused].any() and not got[4][refused].any()


def detect_words(rng, receivers):
    words = [VALID[int(i)] for i in rng.integers(0, len(VALID), receivers)]
    words[1] = S | SN
    words[2] = 0x40 | CF
    return words


def test_detect_mixed_candidates_and_words(cb, entries):
    """auto sessions (every mode) and sessions locked to one mode, with mixed words, three batches back to back, against one existing
    detect receivers call per word on fresh contexts and tables"""
    import torch
    pics = exact_pictures(cb)
    n, receivers, K = 2 * len(pics), 10, len(RECV)
    ctxs, refs = contexts(cb, RECV, n), contexts(cb, RECV, n)
    ents = [entries[i % 4] for i in range(receivers)]
    tables, ref_tables = [cb.receiver_states(ents) for _ in RECV], [cb.receiver_states(ents) for _ in RECV]
    before = [t.clone() for t in tables]
    rng = np.random.default_rng(21)
    locks = [(1 << K) - 1 if r % 3 == 0 else 1 << (r % K) for r in range(receivers)]
    try:
        for batch in range(3):
            words = detect_words(rng, receivers)
            d_words = table(words)
            order = rng.permutation(n)
            ts, orders = fresh([pics[i % len(pics)] for i in order], rng)
            of = rng.integers(0, receivers, n)
            of[:receivers] = np.arange(receivers)
            rng.shuffle(of)
            cand = np.array([locks[r] for r in of], np.uint32)
            got = run_detect(cb, ctxs, ts, orders, of, tables, cand, 0, d_words)
            want, refused = detect_grouped(cb, refs, ts, orders, of, cand, words, ref_tables)
            assert refused.any() and (got[3] >= 0).any()
            check_detect(cb, got, want, refused)
            for t, u in zip(tables, ref_tables):
                assert torch.equal(t, u)
        for t, t0 in zip(tables, before):                 # the refused receivers' rows are untouched in every mode
            assert torch.equal(t.view(torch.int32).reshape(-1, 10)[1:3], t0.view(torch.int32).reshape(-1, 10)[1:3])
    finally:
        for c in ctxs + refs:
            c.close()


def test_detect_plan_over_launches(cb, entries):
    """the detect plan over device descriptors with a flags table: the table, the map, the candidates and the descriptors change
    between launches; each launch equals the grouped existing detect receivers calls, empty slots included; one graph launch"""
    import torch
    pics = exact_pictures(cb)
    n, receivers, K = len(pics), 8, len(RECV)
    ctxs, refs = contexts(cb, RECV, n), contexts(cb, RECV, n)
    ents = [entries[i % 4] for i in range(receivers)]
    tables, ref_tables = [cb.receiver_states(ents) for _ in RECV], [cb.receiver_states(ents) for _ in RECV]
    d_pics = torch.zeros((n, 40), dtype=torch.uint8, device="cuda")
    of_t = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    cand_t = torch.zeros(n, dtype=torch.int32, device="cuda")
    words_t = table([0] * receivers)
    out = Out(ctxs, n)
    torch.cuda.synchronize()
    bounds = bounds_of(pics)
    plan = cb.detect_receivers_camera_plan_pictures_dev(ctxs, d_pics, bounds, cand_t, of_t, tables, out.chunks.data_ptr(), out.mask.data_ptr(),
                                                        out.status.data_ptr(), out.mode.data_ptr(), out.mode_masks.data_ptr(),
                                                        receiver_flags=words_t)
    rng = np.random.default_rng(33)
    keep = []
    try:
        for k in range(4):
            ts, orders = fresh([pics[i] for i in rng.permutation(n)], rng)
            keep.append(ts)
            of = rng.integers(0, receivers, n)
            of[rng.choice(n, 2, replace=False)] = -1
            cand = np.where(rng.random(n) < 0.5, (1 << K) - 1, 1 << rng.integers(0, K, n)).astype(np.uint32)
            words = detect_words(rng, receivers)
            d_pics.copy_(torch.from_numpy(np.ascontiguousarray(cb.picture_descriptors(ts, orders))))
            of_t.copy_(torch.from_numpy(of.astype(np.int32)))
            cand_t.copy_(torch.from_numpy(cand.view(np.int32)))
            words_t.copy_(table(words))
            torch.cuda.synchronize()
            before = cb.launch_count()
            plan.launch()
            assert cb.launch_count() - before == graph_kernel_nodes(plan.graph)
            ctxs[0].sync()
            torch.cuda.synchronize()
            got = out.host()
            inside = of >= 0
            take = np.flatnonzero(inside)
            want, refused = detect_grouped(cb, refs, [ts[i] for i in take], [orders[i] for i in take], of[take], cand[take], words, ref_tables)
            check_detect(cb, [g[take] for g in got], want, refused)
            assert (got[2][~inside] == cb.EXTRACT_EMPTY).all() and (got[3][~inside] == -1).all() and (got[1][~inside] == 0).all()
            for t, u in zip(tables, ref_tables):
                assert torch.equal(t, u)
    finally:
        plan.close()
        for c in ctxs + refs:
            c.close()
