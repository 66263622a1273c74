"""The grouped history call (cb200_scan_extract_decode_chunks_grouped_history_dev) on the GPU, in modes 68, 67, 66, 4 and 8.

A sequence of batches of sizes 1, 2 and mixed goes through one context with a history, while a twin context takes the same batches
through cb200_scan_extract_decode_chunks_pictures_dev.  Per call the per-picture outputs must be the twin's bit for bit; group_of,
the count and the history's tags must be tests/history_fixtures.history_rule on the oracle's cells (under CC_FIT the fitted cells of
one decoder over the whole sequence); slots [0, count) the oracle's decode of the vote over the members, and without CC_FIT also the
combined call's on a third context given the member pictures again; the slots past the count zero."""
import numpy as np
import pytest

from combine_fixtures import ORA, clean_picture, fitted_cells, group_expectation, picture_cells
from group_fixtures import capture_of, frame_captures, match_matrix, seeded_frame
from history_fixtures import history_rule
from gpu_support import cb  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

MODES = [68, 67, 66, 4, 8]
FLAGS = ["none", "SHARPEN_IF_NEEDED", "CC_SIMPLE", "CC_FIT"]


def flag_bits(cb, name):
    return 0 if name == "none" else getattr(cb, "FLAG_" + name)


def noise():
    return np.random.default_rng(7).integers(0, 256, (700, 900, 3), dtype=np.uint8)


_sequences = {}


def sequence(mode_val):
    """captures of four seeded frames (2, 3, 2 and 1 of them), a noise picture and the clean picture, in batches of 1, 2, 1, 3, 1
    and 2 pictures: frames A and B are split across calls, D is a lone capture"""
    if mode_val not in _sequences:
        pics, _ = frame_captures(mode_val, [2, 3, 2, 1], seed=5)
        a, b, c, d = pics[0:2], pics[2:5], pics[5:7], pics[7:8]
        _sequences[mode_val] = [[a[0]], [a[1], b[0]], [b[1]], [noise(), b[2], c[0]], [clean_picture(mode_val)], [c[1], d[0]]]
    return _sequences[mode_val]


def tensors(pics):
    import torch
    return [torch.from_numpy(np.ascontiguousarray(p)).cuda() for p in pics]


class Out:
    def __init__(self, ctx, n, m):
        import torch
        db = ctx.info.data_bytes
        z = lambda shape, v, dt: torch.full(shape, v, dtype=dt, device="cuda")
        self.chunks, self.mask = z((max(n, 1), db), 0xA5, torch.uint8), z((max(n, 1),), -1, torch.int32)
        self.status, self.flags = z((max(n, 1),), 7, torch.int32), z((max(n, 1),), 0xEE, torch.uint8)
        self.gchunks, self.gmask = z((max(m, 1), db), 0x5A, torch.uint8), z((max(m, 1),), -1, torch.int32)
        self.gused, self.gof, self.count = z((max(m, 1),), 9, torch.int32), z((max(n, 1),), -9, torch.int32), z((1,), -9, torch.int32)
        self.n, self.m = n, m

    def pictures(self, ctx, d, flags):
        ctx.scan_extract_decode_chunks_pictures_dev(d, self.chunks.data_ptr(), self.mask.data_ptr(), self.status.data_ptr(),
                                                    self.flags.data_ptr(), flags=flags)

    def history(self, ctx, hist, d, flags):
        ctx.scan_extract_decode_chunks_grouped_history_dev(d, hist, self.chunks.data_ptr(), self.mask.data_ptr(), self.status.data_ptr(),
                                                           self.gof.data_ptr(), self.count.data_ptr(), self.gchunks.data_ptr(),
                                                           self.gmask.data_ptr(), self.gused.data_ptr(), self.flags.data_ptr(), flags=flags)

    def grouped(self, ctx, d, flags):
        ctx.scan_extract_decode_chunks_grouped_dev(d, self.chunks.data_ptr(), self.mask.data_ptr(), self.status.data_ptr(),
                                                   self.gof.data_ptr(), self.count.data_ptr(), self.gchunks.data_ptr(),
                                                   self.gmask.data_ptr(), self.gused.data_ptr(), self.flags.data_ptr(), flags=flags)

    def combined(self, ctx, d, of, m, flags):
        ctx.scan_extract_decode_chunks_combined_dev(d, of, m, self.chunks.data_ptr(), self.mask.data_ptr(), self.status.data_ptr(),
                                                    self.gchunks.data_ptr(), self.gmask.data_ptr(), self.gused.data_ptr(),
                                                    self.flags.data_ptr(), flags=flags)

    def host(self):
        n, m = self.n, self.m
        return dict(chunks=self.chunks[:n].cpu().numpy(), mask=self.mask[:n].cpu().numpy(), status=self.status[:n].cpu().numpy(),
                    flags=self.flags[:n].cpu().numpy(), gchunks=self.gchunks[:m].cpu().numpy(), gmask=self.gmask[:m].cpu().numpy(),
                    gused=self.gused[:m].cpu().numpy(), group_of=self.gof[:n].cpu().numpy(), count=int(self.count[0]))


def state(cb, ctx, n):
    s = {"ccm": ctx.get_ccm(), "transforms": ctx.camera_transforms(n)}
    try:
        s["frame_ccms"] = ctx.frame_ccms(n)
    except cb.Cb200Error as e:
        s["frame_ccms"] = str(e)
    return s


def same(a, b):
    if isinstance(a, str) or isinstance(b, str):
        return a == b
    return np.array_equal(a, b, equal_nan=np.asarray(a).dtype.kind == "f")


def oracle_cells(mode_val, flat, flagname):
    sharpen = "needed" if flagname == "SHARPEN_IF_NEEDED" else "no"
    if flagname == "CC_FIT":
        return [p[:3] for p in fitted_cells(mode_val, flat, sharpen)]
    return [picture_cells(mode_val, p, sharpen, 1 if flagname == "CC_SIMPLE" else 0) for p in flat]


def full_mask(ctx):
    return (1 << ctx.info.chunks_per_frame) - 1


def check_record(mo, got, g, rec, mask, used, what):
    assert (int(got["gmask"][g]), int(got["gused"][g])) == (mask, used), what
    if rec is not None:
        rows = got["gchunks"][g].reshape(mo.chunks_per_frame, mo.chunk_size)[[q for q in range(mo.chunks_per_frame) if mask >> q & 1]]
        assert rec[0] == len(rows) * mo.chunk_size and np.array_equal(rows, rec[1][:len(rows)]), what


def run_sequence(cb, mode_val, batches, flagname, capacity):
    """the sequence through a history call, checked call by call; returns each call's outputs"""
    import torch
    flags = flag_bits(cb, flagname)
    flat = [p for b in batches for p in b]
    per = oracle_cells(mode_val, flat, flagname)
    mo = ORA.mode(mode_val)
    nmax = max(len(b) for b in batches)
    ctx, twin = cb.Context(mode_val, max_frames=nmax), cb.Context(mode_val, max_frames=nmax)
    hist = ctx.group_history(capacity)
    full = full_mask(ctx)
    history = []                                     # (tag, index into flat) of the expected history, oldest first
    results, at = [], 0
    for call, pics in enumerate(batches):
        n = len(pics)
        d = tensors(pics)
        out, ref = Out(ctx, n, n), Out(twin, n, n)
        torch.cuda.synchronize()
        out.history(ctx, hist, d, flags)
        ref.pictures(twin, d, flags)
        ctx.sync()
        twin.sync()
        got, want = out.host(), ref.host()
        for k in ("chunks", "mask", "status", "flags"):
            assert np.array_equal(got[k], want[k]), (call, k)
        gs, ws = state(cb, ctx, n), state(cb, twin, n)
        for k in gs:
            assert same(gs[k], ws[k]), (call, k)
        # the rule on the oracle's cells
        idx = [i for _, i in history] + list(range(at, at + n))
        pos = [(1,) + tuple(per[i][1:3]) if q < len(history) else per[i] for q, i in enumerate(idx)]
        assert got["status"].tolist() == [per[i][0] for i in range(at, at + n)], call
        match = match_matrix([p[1] for p in pos], [p[0] for p in pos], mo.symbol_bits, mo.total_cells)
        own = [int(m) == full for m in got["mask"]]
        expect = {}

        def group_complete(g, members):
            expect[g] = group_expectation(mode_val, pos, members)
            return expect[g][1] == full
        of, count, groups, kept = history_rule(match, len(history), [s in (1, 2) for s in got["status"]], own, group_complete, capacity)
        assert (got["group_of"].tolist(), got["count"]) == (of, count), call
        for g in range(count):
            check_record(mo, got, g, *expect[g], (call, g))
        assert not got["gchunks"][count:].any() and not got["gmask"][count:].any() and not got["gused"][count:].any(), call
        if count and flagname != "CC_FIT":
            members = [p for g in groups for p in g]
            third = cb.Context(mode_val, max_frames=len(members))
            cout = Out(third, len(members), count)
            torch.cuda.synchronize()
            cout.combined(third, tensors([flat[idx[p]] for p in members]), [g for g, m in enumerate(groups) for _ in m], count, flags)
            third.sync()
            ch = cout.host()
            third.close()
            for k in ("gchunks", "gmask", "gused"):
                assert np.array_equal(ch[k], got[k][:count]), (call, k)
        tags = [t for t, _ in history] + [call << 32 | i for i in range(n)]
        history = [(tags[p], idx[p]) for p in kept]
        assert hist.tags().tolist() == [t for t, _ in history], call
        results.append(got)
        at += n
    hist.close()
    ctx.close()
    twin.close()
    return results


@pytest.mark.parametrize("flagname", FLAGS)
@pytest.mark.parametrize("mode_val", MODES)
def test_a_sequence_of_batches_follows_the_rule(cb, mode_val, flagname):
    res = run_sequence(cb, mode_val, sequence(mode_val), flagname, capacity=4)
    assert sum(r["count"] for r in res) >= 2                                 # premise: groups across calls
    assert 0 in res[3]["status"].tolist()                                    # premise: the noise picture fails


@pytest.mark.parametrize("mode_val", MODES)
def test_a_frame_whose_blocks_all_decode_has_the_complete_mask(cb, mode_val):
    """the clean picture decodes every block (the oracle says so) and its mask is then all chunks_per_frame bits"""
    import torch
    mo = ORA.mode(mode_val)
    st, values, _ = picture_cells(mode_val, clean_picture(mode_val))
    ok = ORA.decode(mo, ORA.render_frame(mo, values))[1]
    assert st in (1, 2) and np.asarray(ok).all()
    ctx = cb.Context(mode_val, max_frames=1)
    out = Out(ctx, 1, 1)
    d = tensors([clean_picture(mode_val)])
    torch.cuda.synchronize()
    out.pictures(ctx, d, 0)
    ctx.sync()
    assert int(out.mask[0]) == full_mask(ctx)
    ctx.close()


def test_a_new_history_gives_the_grouped_call(cb):
    import torch
    pics, _ = frame_captures(68, [2, 3, 1, 2], seed=9)
    pics += [noise(), clean_picture(68)]
    pics = [pics[i] for i in np.random.default_rng(68).permutation(len(pics))]
    n = len(pics)
    d = tensors(pics)
    ctx, gctx = cb.Context(68, max_frames=n), cb.Context(68, max_frames=n)
    hist = ctx.group_history(32)
    out, gout = Out(ctx, n, n), Out(gctx, n, n // 2)
    torch.cuda.synchronize()
    out.history(ctx, hist, d, 0)
    gout.grouped(gctx, d, 0)
    ctx.sync()
    gctx.sync()
    got, want = out.host(), gout.host()
    count = want["count"]
    assert count >= 3 and (got["group_of"].tolist(), got["count"]) == (want["group_of"].tolist(), count)
    for k in ("gchunks", "gmask", "gused"):
        assert np.array_equal(got[k][:count], want[k][:count]), k
    assert not got["gchunks"][count:].any() and not got["gmask"][count:].any() and not got["gused"][count:].any()
    hist.close()
    ctx.close()
    gctx.close()


def test_eviction_and_reset(cb):
    """H = 2 after five lone captures of five frames, one per call: the last two stay; reset empties it and restarts the count"""
    import torch
    pics = [capture_of(68, seeded_frame(68, 500 + f), [500, f]) for f in range(5)]
    res = run_sequence(cb, 68, [[p] for p in pics], "none", capacity=2)
    assert all(r["count"] == 0 and r["mask"][0] != (1 << ORA.mode(68).chunks_per_frame) - 1 for r in res)
    ctx = cb.Context(68, max_frames=2)
    hist = ctx.group_history(2)
    out = Out(ctx, 1, 1)
    d = tensors(pics)
    torch.cuda.synchronize()
    for t in d:
        out.history(ctx, hist, [t], 0)
    assert hist.tags().tolist() == [3 << 32, 4 << 32]
    out.history(ctx, hist, [], 0)                                            # counted, nothing changes
    assert hist.tags().tolist() == [3 << 32, 4 << 32]
    hist.reset()
    assert hist.tags().tolist() == []
    out.history(ctx, hist, d[:1], 0)
    assert hist.tags().tolist() == [0]
    hist.close()
    ctx.close()


@pytest.mark.parametrize("mode_val", [68, 4])
def test_one_picture_per_call_recovers_a_frame_no_capture_decodes(cb, mode_val):
    """three captures of a frame, each failing alone, one per call: a group record holds the whole frame, and the frame's pictures
    then leave the history"""
    frame = seeded_frame(mode_val, 4242)
    pics = [capture_of(mode_val, frame, [4242, s]) for s in range(3)]
    res = run_sequence(cb, mode_val, [[p] for p in pics], "none", capacity=32)
    ctx = cb.Context(mode_val, max_frames=1)
    full = full_mask(ctx)
    ctx.close()
    assert all(int(r["mask"][0]) != full for r in res)                      # premise: no capture decodes alone
    assert any(r["count"] == 1 and int(r["gmask"][0]) == full for r in res)


def test_launches_and_refusals_that_need_a_context(cb):
    """nine launches more than the pictures call; another context's history, no history and n > max_frames are refused"""
    import torch
    lib = cb.load_library()
    pics = sequence(68)[1]
    d = tensors(pics)
    ctx, other = cb.Context(68, max_frames=2), cb.Context(68, max_frames=2)
    hist, foreign = ctx.group_history(8), other.group_history(8)
    out = Out(ctx, 2, 2)
    torch.cuda.synchronize()
    out.history(ctx, hist, d, 0)
    out.pictures(ctx, d, 0)
    ctx.sync()
    n0 = lib.cb200_launch_count()
    out.pictures(ctx, d, 0)
    n1 = lib.cb200_launch_count()
    out.history(ctx, hist, d, 0)
    n2 = lib.cb200_launch_count()
    ctx.sync()
    assert n2 - n1 == (n1 - n0) + 9
    with pytest.raises(cb.Cb200Error, match="another context"):
        out.history(ctx, foreign, d, 0)
    with pytest.raises(cb.Cb200Error, match="null history"):
        out.history(ctx, None, d, 0)
    with pytest.raises(cb.Cb200Error, match=r"n = 3 > max_frames = 2"):
        out.history(ctx, hist, d + d[:1], 0)
    hist.close()
    foreign.close()
    ctx.close()
    other.close()
