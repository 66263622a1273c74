"""The grouped receivers call (cb200_scan_extract_decode_chunks_grouped_receivers_dev and its _flags_ form) on the GPU, in modes 68,
67, 66, 4 and 8 under no CC, SHARPEN_IF_NEEDED, CC_SIMPLE and CC_FIT, with a distinct entry state per receiver.

Per picture, and for every receiver's state afterwards, it must give exactly what the receivers call gives on a twin context.  Each
receiver's groups, in slot order, must be exactly what the grouped call gives on that receiver's pictures alone on a context whose CCM
is set to the receiver's entry state: records, masks, used counts and members.  The batches hold captures of seeded frames
(group_fixtures.frame_captures); two receivers hold captures of one frame, which must form one group in each receiver, never one
across them."""
import time

import numpy as np
import pytest

from combine_fixtures import ORA, clean_picture, picture_cells
from group_fixtures import assign, frame_captures, match_matrix, rule_groups
from gpu_support import cb, entry_states  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

MODES = [68, 67, 66, 4, 8]
FLAGS = ["none", "SHARPEN_IF_NEEDED", "CC_SIMPLE", "CC_FIT"]
R = 4


def flag_bits(cb, name):
    return 0 if name == "none" else getattr(cb, "FLAG_" + name)


def noise():
    return np.random.default_rng(7).integers(0, 256, (700, 900, 3), dtype=np.uint8)


_batches = {}


def batch(mode_val):
    """(pictures, receiver of each) in a seeded order: frame 0's four captures split between receivers 0 and 1, two more frames of
    receiver 0 and 1, a frame and a noise picture of receiver 2, a lone capture and the clean picture of receiver 3"""
    if mode_val not in _batches:
        pics, frame_of = frame_captures(mode_val, [4, 2, 3, 2, 1], seed=5)
        recv = [0, 0, 1, 1] + [0, 0] + [1, 1, 1] + [2, 2] + [3]
        pics += [noise(), clean_picture(mode_val)]
        recv += [2, 3]
        order = np.random.default_rng(mode_val + 100).permutation(len(pics))
        _batches[mode_val] = ([pics[i] for i in order], np.array([recv[i] for i in order], np.int32),
                              [frame_of[i] if i < len(frame_of) else -1 for i in order])
    return _batches[mode_val]


def tensors(pics):
    import torch
    return [torch.from_numpy(np.ascontiguousarray(p)).cuda() for p in pics]


class Out:
    def __init__(self, ctx, n):
        import torch
        db = ctx.info.data_bytes
        m = n // 2
        z = lambda shape, v, dt: torch.full(shape, v, dtype=dt, device="cuda")
        self.chunks, self.mask = z((max(n, 1), db), 0xA5, torch.uint8), z((max(n, 1),), -1, torch.int32)
        self.status, self.flags = z((max(n, 1),), 7, torch.int32), z((max(n, 1),), 0xEE, torch.uint8)
        self.gchunks, self.gmask = z((max(m, 1), db), 0x5A, torch.uint8), z((max(m, 1),), -1, torch.int32)
        self.gused, self.gof, self.count = z((max(m, 1),), 9, torch.int32), z((max(n, 1),), -9, torch.int32), z((1,), -9, torch.int32)
        self.grec = z((max(m, 1),), -9, torch.int32)
        self.n, self.m = n, m

    def receivers(self, ctx, d, of, states, flags, words=None):
        ctx.scan_extract_decode_chunks_receivers_dev(d, of, states, self.chunks.data_ptr(), self.mask.data_ptr(), self.status.data_ptr(),
                                                     self.flags.data_ptr(), flags=flags, receiver_flags=words)

    def grouped_receivers(self, ctx, d, of, states, flags, words=None):
        ctx.scan_extract_decode_chunks_grouped_receivers_dev(d, of, states, self.chunks.data_ptr(), self.mask.data_ptr(),
                                                             self.status.data_ptr(), self.gof.data_ptr(), self.count.data_ptr(),
                                                             self.gchunks.data_ptr(), self.gmask.data_ptr(), self.gused.data_ptr(),
                                                             self.grec.data_ptr(), self.flags.data_ptr(), flags=flags,
                                                             receiver_flags=words)

    def grouped(self, ctx, d, flags):
        ctx.scan_extract_decode_chunks_grouped_dev(d, self.chunks.data_ptr(), self.mask.data_ptr(), self.status.data_ptr(),
                                                   self.gof.data_ptr(), self.count.data_ptr(), self.gchunks.data_ptr(),
                                                   self.gmask.data_ptr(), self.gused.data_ptr(), self.flags.data_ptr(), flags=flags)

    def host(self):
        n, m = self.n, self.m
        return dict(chunks=self.chunks[:n].cpu().numpy(), mask=self.mask[:n].cpu().numpy(), status=self.status[:n].cpu().numpy(),
                    flags=self.flags[:n].cpu().numpy(), gchunks=self.gchunks[:m].cpu().numpy(), gmask=self.gmask[:m].cpu().numpy(),
                    gused=self.gused[:m].cpu().numpy(), group_of=self.gof[:n].cpu().numpy(), count=int(self.count[0]),
                    grec=self.grec[:m].cpu().numpy())


def run(cb, mode_val, pics, kind, flags, of=None, ccms=None, words=None, ccm=None):
    """one call of `kind` ("receivers", "grouped_receivers" or "grouped") on a fresh context: its outputs, the states afterwards,
    the transforms and the frame CCMs.  ccm: the context's CCM before a grouped call"""
    import torch
    n = len(pics)
    d = tensors(pics)
    ctx = cb.Context(mode_val, max_frames=max(n, 1))
    out = Out(ctx, n)
    states = cb.receiver_states(ccms) if ccms is not None else None
    table = None if words is None else torch.tensor(np.array(words, np.uint32).view(np.int32), device="cuda")
    if ccm is not None:
        ctx.set_ccm(ccm)
    torch.cuda.synchronize()
    if kind == "receivers":
        out.receivers(ctx, d, of, states, flags, table)
    elif kind == "grouped_receivers":
        out.grouped_receivers(ctx, d, of, states, flags, table)
    else:
        out.grouped(ctx, d, flags)
    ctx.sync()
    h = out.host()
    h["states"] = None if states is None else states.cpu().numpy()
    h["transforms"] = ctx.camera_transforms(n) if n else None
    try:
        h["frame_ccms"] = ctx.frame_ccms(n)
    except cb.Cb200Error as e:
        h["frame_ccms"] = str(e)
    h["ccm"] = ctx.get_ccm()
    ctx.close()
    return h


def same(a, b):
    if isinstance(a, str) or isinstance(b, str):
        return a == b
    return (a is None) == (b is None) and (a is None or np.array_equal(a, b, equal_nan=np.asarray(a).dtype.kind == "f"))


PER_PICTURE = ("chunks", "mask", "status", "flags", "states", "transforms", "frame_ccms", "ccm")


def check_receiver_groups(cb, mode_val, pics, of, ccms, flags, got, words=None):
    """each receiver's groups equal the grouped call on its pictures alone on a context set to its entry state"""
    count = got["count"]
    grec = got["grec"]
    assert (grec[count:] == -1).all() and (grec[:count] >= 0).all()
    assert not got["gchunks"][count:].any() and not got["gmask"][count:].any() and not got["gused"][count:].any()
    for r in range(len(ccms)):
        idx = np.flatnonzero(of == r)
        slots = [g for g in range(count) if grec[g] == r]
        if len(idx) == 0:
            assert not slots
            continue
        f = flags | (0 if words is None else int(words[r]))
        alone = run(cb, mode_val, [pics[i] for i in idx], "grouped", f, ccm=ccms[r])
        assert alone["count"] == len(slots), r
        for k, g in enumerate(slots):
            assert np.array_equal(got["gchunks"][g], alone["gchunks"][k]), (r, k)
            assert got["gmask"][g] == alone["gmask"][k] and got["gused"][g] == alone["gused"][k], (r, k)
            assert np.flatnonzero(got["group_of"] == g).tolist() == idx[alone["group_of"] == k].tolist(), (r, k)
        mine = got["group_of"][idx]
        assert np.isin(mine, slots + [-1]).all(), r


@pytest.mark.parametrize("flagname", FLAGS)
@pytest.mark.parametrize("mode_val", MODES)
def test_per_picture_the_receivers_call_per_receiver_the_grouped_call(cb, mode_val, flagname):
    pics, of, frame_of = batch(mode_val)
    ccms = entry_states(R, mode_val)
    flags = flag_bits(cb, flagname)
    want = run(cb, mode_val, pics, "receivers", flags, of, ccms)
    got = run(cb, mode_val, pics, "grouped_receivers", flags, of, ccms)
    for k in PER_PICTURE:
        assert same(want[k], got[k]), k
    check_receiver_groups(cb, mode_val, pics, of, ccms, flags, got)
    # frame 0's captures in receivers 0 and 1: one group in each, never one across them
    f0 = [i for i in range(len(pics)) if frame_of[i] == 0]
    g0 = {int(got["group_of"][i]) for i in f0 if of[i] == 0}
    g1 = {int(got["group_of"][i]) for i in f0 if of[i] == 1}
    assert len(g0) == 1 and len(g1) == 1 and g0 != g1 and -1 not in g0 | g1
    assert got["count"] >= 4                                       # premise: the planted frames group


@pytest.mark.parametrize("mode_val", MODES)
def test_no_cc_groups_are_the_rule_on_the_oracles_cells(cb, mode_val):
    """the rule per receiver on the oracle's cells, numbered in the leaders' batch order (inactive states: the oracle's cells)"""
    pics, of, _ = batch(mode_val)
    got = run(cb, mode_val, pics, "grouped_receivers", 0, of, [None] * R)
    per = [picture_cells(mode_val, p) for p in pics]
    n = len(pics)
    local, leaders = np.full(n, -1), []
    for r in range(R):
        idx = np.flatnonzero(of == r)
        sub, _ = rule_groups(mode_val, [per[i] for i in idx])
        for k, g in enumerate(sub):
            local[idx[k]] = g
        leaders += [(int(idx[sub.index(g)]), r, g) for g in range(max(sub, default=-1) + 1)]
    leaders.sort()
    number = {(r, g): k for k, (_, r, g) in enumerate(leaders)}
    want = [number[(int(of[i]), int(local[i]))] if local[i] >= 0 else -1 for i in range(n)]
    assert (got["group_of"].tolist(), got["count"]) == (want, len(leaders))
    assert got["grec"][:len(leaders)].tolist() == [r for _, r, _ in leaders]
    assert got["status"].tolist() == [p[0] for p in per]


WORDS = {"valid": [0x20 | 0x8, 0x0, 0x4, 0x2]}


@pytest.mark.parametrize("mode_val", [68, 4])
def test_the_flags_form(cb, mode_val):
    pics, of, _ = batch(mode_val)
    ccms = entry_states(R, mode_val + 1)
    words = WORDS["valid"]
    want = run(cb, mode_val, pics, "receivers", 0, of, ccms, words=words)
    got = run(cb, mode_val, pics, "grouped_receivers", 0, of, ccms, words=words)
    for k in PER_PICTURE:
        assert same(want[k], got[k]), k
    check_receiver_groups(cb, mode_val, pics, of, ccms, 0, got, words=words)


def test_an_invalid_word_leaves_its_receiver_out_and_the_others_alone(cb):
    pics, of, _ = batch(68)
    ccms = entry_states(R, 9)
    words = list(WORDS["valid"])
    good = run(cb, 68, pics, "grouped_receivers", 0, of, ccms, words=words)
    words[1] = 0x2 | 0x20                                          # both sharpen bits: refused
    bad = run(cb, 68, pics, "grouped_receivers", 0, of, ccms, words=words)
    want = run(cb, 68, pics, "receivers", 0, of, ccms, words=words)
    for k in PER_PICTURE:
        assert same(want[k], bad[k]), k
    mine = of == 1
    assert (bad["status"][mine] == cb.EXTRACT_REFUSED).all() and (bad["group_of"][mine] == -1).all()
    assert 1 not in bad["grec"][:bad["count"]].tolist() and 1 in good["grec"][:good["count"]].tolist()
    # every other receiver: the same groups, members and records, in the same order
    for r in (0, 2, 3):
        sg = [g for g in range(good["count"]) if good["grec"][g] == r]
        sb = [g for g in range(bad["count"]) if bad["grec"][g] == r]
        assert len(sg) == len(sb)
        for a, b in zip(sg, sb):
            assert np.flatnonzero(good["group_of"] == a).tolist() == np.flatnonzero(bad["group_of"] == b).tolist()
            for k in ("gchunks", "gmask", "gused"):
                assert np.array_equal(good[k][a], bad[k][b]), (r, k)
    for k in ("chunks", "mask", "status"):
        assert np.array_equal(good[k][~mine], bad[k][~mine]), k


@pytest.mark.parametrize("flagname", ["none", "CC_FIT"])
def test_one_receiver_is_the_grouped_call(cb, flagname):
    pics, _, _ = batch(4)
    of = np.zeros(len(pics), np.int32)
    flags = flag_bits(cb, flagname)
    want = run(cb, 4, pics, "grouped", flags)
    got = run(cb, 4, pics, "grouped_receivers", flags, of, [None])
    for k in ("chunks", "mask", "status", "flags", "transforms", "gchunks", "gmask", "gused", "group_of", "count"):
        assert same(want[k], got[k]), k
    assert (got["grec"][:got["count"]] == 0).all() and (got["grec"][got["count"]:] == -1).all()


@pytest.mark.parametrize("n", [0, 1])
def test_fewer_than_two_pictures_give_no_group(cb, n):
    pics, of, _ = batch(68)
    want = run(cb, 68, pics[:n], "receivers", 0, of[:n], [None] * R)
    got = run(cb, 68, pics[:n], "grouped_receivers", 0, of[:n], [None] * R)
    assert got["count"] == 0 and got["group_of"].tolist() == [-1] * n
    for k in ("chunks", "mask", "status", "states"):
        assert same(want[k], got[k]), k


def test_a_large_batch_of_many_receivers(cb):
    """1024 pictures of 64 receivers (12 captures of four frames, repeated as the same tensors): many segments at once, the tile
    list, groups cut at 16 within a receiver and frames shared by every receiver"""
    import torch
    n, K = 1024, 64
    base, _ = frame_captures(4, [3, 3, 3, 3], seed=11)
    per = [picture_cells(4, p) for p in base]
    rng = np.random.default_rng(1024)
    pick = rng.integers(0, len(base), n)
    of = rng.integers(0, K, n).astype(np.int32)
    of[rng.random(n) < 0.25] = 5                                   # one large receiver: a segment across several tiles
    mode = ORA.mode(4)
    m = match_matrix([per[i][1] for i in pick], [per[i][0] for i in pick], mode.symbol_bits, mode.total_cells)
    elig = np.array([per[i][0] in (1, 2) for i in pick])
    local, leaders = np.full(n, -1), []
    for r in range(K):
        idx = np.flatnonzero(of == r)
        sub, _ = assign(m[np.ix_(idx, idx)], elig[idx])
        for k, g in enumerate(sub):
            local[idx[k]] = g
        leaders += [(int(idx[sub.index(g)]), r, g) for g in range(max(sub, default=-1) + 1)]
    leaders.sort()
    number = {(r, g): k for k, (_, r, g) in enumerate(leaders)}
    want = [number[(int(of[i]), int(local[i]))] if local[i] >= 0 else -1 for i in range(n)]
    d12 = tensors(base)
    d = [d12[i] for i in pick]
    ctx = cb.Context(4, max_frames=n)
    out = Out(ctx, n)
    out.grouped_receivers(ctx, d, of, cb.receiver_states([None] * K), 0)
    ctx.sync()
    got = out.host()
    ctx.close()
    assert (got["group_of"].tolist(), got["count"]) == (want, len(leaders))
    assert got["grec"][:len(leaders)].tolist() == [r for _, r, _ in leaders]
    assert len(leaders) >= K and max(np.bincount(got["group_of"][got["group_of"] >= 0])) == 16
    count = got["count"]
    comb = cb.Context(4, max_frames=n)
    cout = Out(comb, n)
    gchunks = torch.zeros((count, comb.info.data_bytes), dtype=torch.uint8, device="cuda")
    gmask, gused = (torch.full((count,), -1, dtype=torch.int32, device="cuda") for _ in range(2))
    comb.scan_extract_decode_chunks_combined_dev(d, got["group_of"], count, cout.chunks.data_ptr(), cout.mask.data_ptr(),
                                                 cout.status.data_ptr(), gchunks.data_ptr(), gmask.data_ptr(), gused.data_ptr())
    comb.sync()
    assert np.array_equal(gchunks.cpu().numpy(), got["gchunks"][:count])
    assert np.array_equal(gmask.cpu().numpy(), got["gmask"][:count]) and np.array_equal(gused.cpu().numpy(), got["gused"][:count])
    assert np.array_equal(cout.chunks[:n].cpu().numpy(), got["chunks"])
    comb.close()


def test_calls_only_enqueue_with_six_launches_more(cb):
    """two grouped receivers calls queued behind a sleeping stream return at once, equal the same calls run alone, and each launches
    six kernels more than the receivers call on the same batch"""
    import torch
    pics, of, _ = batch(4)
    ccms = entry_states(R, 3)
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    lib = cb.load_library()
    d = tensors(pics)
    n = len(pics)
    ctx = cb.Context(4, max_frames=n)
    twin = cb.Context(4, max_frames=n)
    outs = [Out(ctx, n) for _ in range(2)]
    ref = Out(twin, n)
    twin_states = cb.receiver_states(ccms)

    def start(c, st):                                               # every buffer at its size
        outs[0].grouped_receivers(c, d, of, st, flags)
        c.sync()
    start(twin, cb.receiver_states(ccms))
    want = []
    for _ in range(2):
        outs[0].grouped_receivers(twin, d, of, twin_states, flags)
        twin.sync()
        want.append(outs[0].host())
    n0 = lib.cb200_launch_count()
    ref.receivers(twin, d, of, cb.receiver_states(ccms), flags)
    n1 = lib.cb200_launch_count()
    twin.sync()
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    start(ctx, cb.receiver_states(ccms))
    torch.cuda.synchronize()
    shared = cb.receiver_states(ccms)
    with torch.cuda.stream(stream):
        torch.cuda._sleep(int(1.5e9))
    t0 = time.perf_counter()
    c0 = lib.cb200_launch_count()
    for o in outs:
        o.grouped_receivers(ctx, d, of, shared, flags)
    c1 = lib.cb200_launch_count()
    spent = time.perf_counter() - t0
    busy = not stream.query()
    ctx.sync()
    assert busy, "the stream finished before the calls returned"
    assert spent < 0.25, spent
    assert c1 - c0 == 2 * ((n1 - n0) + 6)
    for o, w in zip(outs, want):
        h = o.host()
        for k in w:
            assert np.array_equal(h[k], w[k]), k
    assert np.array_equal(shared.cpu().numpy(), twin_states.cpu().numpy())
    ctx.close()
    twin.close()


def test_refusals_that_need_a_context(cb):
    pics, of, _ = batch(68)
    d = tensors(pics)
    ctx = cb.Context(68, max_frames=len(pics) - 1)
    out = Out(ctx, len(pics))
    states = cb.receiver_states([None] * R)
    with pytest.raises(cb.Cb200Error, match=r"n = %d > max_frames = %d" % (len(pics), len(pics) - 1)):
        out.grouped_receivers(ctx, d, of, states, 0)
    with pytest.raises(cb.Cb200Error, match="null output"):
        ctx.scan_extract_decode_chunks_grouped_receivers_dev(d[:2], of[:2], states, 0, out.mask.data_ptr(), out.status.data_ptr(),
                                                             out.gof.data_ptr(), out.count.data_ptr(), out.gchunks.data_ptr(),
                                                             out.gmask.data_ptr(), out.gused.data_ptr(), out.grec.data_ptr())
    ctx.close()
    chained = cb.Context(68, max_frames=len(pics))
    chained.ccm_chain_root_create(1)
    chained.ccm_chain_attach(0, 1)
    out = Out(chained, len(pics))
    before = cb.launch_count()
    with pytest.raises(cb.Cb200Error, match="linked to a CCM chain"):
        out.grouped_receivers(chained, d, of, states, 0)
    assert cb.launch_count() == before
    chained.close()
