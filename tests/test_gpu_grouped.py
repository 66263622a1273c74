"""The grouped camera call (cb200_scan_extract_decode_chunks_grouped_dev) on the GPU, in modes 68, 67, 66, 4 and 8.

Per picture it must give exactly what cb200_scan_extract_decode_chunks_pictures_dev gives on a twin context.  Its group_of and count
must be the rule of include/cb200.h on the oracle's cells (tests/group_fixtures.py; under CC_FIT the cells of the oracle's CC 2
route), and its first `count` slots exactly what cb200_scan_extract_decode_chunks_combined_dev gives on a third context with the
device's group_of; the slots past the count are zero.  The batches mix captures of distinct seeded frames, a lone capture, a picture
that fails extraction and a clean picture (in mode 4 also the six photographs), shuffled."""
import time

import numpy as np
import pytest

from combine_fixtures import clean_picture, fitted_cells, picture_cells
from group_fixtures import capture_of, frame_captures, rule_groups, seeded_frame
from ragged_samples import sample

pytestmark = pytest.mark.gpu

MODES = [68, 67, 66, 4, 8]
FLAGS = ["none", "SHARPEN_IF_NEEDED", "CC_SIMPLE", "CC_FIT"]
PHOTOS = ["6bit/4_30_f0_627.jpg", "6bit/4_30_f0_177_ccm.jpg", "6bit/4_30_f1_360.jpg", "6bit/4_30_f2_246.jpg", "6bit/4_30_f2_734.jpg",
          "6bit/4_30_802.jpg"]


@pytest.fixture(scope="module")
def cb():
    import libcimbar_b200 as cb
    return cb


def flag_bits(cb, name):
    return 0 if name == "none" else getattr(cb, "FLAG_" + name)


def noise():
    return np.random.default_rng(7).integers(0, 256, (700, 900, 3), dtype=np.uint8)


_batches = {}


def batch(mode_val):
    """2, 3, 4 and 2 captures of four seeded frames, one capture of a fifth, a noise picture, the clean picture and, in mode 4, the
    six photographs, in a seeded order"""
    if mode_val not in _batches:
        pics, _ = frame_captures(mode_val, [2, 3, 4, 2, 1], seed=3)
        pics += [noise(), clean_picture(mode_val)]
        if mode_val == 4:
            pics += [sample(nm) for nm in PHOTOS]
        order = np.random.default_rng(mode_val).permutation(len(pics))
        _batches[mode_val] = [pics[i] for i in order]
    return _batches[mode_val]


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


def run(cb, mode_val, pics, kind, flags, of=None, m=None):
    """one call of `kind` on a fresh context: its outputs, the CCM afterwards, the transforms and the frame CCMs"""
    import torch
    n = len(pics)
    d = tensors(pics)
    slots = n // 2 if m is None else m
    ctx = cb.Context(mode_val, max_frames=max(n, slots, 1))
    out = Out(ctx, n, slots)
    torch.cuda.synchronize()
    if kind == "pictures":
        out.pictures(ctx, d, flags)
    elif kind == "grouped":
        out.grouped(ctx, d, flags)
    else:
        out.combined(ctx, d, of, m, flags)
    ctx.sync()
    h = out.host()
    h["ccm"] = ctx.get_ccm()
    h["transforms"] = ctx.camera_transforms(n) if n else None
    try:
        h["frame_ccms"] = ctx.frame_ccms(n)
    except cb.Cb200Error as e:
        h["frame_ccms"] = str(e)
    ctx.close()
    return h


def same(a, b):
    if isinstance(a, str) or isinstance(b, str):
        return a == b
    return (a is None) == (b is None) and (a is None or np.array_equal(a, b, equal_nan=np.asarray(a).dtype.kind == "f"))


PER_PICTURE = ("chunks", "mask", "status", "flags", "ccm", "transforms", "frame_ccms")


def expected_groups(mode_val, pics, flagname):
    sharpen = "needed" if flagname == "SHARPEN_IF_NEEDED" else "no"
    if flagname == "CC_FIT":
        per = fitted_cells(mode_val, pics, sharpen)
    else:
        per = [picture_cells(mode_val, p, sharpen, 1 if flagname == "CC_SIMPLE" else 0) for p in pics]
    return rule_groups(mode_val, per), [p[0] for p in per]


def check_grouped(cb, mode_val, pics, flags, want_of, want_count):
    """the grouped call against the pictures call and the combined call given the device's groups; returns the grouped outputs"""
    want = run(cb, mode_val, pics, "pictures", flags)
    got = run(cb, mode_val, pics, "grouped", flags)
    for k in PER_PICTURE:
        assert same(want[k], got[k]), k
    assert (got["group_of"].tolist(), got["count"]) == (want_of, want_count)
    count = got["count"]
    if count:
        comb = run(cb, mode_val, pics, "combined", flags, of=got["group_of"], m=count)
        for k in ("gchunks", "gmask", "gused"):
            assert np.array_equal(comb[k], got[k][:count]), k
    assert not got["gchunks"][count:].any() and not got["gmask"][count:].any() and not got["gused"][count:].any()
    return got


@pytest.mark.parametrize("flagname", FLAGS)
@pytest.mark.parametrize("mode_val", MODES)
def test_groups_are_the_rule_and_slots_the_combined_call(cb, mode_val, flagname):
    pics = batch(mode_val)
    (of, count), statuses = expected_groups(mode_val, pics, flagname)
    got = check_grouped(cb, mode_val, pics, flag_bits(cb, flagname), of, count)
    assert got["status"].tolist() == statuses
    assert 0 in statuses and count >= 4                              # premise: a picture that fails, the planted frames
    assert all(got["gused"][g] == of.count(g) for g in range(count))


def test_no_interleave(cb):
    pics = batch(68)
    (of, count), _ = expected_groups(68, pics, "none")
    check_grouped(cb, 68, pics, cb.FLAG_NO_INTERLEAVE, of, count)


def test_the_cap_of_sixteen_on_the_device(cb):
    frame = seeded_frame(4, 77)
    pics = [capture_of(4, frame, [77, s]) for s in range(18)]
    got = check_grouped(cb, 4, pics, 0, [0] * 16 + [1] * 2, 2)
    assert got["gused"].tolist()[:2] == [16, 2]


@pytest.mark.parametrize("n", [0, 1])
def test_fewer_than_two_pictures_give_no_group(cb, n):
    pics = batch(68)[:n]
    want = run(cb, 68, pics, "pictures", 0)
    got = run(cb, 68, pics, "grouped", 0)
    assert got["count"] == 0 and got["group_of"].tolist() == [-1] * n
    for k in ("chunks", "mask", "status"):
        assert same(want[k], got[k]), k


def test_pictures_that_all_fail_give_no_group(cb):
    pics = [noise(), noise()[::-1].copy(), noise()[:, ::-1].copy()]
    got = check_grouped(cb, 68, pics, cb.FLAG_CC_FIT, [-1] * 3, 0)
    assert (got["status"] == 0).all()


@pytest.mark.parametrize("n", [97, 301])
def test_a_large_batch_of_repeated_pictures(cb, n):
    """12 captures (four frames, three each) repeated as the same tensors in a seeded order: partial pairing tiles, groups cut at 16"""
    import torch
    base, _ = frame_captures(4, [3, 3, 3, 3], seed=11)
    per = [picture_cells(4, p) for p in base]
    pick = np.random.default_rng(n).integers(0, len(base), n)
    (of, count) = rule_groups(4, [per[i] for i in pick])
    d12 = tensors(base)
    d = [d12[i] for i in pick]
    ctx = cb.Context(4, max_frames=n)
    out = Out(ctx, n, n // 2)
    out.grouped(ctx, d, 0)
    ctx.sync()
    got = out.host()
    ctx.close()
    assert (got["group_of"].tolist(), got["count"]) == (of, count)
    assert count >= 8 and not got["gused"][count:].any()
    comb = cb.Context(4, max_frames=n)
    cout = Out(comb, n, count)
    cout.combined(comb, d, got["group_of"], count, 0)
    comb.sync()
    ch = cout.host()
    comb.close()
    for k in ("gchunks", "gmask", "gused"):
        assert np.array_equal(ch[k], got[k][:count]), k
    assert np.array_equal(ch["chunks"], got["chunks"]) and np.array_equal(ch["mask"], got["mask"])
    torch.cuda.synchronize()


def test_calls_only_enqueue_with_six_launches_more(cb):
    """two grouped calls queued behind a sleeping stream return at once, equal the same calls run alone, and each launches six
    kernels more than the pictures call on the same batch (the pairing and the assignment, then the combined call's four)"""
    import torch
    pics = batch(4)
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    lib = cb.load_library()
    d = tensors(pics)
    n = len(pics)
    ctx = cb.Context(4, max_frames=n)
    twin = cb.Context(4, max_frames=n)
    outs = [Out(ctx, n, n // 2) for _ in range(2)]
    ref = Out(twin, n, n // 2)

    def start(c):                                                   # every buffer at its size, then no CCM
        outs[0].grouped(c, d, flags)
        c.sync()
        c.set_ccm(None)
        c.sync()
    start(twin)
    want = []
    for _ in range(2):
        outs[0].grouped(twin, d, flags)
        twin.sync()
        want.append(outs[0].host())
    n0 = lib.cb200_launch_count()
    ref.pictures(twin, d, flags)
    n1 = lib.cb200_launch_count()
    twin.sync()
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    start(ctx)
    torch.cuda.synchronize()
    with torch.cuda.stream(stream):
        torch.cuda._sleep(int(1.5e9))
    t0 = time.perf_counter()
    c0 = lib.cb200_launch_count()
    for o in outs:
        o.grouped(ctx, d, flags)
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
    ctx.close()
    twin.close()


def test_refusals_that_need_a_context(cb):
    pics = batch(68)
    ctx = cb.Context(68, max_frames=len(pics) - 1)
    out = Out(ctx, len(pics), len(pics) // 2)
    d = tensors(pics)
    with pytest.raises(cb.Cb200Error, match=r"n = %d > max_frames = %d" % (len(pics), len(pics) - 1)):
        out.grouped(ctx, d, 0)
    with pytest.raises(cb.Cb200Error, match="null output"):
        ctx.scan_extract_decode_chunks_grouped_dev(d[:2], 0, out.mask.data_ptr(), out.status.data_ptr(), out.gof.data_ptr(),
                                                   out.count.data_ptr(), out.gchunks.data_ptr(), out.gmask.data_ptr(), out.gused.data_ptr())
    ctx.close()
