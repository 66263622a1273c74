"""The combined camera call (cb200_scan_extract_decode_chunks_combined_dev) on the GPU, in modes 68, 67, 66, 4 and 8.

Per picture it must give exactly what cb200_scan_extract_decode_chunks_pictures_dev gives on a twin context (records, masks, frame
flags, statuses, transforms, the CCM afterwards).  Per group the record, mask and count must be the rule of include/cb200.h applied
to the oracle's cells (tests/combine_fixtures.py) under every flag set, CC_FIT included (fitted_cells: the cells of the oracle's CC 2
route).  A group of one picture, or of one picture repeated, gives that picture's record.  The synthetic rescue groups decode every block on the device, and the call only enqueues, with four launches more than the
pictures call."""
import time

import numpy as np
import pytest

from combine_fixtures import ORA, capture, clean_picture, fitted_cells, group_expectation, picture_cells
from ragged_samples import sample
from gpu_support import cb  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

MODES = [68, 67, 66, 4, 8]
FLAGS = ["none", "SHARPEN_IF_NEEDED", "CC_SIMPLE", "CC_FIT"]


def flag_bits(cb, name):
    return 0 if name == "none" else getattr(cb, "FLAG_" + name)


_batches = {}


def batch(mode_val):
    """pictures and their groups: six synthetic captures in groups {0, 1}, {2, 3, 4} and {5}; a noise picture (FAILURE) alone in
    group 3; a capture outside every group; group 4 without pictures; in mode 4 the two real pairs as groups 5 and 6; last, alone in
    the last group, a clean picture (clean_picture) that K1 decodes without flags, so that the walk over every picture also takes a
    frame the pictures call does not walk"""
    if mode_val not in _batches:
        pics = [capture(mode_val, 1000 * mode_val + s) for s in range(6)]
        pics.append(np.random.default_rng(7).integers(0, 256, (700, 900, 3), dtype=np.uint8))
        pics.append(capture(mode_val, 1000 * mode_val + 6))
        of, m = [0, 0, 1, 1, 1, 2, 3, -1], 5
        if mode_val == 4:
            pics += [sample(n) for n in ("6bit/4_30_f0_627.jpg", "6bit/4_30_f2_246.jpg", "6bit/4_30_f0_177_ccm.jpg", "6bit/4_30_f2_734.jpg")]
            of += [5, 6, 5, 6]
            m = 7
        pics.append(clean_picture(mode_val))
        of.append(m)
        m += 1
        _batches[mode_val] = (pics, of, m)
    return _batches[mode_val]


def tensors(pics):
    import torch
    return [torch.from_numpy(np.ascontiguousarray(p)).cuda() for p in pics]


class Out:
    def __init__(self, ctx, n, m):
        import torch
        self.db = ctx.info.data_bytes
        self.chunks = torch.full((max(n, 1), self.db), 0xA5, dtype=torch.uint8, device="cuda")
        self.mask = torch.full((max(n, 1),), -1, dtype=torch.int32, device="cuda")
        self.status = torch.full((max(n, 1),), 7, dtype=torch.int32, device="cuda")
        self.flags = torch.full((max(n, 1),), 0xEE, dtype=torch.uint8, device="cuda")
        self.gchunks = torch.full((max(m, 1), self.db), 0x5A, dtype=torch.uint8, device="cuda")
        self.gmask = torch.full((max(m, 1),), -1, dtype=torch.int32, device="cuda")
        self.gused = torch.full((max(m, 1),), 9, dtype=torch.int32, device="cuda")
        self.n, self.m = n, m

    def pictures(self, ctx, d, flags):
        ctx.scan_extract_decode_chunks_pictures_dev(d, self.chunks.data_ptr(), self.mask.data_ptr(), self.status.data_ptr(),
                                                    self.flags.data_ptr(), flags=flags)

    def combined(self, ctx, d, of, m, flags):
        ctx.scan_extract_decode_chunks_combined_dev(d, of, m, self.chunks.data_ptr(), self.mask.data_ptr(), self.status.data_ptr(),
                                                    self.gchunks.data_ptr(), self.gmask.data_ptr(), self.gused.data_ptr(),
                                                    self.flags.data_ptr(), flags=flags)

    def host(self):
        n, m = self.n, self.m
        return dict(chunks=self.chunks[:n].cpu().numpy(), mask=self.mask[:n].cpu().numpy().view(np.uint32), status=self.status[:n].cpu().numpy(),
                    flags=self.flags[:n].cpu().numpy(), gchunks=self.gchunks[:m].cpu().numpy(), gmask=self.gmask[:m].cpu().numpy().view(np.uint32),
                    gused=self.gused[:m].cpu().numpy())


def twin_run(cb, mode_val, pics, of, m, flags):
    """the pictures call on one context and the combined call on its twin: both outputs, both contexts' CCM states and transforms"""
    import torch
    d = tensors(pics)
    res = []
    for combined in (False, True):
        ctx = cb.Context(mode_val, max_frames=max(len(pics), m, 1))
        out = Out(ctx, len(pics), m)
        torch.cuda.synchronize()
        if combined:
            out.combined(ctx, d, of, m, flags)
        else:
            out.pictures(ctx, d, flags)
        ctx.sync()
        h = out.host()
        h["ccm"] = ctx.get_ccm()
        h["transforms"] = ctx.camera_transforms(len(pics)) if pics else None
        try:                                                        # the matrices, or the refusal when the call took no fitted route
            h["frame_ccms"] = ctx.frame_ccms(len(pics))
        except cb.Cb200Error as e:
            h["frame_ccms"] = str(e)
        ctx.close()
        res.append(h)
    return res


def same(a, b):
    if isinstance(a, str) or isinstance(b, str):
        return a == b
    return (a is None) == (b is None) and (a is None or np.array_equal(a, b, equal_nan=np.asarray(a).dtype.kind == "f"))


@pytest.mark.parametrize("flagname", FLAGS)
@pytest.mark.parametrize("mode_val", MODES)
def test_pictures_equal_the_pictures_call_and_groups_the_rule(cb, mode_val, flagname):
    flags = flag_bits(cb, flagname)
    pics, of, m = batch(mode_val)
    want, got = twin_run(cb, mode_val, pics, of, m, flags)
    for k in ("chunks", "mask", "status", "flags", "ccm", "transforms", "frame_ccms"):
        assert same(want.get(k), got.get(k)), (mode_val, flagname, k)
    assert want["status"][6] == 0 and (want["status"][:6] > 0).all()                   # premise: a FAILURE picture, six captures
    assert got["gused"].tolist()[:5] == [2, 3, 1, 0, 0]
    assert got["gmask"][3] == 0 and got["gmask"][4] == 0 and not got["gchunks"][3:5].any()
    if flagname != "SHARPEN_IF_NEEDED":                     # premise: a picture K1 does not flag (the clean one, not sharpened)
        assert want["flags"][-1] == 0, (mode_val, flagname)
    sharpen = "needed" if flagname == "SHARPEN_IF_NEEDED" else "no"
    if flagname == "CC_FIT":
        per = fitted_cells(mode_val, pics, sharpen)
    else:
        per = [picture_cells(mode_val, p, sharpen, 1 if flagname == "CC_SIMPLE" else 0) for p in pics]
    assert [p[0] for p in per] == got["status"].tolist()
    mo = ORA.mode(mode_val)
    for g in range(m):
        rec, mask, used = group_expectation(mode_val, per, [i for i in range(len(pics)) if of[i] == g])
        assert (int(got["gmask"][g]), int(got["gused"][g])) == (mask, used), (mode_val, flagname, g)
        if rec is not None:
            rows = got["gchunks"][g].reshape(mo.chunks_per_frame, mo.chunk_size)[[q for q in range(mo.chunks_per_frame) if mask >> q & 1]]
            assert rec[0] == len(rows) * mo.chunk_size and np.array_equal(rows, rec[1][:len(rows)]), (mode_val, flagname, g)
    if mode_val in (68, 4) and flagname in ("none", "SHARPEN_IF_NEEDED"):            # the rescue groups decode every block
        full = (1 << mo.chunks_per_frame) - 1
        assert got["gmask"][:2].tolist() == [full] * 2
        if flagname == "none":                                                     # premise (the oracle's, test_combine_fixtures)
            assert all(want["mask"][i] != full for i in range(6))


@pytest.mark.parametrize("flagname", FLAGS)
@pytest.mark.parametrize("mode_val", [68, 4])
def test_one_picture_and_repeated_pictures_give_that_pictures_record(cb, mode_val, flagname):
    """groups {0}, {1, 1, 1} (one tensor three times), {2}, and the FAILURE picture's group; two pictures outside every group"""
    flags = flag_bits(cb, flagname)
    pics, _, _ = batch(mode_val)
    sel = [pics[0], pics[1], pics[1], pics[1], pics[7], pics[2], pics[6], pics[3]]
    of = [0, 1, 1, 1, -1, 2, 3, -1]
    want, got = twin_run(cb, mode_val, sel, of, 4, flags)
    assert same(want["chunks"], got["chunks"]) and same(want["mask"], got["mask"])
    assert got["gused"].tolist() == [1, 3, 1, 0]
    for g, i in ((0, 0), (1, 1), (2, 5)):
        assert got["gmask"][g] == want["mask"][i] and np.array_equal(got["gchunks"][g], want["chunks"][i]), (mode_val, flagname, g)
    assert got["gmask"][3] == 0 and not got["gchunks"][3].any()
    # pictures outside every group touch no group: the same groups without them
    keep = [i for i in range(len(sel)) if of[i] >= 0]
    _, alone = twin_run(cb, mode_val, [sel[i] for i in keep], [of[i] for i in keep], 4, flags)
    for k in ("gchunks", "gmask", "gused"):
        assert same(alone[k], got[k]), k


def test_without_groups_it_is_the_pictures_call(cb):
    pics, _, _ = batch(68)
    want, got = twin_run(cb, 68, pics, None, 0, cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT)
    for k in ("chunks", "mask", "status", "flags", "ccm", "transforms", "frame_ccms"):
        assert same(want.get(k), got.get(k)), k
    lib = cb.load_library()
    ctx = cb.Context(68, max_frames=len(pics))
    out = Out(ctx, len(pics), 3)
    d = tensors(pics)
    before = lib.cb200_launch_count()
    out.pictures(ctx, d, 0)
    mid = lib.cb200_launch_count()
    out.combined(ctx, d, [-1] * len(pics), 0, 0)
    end = lib.cb200_launch_count()
    ctx.sync()
    assert end - mid == mid - before
    ctx.close()


def test_groups_of_an_empty_batch_are_empty(cb):
    ctx = cb.Context(68, max_frames=4)
    out = Out(ctx, 0, 3)
    out.combined(ctx, [], [], 3, 0)
    ctx.sync()
    h = out.host()
    assert h["gmask"].tolist() == [0, 0, 0] and h["gused"].tolist() == [0, 0, 0] and not h["gchunks"].any()
    ctx.close()


def test_refusals_that_need_a_context(cb):
    pics, of, m = batch(68)
    ctx = cb.Context(68, max_frames=len(pics))
    out = Out(ctx, len(pics), len(pics) + 1)
    d = tensors(pics)
    with pytest.raises(cb.Cb200Error, match=r"m = %d > max_frames = %d" % (len(pics) + 1, len(pics))):
        out.combined(ctx, d, of, len(pics) + 1, 0)
    with pytest.raises(cb.Cb200Error, match="null output"):
        ctx.scan_extract_decode_chunks_combined_dev(d, of, m, 0, out.mask.data_ptr(), out.status.data_ptr(), out.gchunks.data_ptr(),
                                                    out.gmask.data_ptr(), out.gused.data_ptr())
    ctx.close()


def test_calls_only_enqueue_with_four_launches_more(cb):
    """two combined calls queued behind a sleeping stream return at once, equal the same calls run alone, and each launches four
    kernels more than the pictures call on the same batch"""
    import torch
    pics, of, m = batch(4)
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    lib = cb.load_library()
    d = tensors(pics)
    ctx = cb.Context(4, max_frames=len(pics))
    twin = cb.Context(4, max_frames=len(pics))
    outs = [Out(ctx, len(pics), m) for _ in range(2)]
    ref = Out(twin, len(pics), m)
    def start(c):                                                   # every buffer at its size, then no CCM
        outs[0].combined(c, d, of, m, flags)
        c.sync()
        c.set_ccm(None)
        c.sync()
    start(twin)
    want = []
    for _ in range(2):
        outs[0].combined(twin, d, of, m, flags)
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
        o.combined(ctx, d, of, m, flags)
    c1 = lib.cb200_launch_count()
    spent = time.perf_counter() - t0
    busy = not stream.query()
    ctx.sync()
    assert busy, "the stream finished before the calls returned"
    assert spent < 0.25, spent
    assert c1 - c0 == 2 * ((n1 - n0) + 4)
    for o, w in zip(outs, want):
        h = o.host()
        for k in w:
            assert np.array_equal(h[k], w[k]), k
    ctx.close()
    twin.close()
