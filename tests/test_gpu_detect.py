"""The receiver's auto mode (cb200_detect_scan_extract_decode_chunks_dev): one call decodes a camera batch under several candidate
modes, with the scan done once and one exact walk per frame geometry.
  - mixed mode-B and 4C photographs and a noise picture are detected as 68, 4 and -1, with the records of the reference CLI's loop
    in the detected mode;
  - rendered 66 and 67 frames, as camera pictures, are detected as their own modes;
  - for every flag combination of the camera tests and several candidate sets, each context ends exactly where a direct call on
    it would: masks, records, statuses, transforms and the CCM carried over two calls;
  - the walk runs once per geometry (one for 68 / 4 / 8, three for 66 / 68 / 67 / 4), and the geometries' walks overlap."""
import numpy as np
import pytest

from oracle_lib import load_sample
from ragged_samples import GLOB, sample
from gpu_support import cb  # noqa: F401  (fixtures)
from gpu_support import Detect, FLAGS, ORA, RECV, cli_loop, contexts, dense, detect, exact_pictures, mixed_pictures, packed, rendered

pytestmark = pytest.mark.gpu


def direct(cb, ctx, pics, flags):
    import torch
    d, wh = packed(pics)
    n, db = len(pics), ctx.info.data_bytes
    chunks = torch.zeros(n * db, dtype=torch.uint8, device="cuda")
    mask = torch.zeros(n, dtype=torch.int32, device="cuda")
    status = torch.zeros(n, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    ctx.scan_extract_decode_chunks_dev(d.data_ptr(), wh, chunks.data_ptr(), mask.data_ptr(), status.data_ptr(), flags=flags)
    ctx.sync()
    return chunks.cpu().numpy().reshape(n, db), mask.cpu().numpy().view(np.uint32), status.cpu().numpy()


def check_selected(ctxs, got, want):
    """the selection rule over the direct results `want` (one (chunks, mask, status) per context)"""
    chunks, mask, status, mode, mode_masks = got
    for i in range(len(mode)):
        masks = [int(w[1][i]) for w in want]
        assert mode_masks[i].tolist() == masks, i
        first = next((k for k, v in enumerate(masks) if v), -1)
        assert mode[i] == first, i
        k = max(first, 0)
        assert status[i] == want[k][2][i], i
        if first < 0:
            assert mask[i] == 0 and not chunks[i].any(), i
            continue
        db = ctxs[first].info.data_bytes
        assert mask[i] == masks[first], i
        assert np.array_equal(chunks[i, :db], want[first][0][i]), i
        assert not chunks[i, db:].any(), i


# ------------------------------------------------------------------------------------------------ detection
def test_mixed_photographs_are_detected_with_the_cli_records(cb):
    pics, kinds = mixed_pictures()
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    ctxs = contexts(cb, RECV, len(pics))
    try:
        chunks, mask, status, mode, _ = detect(cb, ctxs, pics, flags)
        loops = {m: cli_loop(m, "detect-mixed", pics, 2, "needed")[0] for m in (68, 4)}
        found = {"b": 0, "4c": 0}
        for i, kind in enumerate(kinds):
            if kind == "noise":
                assert mode[i] == -1 and mask[i] == 0, i
                continue
            mv = 68 if kind == "b" else 4
            st, _, wd = loops[mv][i]
            if st == 0 or wd[0] == 0:                    # the CLI gets nothing from this picture in its own mode either
                assert mode[i] == -1 or RECV[mode[i]] != mv, i
                continue
            assert RECV[mode[i]] == mv, (i, kind, mode[i])
            found[kind] += 1
            m = ORA.mode(mv)
            cnt, rows = dense(m, chunks[i, :ctxs[RECV.index(mv)].info.data_bytes], int(mask[i]))
            good, wchunks, wmask = wd
            assert status[i] == st and mask[i] == wmask and cnt * m.chunk_size == good, i
            assert np.array_equal(rows, wchunks[:cnt]), i
        assert found["b"] >= 4 and found["4c"] >= 3, found          # premise: both kinds decode
    finally:
        for c in ctxs:
            c.close()


@pytest.mark.parametrize("mode_val", [66, 67])
def test_rendered_frames_are_detected_as_their_mode(cb, mode_val):
    pics = rendered(cb, mode_val)
    flags = cb.FLAG_SHARPEN_IF_NEEDED
    ctxs = contexts(cb, RECV, len(pics))
    refs = [cb.Context(m, max_frames=len(pics)) for m in RECV]
    try:
        got = detect(cb, ctxs, pics, flags)
        want = [direct(cb, r, pics, flags) for r in refs]
        assert all(want[RECV.index(mode_val)][1] != 0)                # premise: the pictures decode in their own mode
        assert [RECV[k] for k in got[3]] == [mode_val] * len(pics)
        check_selected(ctxs, got, want)
    finally:
        for c in ctxs + refs:
            c.close()


# ------------------------------------------------------------------------------------------------ exactness
SETS = [RECV, [4, 67, 68, 66], [68, 4, 8]]


@pytest.mark.parametrize("modes", SETS, ids=lambda s: "-".join(map(str, s)))
@pytest.mark.parametrize("sflag,ccflag", FLAGS)
def test_each_context_ends_where_a_direct_call_leaves_it(cb, modes, sflag, ccflag):
    flags = (getattr(cb, "FLAG_" + sflag) if sflag else 0) | (getattr(cb, "FLAG_" + ccflag) if ccflag else 0)
    pics = exact_pictures(cb)
    batches = [pics, pics[5:] + pics[:5]]                 # two calls: the CCM carries from the first into the second
    n = len(pics)
    ctxs = contexts(cb, modes, n)
    refs = [cb.Context(m, max_frames=n) for m in modes]
    try:
        for b in batches:
            got = detect(cb, ctxs, b, flags)
            want = [direct(cb, r, b, flags) for r in refs]
            check_selected(ctxs, got, want)
            for c, r in zip(ctxs, refs):
                assert np.array_equal(c.camera_transforms(n), r.camera_transforms(n)), c.info.mode_val
        assert any(got[3] >= 0) and any(got[3] < 0)              # premise: some pictures are detected, the noise is not
        for c, r in zip(ctxs, refs):
            a, b = c.get_ccm(), r.get_ccm()
            assert (a is None) == (b is None) and (a is None or np.array_equal(a, b)), c.info.mode_val
            if ccflag == "CC_FIT" and not c.info.legacy_mode:
                fa, fb = c.frame_ccms(n), r.frame_ccms(n)
                assert all(np.array_equal(x, y) for x, y in zip(fa, fb)), c.info.mode_val
    finally:
        for c in ctxs + refs:
            c.close()


# ------------------------------------------------------------------------------------------------ sharing
def walks(cb, fn):
    """the exact-walk kernels fn() launches: their (start, end) in the trace"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = []
    for e in prof.events():
        if "k_flood_walk" in e.name and e.device_type == torch.autograd.DeviceType.CUDA:
            out.append((e.time_range.start, e.time_range.end))
    return sorted(out)


@pytest.mark.parametrize("modes,geometries", [([68, 4, 8], 1), (RECV, 3)], ids=["one-geometry", "three-geometries"])
def test_one_walk_per_geometry(cb, modes, geometries):
    import torch
    pics = [load_sample("b/ex2434.jpg"), sample(GLOB[0])]
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    d, wh = packed(pics)
    ctxs = contexts(cb, modes, len(pics))
    out = Detect(ctxs, len(pics))
    try:
        for _ in range(2):                                # warm-up: buffers grown, side streams created
            out.call(cb, ctxs, d, wh, flags)
        ctxs[0].sync()
        got = walks(cb, lambda: (out.call(cb, ctxs, d, wh, flags), ctxs[0].sync()))
        assert len(got) == geometries, got
        outs = [torch.zeros(len(pics) * 8750, dtype=torch.uint8, device="cuda") for _ in ctxs]
        words = torch.zeros(4 * len(pics), dtype=torch.int32, device="cuda")

        def directs():
            for c, o in zip(ctxs, outs):
                c.scan_extract_decode_chunks_dev(d.data_ptr(), wh, o.data_ptr(), words.data_ptr(), words.data_ptr(), flags=flags)
            ctxs[0].sync()
        assert len(walks(cb, directs)) == len(modes)
        if geometries > 1:                                # the walks of the geometries overlap on the device
            got = walks(cb, lambda: (out.call(cb, ctxs, d, wh, flags), ctxs[0].sync()))
            assert max(s for s, _ in got) < min(e for _, e in got), got
    finally:
        for c in ctxs:
            c.close()
