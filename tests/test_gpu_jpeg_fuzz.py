"""The generated JPEG corpus of tests/jpeg_fuzz.py decoded on the device (cb200_jpeg_decode_dev): every picture the call accepts
(short side 60 or more) is cv2.imread + cvtColor(BGR2RGB)'s bytes with status 0, and nothing is written past the last picture --
the whole corpus in one call, the largest files among the smallest, and one call per restart interval.  The damaged files of the
host test, and every byte value after an orphaned FF, get the host build's verdict: status -2, or status 0 and cv2's picture of
the same bytes (unless the host build finds IDCT blocks outside the range where libjpeg-turbo's C and SIMD IDCTs agree)."""
import numpy as np
import pytest

from jpeg_fuzz import corpus, mutations, orphaned_ff, restart_class, walk
from jpeg_matrix import cv2_rgb
from cpu_support import core, decode_wide  # noqa: F401

pytestmark = pytest.mark.gpu

FILES = corpus()
DEV = [(n, d) for n, d in FILES if min(walk(d)["size"]) >= 60]
SLACK = 4096


@pytest.fixture(scope="module")
def ctx():
    import libcimbar_b200 as cb
    c = cb.Context(4, max_frames=1)
    yield c
    c.close()


def decode_dev(ctx, files):
    """[(rgb, status)] of one cb200_jpeg_decode_dev call into a buffer of 0xA5 bytes; asserts the SLACK bytes after the last
    picture are untouched"""
    import libcimbar_b200 as cb
    import torch
    shapes = [cb.jpeg_info(f) for f in files]
    total = sum(3 * w * h for w, h in shapes)
    out = torch.full((total + SLACK,), 0xA5, dtype=torch.uint8, device="cuda")
    status = torch.full((len(files),), 7, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    ctx.jpeg_decode_dev(files, out.data_ptr(), status.data_ptr())
    ctx.sync()
    host, st = out.cpu().numpy(), status.cpu().numpy()
    assert (host[total:] == 0xA5).all(), "written past the last picture"
    res, at = [], 0
    for (w, h), s in zip(shapes, st):
        res.append((host[at:at + 3 * w * h].reshape(h, w, 3), int(s)))
        at += 3 * w * h
    return res


def check(ctx, files):
    got = decode_dev(ctx, [d for _, d in files])
    for (name, data), (rgb, st) in zip(files, got):
        want = cv2_rgb(data)
        assert st == 0, name
        assert rgb.shape == want.shape and np.array_equal(rgb, want), (name, int(np.count_nonzero(rgb != want)))


def test_premise_the_device_gets_most_of_the_corpus():
    assert len(DEV) >= 150 and {restart_class(walk(d)["restart"]) for _, d in DEV} == {0, 1, 2, 7, "large"}


def test_whole_corpus_in_one_call(ctx):
    check(ctx, DEV)


def test_largest_among_smallest(ctx):
    by_size = sorted(DEV, key=lambda f: np.prod(walk(f[1])["size"]))
    small, large = by_size[:4], by_size[-4:]
    assert min(np.prod(walk(d)["size"]) for _, d in large) >= 3000 * 2000 and max(np.prod(walk(d)["size"]) for _, d in small) <= 61 * 61
    check(ctx, [small[0], large[0], small[1], small[2], large[1], large[2], small[3], large[3]])


@pytest.mark.parametrize("rst", [0, 1, 2, 7, "large"])
def test_one_call_per_restart_interval(ctx, rst):
    files = [(n, d) for n, d in DEV if restart_class(walk(d)["restart"]) == rst]
    assert len(files) >= 10
    check(ctx, files)


@pytest.mark.parametrize("which", ["mutations", "orphaned_ff"])
def test_damaged_files_get_the_host_verdict(ctx, core, which):  # noqa: F811
    """status -2, or status 0 and cv2's picture of the same bytes -- and the same status as the host build of the decoder"""
    damaged = mutations(FILES) if which == "mutations" else orphaned_ff(FILES)
    got = decode_dev(ctx, [d for _, d in damaged])
    for (name, data), (rgb, st) in zip(damaged, got):
        rc, wide, want = decode_wide(core, data)
        assert st == rc and st in (0, -2), (name, st, rc)
        if st == 0:
            assert np.array_equal(rgb, want), name
            if wide == 0:
                assert np.array_equal(rgb, cv2_rgb(data)), name
    assert {st for _, st in got} == {0, -2}
