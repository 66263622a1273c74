"""The fixtures of the combined camera call, on the CPU oracle (tests/combine_fixtures.py).

Synthetic captures: every capture alone fails some Reed-Solomon blocks and every group of two or three decodes all of them, in
modes 68 and 4, so the GPU tests' rescue groups cannot silently stop being rescues.

The sample photographs hold two pairs of pictures of one frame (mode 4).  Per-block ok counts, sharpened as the CLI's default
`--preprocess -1` does, under colour correction 0 and 1 (the oracle restates no other per cell):

| pair | cc | first alone | second alone | combined |
|---|---|---|---|---|
| f0_627 + f0_177_ccm | 0 | 60 | 0 | 0 |
| f0_627 + f0_177_ccm | 1 | 60 | 28 | 58 |
| f2_246 + f2_734 | 0, 1 | 60 | 60 | 60 |

So the frame-0 pair is no rescue: with two pictures a cell goes to the lower symbol distance, which cannot see that 177_ccm's
colours are wrong.  The frame-2 pictures decode fully on their own, and their group record is theirs."""
import numpy as np
import pytest

from combine_fixtures import ORA, capture, cells_record, clean_picture, extract, fitted_cells, picture_cells, vote
from ragged_samples import sample

SEEDS = 6
GROUPS = [[0, 1], [2, 3], [4, 5], [0, 2, 4], [1, 3, 5]]


def synthetic(mode_val):
    return [picture_cells(mode_val, capture(mode_val, 1000 * mode_val + s)) for s in range(SEEDS)]


def blocks(mode_val, values):
    return int(cells_record(mode_val, values)[3].sum())


def combined(mode_val, pp):
    return vote(np.stack([p[1] for p in pp]), np.stack([p[2] for p in pp]))


@pytest.mark.parametrize("mode_val", [68, 4])
def test_synthetic_captures_fail_alone_and_decode_combined(mode_val):
    m = ORA.mode(mode_val)
    nblocks = ORA.capacity(m) // m.ecc_block_size
    pp = synthetic(mode_val)
    assert all(p[0] in (1, 2) for p in pp)
    alone = [blocks(mode_val, p[1]) for p in pp]
    assert all(a < nblocks for a in alone), alone
    for g in GROUPS:
        assert blocks(mode_val, combined(mode_val, [pp[i] for i in g])) == nblocks, (g, alone)


PAIRS = {"f0": ["6bit/4_30_f0_627.jpg", "6bit/4_30_f0_177_ccm.jpg"], "f2": ["6bit/4_30_f2_246.jpg", "6bit/4_30_f2_734.jpg"]}
PINNED = {("f0", 0): (60, 0, 0), ("f0", 1): (60, 28, 58), ("f2", 0): (60, 60, 60), ("f2", 1): (60, 60, 60)}


@pytest.mark.parametrize("pair,cc", sorted(PINNED))
def test_real_pairs(pair, cc):
    pp = [picture_cells(4, sample(name), "needed", cc) for name in PAIRS[pair]]
    assert [p[0] for p in pp] == [2, 2]
    v = combined(4, pp)
    assert (blocks(4, pp[0][1]), blocks(4, pp[1][1]), blocks(4, v)) == PINNED[(pair, cc)]
    if pair == "f2":                                                 # both decode fully: the group record is theirs
        good, chunks, mask, _ = cells_record(4, v)
        for p in pp:
            g1, c1, m1, _ = cells_record(4, p[1])
            assert (good, mask) == (g1, m1) and np.array_equal(chunks, c1)


@pytest.mark.parametrize("mode_val,sharpen", [(68, "no"), (68, "needed"), (4, "needed"), (67, "no")])
def test_fitted_cells_give_the_cc2_records(mode_val, sharpen):
    """the colour correction 2 cells (fitted_cells: the oracle's CC 2 route, then its cells with the matrix that route installed)
    decode to exactly the record cbo_decode_fountain_cc gives each picture of a CLI-style batch"""
    pics = [capture(mode_val, 1000 * mode_val + s) for s in range(3)] + [clean_picture(mode_val)]
    if mode_val == 4:
        pics += [sample("6bit/4_30_f0_627.jpg"), sample("6bit/4_30_f0_177_ccm.jpg")]
    m = ORA.mode(mode_val)
    for i, (status, values, _, rec) in enumerate(fitted_cells(mode_val, pics, sharpen)):
        assert status in (1, 2), i
        good, chunks, mask, _ = cells_record(mode_val, values)
        k = good // m.chunk_size
        assert (good, mask) == rec[0::2] and np.array_equal(chunks[:k], rec[1][:k]), (mode_val, sharpen, i)


@pytest.mark.parametrize("mode_val", [68, 67, 66, 4, 8])
def test_the_clean_picture_extracts_to_its_frame(mode_val):
    """clean_picture's deskew is a whole-pixel translation of the cells, and the walk keeps every cell at the centre hash"""
    from combine_fixtures import base_frame
    f = base_frame(mode_val)
    status, frame = extract(mode_val, clean_picture(mode_val))
    assert status in (1, 2) and np.array_equal(frame[70:-70, 70:-70], f[70:-70, 70:-70])
    _, cells = ORA.decode_raw(ORA.mode(mode_val), frame, want_cells=True)
    assert (cells["drift_offset"] == 4).all()
