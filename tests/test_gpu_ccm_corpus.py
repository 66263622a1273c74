"""The kernels of the colour-correction side path against cv2 and the numpy models of ccm_corpus.py, on its corpus: k_ccm_fit
(through cb200_fit_ccm with a given header, on painted frames of every mode with colour bits, every row count the header search
reaches), the CC_FIT batch path with grey and channel-saturated frames (the carry of a 1e7 fit), k_ccm_simple on anchor whites whose
von Kries denominator is 0.0f, and best_color_ccm (cb200_best_colors, K1's CM = 1 variant, k_flood_colour) under every corpus
matrix.  Every comparison is exact, NaN positions included.  tests/test_ccm_contract.py pins the oracle and the models to cv2 on
the CPU."""
import cv2
import numpy as np
import pytest

import ccm_corpus as cc
from gpu_support import synth_frames
from oracle_lib import Oracle, load_sample

pytestmark = pytest.mark.gpu

ORA = Oracle()
FITS = cc.fit_cases()
PALETTE = {68: (4, 1), 4: (4, 0), 8: (8, 0)}
FULL_GRID = ["fit-grey-0-n5-c8m0", "nan-row0", "nan-row2", "identity", "minus-identity", "1e30 I", "simple-zero-row1-issue"]


def same(a, b):
    a, b = np.asarray(a, np.float32).reshape(-1), np.asarray(b, np.float32).reshape(-1)
    na, nb = np.isnan(a), np.isnan(b)
    return a.shape == b.shape and np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))


def grey(rgb):
    return cv2.cvtColor(cv2.cvtColor(rgb, cv2.COLOR_RGB2GRAY), cv2.COLOR_GRAY2RGB)


def saturated(rgb):
    out = rgb.copy()
    out[..., 1] = 255
    out[..., 2] = 0
    return out


@pytest.fixture(scope="module")
def cb():
    import libcimbar_b200 as cb
    return cb


@pytest.mark.parametrize("mode_val", cc.COLOUR_MODES)
def test_fit_ccm_on_painted_frames(cb, mode_val):
    m = ORA.mode(mode_val)
    ctx = cb.Context(mode_val, max_frames=1)
    frames = cc.painted_frames(mode_val)
    reached = sorted({int(p.name.split("-")[1][4:]) for p in frames})
    print(f"mode {mode_val}: row counts reached {reached}")
    for p in frames:
        hdr = np.frombuffer(p.hdr, np.uint8)
        got = ctx.fit_ccm(p.frame, hdr, p.radioactive)
        want = ORA.init_ccm(m, p.frame, hdr, p.radioactive)
        if p.actual is None:
            assert got is None and want is None, p.name
            continue
        ref = cc.cv2_fit(p.actual, p.desired)
        assert same(want, ref), f"{p.name}: oracle\n{want}\ncv2\n{ref}"
        if m.legacy_mode:
            # the legacy modes decode symbol and colour bits coupled (Decoder::do_decode_coupled), which never calls init_ccm:
            # the context has no colour stream to fit from and reports no fit
            assert got is None, p.name
            continue
        assert got is not None, p.name
        assert same(got, ref), f"{p.name}: device\n{got}\ncv2\n{ref}\nrows\n{p.actual}"
    ctx.close()


def _oracle_batch(m, frames, initial=None):
    ORA.set_ccm(initial)
    out = []
    try:
        for fr in frames:
            good, chunks, mask = ORA.decode_fountain(m, fr, color_correction=2)
            out.append((good, chunks.copy(), mask, ORA.get_ccm()))
    finally:
        ORA.set_ccm(None)
    return out


def test_cc_fit_batches_with_grey_and_saturated_frames(cb):
    """a frame without a header after a grey one decodes with the grey frame's ~1e7 fit, in the batch and into the next call"""
    m = ORA.mode(68)
    rng = np.random.default_rng(3)
    tr0, tr1, ex = (load_sample(s) for s in ("b/tr_0.png", "b/tr_1.png", "b/ex380.jpg"))
    noise = rng.integers(0, 256, tr0.shape, dtype=np.uint8)
    frames = np.stack([tr0, grey(tr0), noise, tr1, saturated(tr1), grey(ex), noise, ex, grey(tr1), saturated(tr0)])
    want = _oracle_batch(m, frames)
    assert np.abs(want[2][3]).max() > 1e5                       # the carried wild fit
    ctx = cb.Context(68, max_frames=len(frames))
    chunks, counts, masks, _ = ctx.decode_fountain(frames, flags=cb.FLAG_CC_FIT)
    used = ctx.frame_ccms(len(frames))
    for f, (good, wchunks, wmask, wccm) in enumerate(want):
        assert masks[f] == wmask and counts[f] * m.chunk_size == good, (f, hex(masks[f]), hex(wmask))
        assert np.array_equal(chunks[f][:counts[f]], wchunks[:counts[f]]), f
        assert wccm is not None and same(used[f], wccm), (f, used[f], wccm)
    assert same(ctx.get_ccm(), want[-1][3])
    again = _oracle_batch(m, frames[2:3], initial=want[1][3])   # a grey frame's fit carried into the next call
    ctx.set_ccm(want[1][3])
    chunks2, counts2, masks2, _ = ctx.decode_fountain(frames[2:3], flags=cb.FLAG_CC_FIT)
    assert masks2[0] == again[0][2] and same(ctx.get_ccm(), again[0][3])
    ctx.close()


def _anchor_white_frame(base, white):
    frame = base.copy()
    for ax, ay in ((28, 28), (28, 992), (992, 28)):
        for c in range(3):
            s = int(round(white[c] * 16))
            px = np.full(16, s // 16, np.uint8)
            px[: s % 16] += 1
            frame[ay:ay + 4, ax:ax + 4, c] = px.reshape(4, 4)
    return frame


def test_cc_simple_on_corpus_whites(cb):
    m = ORA.mode(68)
    _, _, clean = synth_frames(68, 1, seed=71)
    whites = cc.simple_whites()
    frames = np.stack([_anchor_white_frame(clean[0], w) for _, w, _ in whites])
    ctx = cb.Context(68, max_frames=1)
    for f, (name, white, premise) in enumerate(whites):
        raw, _ = ctx.decode_raw(frames[f], flags=cb.FLAG_CC_SIMPLE)
        want_m = cc.von_kries(white)
        assert same(ctx.get_ccm(), want_m), f"{name}: device\n{ctx.get_ccm()}\nmodel\n{want_m.reshape(3, 3)}"
        try:
            want = ORA.decode_raw(m, frames[f], color_correction=1)
        finally:
            ORA.set_ccm(None)
        bad = np.nonzero(raw[0] != want)[0]
        assert bad.size == 0, f"{name}: byte {bad[0]}: device {raw[0][bad[0]]}, oracle {want[bad[0]]}"
    ctx.close()


def _classify(cb, ctx, mode_val, name, M, means):
    ctx.set_ccm(M.reshape(3, 3))
    got = ctx.best_colors(means)
    for lo in range(0, len(means), 1 << 20):
        want = cc.best_color(M, means[lo:lo + (1 << 20)], *PALETTE[mode_val])
        bad = np.nonzero(got[lo:lo + len(want)] != want)[0]
        if bad.size:
            i = lo + int(bad[0])
            r, g, b = (float(x) for x in means[i])
            row = [float(np.float32(np.float32(np.float32(M[3 * k] * r) + np.float32(M[3 * k + 1] * g)) + np.float32(M[3 * k + 2] * b)))
                   for k in range(3)]
            pytest.fail(f"{name} mode {mode_val}: mean {means[i].tolist()} (transformed {row}): device {got[i]}, model {want[bad[0]]}")


def test_best_colors_on_every_mean_for_the_edge_matrices(cb):
    mats = dict(cc.classifier_matrices(FITS))
    v = np.arange(256, dtype=np.uint8)
    means = np.stack(np.meshgrid(v, v, v, indexing="ij"), -1).reshape(-1, 3)
    ctx = cb.Context(68, max_frames=1)
    for name in FULL_GRID:
        _classify(cb, ctx, 68, name, mats[name], means)
    ctx.close()


@pytest.mark.parametrize("mode_val", [68, 8])
def test_best_colors_on_seeded_means_for_every_matrix(cb, mode_val):
    rng = np.random.default_rng(mode_val)
    means = rng.integers(0, 256, (1 << 16, 3), dtype=np.uint8)
    ctx = cb.Context(mode_val, max_frames=1)
    for name, M in cc.classifier_matrices(FITS):
        _classify(cb, ctx, mode_val, name, M, means)
    ctx.close()


@pytest.mark.parametrize("mode_val", [68, 8])
def test_decode_raw_under_corpus_matrices(cb, mode_val):
    """K1's CM = 1 variant on a clean synthetic frame and, in mode 68, k_flood_colour on a camera frame"""
    m = ORA.mode(mode_val)
    _, _, clean = synth_frames(mode_val, 1, seed=73)
    frames = [("clean", clean[0])] + ([("ex380", load_sample("b/ex380.jpg"))] if mode_val == 68 else [])
    mats = cc.hand_matrices() + [(n, M) for n, M in cc.classifier_matrices(FITS) if n in FULL_GRID or n.startswith("simple-zero")][:12]
    ctx = cb.Context(mode_val, max_frames=1)
    for name, M in mats:
        ctx.set_ccm(M.reshape(3, 3))
        ORA.set_ccm(M)
        try:
            for what, fr in frames:
                raw, ff = ctx.decode_raw(fr)
                want = ORA.decode_raw(m, fr)
                bad = np.nonzero(raw[0] != want)[0]
                assert bad.size == 0, f"{name} on {what}: byte {bad[0]}: device {raw[0][bad[0]]}, oracle {want[bad[0]]}"
        finally:
            ORA.set_ccm(None)
    ctx.close()
