"""The colour-correction side path of the CPU oracle (oracle/cimbar_oracle.c) against OpenCV and plain numpy, on the corpus of
ccm_corpus.py: the CC_FIT least-squares fit against cv2.invert(DECOMP_SVD) + cv2.gemm, the CC_SIMPLE von Kries matrix and the
colour decision under a CCM against float32 numpy models, init_ccm on painted frames, and the fit a colour_correction = 2
decode leaves on grey versions of the sample frames.  Every comparison is exact (NaN positions included).  The GPU side
(tests/test_gpu_ccm_corpus.py) compares the kernels with the same references.

The grey family and the grey sample decodes are the ones that catch a back-substitution threshold of FLT_EPSILON's scale: their
residual singular value (~1e-8 of the sum) lies in the band OpenCV inverts and that threshold drops."""
import cv2
import numpy as np
import pytest

import ccm_corpus as cc
from oracle_lib import Oracle, load_sample, manifest

ORA = Oracle()
FITS = cc.fit_cases()


def _fmt_matx(mat):
    """operator<<(std::ostream&, cv::Matx<float,3,3>): "%.8g" elements, ", " / ";\n " separators"""
    return "[" + ";\n ".join(", ".join("%.8g" % float(x) for x in row) for row in np.asarray(mat).reshape(3, 3)) + "]"


def same(a, b):
    """bit for bit, with every NaN equal to every NaN"""
    a, b = np.asarray(a, np.float32).reshape(-1), np.asarray(b, np.float32).reshape(-1)
    na, nb = np.isnan(a), np.isnan(b)
    return a.shape == b.shape and np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))


def grey(rgb):
    return cv2.cvtColor(cv2.cvtColor(rgb, cv2.COLOR_RGB2GRAY), cv2.COLOR_GRAY2RGB)


@pytest.mark.parametrize("idx", range(2))
def test_cv2_fit_reproduces_the_reference_strings(idx):
    """cv2_fit is the reference's arithmetic: color_correctionTest.cpp's printed matrices, digit for digit"""
    g = manifest()["moore_penrose_goldens"][idx]
    assert _fmt_matx(cc.cv2_fit(g["actual"], g["desired"])) == g["matrix_str"]


@pytest.mark.parametrize("family", cc.FAMILIES)
def test_oracle_fit_equals_cv2(family):
    cases = [c for c in FITS if c.family == family]
    assert len(cases) >= 40 and {c.rows for c in cases} == set(range(5, 10))
    for c in cases:
        assert c.holds(), f"{c.name}: the premise '{c.premise}' does not hold: W = {cc.singular_values(c.actual)}"
        got, want = ORA.moore_penrose_lsm(c.actual, c.desired), cc.cv2_fit(c.actual, c.desired)
        assert same(got, want), f"{c.name}: oracle\n{got}\ncv2\n{want}\nW = {cc.singular_values(c.actual)}"


def test_the_corpus_reaches_every_edge_of_the_back_substitution():
    per = {f: cc.premise_counts([c for c in FITS if c.family == f]) for f in cc.FAMILIES}
    total = cc.premise_counts(FITS)
    assert all(v > 0 for v in total.values()), total
    for f in ("grey", "near_grey", "low_channels", "high_channels"):
        assert per[f]["band"] > 0, (f, per[f])
    # the fits in the band are the wild ones: entries of 1e5 and more
    wild = [c for c in FITS if cc.PREMISES["band"][1](cc.singular_values(c.actual))]
    assert all(np.abs(cc.cv2_fit(c.actual, c.desired)).max() > 1e5 for c in wild if c.family == "grey")


def test_simple_ccm_equals_von_kries():
    g = manifest()["adaptation_golden"]
    assert same(ORA.adaptation_matrix(g["actual"], g["desired"]), cc.von_kries(g["actual"], g["desired"]))
    whites = cc.simple_whites()
    assert sum(p == "zero" for _, _, p in whites) >= 20
    for name, white, premise in whites:
        want = cc.von_kries(white)
        assert same(ORA.adaptation_matrix(white, (255, 255, 255)), want), name
        zero = (cc.von_kries_denominators(white) == 0).any()
        assert zero == (premise == "zero"), name
        assert np.isfinite(want).all() != zero, name
    # the oracle's CC_SIMPLE entry computes its white from the anchor patches: the same matrix
    m = ORA.mode(68)
    frame = np.zeros((1024, 1024, 3), np.uint8)
    for name, white, _ in whites:
        for ax, ay in ((28, 28), (28, 992), (992, 28)):
            for c in range(3):
                s = int(round(white[c] * 16))
                px = np.full(16, s // 16, np.uint8)
                px[: s % 16] += 1
                frame[ay:ay + 4, ax:ax + 4, c] = px.reshape(4, 4)
        assert same(ORA.simple_ccm(m, frame), cc.von_kries(white)), name


@pytest.mark.parametrize("key", [(4, 1), (4, 0), (8, 0)], ids=lambda k: f"{k[0]}colours-mode{k[1]}")
def test_best_color_equals_the_model(key):
    rng = np.random.default_rng(7)
    means = np.concatenate([rng.integers(0, 256, (4096, 3)), [[0, 0, 0], [255, 255, 255], [1, 1, 1], [48, 48, 48], [0, 255, 0]]]).astype(np.uint8)
    mats = cc.classifier_matrices(FITS)
    nan0 = 0
    for name, M in mats:
        want = cc.best_color(M, means, *key)
        got = ORA.best_colors(means, *key, M)
        bad = np.nonzero(got != want)[0]
        assert bad.size == 0, f"{name}: mean {means[bad[0]].tolist()}: oracle {got[bad[0]]}, model {want[bad[0]]}"
        nan0 += bool(np.isnan(M[:3]).any())
    assert nan0 >= 2                       # the NaN-in-r rule is exercised (hand-made and CC_SIMPLE matrices)


@pytest.mark.parametrize("mode_val", cc.COLOUR_MODES)
def test_init_ccm_on_painted_frames(mode_val):
    m = ORA.mode(mode_val)
    frames = cc.painted_frames(mode_val)
    rows = {p.name.split("-")[1] for p in frames}
    assert rows == ({"rows6", "rows7", "rows8", "rows9"} if mode_val == 8 else {"rows0", "rows5"}), rows
    for p in frames:
        got = ORA.init_ccm(m, p.frame, np.frombuffer(p.hdr, np.uint8), p.radioactive)
        if p.actual is None:
            assert got is None, p.name
            continue
        a, d = ORA.last_fit_rows()
        assert np.array_equal(a, p.actual) and np.array_equal(d, p.desired), p.name
        assert got is not None and same(got, cc.cv2_fit(p.actual, p.desired)), p.name


@pytest.mark.parametrize("sample", ["b/tr_0.png", "b/tr_1.png", "b/ex380.jpg"])
def test_grey_sample_decode_leaves_cv2s_fit(sample):
    """a monochrome capture of a colour frame: init_ccm's rows are grey, so the fit is in the band (entries ~1e6..1e7)"""
    m = ORA.mode(68)
    ORA.set_ccm(None)
    try:
        good, _, mask = ORA.decode_fountain(m, grey(load_sample(sample)), color_correction=2)
        mat = ORA.get_ccm()
        actual, desired = ORA.last_fit_rows()
    finally:
        ORA.set_ccm(None)
    assert mat is not None and len(actual) == 5
    assert cc.PREMISES["band"][1](cc.singular_values(actual)), cc.singular_values(actual)
    assert same(mat, cc.cv2_fit(actual, desired)) and np.abs(mat).max() > 1e5, mat
    assert mask == 0xFF and good == 8 * m.chunk_size
