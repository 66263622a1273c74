"""Camera pictures in the caller's layout (cb200_scan_extract_decode_chunks_pictures_dev): BGR, RGBA, BGRA, planar and pitched RGB
pictures, each in its own allocation, at unaligned addresses and with rows padded with 0xFF, must give byte for byte what
cb200_scan_extract_decode_chunks_ragged_dev gives on the packed RGB batch -- chunks, masks, frame flags, statuses, transforms, the
CCM carried from batch to batch and the per-frame CCMs -- under every sharpen and colour-correction flag, with as many kernel
launches."""
import cv2
import numpy as np
import pytest

from oracle_lib import load_sample
from ragged_samples import GLOB, sample
from gpu_support import cb  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu


def odd_crop(rgb):
    return np.ascontiguousarray(rgb[3:-2, 1:-2])


def batches_4c():
    """the ragged samples (the golden photographs in glob order, with the 9-tap stand-in), an odd-sized crop and a noise picture of
    odd width, as two consecutive batches"""
    noise = np.random.default_rng(61).integers(0, 256, (899, 1201, 3), dtype=np.uint8)
    a = [sample(s) for s in GLOB[:4]] + [noise]
    b = [sample(s) for s in GLOB[4:]] + [odd_crop(load_sample("6bit/4_30_f0_627.jpg"))]
    return a, b


def batches_b():
    noise = np.random.default_rng(67).integers(0, 256, (700, 903, 3), dtype=np.uint8)
    ex1, ex2 = load_sample("b/ex2434.jpg"), load_sample("b/ex380.jpg")
    return [ex1, noise, ex2], [odd_crop(ex2), cv2.resize(ex1, None, fx=1.3, fy=1.3)]


LAYOUTS = ["rgb", "bgr", "rgba", "bgra", "planar"]


def placed(rgb, layout, shift, pad, seed=0):
    """rgb as a CUDA tensor in `layout` (cvtColor'd; alpha random), in an allocation of its own, starting `shift` bytes past an
    aligned address, each row (each plane's row) followed by `pad` bytes of 0xFF; returns (tensor, order)"""
    import torch
    h, w, _ = rgb.shape
    if layout == "planar":
        pitch = w + pad
        plane = h * pitch + 3 * pad
        buf = torch.full((shift + 3 * plane,), 0xFF, dtype=torch.uint8, device="cuda")
        t = torch.as_strided(buf, (3, h, w), (plane, pitch, 1), shift)
        t.copy_(torch.from_numpy(np.ascontiguousarray(rgb.transpose(2, 0, 1))))
        return t, "rgb"
    conv = {"rgb": rgb, "bgr": cv2.cvtColor(rgb, cv2.COLOR_RGB2BGR), "rgba": cv2.cvtColor(rgb, cv2.COLOR_RGB2RGBA),
            "bgra": cv2.cvtColor(rgb, cv2.COLOR_RGB2BGRA)}[layout]
    ch = conv.shape[2]
    if ch == 4:
        conv[:, :, 3] = np.random.default_rng(seed).integers(0, 256, (h, w), dtype=np.uint8)
    pitch = w * ch + pad
    buf = torch.full((shift + h * pitch,), 0xFF, dtype=torch.uint8, device="cuda")
    t = torch.as_strided(buf, (h, w, ch), (pitch, ch, 1), shift)
    t.copy_(torch.from_numpy(np.ascontiguousarray(conv)))
    return t, ("bgr" if layout in ("bgr", "bgra") else "rgb")


class Outputs:
    def __init__(self, ctx, n):
        import torch
        self.n, self.db = n, ctx.info.data_bytes
        self.chunks = torch.full((n * self.db,), 0xA5, dtype=torch.uint8, device="cuda")
        self.mask = torch.full((n,), -1, dtype=torch.int32, device="cuda")
        self.status = torch.full((n,), 7, dtype=torch.int32, device="cuda")
        self.flags = torch.full((n,), 0xEE, dtype=torch.uint8, device="cuda")

    def args(self):
        return self.chunks.data_ptr(), self.mask.data_ptr(), self.status.data_ptr(), self.flags.data_ptr()

    def host(self):
        return (self.chunks.cpu().numpy().reshape(self.n, self.db), self.mask.cpu().numpy(), self.status.cpu().numpy(),
                self.flags.cpu().numpy())


def results(cb, ctx, out, flags):
    """everything the call leaves behind, after it has run (the per-frame CCMs where CC_FIT fits them: not in the legacy 4C layout)"""
    ctx.sync()
    n = out.n
    r = {"out": out.host(), "transforms": ctx.camera_transforms(n), "ccm": ctx.get_ccm()}
    if flags & cb.FLAG_CC_FIT and ctx.info.legacy_mode == 0:
        r["frame_ccms"] = ctx.frame_ccms(n)
    return r


def run_packed(cb, ctx, pics, flags):
    import torch
    d = torch.cat([torch.from_numpy(np.ascontiguousarray(p).reshape(-1)) for p in pics]).cuda()
    wh = np.array([(p.shape[1], p.shape[0]) for p in pics], np.int32)
    out = Outputs(ctx, len(pics))
    torch.cuda.synchronize()
    before = cb.launch_count()
    ctx.scan_extract_decode_chunks_dev(d.data_ptr(), wh, *out.args()[:3], d_flags=out.args()[3], flags=flags)
    launches = cb.launch_count() - before
    return results(cb, ctx, out, flags), launches


def run_pictures(cb, ctx, pics, layouts, flags, seed):
    import torch
    placed_ = [placed(p, lay, (seed + i) % 4, (0, 1, 4, 7, 13)[(seed + 2 * i) % 5], seed + i) for i, (p, lay) in enumerate(zip(pics, layouts))]
    tensors = [t for t, _ in placed_]
    out = Outputs(ctx, len(pics))
    torch.cuda.synchronize()
    before = cb.launch_count()
    ctx.scan_extract_decode_chunks_pictures_dev(tensors, *out.args()[:3], d_flags=out.args()[3], flags=flags, order=[o for _, o in placed_])
    launches = cb.launch_count() - before
    return results(cb, ctx, out, flags), launches


def same(a, b, what):
    for x, y in zip(a["out"], b["out"]):
        assert np.array_equal(x, y), what
    assert np.array_equal(a["transforms"], b["transforms"]), what
    assert (a["ccm"] is None) == (b["ccm"] is None) and (a["ccm"] is None or np.array_equal(a["ccm"], b["ccm"])), what
    if "frame_ccms" in a:
        assert np.array_equal(a["frame_ccms"], b["frame_ccms"], equal_nan=True), what


_refs = {}


def reference(cb, mode_val, batches, name, flags):
    """the packed RGB call on each batch in turn, on one context (the CCM carries from the first batch into the second)"""
    key = (mode_val, name, flags)
    if key not in _refs:
        ctx = cb.Context(mode_val, max_frames=max(len(b) for b in batches))
        _refs[key] = [run_packed(cb, ctx, b, flags) for b in batches]
        ctx.close()
    return _refs[key]


def compare(cb, mode_val, batches, name, flags, layouts_of):
    want = reference(cb, mode_val, batches, name, flags)
    ctx = cb.Context(mode_val, max_frames=max(len(b) for b in batches))
    for k, b in enumerate(batches):
        got, launches = run_pictures(cb, ctx, b, layouts_of(k, len(b)), flags, seed=7 * k + flags)
        same(got, want[k][0], (name, flags, k))
        assert launches == want[k][1], (launches, want[k][1])
    ctx.close()
    return want


FLAGS = [("none", []), ("SHARPEN", ["SHARPEN"]), ("SHARPEN_IF_NEEDED", ["SHARPEN_IF_NEEDED"]),
         ("CC_SIMPLE", ["SHARPEN_IF_NEEDED", "CC_SIMPLE"]), ("CC_FIT", ["SHARPEN_IF_NEEDED", "CC_FIT"])]


def flag_bits(cb, names):
    f = 0
    for n in names:
        f |= getattr(cb, "FLAG_" + n)
    return f


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("fname,fnames", FLAGS, ids=[f[0] for f in FLAGS])
def test_each_layout_equals_the_packed_rgb_call(cb, layout, fname, fnames):
    flags = flag_bits(cb, fnames)
    want = compare(cb, 4, batches_4c(), "4c", flags, lambda k, n: [layout] * n)
    statuses = set(np.concatenate([w[0]["out"][2] for w in want]).tolist())
    assert statuses == {0, 1, 2}                                     # premise: failures, clean and NEEDS_SHARPEN pictures
    if flags & cb.FLAG_CC_SIMPLE:
        assert want[0][0]["ccm"] is not None                         # premise: a CCM carries into the second batch


@pytest.mark.parametrize("fname,fnames", [FLAGS[2], FLAGS[4]], ids=["SHARPEN_IF_NEEDED", "CC_FIT"])
def test_mixed_layouts_in_one_batch(cb, fname, fnames):
    flags = flag_bits(cb, fnames)
    compare(cb, 4, batches_4c(), "4c", flags, lambda k, n: [LAYOUTS[(i + 2 * k) % 5] for i in range(n)])


def test_mode_b_mixed_layouts(cb):
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    want = compare(cb, 68, batches_b(), "b", flags, lambda k, n: [LAYOUTS[(4 - i - k) % 5] for i in range(n)])
    assert (want[0][0]["out"][1] != 0).sum() >= 2                   # premise: chunks decode
    assert want[0][0]["ccm"] is not None and (~np.isnan(want[1][0]["frame_ccms"][:, 0, 0])).sum() >= 1   # premise: fits carried and used


def test_refusals_that_need_a_context_and_empty_batches(cb):
    import torch
    pics = [placed(sample(GLOB[0]), "bgr", 1, 3)[0], placed(sample(GLOB[2]), "planar", 2, 5)[0]]
    small = cb.Context(4, max_frames=1)
    out = Outputs(small, 2)
    with pytest.raises(cb.Cb200Error, match="max_frames"):
        small.scan_extract_decode_chunks_pictures_dev(pics, *out.args()[:3], order=["bgr", "rgb"])
    with pytest.raises(cb.Cb200Error, match="null output"):
        small.scan_extract_decode_chunks_pictures_dev(pics[:1], out.chunks.data_ptr(), None, out.status.data_ptr(), order="bgr")
    small.scan_extract_decode_chunks_pictures_dev([], *out.args()[:3])          # n = 0: nothing to do, no error
    torch.cuda.synchronize()
    small.close()
