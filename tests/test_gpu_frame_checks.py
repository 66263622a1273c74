"""A frame call refused for CC_SIMPLE together with CC_FIT fails before any CUDA call: it launches nothing and leaves the context's
staging buffer as the last accepted host-pointer call left it, so cb200_fit_ccm(ctx, NULL, ...) still fits that call's frame."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _frame_with_header(ora, info, header, seed):
    """a mode-68 frame whose colour-stream chunks start with `header`, its block id counted up per chunk as the fit predicts"""
    m = ora.mode(68)
    payload = np.random.default_rng(seed).integers(0, 256, info.data_bytes, dtype=np.uint8)
    colours_at = info.raw_symbol_bytes // info.ecc_block_size * (info.ecc_block_size - info.ecc_bytes)
    for c, at in enumerate(range(colours_at, info.data_bytes, info.chunk_size)):
        block_id = (header[4] << 8 | header[5]) + c
        payload[at:at + 6] = header[:4] + [block_id >> 8, block_id & 0xFF]
    return ora.render_frame(m, ora.payload_to_cells(m, payload))


def test_refused_flags_leave_the_staged_frames_in_place():
    import libcimbar_b200 as cb
    from gpu_support import ORA, tint
    ctx = cb.Context(68, max_frames=2)
    header = [0x00, 0x01, 0x86, 0xA0, 0x00, 0x05]
    frame = _frame_with_header(ORA, ctx.info, header, seed=61)
    a = np.stack([tint(frame[None], (0.8, 0.6, 1.0))[0]] * 2)
    b = np.stack([tint(frame[None], (1.0, 0.7, 0.55))[0]] * 2)
    ctx.decode_fountain(a)
    launches = cb.launch_count()
    both = cb.FLAG_CC_SIMPLE | cb.FLAG_CC_FIT
    for refused in (lambda: ctx.decode(b, flags=both),
                    lambda: ctx.decode_fountain(b, flags=both),
                    lambda: ctx.decode_fountain(b, flags=both, sharpen=[True, False])):
        with pytest.raises(cb.Cb200Error, match="CC_SIMPLE and CC_FIT are exclusive"):
            refused()
        assert cb.launch_count() == launches
    got = ctx.fit_ccm(None, header, 0)
    fresh = cb.Context(68, max_frames=1)
    want = fresh.fit_ccm(a[0], header, 0)
    other = fresh.fit_ccm(b[0], header, 0)
    assert want is not None and np.array_equal(got, want)
    assert other is None or not np.array_equal(other, want)       # the premise: a fit of B's frame would tell
    fresh.close()
    ctx.close()
