"""A camera or corner call refused for CC_SIMPLE together with CC_FIT fails before any CUDA call: it launches nothing and leaves the
context as the earlier camera call left it (cb200_camera_transforms still reports that call's pictures)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def test_refused_flags_leave_the_last_camera_call_in_place():
    import libcimbar_b200 as cb
    ctx = cb.Context(68, max_frames=8)
    rng = np.random.default_rng(11)
    pics = rng.integers(0, 256, (3, 960, 1280, 3), dtype=np.uint8)
    ctx.scan_extract_decode_fountain(pics)
    want = ctx.camera_transforms(3)
    launches = cb.launch_count()
    both = cb.FLAG_CC_SIMPLE | cb.FLAG_CC_FIT
    corners = np.tile(np.array([0, 0, 1279, 0, 0, 959, 1279, 959], np.float32), (2, 1))
    for refused in (lambda: ctx.scan_extract_decode_fountain(pics[:2], flags=both),
                    lambda: ctx.scan_extract_decode_fountain_ragged(list(pics[:2]), flags=both),
                    lambda: ctx.extract_decode_fountain(pics[:2], corners, flags=both)):
        with pytest.raises(cb.Cb200Error, match="CC_SIMPLE and CC_FIT are exclusive"):
            refused()
        assert cb.launch_count() == launches
        assert np.array_equal(ctx.camera_transforms(3), want)
    ctx.close()
