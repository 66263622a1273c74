"""libcimbar_b200 -- H100 (sm_90a) implementation of libcimbar's per-frame decode hot path.

This Python module is only plumbing around the C ABI of lib/libcb200.so (include/cb200.h): it loads the
shared library with ctypes and passes raw pointers (numpy host buffers or torch device pointers).  There is
no Python or CPU decode path here: if the CUDA library is missing or no GPU is present, calls fail loudly."""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "lib", "libcb200.so")

FLAG_NO_FALLBACK = 0x1
FLAG_SHARPEN = 0x2
FLAG_CC_SIMPLE = 0x4
FLAG_CC_FIT = 0x8
FLAG_NO_INTERLEAVE = 0x10
FLAG_SHARPEN_IF_NEEDED = 0x20     # camera entry points only: sharpen the pictures Extractor::extract calls NEEDS_SHARPEN
FRAME_FALLBACK = 0x1
FRAME_INEXACT = 0x2

EXPORTS = [
    "cb200_last_error", "cb200_version", "cb200_create", "cb200_destroy", "cb200_get_info", "cb200_set_stream",
    "cb200_sync", "cb200_decode_raw_dev", "cb200_rs_correct_dev", "cb200_decode_chunks_dev", "cb200_decode_raw",
    "cb200_decode", "cb200_decode_fountain", "cb200_decode_symbols", "cb200_best_colors", "cb200_render_frames_dev",
    "cb200_mode_info", "cb200_interleave_indices", "cb200_encode_cells_dev", "cb200_set_timing", "cb200_get_timing", "cb200_decode_cells",
    "cb200_sink_create", "cb200_sink_create_wirehair", "cb200_sink_destroy", "cb200_sink_decode_frame", "cb200_sink_ingest", "cb200_sink_file_size",
    "cb200_sink_file_read", "cb200_selfcheck", "cb200_set_ccm", "cb200_get_ccm", "cb200_launch_count", "cb200_decode_fountain_from_dev", "cb200_perspective_transform", "cb200_deskew_dev", "cb200_deskew",
    "cb200_extract_decode_fountain", "cb200_extract_decode_fountain_dev", "cb200_scan", "cb200_scan_dev", "cb200_scan_blurred",
    "cb200_scan_extract_decode_fountain", "cb200_decode_cells_means", "cb200_fit_ccm", "cb200_palette_color",
    "cb200_gather_root_create", "cb200_gather_peer_open", "cb200_gather_slot", "cb200_gather_publish", "cb200_gather_push", "cb200_gather_wait",
    "cb200_gather_release", "cb200_gather_acquire",
    "cb200_gather_status", "cb200_comm_unique_id", "cb200_comm_init", "cb200_gather_chunks", "cb200_gather_chunks_wait",
    "cb200_decode_chunks_sharpen_dev", "cb200_decode_fountain_sharpen",
    "cb200_scan_ragged", "cb200_scan_ragged_dev", "cb200_scan_blurred_ragged", "cb200_extract_decode_fountain_ragged_dev",
    "cb200_scan_extract_decode_fountain_ragged", "cb200_scan_extract_decode_chunks_ragged_dev", "cb200_scan_extract_decode_chunks_dev",
    "cb200_camera_transforms", "cb200_jpeg_info", "cb200_jpeg_decode_dev", "cb200_jpeg_scan_extract_decode_chunks_dev",
    "cb200_png_info", "cb200_png_decode_dev", "cb200_png_scan_extract_decode_chunks_dev",
    "cb200_ccm_chain_root_create", "cb200_ccm_chain_peer_open", "cb200_ccm_chain_attach", "cb200_ccm_chain_step", "cb200_ccm_chain_status",
    "cb200_ccm_chain_link_ms", "cb200_get_frame_ccms",
    "cb200_camera_plan_create", "cb200_camera_plan_launch", "cb200_camera_plan_graph", "cb200_camera_plan_destroy",
]


class Info(C.Structure):
    _fields_ = [(n, C.c_int) for n in (
        "mode_val", "image_size_x", "image_size_y", "frame_bytes", "total_cells", "symbol_bits", "color_bits",
        "raw_bytes", "raw_symbol_bytes", "ecc_bytes", "ecc_block_size", "rs_blocks", "data_bytes", "chunk_size",
        "chunks_per_frame", "legacy_mode", "max_frames", "sm_count")]


TRACE_DTYPE = np.dtype([("order", "<u2"), ("x", "<i2"), ("y", "<i2"), ("drift_offset", "u1"), ("distance", "u1")])


class Cb200Error(RuntimeError):
    pass


_lib = None


def load_library():
    """Load libcb200.so (building it is __graft_entry__.build()'s / libcimbar_b200.build's job)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise Cb200Error(f"{LIB_PATH} is missing: build it with `python -m libcimbar_b200.build` "
                         "(there is no fallback implementation)")
    lib = C.CDLL(LIB_PATH)
    vp, u8p, u32p, u16p = C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p
    lib.cb200_last_error.restype = C.c_char_p
    lib.cb200_create.argtypes = [C.POINTER(vp), C.c_int, C.c_int, C.c_int]
    lib.cb200_destroy.argtypes = [vp]
    lib.cb200_get_info.argtypes = [vp, C.POINTER(Info)]
    lib.cb200_set_stream.argtypes = [vp, vp]
    lib.cb200_sync.argtypes = [vp]
    lib.cb200_decode_raw_dev.argtypes = [vp, u8p, C.c_int, C.c_uint32, u8p, u8p]
    lib.cb200_rs_correct_dev.argtypes = [vp, u8p, C.c_int, u8p, u8p]
    lib.cb200_decode_chunks_dev.argtypes = [vp, u8p, C.c_int, C.c_uint32, u8p, u32p, u8p]
    lib.cb200_decode_raw.argtypes = [vp, u8p, C.c_int, C.c_uint32, u8p, u8p]
    lib.cb200_decode.argtypes = [vp, u8p, C.c_int, C.c_uint32, u8p, u8p, u8p]
    lib.cb200_decode_fountain.argtypes = [vp, u8p, C.c_int, C.c_uint32, u8p, u32p, u32p, u8p]
    lib.cb200_decode_chunks_sharpen_dev.argtypes = [vp, u8p, C.c_int, C.c_uint32, u8p, u8p, u32p, u8p]
    lib.cb200_decode_fountain_sharpen.argtypes = [vp, u8p, C.c_int, C.c_uint32, u8p, u8p, u32p, u32p, u8p]
    lib.cb200_decode_cells.argtypes = [vp, u8p, C.c_int, C.c_uint32, u8p, vp]
    lib.cb200_decode_symbols.argtypes = [vp, u16p, u8p, C.c_int, u8p, u8p, u8p]
    lib.cb200_best_colors.argtypes = [vp, u8p, C.c_int, u8p]
    lib.cb200_set_ccm.argtypes = [vp, C.c_void_p]
    lib.cb200_get_ccm.argtypes = [vp, C.c_void_p]
    lib.cb200_render_frames_dev.argtypes = [vp, u8p, C.c_int, u8p]
    lib.cb200_encode_cells_dev.argtypes = [vp, u8p, C.c_int, u8p]
    lib.cb200_set_timing.argtypes = [vp, C.c_int]
    lib.cb200_get_timing.argtypes = [vp, C.c_int, C.POINTER(C.c_float), C.c_int, C.POINTER(C.c_int)]
    lib.cb200_sink_create.restype = vp
    lib.cb200_sink_create.argtypes = [C.c_uint, vp, vp, vp, vp]
    lib.cb200_sink_create_wirehair.restype = vp
    lib.cb200_sink_create_wirehair.argtypes = [C.c_uint, C.c_char_p]
    lib.cb200_sink_destroy.argtypes = [vp]
    lib.cb200_sink_decode_frame.restype = C.c_int64
    lib.cb200_sink_decode_frame.argtypes = [vp, u8p, C.c_uint]
    lib.cb200_sink_ingest.restype = C.c_int64
    lib.cb200_sink_ingest.argtypes = [vp, u8p, u32p, C.c_int, C.c_int]
    lib.cb200_sink_file_size.restype = C.c_int64
    lib.cb200_sink_file_size.argtypes = [vp, C.c_uint32]
    lib.cb200_sink_file_read.argtypes = [vp, C.c_uint32, u8p, C.c_uint64]
    lib.cb200_launch_count.restype = C.c_ulonglong
    lib.cb200_decode_fountain_from_dev.argtypes = [vp, u8p, C.c_int, C.c_uint32, u8p, u32p, u32p, u8p]
    lib.cb200_perspective_transform.argtypes = [vp, vp, vp]
    lib.cb200_deskew_dev.argtypes = [vp, u8p, C.c_int, C.c_int, C.c_int, vp, u8p]
    lib.cb200_deskew.argtypes = [vp, u8p, C.c_int, C.c_int, C.c_int, vp, u8p]
    lib.cb200_extract_decode_fountain.argtypes = [vp, u8p, C.c_int, C.c_int, C.c_int, vp, C.c_uint32, u8p, u32p, u32p, u8p]
    lib.cb200_extract_decode_fountain_dev.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, vp, C.c_uint32, u8p, u32p, u32p, u8p]
    lib.cb200_scan.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, vp, vp, vp]
    lib.cb200_scan_dev.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, vp, vp, vp]
    lib.cb200_scan_blurred.argtypes = [vp, vp, vp, C.c_int, C.c_int, C.c_int]
    lib.cb200_scan_extract_decode_fountain.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.c_uint32, vp, vp, vp, vp, vp]
    lib.cb200_scan_ragged.argtypes = [vp, vp, vp, C.c_int, vp, vp, vp]
    lib.cb200_scan_ragged_dev.argtypes = [vp, vp, vp, C.c_int, vp, vp, vp]
    lib.cb200_scan_blurred_ragged.argtypes = [vp, vp, vp, vp, C.c_int]
    lib.cb200_extract_decode_fountain_ragged_dev.argtypes = [vp, vp, vp, C.c_int, vp, C.c_uint32, vp, vp, vp, vp]
    lib.cb200_scan_extract_decode_fountain_ragged.argtypes = [vp, vp, vp, C.c_int, C.c_uint32, vp, vp, vp, vp, vp]
    lib.cb200_scan_extract_decode_chunks_ragged_dev.argtypes = [vp, vp, vp, C.c_int, C.c_uint32, vp, vp, vp, vp]
    lib.cb200_scan_extract_decode_chunks_dev.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.c_uint32, vp, vp, vp, vp]
    lib.cb200_camera_transforms.argtypes = [vp, vp, C.c_int]
    lib.cb200_jpeg_info.argtypes = [vp, C.c_uint64, vp, vp]
    lib.cb200_jpeg_decode_dev.argtypes = [vp, vp, vp, C.c_int, vp, vp]
    lib.cb200_jpeg_scan_extract_decode_chunks_dev.argtypes = [vp, vp, vp, C.c_int, C.c_uint32, vp, vp, vp, vp]
    lib.cb200_png_info.argtypes = [vp, C.c_uint64, vp, vp]
    lib.cb200_png_decode_dev.argtypes = [vp, vp, vp, C.c_int, vp, vp]
    lib.cb200_png_scan_extract_decode_chunks_dev.argtypes = [vp, vp, vp, C.c_int, C.c_uint32, vp, vp, vp, vp]
    lib.cb200_decode_cells_means.argtypes = [vp, u8p, C.c_int, C.c_uint32, u8p, vp, vp]
    lib.cb200_fit_ccm.argtypes = [vp, u8p, u8p, C.c_uint32, C.c_uint32, C.c_void_p]
    lib.cb200_palette_color.argtypes = [C.c_int, C.c_uint, C.c_int, u8p]
    lib.cb200_gather_root_create.argtypes = [vp, C.c_int, u8p]
    lib.cb200_gather_peer_open.argtypes = [vp, C.c_int, C.c_int, u8p]
    lib.cb200_gather_slot.argtypes = [vp, C.c_int, C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p)]
    lib.cb200_gather_publish.argtypes = [vp, C.c_int, C.c_uint32]
    lib.cb200_gather_push.argtypes = [vp, C.c_int, u8p, u32p, C.c_int, C.c_uint32, C.c_uint32]
    lib.cb200_gather_wait.argtypes = [vp, C.c_int, C.c_uint32, C.c_double]
    lib.cb200_gather_release.argtypes = [vp, C.c_int, C.c_uint32]
    lib.cb200_gather_acquire.argtypes = [vp, C.c_int, C.c_uint32, C.c_double]
    lib.cb200_gather_status.argtypes = [vp]
    lib.cb200_comm_unique_id.argtypes = [u8p]
    lib.cb200_comm_init.argtypes = [vp, u8p, C.c_int, C.c_int]
    lib.cb200_gather_chunks.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, u8p, u32p, C.c_int, u8p, u32p]
    lib.cb200_gather_chunks_wait.argtypes = [vp, C.c_int]
    lib.cb200_ccm_chain_root_create.argtypes = [vp, C.c_int, u8p]
    lib.cb200_ccm_chain_peer_open.argtypes = [vp, C.c_int, C.c_int, u8p]
    lib.cb200_ccm_chain_attach.argtypes = [vp, C.c_int, C.c_int]
    lib.cb200_ccm_chain_step.argtypes = [vp, C.c_uint32]
    lib.cb200_ccm_chain_status.argtypes = [vp]
    lib.cb200_ccm_chain_link_ms.argtypes = [vp, C.POINTER(C.c_float)]
    lib.cb200_get_frame_ccms.argtypes = [vp, C.c_int, vp, vp]
    lib.cb200_camera_plan_create.argtypes = [vp, vp, C.c_int, C.c_uint32, vp, vp, vp, vp, vp, C.POINTER(C.c_void_p)]
    lib.cb200_camera_plan_launch.argtypes = [vp]
    lib.cb200_camera_plan_graph.argtypes = [vp, C.POINTER(C.c_void_p)]
    lib.cb200_camera_plan_destroy.argtypes = [vp]
    lib.cb200_selfcheck.argtypes = [C.c_int]
    lib.cb200_mode_info.argtypes = [C.c_int, C.POINTER(Info)]
    lib.cb200_interleave_indices.argtypes = [C.c_int, u16p]
    _lib = lib
    return lib


def _check(rc):
    if rc != 0:
        raise Cb200Error(f"cb200 error {rc}: {load_library().cb200_last_error().decode()}")


def launch_count():
    """kernels launched by libcb200 in this process so far"""
    return int(load_library().cb200_launch_count())


def comm_unique_id():
    """ncclGetUniqueId through the library's run-time NCCL binding: 128 bytes to broadcast to the other ranks"""
    h = (C.c_uint8 * 128)()
    _check(load_library().cb200_comm_unique_id(C.cast(h, C.c_void_p)))
    return bytes(h)


def perspective_transform(src_xy, dst_xy):
    """cv::getPerspectiveTransform restated (host): 4 source and 4 destination points -> 3x3 float64"""
    a = np.ascontiguousarray(src_xy, dtype=np.float32).reshape(8)
    b = np.ascontiguousarray(dst_xy, dtype=np.float32).reshape(8)
    out = np.zeros(9, dtype=np.float64)
    _check(load_library().cb200_perspective_transform(a.ctypes.data, b.ctypes.data, out.ctypes.data))
    return out.reshape(3, 3)


def mode_info(mode_val=68):
    info = Info()
    _check(load_library().cb200_mode_info(mode_val, C.byref(info)))
    return info


def interleave_indices(mode_val=68):
    info = mode_info(mode_val)
    idx = np.zeros(info.total_cells, dtype=np.uint16)
    _check(load_library().cb200_interleave_indices(mode_val, idx.ctypes.data))
    return idx


def _hptr(a):
    return a.ctypes.data if a is not None else None


def _ragged(pictures):
    """a list of (h, w, 3) uint8 pictures of any sizes -> (contiguous pictures, n host pointers, wh n x 2 int32 = (w, h))"""
    pics = [np.ascontiguousarray(p, dtype=np.uint8) for p in pictures]
    for i, p in enumerate(pics):
        if p.ndim != 3 or p.shape[2] != 3:
            raise Cb200Error(f"picture {i} must be (h, w, 3) RGB8, got {p.shape}")
    ptrs = (C.c_void_p * max(len(pics), 1))(*[p.ctypes.data for p in pics])
    wh = np.array([(p.shape[1], p.shape[0]) for p in pics], dtype=np.int32).reshape(-1, 2)
    return pics, ptrs, wh


def jpeg_info(data):
    """(w, h) of a JPEG file (bytes) after its EXIF orientation, as cb200_jpeg_info: host only, no GPU.  Raises Cb200Error with
    the reason for a file the device decoder refuses"""
    w, h = C.c_int32(), C.c_int32()
    _check(load_library().cb200_jpeg_info(data, len(data), C.byref(w), C.byref(h)))
    return w.value, h.value


def png_info(data):
    """(w, h) of a PNG file (bytes) after its eXIf orientation, as cb200_png_info: host only, no GPU.  Raises Cb200Error with the
    reason for a file the device decoder refuses"""
    w, h = C.c_int32(), C.c_int32()
    _check(load_library().cb200_png_info(data, len(data), C.byref(w), C.byref(h)))
    return w.value, h.value


def _files(files):
    """a list of bytes -> (kept objects, n host pointers, n sizes)"""
    files = [bytes(f) for f in files]
    ptrs = (C.c_char_p * max(len(files), 1))(*files)
    sizes = (C.c_uint64 * max(len(files), 1))(*[len(f) for f in files])
    return files, ptrs, sizes


def _selection(sharpen, n):
    """a per-frame sharpen choice as the C ABI takes it: n bytes, nonzero = should_preprocess"""
    sel = np.ascontiguousarray(np.asarray(sharpen).astype(bool), dtype=np.uint8).reshape(-1)
    if sel.size != n:
        raise Cb200Error(f"sharpen must have one entry per frame ({n}), got {sel.size}")
    return sel


class Context:
    """One decode context = one GPU + one stream (cb200_create / cb200_destroy)."""

    def __init__(self, mode_val=68, max_frames=64, device=-1):
        self.lib = load_library()
        self._h = C.c_void_p()
        _check(self.lib.cb200_create(C.byref(self._h), device, mode_val, max_frames))
        self.info = Info()
        _check(self.lib.cb200_get_info(self._h, C.byref(self.info)))

    def close(self):
        if self._h:
            self.lib.cb200_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_stream(self, cuda_stream_ptr):
        _check(self.lib.cb200_set_stream(self._h, cuda_stream_ptr))

    def sync(self):
        _check(self.lib.cb200_sync(self._h))

    # ---- host-pointer entry points (numpy in / numpy out)
    def _frames(self, rgb):
        rgb = np.ascontiguousarray(rgb, dtype=np.uint8)
        if rgb.ndim == 3:
            rgb = rgb[None]
        n = rgb.shape[0]
        if rgb.shape[1:] != (self.info.image_size_y, self.info.image_size_x, 3):
            raise Cb200Error(f"frames must be {self.info.image_size_y}x{self.info.image_size_x}x3 RGB8, got {rgb.shape[1:]}")
        return rgb, n

    def decode_raw(self, rgb, flags=0):
        rgb, n = self._frames(rgb)
        raw = np.zeros((n, self.info.raw_bytes), dtype=np.uint8)
        ff = np.zeros(n, dtype=np.uint8)
        _check(self.lib.cb200_decode_raw(self._h, rgb.ctypes.data, n, flags, raw.ctypes.data, ff.ctypes.data))
        return raw, ff

    def decode(self, rgb, flags=0):
        rgb, n = self._frames(rgb)
        data = np.zeros((n, self.info.data_bytes), dtype=np.uint8)
        ok = np.zeros((n, self.info.rs_blocks), dtype=np.uint8)
        ff = np.zeros(n, dtype=np.uint8)
        _check(self.lib.cb200_decode(self._h, rgb.ctypes.data, n, flags, data.ctypes.data, ok.ctypes.data, ff.ctypes.data))
        return data, ok, ff

    def decode_fountain(self, rgb, flags=0, sharpen=None):
        """Decoder::decode_fountain over a batch.  sharpen: None = as `flags` says for every frame; else one bool per frame
        (should_preprocess of that frame; `flags` must not contain FLAG_SHARPEN then)"""
        rgb, n = self._frames(rgb)
        chunks = np.zeros((n, self.info.chunks_per_frame, self.info.chunk_size), dtype=np.uint8)
        count = np.zeros(n, dtype=np.uint32)
        mask = np.zeros(n, dtype=np.uint32)
        ff = np.zeros(n, dtype=np.uint8)
        if sharpen is None:
            _check(self.lib.cb200_decode_fountain(self._h, rgb.ctypes.data, n, flags, chunks.ctypes.data, count.ctypes.data,
                                                  mask.ctypes.data, ff.ctypes.data))
        else:
            sel = _selection(sharpen, n)
            _check(self.lib.cb200_decode_fountain_sharpen(self._h, rgb.ctypes.data, n, flags, sel.ctypes.data, chunks.ctypes.data,
                                                          count.ctypes.data, mask.ctypes.data, ff.ctypes.data))
        return chunks, count, mask, ff

    def deskew(self, src, m9):
        """cv::warpPerspective(src, M, mode size, INTER_LINEAR) on the device; src: (n, h, w, 3) or (h, w, 3) uint8, m9: (n, 3, 3) float64"""
        src = np.ascontiguousarray(src, dtype=np.uint8)
        if src.ndim == 3:
            src = src[None]
        n, h, w, _ = src.shape
        m = np.ascontiguousarray(m9, dtype=np.float64).reshape(n, 9)
        out = np.zeros((n, self.info.image_size_y, self.info.image_size_x, 3), dtype=np.uint8)
        _check(self.lib.cb200_deskew(self._h, src.ctypes.data, w, h, n, m.ctypes.data, out.ctypes.data))
        return out

    def extract_decode_fountain(self, src, corners, flags=0):
        """camera images + their four anchor centres (tl, tr, bl, br) -> fountain chunks; the deskewed frames stay on the device"""
        src = np.ascontiguousarray(src, dtype=np.uint8)
        if src.ndim == 3:
            src = src[None]
        n, h, w, _ = src.shape
        cr = np.ascontiguousarray(corners, dtype=np.float32).reshape(n, 8)
        chunks = np.zeros((n, self.info.chunks_per_frame, self.info.chunk_size), dtype=np.uint8)
        count = np.zeros(n, dtype=np.uint32)
        mask = np.zeros(n, dtype=np.uint32)
        ff = np.zeros(n, dtype=np.uint8)
        _check(self.lib.cb200_extract_decode_fountain(self._h, src.ctypes.data, w, h, n, cr.ctypes.data, flags, chunks.ctypes.data,
                                                      count.ctypes.data, mask.ctypes.data, ff.ctypes.data))
        return chunks, count, mask, ff

    def scan(self, pictures):
        """Scanner(img).scan() on the device for pictures (n, h, w, 3) or (h, w, 3) uint8 ->
        anchors (n, 4, 4) int32 rows of (x, xmax, y, ymax), count (n,) int32 (-1: capacity overflow), cutoff (n,) uint32"""
        pics = np.ascontiguousarray(pictures, dtype=np.uint8)
        if pics.ndim == 3:
            pics = pics[None]
        n, h, w, _ = pics.shape
        anchors = np.zeros((n, 4, 4), dtype=np.int32)
        count = np.zeros(n, dtype=np.int32)
        cutoff = np.zeros(n, dtype=np.uint32)
        _check(self.lib.cb200_scan(self._h, pics.ctypes.data, w, h, n, anchors.ctypes.data, count.ctypes.data, cutoff.ctypes.data))
        return anchors, count, cutoff

    def scan_blurred(self, n, h, w):
        """the blurred gray pictures and Otsu thresholds of the last scan call"""
        blurred = np.zeros((n, h, w), dtype=np.uint8)
        thr = np.zeros(n, dtype=np.int32)
        _check(self.lib.cb200_scan_blurred(self._h, blurred.ctypes.data, thr.ctypes.data, w, h, n))
        return blurred, thr

    def scan_ragged(self, pictures):
        """scan() for a list of (h, w, 3) uint8 pictures of any sizes, in one call"""
        pics, ptrs, wh = _ragged(pictures)
        n = len(pics)
        anchors = np.zeros((n, 4, 4), dtype=np.int32)
        count = np.zeros(n, dtype=np.int32)
        cutoff = np.zeros(n, dtype=np.uint32)
        _check(self.lib.cb200_scan_ragged(self._h, ptrs, wh.ctypes.data, n, anchors.ctypes.data, count.ctypes.data, cutoff.ctypes.data))
        return anchors, count, cutoff

    def scan_blurred_ragged(self, shapes):
        """the blurred gray pictures (a list, one (h, w) array each) and Otsu thresholds of the last scan call; shapes: its (h, w)s"""
        wh = np.array([(w, h) for h, w in (tuple(s)[:2] for s in shapes)], dtype=np.int32).reshape(-1, 2)
        n = wh.shape[0]
        flat = np.zeros(int((wh[:, 0].astype(np.int64) * wh[:, 1]).sum()), dtype=np.uint8)
        thr = np.zeros(n, dtype=np.int32)
        _check(self.lib.cb200_scan_blurred_ragged(self._h, flat.ctypes.data, thr.ctypes.data, wh.ctypes.data, n))
        out, at = [], 0
        for w, h in wh.tolist():
            out.append(flat[at:at + w * h].reshape(h, w))
            at += w * h
        return out, thr

    def scan_extract_decode_fountain_ragged(self, pictures, flags=0):
        """scan_extract_decode_fountain for a list of (h, w, 3) uint8 pictures of any sizes, in order (the CLI's decode loop)"""
        pics, ptrs, wh = _ragged(pictures)
        n = len(pics)
        chunks = np.zeros((n, self.info.chunks_per_frame, self.info.chunk_size), dtype=np.uint8)
        count = np.zeros(n, dtype=np.uint32)
        mask = np.zeros(n, dtype=np.uint32)
        ff = np.zeros(n, dtype=np.uint8)
        status = np.zeros(n, dtype=np.int32)
        _check(self.lib.cb200_scan_extract_decode_fountain_ragged(self._h, ptrs, wh.ctypes.data, n, flags, chunks.ctypes.data, count.ctypes.data,
                                                                  mask.ctypes.data, ff.ctypes.data, status.ctypes.data))
        return chunks, count, mask, ff, status

    def scan_extract_decode_fountain(self, pictures, flags=0):
        """Extractor::extract + Decoder::decode_fountain: camera pictures in, chunks out -> (chunks, count, mask, frame_flags, extract_status)"""
        pics = np.ascontiguousarray(pictures, dtype=np.uint8)
        if pics.ndim == 3:
            pics = pics[None]
        n, h, w, _ = pics.shape
        chunks = np.zeros((n, self.info.chunks_per_frame, self.info.chunk_size), dtype=np.uint8)
        count = np.zeros(n, dtype=np.uint32)
        mask = np.zeros(n, dtype=np.uint32)
        ff = np.zeros(n, dtype=np.uint8)
        status = np.zeros(n, dtype=np.int32)
        _check(self.lib.cb200_scan_extract_decode_fountain(self._h, pics.ctypes.data, w, h, n, flags, chunks.ctypes.data, count.ctypes.data,
                                                           mask.ctypes.data, ff.ctypes.data, status.ctypes.data))
        return chunks, count, mask, ff, status

    def decode_cells(self, rgb, flags=0):
        """exact flood walk with per-cell trace (order, x, y, drift_offset, distance) -- CimbReader semantics"""
        rgb, n = self._frames(rgb)
        cells = np.zeros((n, self.info.total_cells), dtype=np.uint8)
        trace = np.zeros((n, self.info.total_cells), dtype=TRACE_DTYPE)
        _check(self.lib.cb200_decode_cells(self._h, rgb.ctypes.data, n, flags, cells.ctypes.data, trace.ctypes.data))
        return cells, trace

    def decode_cells_means(self, rgb, flags=0):
        """like decode_cells, but the colours are left undecided: returns (symbols, trace, means r|g<<8|b<<16)"""
        rgb, n = self._frames(rgb)
        cells = np.zeros((n, self.info.total_cells), dtype=np.uint8)
        trace = np.zeros((n, self.info.total_cells), dtype=TRACE_DTYPE)
        means = np.zeros((n, self.info.total_cells), dtype=np.uint32)
        _check(self.lib.cb200_decode_cells_means(self._h, rgb.ctypes.data, n, flags, cells.ctypes.data, trace.ctypes.data, means.ctypes.data))
        return cells, trace, means

    def fit_ccm(self, rgb, header6, radioactive, flags=0):
        """CimbReader::init_ccm with a header tracked by the caller; returns the fitted 3x3 matrix or None"""
        hdr = np.ascontiguousarray(header6, dtype=np.uint8)
        out = np.zeros(9, dtype=np.float32)
        ptr = None
        if rgb is not None:
            rgb, _ = self._frames(rgb)
            ptr = rgb.ctypes.data
        rc = self.lib.cb200_fit_ccm(self._h, ptr, hdr.ctypes.data, int(radioactive) & 0xFFFFFFFF, flags, out.ctypes.data)
        if rc < 0:
            _check(rc)
        return out.reshape(3, 3) if rc == 1 else None

    def decode_symbols(self, windows, cooldown=None):
        windows = np.ascontiguousarray(windows, dtype=np.uint16).reshape(-1, 10)
        n = windows.shape[0]
        cd = None if cooldown is None else np.ascontiguousarray(cooldown, dtype=np.uint8)
        sym, off, dist = (np.zeros(n, dtype=np.uint8) for _ in range(3))
        _check(self.lib.cb200_decode_symbols(self._h, windows.ctypes.data, _hptr(cd), n, sym.ctypes.data, off.ctypes.data, dist.ctypes.data))
        return sym, off, dist

    def best_colors(self, rgb_means):
        rgb_means = np.ascontiguousarray(rgb_means, dtype=np.uint8).reshape(-1, 3)
        out = np.zeros(rgb_means.shape[0], dtype=np.uint8)
        _check(self.lib.cb200_best_colors(self._h, rgb_means.ctypes.data, rgb_means.shape[0], out.ctypes.data))
        return out

    def set_ccm(self, m9):
        """CimbDecoder::update_color_correction: 3x3 float32 row-major, or None to deactivate"""
        if m9 is None:
            _check(self.lib.cb200_set_ccm(self._h, None))
        else:
            a = np.ascontiguousarray(m9, dtype=np.float32).reshape(9)
            _check(self.lib.cb200_set_ccm(self._h, a.ctypes.data))

    def frame_ccms(self, n):
        """the matrices the first n frames of the last CC_FIT call were decoded with: (n, 3, 3) float32 with NaN for a frame that had
        none (synchronises)"""
        m = np.zeros((n, 9), dtype=np.float32)
        act = np.zeros(n, dtype=np.uint8)
        _check(self.lib.cb200_get_frame_ccms(self._h, n, m.ctypes.data, act.ctypes.data))
        m[act == 0] = np.nan
        return m.reshape(n, 3, 3)

    def get_ccm(self):
        """the active CCM as a 3x3 float32 array, or None"""
        a = np.zeros(9, dtype=np.float32)
        rc = self.lib.cb200_get_ccm(self._h, a.ctypes.data)
        if rc < 0:
            _check(rc)
        return a.reshape(3, 3) if rc == 1 else None

    # ---- device-pointer entry points (raw device addresses, e.g. torch.Tensor.data_ptr())
    def decode_raw_dev(self, d_rgb, n, d_raw_out, d_flags=None, flags=0):
        _check(self.lib.cb200_decode_raw_dev(self._h, d_rgb, n, flags, d_raw_out, d_flags))

    def rs_correct_dev(self, d_raw, n, d_data_out, d_ok=None):
        _check(self.lib.cb200_rs_correct_dev(self._h, d_raw, n, d_data_out, d_ok))

    def decode_chunks_dev(self, d_rgb, n, d_chunks, d_mask, d_flags=None, flags=0, sharpen=None):
        """sharpen: None = as `flags` says; else one bool per frame, host memory (see decode_fountain)"""
        if sharpen is None:
            _check(self.lib.cb200_decode_chunks_dev(self._h, d_rgb, n, flags, d_chunks, d_mask, d_flags))
        else:
            sel = _selection(sharpen, n)
            _check(self.lib.cb200_decode_chunks_sharpen_dev(self._h, d_rgb, n, flags, sel.ctypes.data, d_chunks, d_mask, d_flags))

    def scan_extract_decode_chunks_dev(self, d_pictures, wh, d_chunks, d_mask, d_status, d_flags=None, flags=0):
        """scan_extract_decode_fountain_ragged, enqueue-only: a ragged batch packed in device memory (d_pictures), its sizes wh
        (n x (w, h), host) -> fixed-slot chunks, masks, extract statuses (int32) and frame flags in device memory, on the context's
        stream; returns without waiting for the device"""
        wh = np.ascontiguousarray(wh, dtype=np.int32).reshape(-1, 2)
        _check(self.lib.cb200_scan_extract_decode_chunks_ragged_dev(self._h, d_pictures, wh.ctypes.data, wh.shape[0], flags, d_chunks, d_mask,
                                                                    d_flags, d_status))

    def camera_plan(self, wh, flags, pictures, chunks, mask, frame_flags, status):
        """scan_extract_decode_chunks_dev for pictures of sizes wh (n x (w, h), host) with these flags, captured once in a CUDA graph
        with its device buffers bound (device addresses; frame_flags may be None): a CameraPlan whose launch() replays it on the
        context's stream.  Write each batch's pictures into `pictures` in stream order before its launch"""
        wh = np.ascontiguousarray(wh, dtype=np.int32).reshape(-1, 2)
        h = C.c_void_p()
        _check(self.lib.cb200_camera_plan_create(self._h, wh.ctypes.data, wh.shape[0], flags, pictures, chunks, mask, frame_flags, status,
                                                 C.byref(h)))
        return CameraPlan(self, h)

    jpeg_info = staticmethod(jpeg_info)

    def jpeg_decode_dev(self, files, d_rgb_out, d_status=None):
        """cb200_jpeg_decode_dev, enqueue-only: a list of JPEG files (bytes) -> the packed ragged RGB8 batch at d_rgb_out (picture i at
        3 * sum_{j<i} w_j h_j, sizes as jpeg_info) and n int32 statuses (0, or -2 for corrupt data) at d_status, on the context's stream"""
        keep, ptrs, sizes = _files(files)
        _check(self.lib.cb200_jpeg_decode_dev(self._h, ptrs, sizes, len(keep), d_rgb_out, d_status))

    def jpeg_scan_extract_decode_chunks_dev(self, files, d_chunks, d_mask, d_status, d_flags=None, flags=0):
        """scan_extract_decode_chunks_dev on a list of JPEG files (bytes) decoded on the device; enqueue-only.  A picture with corrupt
        data gets status -2 and mask 0"""
        keep, ptrs, sizes = _files(files)
        _check(self.lib.cb200_jpeg_scan_extract_decode_chunks_dev(self._h, ptrs, sizes, len(keep), flags, d_chunks, d_mask, d_flags, d_status))

    png_info = staticmethod(png_info)

    def png_decode_dev(self, files, d_rgb_out, d_status=None):
        """cb200_png_decode_dev, enqueue-only: a list of PNG files (bytes) -> the packed ragged RGB8 batch at d_rgb_out (picture i at
        3 * sum_{j<i} w_j h_j, sizes as png_info) and n int32 statuses (0, or -2 for corrupt data) at d_status, on the context's
        stream.  Files of the mode's frame size give the frame batch of decode_chunks_dev (the CLI's --no-deskew)"""
        keep, ptrs, sizes = _files(files)
        _check(self.lib.cb200_png_decode_dev(self._h, ptrs, sizes, len(keep), d_rgb_out, d_status))

    def png_scan_extract_decode_chunks_dev(self, files, d_chunks, d_mask, d_status, d_flags=None, flags=0):
        """scan_extract_decode_chunks_dev on a list of PNG files (bytes) decoded on the device; enqueue-only.  A picture with corrupt
        data gets status -2 and mask 0"""
        keep, ptrs, sizes = _files(files)
        _check(self.lib.cb200_png_scan_extract_decode_chunks_dev(self._h, ptrs, sizes, len(keep), flags, d_chunks, d_mask, d_flags, d_status))

    def camera_transforms(self, n):
        """the forward perspective transforms of the first n pictures of the last camera call: (n, 3, 3) float64 (synchronises)"""
        out = np.zeros((n, 3, 3), dtype=np.float64)
        _check(self.lib.cb200_camera_transforms(self._h, out.ctypes.data, n))
        return out

    def encode_cells_dev(self, d_payload, n, d_cellvals):
        _check(self.lib.cb200_encode_cells_dev(self._h, d_payload, n, d_cellvals))

    def set_timing(self, enable=True):
        _check(self.lib.cb200_set_timing(self._h, int(enable)))

    def get_timing(self, calls_back=0):
        """ms per kernel of the pipeline call `calls_back` calls ago: [K1 (both launches of a mixed batch), K1x, pack, RS, mask]"""
        ms = (C.c_float * 8)()
        n = C.c_int(0)
        _check(self.lib.cb200_get_timing(self._h, calls_back, ms, 8, C.byref(n)))
        return [ms[i] for i in range(n.value)]

    # ---- multi-GPU chunk-record exchange (cb200_gather_*): see include/cb200.h
    def gather_root_create(self, nranks):
        h = (C.c_uint8 * 64)()
        _check(self.lib.cb200_gather_root_create(self._h, nranks, C.cast(h, C.c_void_p)))
        return bytes(h)

    def gather_peer_open(self, nranks, rank, handle):
        h = (C.c_uint8 * 64).from_buffer_copy(handle)
        _check(self.lib.cb200_gather_peer_open(self._h, nranks, rank, C.cast(h, C.c_void_p)))

    def gather_slot(self, buffer, rank=-1):
        """device addresses (chunks, masks) of `rank`'s records in window buffer `buffer` (rank < 0: this rank's own slot)"""
        pc, pm = C.c_void_p(), C.c_void_p()
        _check(self.lib.cb200_gather_slot(self._h, buffer, rank, C.byref(pc), C.byref(pm)))
        return pc.value, pm.value

    def gather_publish(self, buffer, epoch):
        _check(self.lib.cb200_gather_publish(self._h, buffer, epoch))

    def gather_push(self, buffer, d_chunks, d_mask, n, epoch, acquire_epoch=0):
        """records in local buffers -> this rank's window slot by a copy-engine transfer on the side stream, then publish"""
        _check(self.lib.cb200_gather_push(self._h, buffer, d_chunks, d_mask, n, epoch, acquire_epoch))

    def gather_wait(self, buffer, epoch, timeout_s=30.0):
        _check(self.lib.cb200_gather_wait(self._h, buffer, epoch, timeout_s))

    def gather_release(self, buffer, epoch):
        _check(self.lib.cb200_gather_release(self._h, buffer, epoch))

    def gather_acquire(self, buffer, epoch, timeout_s=30.0):
        _check(self.lib.cb200_gather_acquire(self._h, buffer, epoch, timeout_s))

    def gather_status(self):
        _check(self.lib.cb200_gather_status(self._h))

    def comm_init(self, uid, nranks, rank):
        h = (C.c_uint8 * 128).from_buffer_copy(uid)
        _check(self.lib.cb200_comm_init(self._h, C.cast(h, C.c_void_p), nranks, rank))

    def gather_chunks(self, nranks, rank, buffer, d_chunks, d_mask, n, d_all_chunks=None, d_all_masks=None, comm=None):
        _check(self.lib.cb200_gather_chunks(self._h, comm, nranks, rank, buffer, d_chunks, d_mask, n, d_all_chunks, d_all_masks))

    def gather_chunks_wait(self, buffer):
        _check(self.lib.cb200_gather_chunks_wait(self._h, buffer))

    # ---- multi-GPU CC_FIT chain (cb200_ccm_chain_*): see include/cb200.h
    def ccm_chain_root_create(self, nranks):
        h = (C.c_uint8 * 64)()
        _check(self.lib.cb200_ccm_chain_root_create(self._h, nranks, C.cast(h, C.c_void_p)))
        return bytes(h)

    def ccm_chain_peer_open(self, nranks, rank, handle):
        h = (C.c_uint8 * 64).from_buffer_copy(handle)
        _check(self.lib.cb200_ccm_chain_peer_open(self._h, nranks, rank, C.cast(h, C.c_void_p)))

    def ccm_chain_attach(self, rank, nranks):
        _check(self.lib.cb200_ccm_chain_attach(self._h, rank, nranks))

    def ccm_chain_step(self, epoch):
        """the epoch of the next CC_FIT call (the same on every rank for the same step, increasing from step to step)"""
        _check(self.lib.cb200_ccm_chain_step(self._h, epoch))

    def ccm_chain_status(self):
        _check(self.lib.cb200_ccm_chain_status(self._h))

    def ccm_chain_link_ms(self):
        """ms of the last chained call's link kernel (set_timing on before the call; synchronises on it)"""
        ms = C.c_float(0)
        _check(self.lib.cb200_ccm_chain_link_ms(self._h, C.byref(ms)))
        return ms.value

    def render_frames_dev(self, d_cellvals, n, d_rgb_out):
        _check(self.lib.cb200_render_frames_dev(self._h, d_cellvals, n, d_rgb_out))


class CameraPlan:
    """a camera plan (cb200_camera_plan_*): launch() is one graph launch on the context's stream, or a child node of the capture
    in progress on it (torch.cuda.graph); `graph` is the cudaGraph_t as an int.  The plan belongs to its context, which must outlive
    it (closing the context destroys its plans)"""

    def __init__(self, ctx, handle):
        self.ctx, self._h = ctx, handle

    def launch(self):
        _check(self.ctx.lib.cb200_camera_plan_launch(self._h))

    @property
    def graph(self):
        g = C.c_void_p()
        _check(self.ctx.lib.cb200_camera_plan_graph(self._h, C.byref(g)))
        return g.value

    def close(self):
        if self._h and self.ctx._h:
            self.ctx.lib.cb200_camera_plan_destroy(self._h)
        self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class FountainSink:
    """Rank-0 fountain ingest (cb200_sink_*): header parse, de-dup and stream bookkeeping on the host, with the
    fountain codec (wirehair) supplied by the caller as a ctypes library exposing wirehair's C API."""

    def __init__(self, chunk_size, codec_lib=None):
        """codec_lib: a ctypes library exposing wirehair's C API, or None / a path for the wirehair build that ships with the
        package (lib/libwirehair.so, built by libcimbar_b200.build.build_wirehair)"""
        self.lib = load_library()
        if codec_lib is None or isinstance(codec_lib, (str, bytes)):
            path = codec_lib or os.path.join(HERE, "lib", "libwirehair.so")
            self._h = self.lib.cb200_sink_create_wirehair(chunk_size, path.encode() if isinstance(path, str) else path)
        else:
            fn = lambda name: C.cast(getattr(codec_lib, name), C.c_void_p)
            self._h = self.lib.cb200_sink_create(chunk_size, fn("wirehair_decoder_create"), fn("wirehair_decode"),
                                                 fn("wirehair_recover"), fn("wirehair_free"))
        if not self._h:
            raise Cb200Error("cb200_sink_create failed (is lib/libwirehair.so built? python -m libcimbar_b200.build)")
        self.chunk_size = chunk_size

    def close(self):
        if self._h:
            self.lib.cb200_sink_destroy(self._h)
            self._h = None

    def decode_frame(self, chunk):
        chunk = np.ascontiguousarray(chunk, dtype=np.uint8)
        return self.lib.cb200_sink_decode_frame(self._h, chunk.ctypes.data, chunk.size)

    def ingest(self, chunks, masks):
        chunks = np.ascontiguousarray(chunks, dtype=np.uint8)
        masks = np.ascontiguousarray(masks, dtype=np.uint32)
        n = masks.size
        return self.lib.cb200_sink_ingest(self._h, chunks.ctypes.data, masks.ctypes.data, n, chunks.size // (n * self.chunk_size))

    def file(self, file_id):
        size = self.lib.cb200_sink_file_size(self._h, file_id)
        if size < 0:
            return None
        out = np.zeros(size, dtype=np.uint8)
        _check(self.lib.cb200_sink_file_read(self._h, file_id, out.ctypes.data, size))
        return out
