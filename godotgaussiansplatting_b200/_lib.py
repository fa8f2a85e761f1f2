"""ctypes binding of the in-tree `libgsr.so` (include/gsr.h).

There is NO fallback: if the shared library is missing or does not load, importing a symbol raises, and
every entry point fails with GSR_ERR_CUDA when no sm_90 device is present.
"""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("GSR_LIB_PATH") or os.path.join(HERE, "libgsr.so")  # env override: kernel-variant experiments only

GSR_OK, GSR_ERR_INVALID, GSR_ERR_CUDA, GSR_ERR_OOM, GSR_ERR_STATE, GSR_ERR_OVERFLOW = range(6)
GSR_FLAG_REFERENCE_QUIRKS, GSR_FLAG_FIXED_RANGES, GSR_FLAG_FAST_REJECT, GSR_FLAG_STATIC_CAPACITY, GSR_FLAG_UNCONTRACTED_BLEND = 0x1, 0x2, 0x4, 0x8, 0x10
GSR_FLAG_ORTHOGRAPHIC = 0x20
GSR_FLAG_SH_HALF = 0x40   # SH coefficients stored as IEEE binary16 (include/gsr.h)
(GSR_BUF_RECORDS, GSR_BUF_KEYS, GSR_BUF_VALUES, GSR_BUF_BOUNDS, GSR_BUF_KEYS_UNSORTED, GSR_BUF_VALUES_UNSORTED,
 GSR_BUF_FRAMEBUFFER, GSR_BUF_COMPOSITOR_TRACE, GSR_BUF_COMPOSITOR_TRACE_COUNT, GSR_BUF_INSTANCES, GSR_BUF_SPLATS, GSR_BUF_DEPTH_WORDS_UNSORTED,
 GSR_BUF_INSTANCE_APPEARANCE, GSR_BUF_EDIT_TRANSFORM, GSR_BUF_EDIT_COLOR) = range(15)
GSR_DEPTH_ORDER_KEY16, GSR_DEPTH_ORDER_VIEW_DEPTH = 0, 1
GSR_MAX_CUTOUTS = 16
GSR_CUTOUT_BOX, GSR_CUTOUT_ELLIPSOID = 0, 1
GSR_CUTOUT_KEEP, GSR_CUTOUT_REMOVE = 0, 1
GSR_CUTOUT_FRAME, GSR_CUTOUT_SOURCE = 0, 1
GSR_MAX_INSTANCES, GSR_INSTANCE_RING = 4096, 8
GSR_TINT_MAX = 16.0
GSR_DRAW_ALL = 0xFFFFFFFFFFFFFFFF   # gsr_instance_appearance.draw_count: every splat of the range
GSR_NO_ID = 0xFFFFFFFF              # gsr_set_splat_ids: no splat / no instance
GSR_MAX_SELECT_VERTICES = 64
GSR_SELECT_SET, GSR_SELECT_ADD, GSR_SELECT_SUBTRACT, GSR_SELECT_TOGGLE = range(4)
GSR_PROP_OPACITY, GSR_PROP_SIZE, GSR_PROP_VOLUME, GSR_PROP_ISOTROPY, GSR_PROP_COLOR_DISTANCE = range(5)
GSR_PROP_CONTRIBUTION, GSR_PROP_PEAK_CONTRIBUTION, GSR_PROP_VIEWS, GSR_PROP_CONTRIBUTING_PIXELS = range(16, 20)   # gsr_set_splat_contribution
GSR_MAX_SPLAT_FILTERS = 8
GSR_MAX_HISTOGRAM_BINS = 1024
GSR_HISTOGRAM_KEPT, GSR_HISTOGRAM_SELECTED = 0, 1
GSR_NEIGHBOR_SPARSE, GSR_NEIGHBOR_GROW, GSR_NEIGHBOR_CONNECTED, GSR_NEIGHBOR_SMALL_CLUSTERS = range(4)
GSR_MAX_NEIGHBOR_CANDIDATES = 1 << 34
GSR_NEIGHBOR_MIN_RADIUS, GSR_NEIGHBOR_MAX_RADIUS = 2.0 ** -60, 2.0 ** 60
GSR_NEIGHBOR_SCRATCH_BYTES_PER_SLOT = 32
GSR_EXPORT_KEPT, GSR_EXPORT_SELECTED = 0, 1
GSR_COMPRESSED_CHUNK = 256
GSR_COMPRESS_STORE_ORDER, GSR_COMPRESS_MORTON = 0, 1

# every symbol include/gsr.h declares (tests/test_abi.py checks the header against this list and the .so)
EXPORTS = [
    "gsr_create", "gsr_destroy", "gsr_set_stream", "gsr_upload_splats_aos", "gsr_upload_ply_raw", "gsr_upload_ply", "gsr_resize", "gsr_set_band", "gsr_set_row_interleave", "gsr_band_sync_word", "gsr_band_fixup", "gsr_render",
    "gsr_render_async", "gsr_render_async_rgb", "gsr_render_async_fmt", "gsr_output_bytes", "gsr_present_device", "gsr_readback_async", "gsr_peer_export_framebuffers", "gsr_peer_import_framebuffers",
    "gsr_stream_join", "gsr_group_export", "gsr_group_attach", "gsr_group_detach", "gsr_group_set_present", "gsr_readback_rows_async", "gsr_sync", "gsr_framebuffer_device_ptr", "gsr_set_framebuffer_external",
    "gsr_set_depth_compositing", "gsr_set_motion_vectors", "gsr_reset_motion", "gsr_set_splat_ids", "gsr_set_instances", "gsr_set_instance_appearance", "gsr_set_sh_degree", "gsr_set_antialiasing", "gsr_set_depth_order", "gsr_set_cutouts", "gsr_upload_ply_filtered", "gsr_pick",
    "gsr_select_all", "gsr_select_polygon", "gsr_select_volume", "gsr_select_ids", "gsr_hide_selection", "gsr_unhide_all", "gsr_clear_splat_masks",
    "gsr_get_splat_masks", "gsr_set_splat_masks", "gsr_splat_mask_counts", "gsr_set_selection_style",
    "gsr_transform_selection", "gsr_splat_store_bytes", "gsr_copy_splat_store", "gsr_restore_splat_store", "gsr_recolor_selection",
    "gsr_delete_hidden", "gsr_duplicate_selection", "gsr_set_splat_count", "gsr_select_where", "gsr_splat_histogram",
    "gsr_select_neighborhood", "gsr_set_splat_contribution", "gsr_reset_splat_contribution", "gsr_splat_contribution_frames", "gsr_export_ply", "gsr_export_compressed_ply", "gsr_upload_compressed_ply",
    "gsr_get_stats", "gsr_get_frame_history", "gsr_debug_copy", "gsr_debug_enable_trace", "gsr_debug_compositor_config", "gsr_debug_pipeline", "gsr_debug_keep_unsorted", "gsr_sorter_create", "gsr_sorter_destroy",
    "gsr_sorter_sort_device", "gsr_sort_pairs_host", "gsr_sorter_last_ms", "gsr_error_string", "gsr_last_error",
    "gsr_device_count", "gsr_version",
]


class GsrConfig(C.Structure):
    _fields_ = [("device", C.c_int32), ("flags", C.c_uint32), ("max_splats", C.c_uint64),
                ("dup_capacity_factor", C.c_uint32), ("sh_bands", C.c_uint32)]


class GsrStats(C.Structure):
    _fields_ = [("num_splats", C.c_uint64), ("duplicates", C.c_uint64), ("visible", C.c_uint64), ("capacity", C.c_uint64),
                ("last_tile", C.c_int64), ("overflow", C.c_uint32), ("width", C.c_uint32), ("height", C.c_uint32),
                ("tiles_x", C.c_uint32), ("tiles_y", C.c_uint32), ("band_y0", C.c_uint32), ("band_y1", C.c_uint32),
                ("kernel_launches", C.c_uint32), ("stage_ms", C.c_float * 5), ("staged", C.c_uint64)]


class GsrPlyLayout(C.Structure):
    _fields_ = [("nprops", C.c_uint32), ("sh_degree", C.c_uint32), ("x", C.c_int32), ("f_dc", C.c_int32), ("f_rest", C.c_int32),
                ("opacity", C.c_int32), ("scale", C.c_int32), ("rot", C.c_int32)]


class GsrInstance(C.Structure):
    _fields_ = [("first", C.c_uint64), ("count", C.c_uint64), ("to_frame", C.c_float * 12)]


class GsrInstanceAppearance(C.Structure):
    _fields_ = [("tint", C.c_float * 3), ("opacity", C.c_float), ("draw_count", C.c_uint64)]


class GsrColorEdit(C.Structure):
    _fields_ = [("matrix", C.c_float * 12), ("band_scale", C.c_float * 3), ("opacity_scale", C.c_float), ("opacity_offset", C.c_float)]


class GsrNeighborhood(C.Structure):
    _fields_ = [("mode", C.c_int32), ("radius", C.c_float), ("count", C.c_uint32), ("instance", C.c_int32)]


class GsrNeighborhoodStats(C.Structure):
    _fields_ = [("participants", C.c_uint64), ("inside", C.c_uint64), ("candidates", C.c_uint64), ("clusters", C.c_uint64),
                ("largest_cluster", C.c_uint64)]


class GsrCompressedPly(C.Structure):
    _fields_ = [("chunks", C.c_void_p), ("packed", C.c_void_p), ("sh", C.c_void_p), ("rows", C.c_uint64), ("chunk_count", C.c_uint64),
                ("sh_degree", C.c_uint32), ("chunk_floats", C.c_uint32)]


class GsrSplatFilter(C.Structure):
    _fields_ = [("property", C.c_int32), ("lo", C.c_float), ("hi", C.c_float), ("rgb", C.c_float * 3)]


class GsrSplatContribution(C.Structure):
    _fields_ = [("weight", C.c_uint64), ("pixels", C.c_uint64), ("peak", C.c_float), ("views", C.c_uint32), ("last_frame", C.c_uint32),
                ("pad", C.c_uint32)]


class GsrCutout(C.Structure):
    _fields_ = [("to_local", C.c_float * 12), ("shape", C.c_int32), ("action", C.c_int32), ("space", C.c_int32)]


GSR_HISTORY_FRAMES = 512
GSR_OUT_RGBA32F, GSR_OUT_RGB32F, GSR_OUT_RGBA16F, GSR_OUT_RGBA8 = range(4)
GSR_OUT_SRGB_TO_LINEAR = 0x100
GSR_GROUP_BLOB_BYTES = 320


class GsrFrameRecord(C.Structure):
    _fields_ = [("frame_index", C.c_uint64), ("duplicates", C.c_uint64), ("visible", C.c_uint64), ("staged", C.c_uint64),
                ("overflow", C.c_uint32), ("reserved", C.c_uint32), ("stage_ms", C.c_float * 5), ("front_ms", C.c_float)]


class GsrError(RuntimeError):
    def __init__(self, code: int, where: str):
        L = lib()
        super().__init__(f"{where}: {L.gsr_error_string(code).decode()} [{code}] -- {L.gsr_last_error().decode()}")
        self.code = code


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(f"{LIB_PATH} is missing: build it with `python -m godotgaussiansplatting_b200.build` "
                              "(nvcc, sm_90a). There is no CPU fallback.")
        L = C.CDLL(LIB_PATH)
        vp, fp, u32 = C.c_void_p, C.POINTER(C.c_float), C.c_uint32
        L.gsr_create.argtypes = [C.POINTER(GsrConfig), C.POINTER(vp)]
        L.gsr_destroy.argtypes = [vp]
        L.gsr_set_stream.argtypes = [vp, vp]
        L.gsr_upload_splats_aos.argtypes = [vp, fp, C.c_uint64, C.c_uint64]
        L.gsr_upload_ply_raw.argtypes = [vp, fp, u32, C.c_uint64, C.c_uint64, C.c_float]
        L.gsr_upload_ply.argtypes = [vp, fp, C.POINTER(GsrPlyLayout), C.c_uint64, C.c_uint64, C.c_float]
        L.gsr_upload_ply_filtered.argtypes = [vp, fp, C.POINTER(GsrPlyLayout), C.c_int32, C.c_uint64, C.c_uint64, C.c_float]
        L.gsr_resize.argtypes = [vp, C.c_int32, C.c_int32]
        L.gsr_set_band.argtypes = [vp, C.c_int32, C.c_int32]
        L.gsr_set_row_interleave.argtypes = [vp, C.c_int32, C.c_int32]
        L.gsr_band_sync_word.argtypes = [vp]
        L.gsr_band_sync_word.restype = vp
        L.gsr_band_fixup.argtypes = [vp]
        L.gsr_render.argtypes = [vp, fp, vp, C.c_float, vp]
        L.gsr_render_async.argtypes = [vp, fp, vp, C.c_float, vp]
        L.gsr_render_async_rgb.argtypes = [vp, fp, vp, C.c_float, vp]
        L.gsr_render_async_fmt.argtypes = [vp, fp, vp, C.c_float, vp, C.c_int32]
        L.gsr_output_bytes.argtypes = [C.c_int32, C.c_int32, C.c_int32]
        L.gsr_output_bytes.restype = C.c_size_t
        L.gsr_present_device.argtypes = [vp, vp, C.c_int32]
        L.gsr_sync.argtypes = [vp]
        L.gsr_stream_join.argtypes = [vp]
        L.gsr_group_export.argtypes = [vp, vp]
        L.gsr_group_attach.argtypes = [vp, C.c_int32, C.c_int32, vp]
        L.gsr_group_detach.argtypes = [vp]
        L.gsr_group_set_present.argtypes = [vp, C.c_int32]
        L.gsr_readback_rows_async.argtypes = [vp, vp]
        L.gsr_readback_async.argtypes = [vp, vp, C.c_int]
        L.gsr_peer_export_framebuffers.argtypes = [vp, vp]
        L.gsr_peer_import_framebuffers.argtypes = [vp, vp]
        L.gsr_framebuffer_device_ptr.argtypes = [vp]
        L.gsr_framebuffer_device_ptr.restype = vp
        L.gsr_set_framebuffer_external.argtypes = [vp, vp]
        L.gsr_set_depth_compositing.argtypes = [vp, vp, vp]
        L.gsr_set_motion_vectors.argtypes = [vp, vp]
        L.gsr_reset_motion.argtypes = [vp]
        L.gsr_set_splat_ids.argtypes = [vp, vp]
        L.gsr_set_splat_contribution.argtypes = [vp, vp, C.c_uint64]
        L.gsr_reset_splat_contribution.argtypes = [vp]
        L.gsr_splat_contribution_frames.argtypes = [vp, C.POINTER(C.c_uint32)]
        L.gsr_set_instances.argtypes = [vp, C.POINTER(GsrInstance), u32]
        L.gsr_set_instance_appearance.argtypes = [vp, C.POINTER(GsrInstanceAppearance), u32]
        L.gsr_set_sh_degree.argtypes = [vp, C.c_int32]
        L.gsr_set_antialiasing.argtypes = [vp, C.c_float]
        L.gsr_set_depth_order.argtypes = [vp, C.c_int32]
        L.gsr_set_cutouts.argtypes = [vp, C.POINTER(GsrCutout), u32]
        L.gsr_pick.argtypes = [vp, u32, C.c_float, fp]
        u32p, u64 = C.POINTER(C.c_uint32), C.c_uint64
        L.gsr_select_all.argtypes = [vp, C.c_int32]
        L.gsr_select_polygon.argtypes = [vp, fp, C.c_float, C.c_int32, fp, u32, C.c_int32]
        L.gsr_select_volume.argtypes = [vp, C.POINTER(GsrCutout), C.c_float, C.c_int32, C.c_int32]
        L.gsr_select_ids.argtypes = [vp, vp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32]
        L.gsr_hide_selection.argtypes = [vp]
        L.gsr_unhide_all.argtypes = [vp]
        L.gsr_clear_splat_masks.argtypes = [vp]
        L.gsr_get_splat_masks.argtypes = [vp, u32p, u32p, u64]
        L.gsr_set_splat_masks.argtypes = [vp, u32p, u32p, u64]
        L.gsr_splat_mask_counts.argtypes = [vp, C.POINTER(u64), C.POINTER(u64)]
        L.gsr_set_selection_style.argtypes = [vp, fp, C.c_float]
        L.gsr_transform_selection.argtypes = [vp, fp, vp]
        L.gsr_recolor_selection.argtypes = [vp, C.POINTER(GsrColorEdit), vp]
        L.gsr_delete_hidden.argtypes = [vp, C.POINTER(u64)]
        L.gsr_duplicate_selection.argtypes = [vp, C.POINTER(u64)]
        L.gsr_set_splat_count.argtypes = [vp, u64]
        L.gsr_select_where.argtypes = [vp, C.POINTER(GsrSplatFilter), u32, C.c_int32, C.c_int32]
        L.gsr_splat_histogram.argtypes = [vp, C.POINTER(GsrSplatFilter), C.c_int32, C.c_int32, fp, u32, C.POINTER(u64), fp]
        L.gsr_select_neighborhood.argtypes = [vp, C.POINTER(GsrNeighborhood), C.c_int32, C.POINTER(GsrNeighborhoodStats)]
        L.gsr_export_ply.argtypes = [vp, C.c_int32, C.c_int32, vp, u64, C.POINTER(u64)]
        L.gsr_export_compressed_ply.argtypes = [vp, C.c_int32, C.c_int32, C.c_int32, C.POINTER(GsrCompressedPly), C.POINTER(u64)]
        L.gsr_upload_compressed_ply.argtypes = [vp, C.POINTER(GsrCompressedPly), u64, C.c_float]
        L.gsr_splat_store_bytes.argtypes = [vp]
        L.gsr_splat_store_bytes.restype = u64
        L.gsr_copy_splat_store.argtypes = [vp, vp]
        L.gsr_restore_splat_store.argtypes = [vp, vp]
        L.gsr_get_stats.argtypes = [vp, C.POINTER(GsrStats)]
        L.gsr_get_frame_history.argtypes = [vp, u32, C.POINTER(GsrFrameRecord), C.POINTER(u32)]
        L.gsr_debug_copy.argtypes = [vp, C.c_int, vp, C.c_size_t]
        L.gsr_debug_keep_unsorted.argtypes = [vp, C.c_int]
        L.gsr_debug_enable_trace.argtypes = [vp, u32]
        L.gsr_debug_compositor_config.argtypes = [vp, C.c_int32, C.c_int32, C.c_int32]
        L.gsr_debug_pipeline.argtypes = [vp, C.c_int32]
        L.gsr_sorter_create.argtypes = [C.c_int32, C.c_uint64, C.POINTER(vp)]
        L.gsr_sorter_destroy.argtypes = [vp]
        L.gsr_sorter_sort_device.argtypes = [vp, vp, vp, C.c_uint64, vp]
        L.gsr_sort_pairs_host.argtypes = [C.c_int32, C.POINTER(u32), C.POINTER(u32), C.c_uint64]
        L.gsr_sorter_last_ms.argtypes = [vp, fp]
        L.gsr_error_string.argtypes = [C.c_int]
        L.gsr_error_string.restype = C.c_char_p
        L.gsr_last_error.restype = C.c_char_p
        L.gsr_version.restype = C.c_char_p
        for name in EXPORTS:
            fn = getattr(L, name)
            if fn.restype is C.c_int and name not in ("gsr_device_count",):
                pass
        _lib = L
    return _lib


def check(code: int, where: str) -> None:
    if code != GSR_OK:
        raise GsrError(code, where)
