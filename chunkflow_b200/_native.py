"""ctypes binding of ``include/chunkflow_b200.h`` (the C-ABI of the CUDA hot path).

The library is loaded lazily and LOUDLY: if ``libchunkflow_b200.so`` is missing (and
cannot be built) or no CUDA device is present, every compute entry point raises --
there is no CPU fallback in the product path.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import numpy as np

OK = 0
ERR_INVALID_ARGUMENT, ERR_CUDA, ERR_WEIGHTS, ERR_OUTPUT_RANGE, ERR_UNSUPPORTED, ERR_CAPACITY = -1, -2, -3, -4, -5, -6
FRAMEWORK_UNET3L, FRAMEWORK_IDENTITY = 0, 1
PRECISION_F32_SIMT, PRECISION_F16X3_UMMA, PRECISION_F16_UMMA, PRECISION_F16F8_UMMA = 0, 1, 2, 3
LAYER_OPS = ("conv3", "conv3_pool", "convT", "maxpool", "first", "head_sigmoid", "head_blend", "conv3_head_blend", "round_trip")
DTYPE_U8, DTYPE_F32, DTYPE_U32, DTYPE_U64, DTYPE_BOOL = 0, 1, 2, 3, 4
AUGMENT_NONE, AUGMENT_REFERENCE, AUGMENT_SPATIAL = 0, 1, 2
QUANTIZE_XY, QUANTIZE_Z = 0, 1
HIST_SLOTS_PER_SLOT = 2   # cfb_region_graph_hist_device: the bin table has 2 x table_slots slots

# every symbol include/chunkflow_b200.h declares
EXPORTS = (
    "cfb_last_error", "cfb_version", "cfb_device_count", "cfb_device_memory", "cfb_create", "cfb_destroy", "cfb_device_name",
    "cfb_set_weight", "cfb_commit_weights", "cfb_patch_mask", "cfb_patch_grid", "cfb_output_shape",
    "cfb_infer_chunk_device", "cfb_infer_chunk_host", "cfb_infer_slab_device", "cfb_normalize_device",
    "cfb_slab_nonzero", "cfb_halo_add_device", "cfb_weight_volume_device",
    "cfb_patch_forward_host", "cfb_make_patch_mask", "cfb_plugin_begin", "cfb_plugin_extract", "cfb_plugin_blend",
    "cfb_plugin_end", "cfb_last_timing", "cfb_set_profiling", "cfb_layer_timing", "cfb_debug_net_forward_host", "cfb_debug_layer_host",
    "cfb_normalize_contrast_device", "cfb_maskout_device", "cfb_crop_margin_device", "cfb_quantize_device",
    "cfb_connected_components_device", "cfb_connected_components_workspace",
    "cfb_watershed_workspace", "cfb_watershed_device", "cfb_region_graph_workspace", "cfb_region_graph_device",
    "cfb_region_graph_read", "cfb_agglomerate_edges_host", "cfb_relabel_device",
    "cfb_region_graph_hist_workspace", "cfb_region_graph_hist_device", "cfb_region_graph_hist_read", "cfb_agglomerate_quantile_host",
    "cfb_evaluate_workspace", "cfb_contingency_device", "cfb_contingency_scores", "cfb_contingency_read",
    "cfb_label_table_workspace", "cfb_label_table_device", "cfb_label_table_read", "cfb_label_table_plan",
    "cfb_label_apply_device", "cfb_downsample_average_device", "cfb_downsample_workspace", "cfb_downsample_segmentation_device",
    "cfb_gaussian_filter_workspace", "cfb_gaussian_filter_device", "cfb_median_filter_device",
    "cfb_clahe_workspace", "cfb_clahe_device",
    "cfb_mesh_workspace", "cfb_mesh_count_device", "cfb_mesh_buffer_bytes", "cfb_mesh_device", "cfb_mesh_read", "cfb_mesh_simplify_host",
    "cfb_skeleton_workspace", "cfb_edt_workspace", "cfb_edt_device", "cfb_skeleton_count_device", "cfb_skeleton_device", "cfb_skeleton_read",
    "cfb_fill_holes_workspace", "cfb_fill_holes_table_workspace", "cfb_fill_holes_components_device", "cfb_fill_holes_graph_device",
    "cfb_fill_holes_enclose", "cfb_fill_holes_apply_device",
)


class Params(C.Structure):
    _fields_ = [
        ("struct_size", C.c_int32), ("device", C.c_int32), ("framework", C.c_int32), ("precision", C.c_int32),
        ("input_patch_size", C.c_int32 * 3), ("output_patch_size", C.c_int32 * 3),
        ("output_patch_overlap", C.c_int32 * 3), ("output_crop_margin", C.c_int32 * 3),
        ("num_input_channels", C.c_int32), ("num_output_channels", C.c_int32), ("batch_size", C.c_int32),
        ("mask_output_chunk", C.c_int32), ("augment", C.c_int32), ("has_myelin_threshold", C.c_int32),
        ("mask_myelin_threshold", C.c_float), ("check_output_range", C.c_int32),
    ]


class SegScores(C.Structure):
    """cfb_seg_scores: the statistics of a contingency table and the five scores of one size threshold."""
    _fields_ = [
        ("struct_size", C.c_int32), ("reserved", C.c_int32),
        ("n", C.c_uint64), ("sum_sq_pairs", C.c_uint64), ("sum_sq_rows", C.c_uint64), ("sum_sq_cols", C.c_uint64),
        ("n_both_nonzero", C.c_uint64), ("seg_ids", C.c_uint64), ("gt_ids", C.c_uint64), ("pairs", C.c_uint64),
        ("pairs_over_threshold", C.c_uint64),
        ("size_threshold", C.c_double), ("xlog_pairs", C.c_double), ("xlog_rows", C.c_double), ("xlog_cols", C.c_double),
        ("rand_index", C.c_double), ("adjusted_rand_index", C.c_double), ("variation_of_information", C.c_double),
        ("fowlkes_mallows_index", C.c_double), ("false_merges", C.c_double), ("false_splits", C.c_double),
    ]

    def as_dict(self) -> dict:
        return {name: getattr(self, name) for name, _ in self._fields_ if name not in ("struct_size", "reserved")}


class LayerArgs(C.Structure):
    """cfb_layer_args: one step of the U-Net layer table for cfb_debug_layer_host."""
    _fields_ = [
        ("struct_size", C.c_int32), ("op", C.c_int32), ("nb", C.c_int32), ("size", C.c_int32 * 3),
        ("ca", C.c_int32), ("cb", C.c_int32), ("cout", C.c_int32), ("relu", C.c_int32),
        ("a", C.c_void_p), ("b", C.c_void_p), ("weight", C.c_void_p), ("bias", C.c_void_p),
        ("head_weight", C.c_void_p), ("head_bias", C.c_void_p), ("head_channels", C.c_int32),
        ("chunk_dtype", C.c_int32), ("chunk", C.c_void_p), ("chunk_size", C.c_int32 * 3),
        ("out_patch", C.c_int32 * 3), ("crop", C.c_int32 * 3), ("out_size", C.c_int32 * 3),
        ("in_origins", C.c_void_p), ("out_origins", C.c_void_p), ("mask", C.c_void_p), ("scale", C.c_float),
        ("out", C.c_void_p), ("pooled", C.c_void_p),
    ]


class NativeError(RuntimeError):
    def __init__(self, code: int, message: str):
        super().__init__(f"chunkflow_b200 native error {code}: {message}")
        self.code = code


_lib: Optional[C.CDLL] = None


def library_path() -> str:
    from .build import LIB_PATH
    return LIB_PATH


def load() -> C.CDLL:
    """Load (building in-tree first if the sources are newer) the native library."""
    global _lib
    if _lib is not None:
        return _lib
    from .build import build_native, LIB_PATH
    path = LIB_PATH
    override = os.environ.get("CFB_NATIVE_LIB")  # development: an instrumented build (python -m chunkflow_b200.build --variant)
    try:
        path = override if override else build_native()
        if override and not os.path.exists(override):
            raise RuntimeError(f"CFB_NATIVE_LIB={override} does not exist")
    except Exception as exc:  # no nvcc on this box: use the prebuilt .so that travelled with the tree
        if override or not os.path.exists(LIB_PATH):
            raise RuntimeError(
                "chunkflow_b200: the CUDA extension libchunkflow_b200.so is missing and could not be built "
                f"({exc}); there is no CPU fallback") from exc
    lib = C.CDLL(path)
    vp, i32, i64, f32p = C.c_void_p, C.c_int32, C.c_int64, C.POINTER(C.c_float)
    lib.cfb_last_error.restype = C.c_char_p
    lib.cfb_device_name.restype = C.c_char_p
    lib.cfb_device_name.argtypes = [vp]
    lib.cfb_version.restype = C.c_int
    lib.cfb_device_count.restype = C.c_int
    lib.cfb_device_memory.argtypes = [i32, C.POINTER(i64), C.POINTER(i64)]
    lib.cfb_create.argtypes = [C.POINTER(Params), C.POINTER(vp)]
    lib.cfb_destroy.argtypes = [vp]
    lib.cfb_set_weight.argtypes = [vp, C.c_char_p, vp, i64]
    lib.cfb_commit_weights.argtypes = [vp]
    lib.cfb_patch_mask.argtypes = [vp, vp]
    lib.cfb_patch_grid.argtypes = [vp, i64, i64, i64, C.POINTER(i64), vp, i64]
    lib.cfb_output_shape.argtypes = [vp, i64, i64, i64, C.POINTER(i64 * 4)]
    lib.cfb_infer_chunk_device.argtypes = [vp, vp, i32, i64, i64, i64, vp, vp]
    lib.cfb_infer_chunk_host.argtypes = [vp, vp, i32, i64, i64, i64, vp]
    lib.cfb_infer_slab_device.argtypes = [vp, vp, i32, i64, i64, i64, i64, i64, vp, vp, vp]
    lib.cfb_normalize_device.argtypes = [vp, vp, vp, i32, i64, i64, i64, i64, i32, vp]
    lib.cfb_slab_nonzero.argtypes = [vp, C.POINTER(i32), vp]
    lib.cfb_halo_add_device.argtypes = [vp, vp, i64, vp]
    lib.cfb_weight_volume_device.argtypes = [vp, i64, i64, i64, i64, i64, i32, vp, vp]
    lib.cfb_patch_forward_host.argtypes = [vp, vp, i32, vp]
    lib.cfb_make_patch_mask.argtypes = [C.POINTER(i32 * 3), C.POINTER(i32 * 3), vp]
    lib.cfb_plugin_begin.argtypes = [vp, vp, i32, i64, i64, i64]
    lib.cfb_plugin_extract.argtypes = [vp, i64, i32, vp]
    lib.cfb_plugin_blend.argtypes = [vp, i64, i32, vp]
    lib.cfb_plugin_end.argtypes = [vp, vp]
    lib.cfb_last_timing.argtypes = [vp, C.POINTER(C.c_float * 5), C.POINTER(i64)]
    lib.cfb_set_profiling.argtypes = [vp, i32]
    lib.cfb_layer_timing.argtypes = [vp, i32, C.POINTER(i32), vp, vp, vp]
    lib.cfb_debug_net_forward_host.argtypes = [vp, vp, vp]
    lib.cfb_debug_layer_host.argtypes = [vp, C.POINTER(LayerArgs)]
    lib.cfb_normalize_contrast_device.argtypes = [vp, i64, i64, i64, C.c_double, C.c_double, i32, i32, i32, vp]
    lib.cfb_maskout_device.argtypes = [vp, i32, i64, i64, i64, i64, vp, i32, i64, i64, i64, vp]
    lib.cfb_crop_margin_device.argtypes = [vp, i32, i64, i64, i64, i64, C.POINTER(i64 * 6), vp, vp]
    lib.cfb_quantize_device.argtypes = [vp, i64, i64, i64, i64, i32, vp, vp]
    lib.cfb_connected_components_device.argtypes = [vp, i32, i64, i64, i64, C.c_float, i32, vp, vp, C.POINTER(C.c_uint32), vp]
    lib.cfb_connected_components_workspace.argtypes = [i64, i64, i64]
    lib.cfb_connected_components_workspace.restype = i64
    lib.cfb_watershed_workspace.argtypes = [i64, i64, i64]
    lib.cfb_watershed_workspace.restype = i64
    lib.cfb_watershed_device.argtypes = [vp, i32, i64, i64, i64, C.c_float, C.c_float, vp, vp, C.POINTER(C.c_uint32), vp]
    lib.cfb_region_graph_workspace.argtypes = [i64]
    lib.cfb_region_graph_workspace.restype = i64
    lib.cfb_region_graph_device.argtypes = [vp, i32, vp, i64, i64, i64, vp, i64, C.POINTER(i64), vp]
    lib.cfb_region_graph_read.argtypes = [vp, i64, i64, vp, vp, vp, vp, vp]
    lib.cfb_agglomerate_edges_host.argtypes = [i64, i64, vp, vp, vp, vp, C.c_float, vp]
    lib.cfb_relabel_device.argtypes = [vp, i64, vp, i64, vp, vp]
    lib.cfb_region_graph_hist_workspace.argtypes = [i64]
    lib.cfb_region_graph_hist_workspace.restype = i64
    lib.cfb_region_graph_hist_device.argtypes = [vp, i32, vp, i64, i64, i64, i32, vp, i64, C.POINTER(i64), C.POINTER(i64), vp]
    lib.cfb_region_graph_hist_read.argtypes = [vp, i64, i64, i64, vp, vp, vp, vp, vp, vp, vp]
    lib.cfb_agglomerate_quantile_host.argtypes = [i64, i64, vp, vp, vp, vp, vp, vp, i32, i32, i32, C.c_float, vp]
    lib.cfb_evaluate_workspace.argtypes = [i64]
    lib.cfb_evaluate_workspace.restype = i64
    lib.cfb_contingency_device.argtypes = [vp, i32, vp, i32, i64, i64, i64, vp, i64, C.POINTER(i64), vp]
    lib.cfb_contingency_scores.argtypes = [vp, i64, C.c_double, C.POINTER(SegScores), vp]
    lib.cfb_contingency_read.argtypes = [vp, i64, i64, vp, vp, vp, vp]
    lib.cfb_label_table_workspace.argtypes = [i64, i64]
    lib.cfb_label_table_workspace.restype = i64
    lib.cfb_label_table_device.argtypes = [vp, i32, i64, i64, i64, vp, i64, C.POINTER(i64), vp]
    lib.cfb_label_table_read.argtypes = [vp, i64, i64, vp, vp, vp, vp]
    lib.cfb_label_table_plan.argtypes = [vp, i64, i64, i32, i64, vp, i64, i32, C.c_uint64, C.POINTER(i64), C.POINTER(i64),
                                         C.POINTER(C.c_uint64), vp]
    lib.cfb_label_apply_device.argtypes = [vp, i32, i64, vp, i64, vp, i32, vp]
    lib.cfb_downsample_average_device.argtypes = [vp, i64, i64, i64, C.POINTER(i64 * 3), vp, vp]
    lib.cfb_downsample_workspace.argtypes = [i32, i64, i64, i64, C.POINTER(i64 * 3), C.POINTER(i64 * 3), C.POINTER(i64)]
    lib.cfb_downsample_segmentation_device.argtypes = [vp, i32, i64, i64, i64, C.POINTER(i64 * 3), vp, vp, vp]
    dp = C.POINTER(C.c_double)
    lib.cfb_gaussian_filter_workspace.argtypes = [i32, i64, i64, i64, i64, C.POINTER(i64)]
    lib.cfb_gaussian_filter_device.argtypes = [vp, i32, i64, i64, i64, i64, dp, i32, dp, i32, dp, i32, vp, i64, vp]
    lib.cfb_median_filter_device.argtypes = [vp, i32, i64, i64, i64, i64, C.POINTER(i64 * 4), i32, vp, vp]
    lib.cfb_clahe_workspace.argtypes = [i64, i64, i64, i32, i32, C.POINTER(i64)]
    lib.cfb_clahe_device.argtypes = [vp, vp, i64, i64, i64, C.c_double, i32, i32, vp, i64, vp]
    bind_mesh(lib)
    bind_skeleton(lib)
    bind_fill_holes(lib)
    for name in EXPORTS:
        getattr(lib, name)   # every declared symbol must be there
    _lib = lib
    return lib


def check(code: int) -> None:
    if code != OK:
        raise NativeError(code, load().cfb_last_error().decode("utf-8", "replace"))


def _ptr(a: np.ndarray) -> C.c_void_p:
    return C.c_void_p(a.ctypes.data)


# ---- operators either side of `inference` on device pointers (include/chunkflow_b200.h, SURVEY section 8 f3) ----
def normalize_contrast_device(d_image: int, zyx, lower_clip_fraction: float, upper_clip_fraction: float, minval: int,
                              maxval: int, per_section: bool, stream: int = 0) -> None:
    check(load().cfb_normalize_contrast_device(C.c_void_p(d_image), *(int(v) for v in zyx), float(lower_clip_fraction),
                                               float(upper_clip_fraction), int(minval), int(maxval), int(bool(per_section)),
                                               C.c_void_p(stream)))


def maskout_device(d_chunk: int, chunk_dtype: int, czyx, d_mask: int, mask_dtype: int, factor, stream: int = 0) -> None:
    check(load().cfb_maskout_device(C.c_void_p(d_chunk), int(chunk_dtype), *(int(v) for v in czyx), C.c_void_p(d_mask),
                                    int(mask_dtype), *(int(v) for v in factor), C.c_void_p(stream)))


def crop_margin_device(d_src: int, dtype: int, czyx, margin6, d_dst: int, stream: int = 0) -> None:
    m = (C.c_int64 * 6)(*(int(v) for v in margin6))
    check(load().cfb_crop_margin_device(C.c_void_p(d_src), int(dtype), *(int(v) for v in czyx), C.byref(m), C.c_void_p(d_dst),
                                        C.c_void_p(stream)))


def quantize_device(d_affinity: int, czyx, mode: int, d_out: int, stream: int = 0) -> None:
    check(load().cfb_quantize_device(C.c_void_p(d_affinity), *(int(v) for v in czyx), int(mode), C.c_void_p(d_out),
                                     C.c_void_p(stream)))


def connected_components_workspace(zyx) -> int:
    return int(load().cfb_connected_components_workspace(*(int(v) for v in zyx)))


def connected_components_device(d_in: int, in_dtype: int, zyx, threshold: float, connectivity: int, d_labels: int, d_workspace: int,
                                stream: int = 0) -> int:
    """-> number of components (synchronises the stream)."""
    n = C.c_uint32()
    check(load().cfb_connected_components_device(C.c_void_p(d_in), int(in_dtype), *(int(v) for v in zyx), float(threshold or 0.0),
                                                 int(connectivity), C.c_void_p(d_labels), C.c_void_p(d_workspace), C.byref(n),
                                                 C.c_void_p(stream)))
    return int(n.value)


# ---- `agglomerate` (include/chunkflow_b200.h, SURVEY section 8 f4) ----
def watershed_workspace(zyx) -> int:
    return int(load().cfb_watershed_workspace(*(int(v) for v in zyx)))


def watershed_device(d_affs: int, flip_channel: bool, zyx, aff_threshold_low: float, aff_threshold_high: float, d_fragments: int,
                     d_workspace: int, stream: int = 0) -> int:
    """-> number of fragments (synchronises the stream)."""
    n = C.c_uint32()
    check(load().cfb_watershed_device(C.c_void_p(d_affs), int(bool(flip_channel)), *(int(v) for v in zyx), float(aff_threshold_low),
                                      float(aff_threshold_high), C.c_void_p(d_fragments), C.c_void_p(d_workspace), C.byref(n),
                                      C.c_void_p(stream)))
    return int(n.value)


def region_graph_workspace(table_slots: int) -> int:
    return int(load().cfb_region_graph_workspace(int(table_slots)))


def region_graph_device(d_affs: int, flip_channel: bool, d_fragments: int, zyx, d_workspace: int, table_slots: int,
                        stream: int = 0) -> int:
    """-> number of edges; raises NativeError with code ERR_CAPACITY when the table is too small."""
    n = C.c_int64()
    check(load().cfb_region_graph_device(C.c_void_p(d_affs), int(bool(flip_channel)), C.c_void_p(d_fragments), *(int(v) for v in zyx),
                                         C.c_void_p(d_workspace), int(table_slots), C.byref(n), C.c_void_p(stream)))
    return int(n.value)


def region_graph_read(d_workspace: int, table_slots: int, num_edges: int, stream: int = 0):
    """-> (u, v, sum_fixed, count) host arrays sorted by (u, v)."""
    u, v = np.empty(num_edges, np.uint32), np.empty(num_edges, np.uint32)
    s, c = np.empty(num_edges, np.uint64), np.empty(num_edges, np.uint32)
    check(load().cfb_region_graph_read(C.c_void_p(d_workspace), int(table_slots), int(num_edges), _ptr(u), _ptr(v), _ptr(s), _ptr(c),
                                       C.c_void_p(stream)))
    return u, v, s, c


def agglomerate_edges_host(num_nodes: int, u, v, sum_fixed, count, threshold: float) -> np.ndarray:
    """The merge loop on the host (no GPU involved) -> root_of (num_nodes,) uint32."""
    u = np.ascontiguousarray(u, np.uint32); v = np.ascontiguousarray(v, np.uint32)
    s = np.ascontiguousarray(sum_fixed, np.uint64); c = np.ascontiguousarray(count, np.uint32)
    if not (u.shape == v.shape == s.shape == c.shape and u.ndim == 1):
        raise ValueError("edge arrays must be one-dimensional and of equal length")
    root = np.empty(int(num_nodes), np.uint32)
    check(load().cfb_agglomerate_edges_host(int(num_nodes), int(u.size), _ptr(u), _ptr(v), _ptr(s), _ptr(c), float(threshold), _ptr(root)))
    return root


def region_graph_hist_workspace(table_slots: int) -> int:
    return int(load().cfb_region_graph_hist_workspace(int(table_slots)))


def region_graph_hist_device(d_affs: int, flip_channel: bool, d_fragments: int, zyx, bins: int, d_workspace: int, table_slots: int,
                             stream: int = 0):
    """-> (edges, histogram entries); raises NativeError with code ERR_CAPACITY when a table is too small."""
    n, nh = C.c_int64(), C.c_int64()
    check(load().cfb_region_graph_hist_device(C.c_void_p(d_affs), int(bool(flip_channel)), C.c_void_p(d_fragments),
                                              *(int(v) for v in zyx), int(bins), C.c_void_p(d_workspace), int(table_slots),
                                              C.byref(n), C.byref(nh), C.c_void_p(stream)))
    return int(n.value), int(nh.value)


def region_graph_hist_read(d_workspace: int, table_slots: int, num_edges: int, num_entries: int, stream: int = 0):
    """-> (u, v, offsets, bins, counts, maxima) host arrays, edges sorted by (u, v), each run of bins sorted."""
    u, v, mx = np.empty(num_edges, np.uint32), np.empty(num_edges, np.uint32), np.empty(num_edges, np.float32)
    off = np.empty(num_edges + 1, np.uint64)
    b, c = np.empty(num_entries, np.uint8), np.empty(num_entries, np.uint32)
    check(load().cfb_region_graph_hist_read(C.c_void_p(d_workspace), int(table_slots), int(num_edges), int(num_entries), _ptr(u),
                                            _ptr(v), _ptr(off), _ptr(b), _ptr(c), _ptr(mx), C.c_void_p(stream)))
    return u, v, off, b, c, mx


def agglomerate_quantile_host(num_nodes: int, u, v, offsets, bins, counts, maxima, threshold: float, quantile: int, num_bins: int,
                              init_with_max: bool) -> np.ndarray:
    """The merge loop with a histogram-quantile score, on the host (no GPU involved) -> root_of (num_nodes,) uint32."""
    u = np.ascontiguousarray(u, np.uint32); v = np.ascontiguousarray(v, np.uint32)
    off = np.ascontiguousarray(offsets, np.uint64)
    b = np.ascontiguousarray(bins, np.uint8); c = np.ascontiguousarray(counts, np.uint32)
    if not (u.shape == v.shape and u.ndim == 1 and off.shape == (u.size + 1,) and b.shape == c.shape and b.ndim == 1):
        raise ValueError("edge arrays must be one-dimensional, offsets one longer than the edges, bins as long as counts")
    if off[-1] != b.size:
        raise ValueError("offsets[-1] must be the number of bins")
    mx = np.ascontiguousarray(maxima if maxima is not None else np.zeros(u.size), np.float32)
    if mx.shape != u.shape:
        raise ValueError("one maximum per edge")
    root = np.empty(int(num_nodes), np.uint32)
    check(load().cfb_agglomerate_quantile_host(int(num_nodes), int(u.size), _ptr(u), _ptr(v), _ptr(off), _ptr(b), _ptr(c), _ptr(mx),
                                               int(quantile), int(num_bins), int(bool(init_with_max)), float(threshold), _ptr(root)))
    return root


def relabel_device(d_labels: int, n: int, d_map: int, map_size: int, d_out: int, stream: int = 0) -> None:
    check(load().cfb_relabel_device(C.c_void_p(d_labels), int(n), C.c_void_p(d_map), int(map_size), C.c_void_p(d_out),
                                    C.c_void_p(stream)))


# ---- `evaluate-segmentation` (include/chunkflow_b200.h, DESIGN.md section 0, row f5) ----
def evaluate_workspace(table_slots: int) -> int:
    return int(load().cfb_evaluate_workspace(int(table_slots)))


def contingency_device(d_seg: int, seg_dtype: int, d_gt: int, gt_dtype: int, zyx, d_workspace: int, table_slots: int,
                       stream: int = 0) -> int:
    """-> number of (seg id, gt id) pairs; raises NativeError with code ERR_CAPACITY when the table is too small."""
    n = C.c_int64()
    check(load().cfb_contingency_device(C.c_void_p(d_seg), int(seg_dtype), C.c_void_p(d_gt), int(gt_dtype), *(int(v) for v in zyx),
                                        C.c_void_p(d_workspace), int(table_slots), C.byref(n), C.c_void_p(stream)))
    return int(n.value)


def contingency_scores(d_workspace: int, table_slots: int, size_threshold: float, stream: int = 0) -> SegScores:
    out = SegScores()
    out.struct_size = C.sizeof(SegScores)
    check(load().cfb_contingency_scores(C.c_void_p(d_workspace), int(table_slots), float(size_threshold), C.byref(out),
                                        C.c_void_p(stream)))
    return out


def contingency_read(d_workspace: int, table_slots: int, num_pairs: int, stream: int = 0):
    """-> (seg ids uint64, gt ids uint64, counts uint32) host arrays sorted by (seg, gt)."""
    s, g, c = np.empty(num_pairs, np.uint64), np.empty(num_pairs, np.uint64), np.empty(num_pairs, np.uint32)
    check(load().cfb_contingency_read(C.c_void_p(d_workspace), int(table_slots), int(num_pairs), _ptr(s), _ptr(g), _ptr(c),
                                      C.c_void_p(stream)))
    return s, g, c


# ---- `mask-out-objects` / `remap-segmentation` (include/chunkflow_b200.h, DESIGN.md section 0, row f6) ----
LABEL_DTYPES = (DTYPE_U8, DTYPE_U32, DTYPE_U64)
MAX_LABEL_VOXELS = 2 ** 32 - 2


def _label_volume(zyx) -> int:
    """Voxel count of a (z, y, x) label volume, checked before the native side reads anything."""
    zyx = tuple(int(v) for v in zyx)
    if len(zyx) != 3 or min(zyx) <= 0:
        raise ValueError(f"a label volume is (z, y, x) with positive sizes, not {zyx}")
    n = zyx[0] * zyx[1] * zyx[2]
    if n > MAX_LABEL_VOXELS:
        raise ValueError("more than 2^32 - 2 voxels")
    return n


def _label_slots(table_slots) -> int:
    slots = int(table_slots)
    if slots < 32 or slots & (slots - 1) or slots >= 1 << 31:
        raise ValueError("table_slots must be a power of two in [32, 2^31)")
    return slots


def _label_dtype(dtype) -> int:
    if dtype not in LABEL_DTYPES:
        raise TypeError("label dtype must be DTYPE_U8, DTYPE_U32 or DTYPE_U64")
    return int(dtype)


def check_base_id(base_id) -> int:
    """``base_id`` of remap as a Python int in [0, 2^64 - 1]."""
    if isinstance(base_id, bool) or not isinstance(base_id, (int, np.integer)):
        raise TypeError(f"base_id must be an integer, not {type(base_id).__name__}")
    base_id = int(base_id)
    if base_id < 0:
        raise ValueError("base_id must not be negative")
    if base_id > 2 ** 64 - 1:
        raise ValueError("base_id must be below 2^64")
    return base_id


def label_table_workspace(voxels: int, table_slots: int) -> int:
    return int(load().cfb_label_table_workspace(int(voxels), _label_slots(table_slots)))


def label_table_device(d_labels: int, dtype: int, zyx, d_workspace: int, table_slots: int, stream: int = 0) -> int:
    """-> number of distinct labels; raises NativeError with code ERR_CAPACITY when the table is too small."""
    _label_volume(zyx)
    dtype, slots = _label_dtype(dtype), _label_slots(table_slots)
    n = C.c_int64()
    check(load().cfb_label_table_device(C.c_void_p(d_labels), dtype, *(int(v) for v in zyx), C.c_void_p(d_workspace), slots,
                                        C.byref(n), C.c_void_p(stream)))
    return int(n.value)


def label_table_read(d_workspace: int, table_slots: int, num_labels: int, stream: int = 0):
    """-> (ids uint64 ascending, voxel counts uint32, linear index of each id's first voxel uint32) host arrays."""
    slots, num = _label_slots(table_slots), int(num_labels)
    if not 0 <= num <= slots:
        raise ValueError("num_labels must be between 0 and table_slots")
    ids, counts, first = np.empty(num, np.uint64), np.empty(num, np.uint32), np.empty(num, np.uint32)
    check(load().cfb_label_table_read(C.c_void_p(d_workspace), slots, num, _ptr(ids), _ptr(counts), _ptr(first), C.c_void_p(stream)))
    return ids, counts, first


def label_table_plan(d_workspace: int, table_slots: int, voxels: int, dust_threshold=None, d_keep_ids: int = 0, num_keep=None,
                     renumber: bool = False, base_id: int = 0, stream: int = 0):
    """Write every table entry's new value: 0 when ``count <= dust_threshold`` (if given) or when the id is not among the
    ``num_keep`` ids at ``d_keep_ids`` (if ``num_keep`` is given; 0 masks everything), else the id, or with ``renumber``
    1 + base_id + the rank of its first voxel.  -> (entries failing the dust test, surviving non-zero ids, new maximum)."""
    slots = _label_slots(table_slots)
    voxels = int(voxels)
    if not 0 < voxels <= MAX_LABEL_VOXELS:
        raise ValueError("voxels must be in [1, 2^32 - 2]")
    base_id = check_base_id(base_id)
    if base_id and not renumber:
        raise ValueError("base_id needs renumber")
    if dust_threshold is not None:
        if isinstance(dust_threshold, bool) or not isinstance(dust_threshold, (int, np.integer)):
            raise TypeError("the dust threshold is an integer number of voxels")
        if not -2 ** 63 <= int(dust_threshold) < 2 ** 63:
            raise ValueError("the dust threshold does not fit in 64 bits")
    if num_keep is not None and (int(num_keep) < 0 or (int(num_keep) > 0 and not d_keep_ids)):
        raise ValueError("a keep-list of num_keep >= 0 ids needs a device pointer when it is not empty")
    dust, survivors, new_max = C.c_int64(), C.c_int64(), C.c_uint64()
    check(load().cfb_label_table_plan(C.c_void_p(d_workspace), slots, voxels, int(dust_threshold is not None),
                                      int(dust_threshold or 0), C.c_void_p(d_keep_ids or None), -1 if num_keep is None else int(num_keep),
                                      int(bool(renumber)), C.c_uint64(base_id), C.byref(dust), C.byref(survivors), C.byref(new_max),
                                      C.c_void_p(stream)))
    return int(dust.value), int(survivors.value), int(new_max.value)


def label_apply_device(d_in: int, in_dtype: int, voxels: int, d_workspace: int, table_slots: int, d_out: int, out_dtype: int,
                       stream: int = 0) -> None:
    """d_out[i] = planned new value of d_in[i]; ``d_out`` may be ``d_in`` when the dtypes are equal."""
    in_dtype, out_dtype, slots = _label_dtype(in_dtype), _label_dtype(out_dtype), _label_slots(table_slots)
    if out_dtype not in (in_dtype, DTYPE_U64):
        raise TypeError("the output is of the input's dtype or uint64")
    if d_in == d_out and in_dtype != out_dtype:
        raise ValueError("in place needs equal dtypes")
    if not 0 < int(voxels) <= MAX_LABEL_VOXELS:
        raise ValueError("voxels must be in [1, 2^32 - 2]")
    check(load().cfb_label_apply_device(C.c_void_p(d_in), in_dtype, int(voxels), C.c_void_p(d_workspace), slots, C.c_void_p(d_out),
                                        out_dtype, C.c_void_p(stream)))


# ---- `downsample` (include/chunkflow_b200.h, DESIGN.md section 0, row f7) ----
SEGMENTATION_DOWNSAMPLE_DTYPES = (DTYPE_U32, DTYPE_U64, DTYPE_BOOL)


def _zyx_and_factor(zyx, factor):
    zyx, factor = tuple(int(v) for v in zyx), tuple(int(v) for v in factor)
    if len(zyx) != 3 or min(zyx) <= 0:
        raise ValueError(f"a volume is (z, y, x) with positive sizes, not {zyx}")
    if len(factor) != 3:
        raise ValueError(f"the factor is (z, y, x), not {factor}")
    if min(factor) <= 0:
        raise ValueError(f"Factors less than one don't make sense. Factor: {factor}")
    return zyx, (C.c_int64 * 3)(*factor)


def _check_refusal(code: int) -> None:
    """A refused factor (the reference raises on it) is a ValueError, like the reference's own refusals."""
    if code == ERR_INVALID_ARGUMENT:
        raise ValueError(load().cfb_last_error().decode("utf-8", "replace"))
    check(code)


def downsample_average_device(d_in: int, zyx, factor, d_out: int, stream: int = 0) -> None:
    """uint8 averaging of the (z, y, x) volume at ``d_in`` into ceil(zyx / factor) voxels at ``d_out``."""
    zyx, f = _zyx_and_factor(zyx, factor)
    _check_refusal(load().cfb_downsample_average_device(C.c_void_p(d_in), *zyx, C.byref(f), C.c_void_p(d_out), C.c_void_p(stream)))


def downsample_workspace(dtype: int, zyx, factor) -> tuple:
    """The plan of a segmentation factor (no device needed) -> (output (z, y, x), workspace bytes); ValueError when refused."""
    if dtype not in SEGMENTATION_DOWNSAMPLE_DTYPES:
        raise TypeError("a segmentation to downsample is DTYPE_U32, DTYPE_U64 or DTYPE_BOOL")
    zyx, f = _zyx_and_factor(zyx, factor)
    out, work = (C.c_int64 * 3)(), C.c_int64()
    _check_refusal(load().cfb_downsample_workspace(int(dtype), *zyx, C.byref(f), C.byref(out), C.byref(work)))
    return tuple(out), int(work.value)


def downsample_segmentation_device(d_in: int, dtype: int, zyx, factor, d_workspace: int, d_out: int, stream: int = 0) -> None:
    """Mode pooling (countless) or striding of the (z, y, x) segmentation at ``d_in``, level after level, into ``d_out``."""
    if dtype not in SEGMENTATION_DOWNSAMPLE_DTYPES:
        raise TypeError("a segmentation to downsample is DTYPE_U32, DTYPE_U64 or DTYPE_BOOL")
    zyx, f = _zyx_and_factor(zyx, factor)
    _check_refusal(load().cfb_downsample_segmentation_device(C.c_void_p(d_in), int(dtype), *zyx, C.byref(f),
                                                             C.c_void_p(d_workspace or None), C.c_void_p(d_out), C.c_void_p(stream)))


# ---- `gaussian-filter` and the median filter (include/chunkflow_b200.h, DESIGN.md section 0, row f8) ----
FILTER_DTYPES = (DTYPE_U8, DTYPE_F32)
FILTER_MODES = {"reflect": 0, "grid-mirror": 0, "nearest": 1, "mirror": 2, "wrap": 3, "grid-wrap": 3, "constant": 4,
                "grid-constant": 4}
MAX_GAUSSIAN_RADIUS = 64
MAX_MEDIAN_WINDOW = 125


def _czyx(shape):
    shape = tuple(int(v) for v in shape)
    if len(shape) not in (3, 4) or min(shape) <= 0:
        raise ValueError(f"a chunk is (z, y, x) or (c, z, y, x) with positive sizes, not {shape}")
    return (1,) + shape if len(shape) == 3 else shape


def _filter_dtype(dtype: int) -> int:
    if dtype not in FILTER_DTYPES:
        raise TypeError("the filters take DTYPE_U8 or DTYPE_F32 chunks")
    return int(dtype)


def gaussian_filter_workspace(dtype: int, shape) -> int:
    """Bytes of device workspace cfb_gaussian_filter_device needs for a chunk of ``shape`` (no device needed)."""
    dtype, czyx, out = _filter_dtype(dtype), _czyx(shape), C.c_int64()
    check(load().cfb_gaussian_filter_workspace(dtype, *czyx, C.byref(out)))
    return int(out.value)


def gaussian_filter_device(d_data: int, dtype: int, shape, weights, d_workspace: int, workspace_bytes: int, stream: int = 0) -> None:
    """In place: every z section of the (z, y, x) or (c, z, y, x) chunk at ``d_data`` filtered along c (4-D only), y and x
    with ``weights`` = one float64 array w[0..r] per axis (w[0] the centre) or None where the axis has no pass."""
    dtype, czyx = _filter_dtype(dtype), _czyx(shape)
    weights = list(weights)
    if len(weights) != (3 if len(tuple(shape)) == 4 else 2):
        raise ValueError("one weight array (or None) per axis of a section")
    if len(weights) == 2:
        weights = [None] + weights
    args, keep = [], []
    for w in weights:
        if w is None:
            args += [None, 0]
            continue
        w = np.ascontiguousarray(w, dtype=np.float64)
        if w.ndim != 1 or not 1 <= w.size <= MAX_GAUSSIAN_RADIUS + 1:
            raise ValueError(f"gaussian filter: a radius of {w.size - 1} exceeds the limit of {MAX_GAUSSIAN_RADIUS}")
        keep.append(w)
        args += [w.ctypes.data_as(C.POINTER(C.c_double)), w.size - 1]
    check(load().cfb_gaussian_filter_device(C.c_void_p(d_data), dtype, *czyx, *args, C.c_void_p(d_workspace),
                                            int(workspace_bytes), C.c_void_p(stream)))


def median_filter_device(d_in: int, dtype: int, shape, size, mode: str, d_out: int, stream: int = 0) -> None:
    """``d_out`` = the median filter of the (z, y, x) or (c, z, y, x) chunk at ``d_in`` with the window ``size`` (one extent
    per axis of the chunk) and boundary ``mode`` (a scipy.ndimage mode name)."""
    ndim, dtype, czyx = len(tuple(shape)), _filter_dtype(dtype), _czyx(shape)
    size = tuple(int(v) for v in size)
    if len(size) != ndim:
        raise ValueError("one window extent per axis of the chunk")
    if mode not in FILTER_MODES:
        raise ValueError(f"unknown mode {mode}")
    s = (C.c_int64 * 4)(*((1,) + size if ndim == 3 else size))
    check(load().cfb_median_filter_device(C.c_void_p(d_in), dtype, *czyx, C.byref(s), FILTER_MODES[mode],
                                          C.c_void_p(d_out), C.c_void_p(stream)))


# ---- `clahe` (include/chunkflow_b200.h, DESIGN.md section 0, row f9) ----
def clahe_args(shape, tile_grid_size) -> tuple:
    """((z, y, x), tiles_x, tiles_y) of a clahe call; ValueError for another ndim or fewer than one tile along an axis."""
    shape = tuple(int(v) for v in shape)
    if len(shape) != 3 or min(shape) <= 0:
        raise ValueError(f"clahe takes a (z, y, x) image with positive sizes, not {shape}")
    tiles = tuple(int(v) for v in tile_grid_size)
    if len(tiles) != 2 or min(tiles) < 1:
        raise ValueError(f"the tile grid (x, y) has at least one tile along each axis, not {tile_grid_size}")
    return shape, tiles[0], tiles[1]


def clahe_workspace(shape, tile_grid_size) -> int:
    """Bytes of device workspace cfb_clahe_device needs for a (z, y, x) chunk and an (x, y) tile grid (no device needed)."""
    zyx, tx, ty = clahe_args(shape, tile_grid_size)
    out = C.c_int64()
    check(load().cfb_clahe_workspace(*zyx, tx, ty, C.byref(out)))
    return int(out.value)


def clahe_device(d_in: int, d_out: int, shape, clip_limit: float, tile_grid_size, d_workspace: int, workspace_bytes: int,
                 stream: int = 0) -> None:
    """``d_out`` = cv2.createCLAHE(clip_limit, tile_grid_size).apply of every z section of the uint8 (z, y, x) chunk at
    ``d_in``; tile_grid_size is (x, y), cv2's order."""
    zyx, tx, ty = clahe_args(shape, tile_grid_size)
    check(load().cfb_clahe_device(C.c_void_p(d_in), C.c_void_p(d_out), *zyx, float(clip_limit), tx, ty,
                                  C.c_void_p(d_workspace or None), int(workspace_bytes), C.c_void_p(stream)))


# ---- `mesh` (include/chunkflow_b200.h) ----
MESH_DTYPES = (DTYPE_U32, DTYPE_U64)


def bind_mesh(lib: C.CDLL) -> None:
    """Argument types of the mesh entry points (also for the host emulation of csrc/mesh.cu)."""
    vp, i32, i64, pi64 = C.c_void_p, C.c_int32, C.c_int64, C.POINTER(C.c_int64)
    lib.cfb_mesh_workspace.argtypes = [i64, i64, i64, i32, pi64]
    lib.cfb_mesh_count_device.argtypes = [vp, i32, i64, i64, i64, vp, i64, i32, vp, pi64, pi64, pi64, vp]
    lib.cfb_mesh_buffer_bytes.argtypes = [i64, i64, i64, pi64]
    lib.cfb_mesh_device.argtypes = [vp, i32, i64, i64, i64, vp, i64, i32, vp, vp, i64, i64, i64, vp, i64, pi64, vp]
    lib.cfb_mesh_read.argtypes = [vp, i64, i64, i64, i64, vp, vp, vp, vp, vp, vp]
    lib.cfb_mesh_simplify_host.argtypes = [i64, vp, i64, vp, i64, C.c_double, pi64, vp, pi64, vp]


def _mesh_dtype(dtype) -> int:
    if dtype not in MESH_DTYPES:
        raise TypeError("a segmentation to mesh is DTYPE_U32 or DTYPE_U64")
    return int(dtype)


def mesh_workspace(zyx, close: bool, lib=None) -> int:
    """Bytes of the count workspace of a (z, y, x) volume (no device needed)."""
    lib, out = lib or load(), C.c_int64()
    _mesh_check(lib, lib.cfb_mesh_workspace(*(int(v) for v in zyx), int(bool(close)), C.byref(out)))
    return int(out.value)


def mesh_count_device(d_labels: int, dtype: int, zyx, d_skip: int, num_skip: int, close: bool, d_workspace: int, stream: int = 0,
                      lib=None):
    """-> ((cube, object) pairs, triangles, vertices) of the segmentation at ``d_labels`` (synchronises the stream)."""
    pairs, tris, verts = C.c_int64(), C.c_int64(), C.c_int64()
    lib = lib or load()
    _mesh_check(lib, lib.cfb_mesh_count_device(C.c_void_p(d_labels), _mesh_dtype(dtype), *(int(v) for v in zyx), C.c_void_p(d_skip or None),
                                               int(num_skip), int(bool(close)), C.c_void_p(d_workspace), C.byref(pairs), C.byref(tris),
                                               C.byref(verts), C.c_void_p(stream)))
    return int(pairs.value), int(tris.value), int(verts.value)


def mesh_buffer_bytes(counts, lib=None) -> int:
    """Bytes of the device buffer of the weld for the counts of mesh_count_device (no device needed)."""
    lib, out = lib or load(), C.c_int64()
    pairs, tris, verts = (int(v) for v in counts)
    _mesh_check(lib, lib.cfb_mesh_buffer_bytes(pairs, tris, verts, C.byref(out)))
    return int(out.value)


def mesh_device(d_labels: int, dtype: int, zyx, d_skip: int, num_skip: int, close: bool, voxel_size, d_workspace: int, counts,
                d_buffer: int, buffer_bytes: int, stream: int = 0, lib=None) -> int:
    """Every mesh welded on the device into ``d_buffer`` -> the number of objects (synchronises the stream)."""
    vs = np.ascontiguousarray(voxel_size, np.float64)
    if vs.shape != (3,):
        raise ValueError("the voxel size is (z, y, x)")
    pairs, tris, verts = (int(v) for v in counts)
    n, lib = C.c_int64(), lib or load()
    _mesh_check(lib, lib.cfb_mesh_device(C.c_void_p(d_labels), _mesh_dtype(dtype), *(int(v) for v in zyx), C.c_void_p(d_skip or None),
                                         int(num_skip), int(bool(close)), _ptr(vs), C.c_void_p(d_workspace), pairs, tris, verts,
                                         C.c_void_p(d_buffer), int(buffer_bytes), C.byref(n), C.c_void_p(stream)))
    return int(n.value)


def mesh_read(d_buffer: int, counts, num_objects: int, stream: int = 0, lib=None) -> dict:
    """The meshes of mesh_device -> {id: (vertices float32 (N, 3) xyz, faces uint32 (M, 3))}, ids ascending."""
    pairs, tris, verts = (int(v) for v in counts)
    n = int(num_objects)
    obj, fo, vo = np.empty(n, np.uint64), np.empty(n + 1, np.int64), np.empty(n + 1, np.int64)
    faces, vertices = np.empty((tris, 3), np.uint32), np.empty((verts, 3), np.float32)
    lib = lib or load()
    _mesh_check(lib, lib.cfb_mesh_read(C.c_void_p(d_buffer), pairs, tris, verts, n, _ptr(obj), _ptr(fo), _ptr(vo), _ptr(faces),
                                       _ptr(vertices), C.c_void_p(stream)))
    return {int(obj[o]): (vertices[vo[o]:vo[o + 1]], faces[fo[o]:fo[o + 1]]) for o in range(n)}


def mesh_simplify_host(vertices, faces, simplification_factor: int, max_simplification_error: float, lib=None):
    """One mesh simplified on the host (no GPU involved) -> (vertices float32 (N, 3), faces uint32 (M, 3))."""
    v, f = np.ascontiguousarray(vertices, np.float32), np.ascontiguousarray(faces, np.uint32)
    if v.ndim != 2 or v.shape[1] != 3 or f.ndim != 2 or f.shape[1] != 3:
        raise ValueError("vertices (N, 3) and faces (M, 3)")
    if isinstance(simplification_factor, bool) or not isinstance(simplification_factor, (int, np.integer)):
        raise TypeError("the simplification factor is an integer")
    ov, of = np.empty_like(v), np.empty_like(f)
    nv, nf = C.c_int64(), C.c_int64()
    lib = lib or load()
    _mesh_check(lib, lib.cfb_mesh_simplify_host(v.shape[0], _ptr(v), f.shape[0], _ptr(f), int(simplification_factor),
                                                float(max_simplification_error), C.byref(nv), _ptr(ov), C.byref(nf), _ptr(of)))
    return ov[:nv.value].copy(), of[:nf.value].copy()


def _mesh_check(lib, code: int) -> None:
    if code != OK:
        raise NativeError(code, lib.cfb_last_error().decode("utf-8", "replace"))


# ---- `skeletonize` (include/chunkflow_b200.h) ----
SKELETON_STATS = ("sweeps", "rounds", "paths", "skeleton_voxels", "relax_ms", "sort_ms", "rounds_ms", "trace_ms")


def bind_skeleton(lib: C.CDLL) -> None:
    """Argument types of the skeleton entry points (also for the host emulation of csrc/skeleton.cu)."""
    vp, i32, i64, pi64 = C.c_void_p, C.c_int32, C.c_int64, C.POINTER(C.c_int64)
    lib.cfb_skeleton_workspace.argtypes = [i64, i64, i64, pi64]
    lib.cfb_edt_workspace.argtypes = [i64, i64, i64, pi64]
    lib.cfb_edt_device.argtypes = [vp, i32, i64, i64, i64, vp, vp, vp, vp]
    lib.cfb_skeleton_count_device.argtypes = [vp, i32, i64, i64, i64, vp, vp, i64, i64, vp, pi64, pi64, pi64, vp]
    lib.cfb_skeleton_device.argtypes = [vp, i32, i64, i64, i64, vp, vp, i32, vp, i64, i64, vp, i64, pi64, vp, vp]
    lib.cfb_skeleton_read.argtypes = [vp, i64, i64, i64, vp, i64, i64, i64, pi64, vp, vp, vp, vp, vp, vp, vp]


def _voxel_size(voxel_size) -> np.ndarray:
    vs = np.ascontiguousarray(voxel_size, np.float64)
    if vs.shape != (3,):
        raise ValueError("the voxel size is (z, y, x)")
    return vs


def skeleton_workspace(zyx, lib=None) -> int:
    """Bytes of the per-voxel workspace of a (z, y, x) volume (no device needed)."""
    lib, out = lib or load(), C.c_int64()
    _mesh_check(lib, lib.cfb_skeleton_workspace(*(int(v) for v in zyx), C.byref(out)))
    return int(out.value)


def edt_workspace(zyx, lib=None) -> int:
    """Bytes of the workspace of the distance transform alone (no device needed)."""
    lib, out = lib or load(), C.c_int64()
    _mesh_check(lib, lib.cfb_edt_workspace(*(int(v) for v in zyx), C.byref(out)))
    return int(out.value)


def edt_device(d_labels: int, dtype: int, zyx, voxel_size, d_out: int, d_workspace: int, stream: int = 0, lib=None) -> None:
    """``d_out`` (float32) = the multi-label distance to the boundary of the segmentation at ``d_labels``."""
    vs, lib = _voxel_size(voxel_size), lib or load()
    _mesh_check(lib, lib.cfb_edt_device(C.c_void_p(d_labels), int(dtype), *(int(v) for v in zyx), _ptr(vs), C.c_void_p(d_out),
                                        C.c_void_p(d_workspace), C.c_void_p(stream)))


def skeleton_count_device(d_labels: int, dtype: int, zyx, voxel_size, d_skip: int, num_skip: int, dust_threshold: int, d_workspace: int,
                          stream: int = 0, lib=None):
    """-> (objects, their voxels, buffer bytes) of the segmentation at ``d_labels`` (synchronises the stream)."""
    vs, lib = _voxel_size(voxel_size), lib or load()
    k, m, nb = C.c_int64(), C.c_int64(), C.c_int64()
    _mesh_check(lib, lib.cfb_skeleton_count_device(C.c_void_p(d_labels), int(dtype), *(int(v) for v in zyx), _ptr(vs),
                                                   C.c_void_p(d_skip or None), int(num_skip), int(dust_threshold), C.c_void_p(d_workspace),
                                                   C.byref(k), C.byref(m), C.byref(nb), C.c_void_p(stream)))
    return int(k.value), int(m.value), int(nb.value)


def skeleton_device(d_labels: int, dtype: int, zyx, voxel_size, scale: float, const: float, pdrf_scale: float, pdrf_exponent: int,
                    d_workspace: int, counts, d_buffer: int, stream: int = 0, lib=None):
    """Every skeleton on the device into ``d_buffer`` -> (skeleton voxels, {stat: value}) (synchronises the stream)."""
    vs, lib = _voxel_size(voxel_size), lib or load()
    prm = np.array([scale, const, pdrf_scale], np.float64)
    st = np.zeros(len(SKELETON_STATS), np.float64)
    K, m, nb = (int(v) for v in counts)
    S = C.c_int64()
    _mesh_check(lib, lib.cfb_skeleton_device(C.c_void_p(d_labels), int(dtype), *(int(v) for v in zyx), _ptr(vs), _ptr(prm), int(pdrf_exponent),
                                             C.c_void_p(d_workspace), K, m, C.c_void_p(d_buffer or None), nb, C.byref(S), _ptr(st),
                                             C.c_void_p(stream)))
    return int(S.value), dict(zip(SKELETON_STATS, st.tolist()))


def skeleton_read(d_buffer: int, zyx, voxel_size, counts, num_skeleton_voxels: int, stream: int = 0, lib=None) -> dict:
    """The skeletons of skeleton_device -> {id: (vertices float32 (N, 3) x y z, edges uint32 (M, 2), radii float32 (N,))}."""
    vs, lib = _voxel_size(voxel_size), lib or load()
    K, m, _ = (int(v) for v in counts)
    S = int(num_skeleton_voxels)
    ids, vo, eo = np.empty(max(K, 1), np.uint64), np.empty(K + 1, np.int64), np.empty(K + 1, np.int64)
    verts, edges, radii = np.empty((S, 3), np.float32), np.empty((max(S - K, 0), 2), np.uint32), np.empty(S, np.float32)
    nl = C.c_int64()
    _mesh_check(lib, lib.cfb_skeleton_read(C.c_void_p(d_buffer or None), *(int(v) for v in zyx), _ptr(vs), K, m, S, C.byref(nl), _ptr(ids),
                                           _ptr(vo), _ptr(eo), _ptr(verts), _ptr(edges), _ptr(radii), C.c_void_p(stream)))
    return {int(ids[i]): (verts[vo[i]:vo[i + 1]], edges[eo[i]:eo[i + 1]], radii[vo[i]:vo[i + 1]]) for i in range(int(nl.value))}


# ---- `fill-segmentation-holes` (include/chunkflow_b200.h) ----
FILL_MODES = ("binary", "keep-enclosed", "remove-enclosed")   # CFB_FILL_BINARY, CFB_FILL_KEEP_ENCLOSED, CFB_FILL_REMOVE_ENCLOSED


def bind_fill_holes(lib: C.CDLL) -> None:
    """Argument types of the fill-holes entry points (also for the host emulation of csrc/fill_holes.cu)."""
    vp, i32, i64, pi64 = C.c_void_p, C.c_int32, C.c_int64, C.POINTER(C.c_int64)
    lib.cfb_fill_holes_workspace.argtypes = [i64, i64, i64, pi64]
    lib.cfb_fill_holes_table_workspace.argtypes = [i64, pi64]
    lib.cfb_fill_holes_components_device.argtypes = [vp, i32, i64, i64, i64, i32, vp, pi64, vp]
    lib.cfb_fill_holes_graph_device.argtypes = [vp, i64, i64, i64, vp, i64, pi64, vp]
    lib.cfb_fill_holes_enclose.argtypes = [vp, i64, i64, i64, vp, i64, i64, vp]
    lib.cfb_fill_holes_apply_device.argtypes = [vp, i32, i64, i64, i64, vp, vp, pi64, vp]


def fill_mode(mode: str) -> int:
    if mode not in FILL_MODES:
        raise ValueError(f"fill holes: the mode is one of {FILL_MODES}, not {mode!r}")
    return FILL_MODES.index(mode)


def fill_holes_workspace(zyx, lib=None) -> int:
    """Bytes of the per-voxel workspace of a (z, y, x) volume (no device needed)."""
    lib, out = lib or load(), C.c_int64()
    _mesh_check(lib, lib.cfb_fill_holes_workspace(*(int(v) for v in zyx), C.byref(out)))
    return int(out.value)


def fill_holes_table_workspace(table_slots: int, lib=None) -> int:
    """Bytes of the pair table of ``table_slots`` slots (no device needed)."""
    lib, out = lib or load(), C.c_int64()
    _mesh_check(lib, lib.cfb_fill_holes_table_workspace(int(table_slots), C.byref(out)))
    return int(out.value)


def fill_holes_components_device(d_in: int, dtype: int, zyx, mode: str, d_workspace: int, stream: int = 0, lib=None) -> int:
    """-> the number of components (of the background in binary mode, of every value otherwise); synchronises the stream."""
    lib, n = lib or load(), C.c_int64()
    _mesh_check(lib, lib.cfb_fill_holes_components_device(C.c_void_p(d_in), int(dtype), *(int(v) for v in zyx), fill_mode(mode),
                                                          C.c_void_p(d_workspace), C.byref(n), C.c_void_p(stream)))
    return int(n.value)


def fill_holes_graph_device(d_workspace: int, zyx, d_table: int, table_slots: int, stream: int = 0, lib=None) -> int:
    """-> the number of touching component pairs; raises NativeError with code ERR_CAPACITY when the table is too small."""
    lib, n = lib or load(), C.c_int64()
    _mesh_check(lib, lib.cfb_fill_holes_graph_device(C.c_void_p(d_workspace), *(int(v) for v in zyx), C.c_void_p(d_table), int(table_slots),
                                                     C.byref(n), C.c_void_p(stream)))
    return int(n.value)


def fill_holes_enclose(d_workspace: int, zyx, d_table: int, table_slots: int, num_edges: int, stream: int = 0, lib=None) -> None:
    """The encloser of every component, on the host (no GPU work but the copies)."""
    lib = lib or load()
    _mesh_check(lib, lib.cfb_fill_holes_enclose(C.c_void_p(d_workspace), *(int(v) for v in zyx), C.c_void_p(d_table), int(table_slots),
                                                int(num_edges), C.c_void_p(stream)))


def fill_holes_apply_device(d_in: int, dtype: int, zyx, d_workspace: int, d_out: int, stream: int = 0, lib=None) -> int:
    """``d_out`` = the filled chunk -> the number of voxels the rule assigned; synchronises the stream."""
    lib, n = lib or load(), C.c_int64()
    _mesh_check(lib, lib.cfb_fill_holes_apply_device(C.c_void_p(d_in), int(dtype), *(int(v) for v in zyx), C.c_void_p(d_workspace),
                                                     C.c_void_p(d_out), C.byref(n), C.c_void_p(stream)))
    return int(n.value)


def device_memory(device: int = 0) -> tuple:
    """(free, total) bytes of device memory."""
    f, t = C.c_int64(), C.c_int64()
    check(load().cfb_device_memory(int(device), C.byref(f), C.byref(t)))
    return f.value, t.value


def make_patch_mask(patch_size, overlap) -> np.ndarray:
    """fp32 bump/patch mask built by the native library (no GPU needed)."""
    ps = (C.c_int32 * 3)(*[int(v) for v in patch_size])
    ov = (C.c_int32 * 3)(*[int(v) for v in overlap])
    out = np.empty(tuple(int(v) for v in patch_size), np.float32)
    check(load().cfb_make_patch_mask(C.byref(ps), C.byref(ov), _ptr(out)))
    return out


def augment_code(augment) -> int:
    """``augment`` as the Inferencer takes it: falsy -> none; True / 'reference' -> the reference's literal arithmetic
    (transform.py:30-52,147-156); 'spatial' -> the 8 spatial flip / transpose variants (explicit opt-in)."""
    if not augment:
        return AUGMENT_NONE
    if augment is True or augment == "reference" or augment == AUGMENT_REFERENCE:
        return AUGMENT_REFERENCE
    if augment == "spatial" or augment == AUGMENT_SPATIAL:
        return AUGMENT_SPATIAL
    raise ValueError(f"augment must be False, True, 'reference' or 'spatial', not {augment!r}")


def halo_add_device(d_dst: int, d_src: int, count: int, stream: int = 0) -> None:
    """d_dst[i] += d_src[i] for `count` float32 on the current device (multi-GPU halo planes)."""
    check(load().cfb_halo_add_device(C.c_void_p(d_dst), C.c_void_p(d_src), int(count), C.c_void_p(stream)))


class Engine:
    """RAII wrapper of a ``cfb_handle``."""

    def __init__(self, *, input_patch_size, output_patch_size, output_patch_overlap, output_crop_margin,
                 num_input_channels=1, num_output_channels=3, batch_size=1, mask_output_chunk=True,
                 framework=FRAMEWORK_UNET3L, precision=PRECISION_F32_SIMT, device=0, augment=False,
                 mask_myelin_threshold=None, check_output_range=True):
        self._h = C.c_void_p()
        self._lib = load()
        p = Params()
        p.struct_size = C.sizeof(Params)
        p.device, p.framework, p.precision = int(device), int(framework), int(precision)
        p.input_patch_size[:] = [int(v) for v in input_patch_size]
        p.output_patch_size[:] = [int(v) for v in output_patch_size]
        p.output_patch_overlap[:] = [int(v) for v in output_patch_overlap]
        p.output_crop_margin[:] = [int(v) for v in output_crop_margin]
        p.num_input_channels, p.num_output_channels = int(num_input_channels), int(num_output_channels)
        p.batch_size, p.mask_output_chunk = int(batch_size), int(bool(mask_output_chunk))
        p.augment = augment_code(augment)
        # truthiness, like the reference (inferencer.py:468: `if self.mask_myelin_threshold:`): None and 0.0 both mean "off"
        p.has_myelin_threshold = int(bool(mask_myelin_threshold))
        p.mask_myelin_threshold = float(mask_myelin_threshold or 0.0)
        p.check_output_range = int(bool(check_output_range))
        self.params = p
        self.input_patch_size = tuple(p.input_patch_size)
        self.output_patch_size = tuple(p.output_patch_size)
        self.num_output_channels = p.num_output_channels
        check(self._lib.cfb_create(C.byref(p), C.byref(self._h)))

    def close(self):
        h = getattr(self, "_h", None)
        if h is not None and h.value:
            try:
                self._lib.cfb_destroy(h)
            finally:
                self._h = None  # (the ctypes module may already be torn down at interpreter exit)

    __del__ = close

    @property
    def device_name(self) -> str:
        return self._lib.cfb_device_name(self._h).decode()

    def load_state_dict(self, state: dict) -> None:
        for name, tensor in state.items():
            a = np.ascontiguousarray(np.asarray(tensor, dtype=np.float32))
            check(self._lib.cfb_set_weight(self._h, name.encode(), _ptr(a), a.size))
        check(self._lib.cfb_commit_weights(self._h))

    def patch_mask(self) -> np.ndarray:
        out = np.empty(self.output_patch_size, np.float32)
        check(self._lib.cfb_patch_mask(self._h, _ptr(out)))
        return out

    def patch_grid(self, chunk_zyx) -> np.ndarray:
        n = C.c_int64()
        cz, cy, cx = (int(v) for v in chunk_zyx)
        check(self._lib.cfb_patch_grid(self._h, cz, cy, cx, C.byref(n), None, 0))
        starts = np.empty((n.value, 3), np.int32)
        check(self._lib.cfb_patch_grid(self._h, cz, cy, cx, C.byref(n), _ptr(starts), n.value))
        return starts

    def output_shape(self, chunk_zyx) -> tuple:
        out = (C.c_int64 * 4)()
        check(self._lib.cfb_output_shape(self._h, *(int(v) for v in chunk_zyx), C.byref(out)))
        return tuple(out)

    @staticmethod
    def _dtype_code(dtype) -> int:
        if np.dtype(dtype) == np.uint8:
            return DTYPE_U8
        if np.dtype(dtype) == np.float32:
            return DTYPE_F32
        raise TypeError(f"input chunk dtype {dtype} is not supported on the device (uint8 or float32)")

    def infer_chunk_host(self, chunk: np.ndarray, out: Optional[np.ndarray] = None) -> np.ndarray:
        chunk = np.ascontiguousarray(chunk)
        if chunk.ndim != 3:
            raise ValueError("expected a (z, y, x) chunk")
        shape = self.output_shape(chunk.shape)
        if out is None:
            out = np.empty(shape, np.float32)
        assert out.shape == shape and out.dtype == np.float32 and out.flags.c_contiguous
        check(self._lib.cfb_infer_chunk_host(self._h, _ptr(chunk), self._dtype_code(chunk.dtype), *chunk.shape, _ptr(out)))
        return out

    def infer_chunk_device(self, d_in: int, dtype, chunk_zyx, d_out: int, stream: int = 0) -> None:
        check(self._lib.cfb_infer_chunk_device(self._h, C.c_void_p(d_in), self._dtype_code(dtype),
                                               *(int(v) for v in chunk_zyx), C.c_void_p(d_out), C.c_void_p(stream)))

    def infer_slab_device(self, d_in: int, dtype, chunk_zyx, zrow_begin: int, zrow_end: int, d_out: int, d_weight: int,
                          stream: int = 0) -> None:
        check(self._lib.cfb_infer_slab_device(self._h, C.c_void_p(d_in), self._dtype_code(dtype),
                                              *(int(v) for v in chunk_zyx), int(zrow_begin), int(zrow_end),
                                              C.c_void_p(d_out), C.c_void_p(d_weight), C.c_void_p(stream)))

    def normalize_device(self, d_out: int, d_weight: int, czyx, stream: int = 0, weight_is_inverse: bool = False,
                         all_zero_input: bool = False) -> None:
        check(self._lib.cfb_normalize_device(self._h, C.c_void_p(d_out), C.c_void_p(d_weight), int(bool(weight_is_inverse)),
                                             *(int(v) for v in czyx), int(bool(all_zero_input)), C.c_void_p(stream)))

    def slab_nonzero(self, stream: int = 0) -> bool:
        flag = C.c_int32()
        check(self._lib.cfb_slab_nonzero(self._h, C.byref(flag), C.c_void_p(stream)))
        return bool(flag.value)

    def weight_volume_device(self, chunk_zyx, z_begin: int, z_end: int, d_weight: int, invert: bool = False, stream: int = 0) -> None:
        check(self._lib.cfb_weight_volume_device(self._h, *(int(v) for v in chunk_zyx), int(z_begin), int(z_end), int(bool(invert)),
                                                 C.c_void_p(d_weight), C.c_void_p(stream)))

    def patch_forward_host(self, patches: np.ndarray) -> np.ndarray:
        patches = np.ascontiguousarray(patches, dtype=np.float32)
        if patches.ndim != 5 or patches.shape[1:] != (1,) + self.input_patch_size:
            raise ValueError(f"expected input patches of shape (batch, 1, {self.input_patch_size}), got {patches.shape}")
        b = patches.shape[0]
        out = np.empty((b, self.num_output_channels) + self.output_patch_size, np.float32)
        check(self._lib.cfb_patch_forward_host(self._h, _ptr(patches), b, _ptr(out)))
        return out

    # plugin level (user-supplied patch backends)
    def plugin_begin(self, chunk: np.ndarray) -> None:
        chunk = np.ascontiguousarray(chunk)
        check(self._lib.cfb_plugin_begin(self._h, _ptr(chunk), self._dtype_code(chunk.dtype), *chunk.shape))

    def plugin_extract(self, first: int, nb: int, out: np.ndarray) -> None:
        assert out.dtype == np.float32 and out.flags.c_contiguous
        if out.shape != (nb, 1) + self.input_patch_size:
            raise ValueError(f"patch buffer must have shape {(nb, 1) + self.input_patch_size}, got {out.shape}")
        check(self._lib.cfb_plugin_extract(self._h, int(first), int(nb), _ptr(out)))

    def plugin_blend(self, first: int, nb: int, masked: np.ndarray) -> None:
        """`masked`: what the user's patch backend returned for patches [first, first+nb) -- already cropped to the output
        patch and bump-masked.  The native side reads nb*C*prod(output_patch_size) floats, so the shape is checked here
        (the reference fails with a numpy broadcasting error on a wrong shape)."""
        masked = np.asarray(masked)
        want = (nb, self.num_output_channels) + self.output_patch_size
        if masked.shape != want:
            raise ValueError(f"the patch backend must return an array of shape {want} (batch, channels, cropped output patch); "
                             f"got {masked.shape}")
        masked = np.ascontiguousarray(masked, dtype=np.float32)
        check(self._lib.cfb_plugin_blend(self._h, int(first), int(nb), _ptr(masked)))

    def plugin_end(self, out: np.ndarray) -> None:
        check(self._lib.cfb_plugin_end(self._h, _ptr(out)))

    def last_timing(self) -> dict:
        ms = (C.c_float * 5)()
        n = C.c_int64()
        check(self._lib.cfb_last_timing(self._h, C.byref(ms), C.byref(n)))
        return dict(total_ms=ms[0], convnet_ms=ms[1], blend_normalize_ms=ms[2], h2d_ms=ms[3], d2h_ms=ms[4],
                    launches=n.value)

    def set_profiling(self, enabled: bool) -> None:
        check(self._lib.cfb_set_profiling(self._h, int(bool(enabled))))

    def layer_timing(self) -> dict:
        """kernel class -> (total ms, launches) since profiling was enabled."""
        cap = 64
        names = (C.c_char * 32 * cap)()
        ms = (C.c_float * cap)()
        launches = (C.c_int64 * cap)()
        n = C.c_int32()
        check(self._lib.cfb_layer_timing(self._h, cap, C.byref(n), C.cast(names, C.c_void_p), C.cast(ms, C.c_void_p),
                                         C.cast(launches, C.c_void_p)))
        return {names[i].value.decode(): (float(ms[i]), int(launches[i])) for i in range(n.value)}

    def debug_net_forward(self, patch: np.ndarray, cnet: int) -> np.ndarray:
        patch = np.ascontiguousarray(patch, dtype=np.float32)
        out = np.empty((cnet,) + self.input_patch_size, np.float32)
        check(self._lib.cfb_debug_net_forward_host(self._h, _ptr(patch), _ptr(out)))
        return out

    def debug_conv3(self, x: np.ndarray, w: np.ndarray, b: np.ndarray, relu: bool) -> np.ndarray:
        """One 3x3x3 convolution of one patch, x (cin, z, y, x) -> (cout, z, y, x), through debug_layer; for cin >= 32 the
        input is fed as two sources of cin / 2 channels (the decoders' concat)."""
        x = np.asarray(x, np.float32)[None]
        cb = x.shape[1] // 2 if x.shape[1] >= 32 else 0
        ca = x.shape[1] - cb
        return self.debug_layer("conv3", x[:, :ca], x[:, ca:] if cb else None, w, b, relu=relu)[0]

    def debug_layer(self, op: str, a: np.ndarray, b: Optional[np.ndarray] = None, weight=None, bias=None, relu: bool = True,
                    head_weight=None, head_bias=None, chunk: Optional[np.ndarray] = None, in_origins=None, out_origins=None,
                    out_patch=None, crop=(0, 0, 0), mask=None, out: Optional[np.ndarray] = None, scale: float = 1.0, size=None):
        """One step of the layer table through the kernels of this engine's precision mode (cfb_debug_layer_host).

        `op` is one of LAYER_OPS.  `a` (nb, ca, z, y, x) and `b` (nb, cb, z, y, x) are the two sources of a concat (`a` is
        (nb, 1, z, y, x) for 'first', or None with `chunk`, `in_origins` (nb, 3) and the patch `size`).  Returns the output array, or (output, pooled)
        for 'conv3_pool'; the blending ops accumulate into `out` (channels, *out_size) and return it."""
        code = LAYER_OPS.index(op)
        keep = []

        def arr(v, dtype=np.float32):
            if v is None:
                return None
            v = np.ascontiguousarray(v, dtype)
            keep.append(v)
            return v

        def ptr(v):
            return None if v is None else v.ctypes.data

        chunk = None if chunk is None else np.ascontiguousarray(chunk)
        a, b, weight, bias = arr(a), arr(b), arr(weight), arr(bias)
        head_weight, head_bias, mask = arr(head_weight), arr(head_bias), arr(mask)
        in_origins, out_origins = arr(in_origins, np.int32), arr(out_origins, np.int32)
        if a is not None:
            nb, ca, z, y, x = a.shape
        else:
            nb, ca, (z, y, x) = len(in_origins), 1, (int(v) for v in size)
        cb = 0 if b is None else b.shape[1]
        cout = {"conv3": None, "conv3_pool": None, "convT": None, "maxpool": ca, "first": 16, "head_sigmoid": None,
                "head_blend": None, "conv3_head_blend": 16, "round_trip": ca}[op]
        if cout is None:
            cout = weight.shape[1] if op == "convT" else weight.shape[0] if weight is not None else 0
        hc = 0 if head_weight is None else head_weight.shape[0]
        p = LayerArgs()
        p.struct_size = C.sizeof(LayerArgs)
        p.op, p.nb, p.ca, p.cb, p.cout, p.relu = code, nb, ca, cb, cout, int(bool(relu))
        p.size[:] = [z, y, x]
        p.a, p.b, p.weight, p.bias = ptr(a), ptr(b), ptr(weight), ptr(bias)
        p.head_weight, p.head_bias, p.head_channels = ptr(head_weight), ptr(head_bias), hc
        if chunk is not None:
            p.chunk, p.chunk_dtype = chunk.ctypes.data, self._dtype_code(chunk.dtype)
            p.chunk_size[:] = list(chunk.shape)
        p.in_origins, p.out_origins, p.mask, p.scale = ptr(in_origins), ptr(out_origins), ptr(mask), float(scale)
        p.crop[:] = [int(v) for v in crop]
        pooled = None
        if op in ("head_blend", "conv3_head_blend"):
            p.out_patch[:] = [int(v) for v in out_patch]
            assert out.dtype == np.float32 and out.flags.c_contiguous and out.shape[0] == hc
            p.out_size[:] = list(out.shape[1:])
        else:
            oc = hc if op == "head_sigmoid" else cout
            shape = (z, 2 * y, 2 * x) if op == "convT" else (z, y // 2, x // 2) if op == "maxpool" else (z, y, x)
            out = np.empty((nb, oc) + shape, np.float32)
            if op == "conv3_pool":
                pooled = np.empty((nb, cout, z, y // 2, x // 2), np.float32)
                p.pooled = pooled.ctypes.data
        p.out = out.ctypes.data
        check(self._lib.cfb_debug_layer_host(self._h, C.byref(p)))
        return (out, pooled) if pooled is not None else out
