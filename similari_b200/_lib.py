"""ctypes binding of libsimilari_b200.so (the C ABI declared in include/similari_b200.h).

The library is the product: hand-written sm_90a CUDA kernels behind an extern "C" boundary.  There is no CPU
fallback -- if the shared library is missing this module raises, and every compute call raises without a GPU.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libsimilari_b200.so")

MAX_CONSTRAINTS = 8
NONE_ID = -(2**63)
KIND_SORT, KIND_BATCH_SORT, KIND_VISUAL_SORT, KIND_BATCH_VISUAL_SORT = 0, 1, 2, 3
POS_MAHA, POS_IOU = 0, 1
VIS_EUCLIDEAN, VIS_COSINE = 0, 1
VOTING_VISUAL, VOTING_POSITIONAL = 0, 1
FEATURE_F32, FEATURE_F16, FEATURE_BF16 = 0, 1, 2


class Sb200Error(RuntimeError):
    pass


class Options(C.Structure):
    """sb200_options (include/similari_b200.h)."""

    _fields_ = [
        ("kind", C.c_int32),
        ("positional_kind", C.c_int32),
        ("iou_threshold", C.c_float),
        ("min_confidence", C.c_float),
        ("max_idle_epochs", C.c_int32),
        ("history_length", C.c_int32),
        ("kalman_position_weight", C.c_float),
        ("kalman_velocity_weight", C.c_float),
        ("n_constraints", C.c_int32),
        ("constraint_epochs", C.c_int32 * MAX_CONSTRAINTS),
        ("constraint_max_dist", C.c_float * MAX_CONSTRAINTS),
        ("visual_kind", C.c_int32),
        ("visual_threshold", C.c_float),
        ("feature_dim", C.c_int32),
        ("visual_max_observations", C.c_int32),
        ("visual_min_votes", C.c_int32),
        ("visual_minimal_track_length", C.c_int32),
        ("visual_minimal_area", C.c_float),
        ("visual_minimal_quality_use", C.c_float),
        ("visual_minimal_quality_collect", C.c_float),
        ("visual_minimal_own_area_percentage_use", C.c_float),
        ("visual_minimal_own_area_percentage_collect", C.c_float),
        ("max_scenes_hint", C.c_int32),
        ("max_tracks_per_scene_hint", C.c_int32),
        ("max_dets_per_scene_hint", C.c_int32),
        ("device", C.c_int32),
    ]


class PredictOut(C.Structure):
    """sb200_predict_out."""

    _fields_ = [
        ("ids", C.c_void_p),
        ("epochs", C.c_void_p),
        ("lengths", C.c_void_p),
        ("voting_types", C.c_void_p),
        ("predicted_boxes", C.c_void_p),
        ("observed_boxes", C.c_void_p),
    ]


class FstoreOptions(C.Structure):
    """sb200_fstore_options."""

    _fields_ = [
        ("metric", C.c_int32),
        ("distance_filter", C.c_float),
        ("max_observations", C.c_int32),
        ("feature_dim", C.c_int32),
        ("topn", C.c_int32),
        ("max_distance", C.c_float),
        ("min_votes", C.c_int32),
        ("device", C.c_int32),
    ]


FSTORE_BLOB_MAGIC, FSTORE_BLOB_VERSION, FSTORE_BLOB_ALIGN, FSTORE_BLOB_SECTIONS = 0x53464253, 1, 256, 4


class FstoreBlobHeader(C.Structure):
    """sb200_fstore_blob_header: the first bytes of a blob of sb200_fstore_save."""

    _fields_ = [
        ("magic", C.c_uint32),
        ("version", C.c_uint32),
        ("total_bytes", C.c_uint64),
        ("metric", C.c_int32),
        ("distance_filter", C.c_float),
        ("max_observations", C.c_int32),
        ("feature_dim", C.c_int32),
        ("topn", C.c_int32),
        ("max_distance", C.c_float),
        ("min_votes", C.c_int32),
        ("d8", C.c_int32),
        ("feature_type", C.c_int32),
        ("storage_type", C.c_int32),
        ("live", C.c_int64),
        ("sec_off", C.c_uint64 * FSTORE_BLOB_SECTIONS),
        ("sec_bytes", C.c_uint64 * FSTORE_BLOB_SECTIONS),
    ]


FSTORE_BLOB_VERSION_GATED, FSTORE_BLOB_SECTIONS_V2 = 2, 7
# track attribute rules of the feature store (sb200_fstore_set_gate)
FSTORE_GATE_NONE, FSTORE_GATE_SAME_SOURCE, FSTORE_GATE_ANY_SOURCE = 0, 1, 2


class FstoreBlobHeaderV2(C.Structure):
    """sb200_fstore_blob_header_v2: the first bytes of the blob of a gated store."""

    _fields_ = FstoreBlobHeader._fields_[:-2] + [
        ("gate", C.c_int32),
        ("reserved", C.c_int32),
        ("sec_off", C.c_uint64 * FSTORE_BLOB_SECTIONS_V2),
        ("sec_bytes", C.c_uint64 * FSTORE_BLOB_SECTIONS_V2),
    ]


FSTORE_BLOB_VERSION_QUALITY, FSTORE_BLOB_SECTIONS_V3 = 3, 10
# retention rules of the feature store (sb200_fstore_set_retention)
FSTORE_KEEP_NEWEST, FSTORE_KEEP_BEST_QUALITY = 0, 1
# voting rules of the feature store (sb200_fstore_set_voting)
FSTORE_VOTING_TOPN, FSTORE_VOTING_BEST_FIT = 0, 1


class FstoreBlobHeaderV3(C.Structure):
    """sb200_fstore_blob_header_v3: the first bytes of the blob of a quality store."""

    _fields_ = FstoreBlobHeader._fields_[:-2] + [
        ("gate", C.c_int32),
        ("retention", C.c_int32),
        ("initial_capacity", C.c_int32),
        ("merge_extension", C.c_float),
        ("sec_off", C.c_uint64 * FSTORE_BLOB_SECTIONS_V3),
        ("sec_bytes", C.c_uint64 * FSTORE_BLOB_SECTIONS_V3),
    ]


class FstoreAttrs(C.Structure):
    """sb200_fstore_attrs: host columns of one source and one [t_start, t_end] window per row."""

    _fields_ = [("source", C.c_void_p), ("t_start", C.c_void_p), ("t_end", C.c_void_p)]


_lib = None

# every symbol include/similari_b200.h declares (checked by tests/test_abi.py without a GPU)
EXPORTS = [
    "sb200_options_default", "sb200_last_error", "sb200_device_count", "sb200_tracker_create", "sb200_tracker_destroy",
    "sb200_tracker_set_stream", "sb200_predict_batch", "sb200_prefetch_inputs", "sb200_predict_batch_device", "sb200_skip_epochs",
    "sb200_current_epoch", "sb200_active_tracks", "sb200_scene_track_counts", "sb200_scene_live_counts", "sb200_set_auto_waste", "sb200_clear_wasted", "sb200_wasted",
    "sb200_idle_tracks", "sb200_scene_tracks", "sb200_last_costs", "sb200_last_stage_ms", "sb200_last_kernel_ms", "sb200_sort_cost_matrix",
    "sb200_visual_cost_matrix", "sb200_sort_voting", "sb200_visual_voting", "sb200_kalman_initiate",
    "sb200_kalman_predict", "sb200_kalman_update", "sb200_nms", "sb200_own_area_shares", "sb200_host_alloc", "sb200_host_free",
    "sb200_predict_batch_async", "sb200_sync", "sb200_frames_in_flight", "sb200_work_counters", "sb200_screen_counters", "sb200_launch_count",
    "sb200_set_feature_dim", "sb200_comm_unique_id", "sb200_comm_create", "sb200_comm_destroy", "sb200_shard_scatter",
    "sb200_shard_gather", "sb200_wasted_history", "sb200_host_counters", "sb200_set_stream_join", "sb200_stream_join",
    "sb200_nms_batch", "sb200_nms_batch_device", "sb200_kalman_distance", "sb200_point_kalman_initiate",
    "sb200_point_kalman_predict", "sb200_point_kalman_update", "sb200_point_kalman_distance", "sb200_box_vertices",
    "sb200_clip_polygons", "sb200_intersection_areas", "sb200_set_feature_history", "sb200_wasted_visual",
    "sb200_feature_history_pool", "sb200_tracker_save", "sb200_tracker_load", "sb200_scenes_export",
    "sb200_scenes_import", "sb200_tracker_options", "sb200_set_feature_type", "sb200_fstore_create",
    "sb200_fstore_destroy", "sb200_fstore_add", "sb200_fstore_search", "sb200_fstore_associate", "sb200_fstore_fetch",
    "sb200_fstore_size", "sb200_fstore_ids", "sb200_fstore_last_stage_ms", "sb200_fstore_set_feature_type",
    "sb200_fstore_get_options", "sb200_fstore_add_device", "sb200_fstore_search_device",
    "sb200_fstore_associate_device", "sb200_fstore_save", "sb200_fstore_load", "sb200_fstore_search_owned",
    "sb200_fstore_merge_owned", "sb200_fstore_set_storage_type", "sb200_fstore_get_storage_type",
    "sb200_fstore_associate_wasted", "sb200_fstore_set_gate", "sb200_fstore_get_gate", "sb200_fstore_add_attr",
    "sb200_fstore_search_attr", "sb200_fstore_associate_attr", "sb200_fstore_fetch_attr",
    "sb200_fstore_set_retention", "sb200_fstore_get_retention", "sb200_fstore_add_quality",
    "sb200_fstore_search_quality", "sb200_fstore_associate_quality", "sb200_fstore_fetch_quality",
    "sb200_fstore_merge_history", "sb200_fstore_find_baked", "sb200_fstore_associate_store",
    "sb200_fstore_set_classes", "sb200_fstore_get_classes", "sb200_fstore_use_class", "sb200_fstore_class_counts",
    "sb200_fstore_set_voting", "sb200_fstore_get_voting", "sb200_scene_observations", "sb200_fstore_search_tracks",
]


def lib():
    """Loads the shared library (never builds it: __graft_entry__.build() / similari_b200._build do that)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise Sb200Error(
            f"{LIB_PATH} is missing: build it with `python -m similari_b200._build` (nvcc, sm_90a). "
            "similari_b200 has no CPU fallback.")
    L = C.CDLL(LIB_PATH)
    vp, i32, i64, u64, f32 = C.c_void_p, C.c_int32, C.c_int64, C.c_uint64, C.c_float
    sig = {
        "sb200_options_default": (None, [C.POINTER(Options)]),
        "sb200_last_error": (C.c_char_p, []),
        "sb200_device_count": (C.c_int, []),
        "sb200_tracker_create": (C.c_int, [C.POINTER(Options), C.POINTER(vp)]),
        "sb200_tracker_destroy": (None, [vp]),
        "sb200_tracker_set_stream": (C.c_int, [vp, vp]),
        "sb200_set_stream_join": (C.c_int, [vp, i32]),
        "sb200_stream_join": (C.c_int, [vp, vp]),
        "sb200_predict_batch": (C.c_int, [vp, i32, vp, vp, vp, vp, vp, vp, vp, vp, C.POINTER(PredictOut)]),
        "sb200_prefetch_inputs": (C.c_int, [vp, i32, vp, vp, vp, vp, vp, vp]),
        "sb200_predict_batch_async": (C.c_int, [vp, i32, vp, vp, vp, vp, vp, vp, vp, vp, C.POINTER(PredictOut)]),
        "sb200_sync": (C.c_int, [vp]),
        "sb200_set_feature_dim": (C.c_int, [vp, i32]),
        "sb200_set_feature_type": (C.c_int, [vp, i32]),
        "sb200_comm_unique_id": (C.c_int, [vp]),
        "sb200_comm_create": (C.c_int, [i32, i32, vp, i32, C.POINTER(vp)]),
        "sb200_comm_destroy": (None, [vp]),
        "sb200_shard_scatter": (C.c_int, [vp, i32, vp, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]),
        "sb200_shard_gather": (C.c_int, [vp, i32, vp, C.POINTER(PredictOut), C.POINTER(PredictOut), vp]),
        "sb200_frames_in_flight": (C.c_int, [vp]),
        "sb200_work_counters": (C.c_int, [vp, vp, vp]),
        "sb200_screen_counters": (C.c_int, [vp, vp]),
        "sb200_launch_count": (u64, []),
        "sb200_host_counters": (C.c_int, [vp, vp]),
        "sb200_predict_batch_device": (C.c_int, [vp, i32, vp, vp, vp, vp, vp, vp, vp, vp, C.POINTER(PredictOut)]),
        "sb200_skip_epochs": (C.c_int, [vp, u64, i32]),
        "sb200_current_epoch": (i64, [vp, u64]),
        "sb200_active_tracks": (i64, [vp]),
        "sb200_scene_track_counts": (C.c_int, [vp, i32, vp, vp]),
        "sb200_scene_live_counts": (C.c_int, [vp, i32, vp, vp, vp]),
        "sb200_set_auto_waste": (C.c_int, [vp, i32]),
        "sb200_clear_wasted": (C.c_int, [vp]),
        "sb200_wasted": (i64, [vp, i64, vp, vp, vp, vp, vp, vp]),
        "sb200_wasted_history": (i64, [vp, i64, vp, vp, vp, vp, vp, vp, i32, vp, vp, vp]),
        "sb200_set_feature_history": (C.c_int, [vp, i32]),
        "sb200_feature_history_pool": (C.c_int, [vp, vp]),
        "sb200_wasted_visual": (i64, [vp, i64, vp, vp, vp, vp, vp, vp, i32, vp, vp, vp, vp, vp]),
        "sb200_tracker_save": (C.c_int, [vp, vp, C.c_size_t, C.POINTER(C.c_size_t)]),
        "sb200_tracker_load": (C.c_int, [vp, C.c_size_t, i32, C.POINTER(vp)]),
        "sb200_scenes_export": (C.c_int, [vp, i32, vp, i32, vp, C.c_size_t, C.POINTER(C.c_size_t)]),
        "sb200_scenes_import": (C.c_int, [vp, vp, C.c_size_t]),
        "sb200_tracker_options": (C.c_int, [vp, C.POINTER(Options), C.POINTER(i32)]),
        "sb200_idle_tracks": (i64, [vp, u64, i64, vp, vp, vp, vp, vp]),
        "sb200_scene_tracks": (i64, [vp, u64, i64, vp, vp, vp, vp]),
        "sb200_last_costs": (i64, [vp, u64, i64, vp, C.POINTER(i32), C.POINTER(i32)]),
        "sb200_last_stage_ms": (C.c_int, [vp, vp]),
        "sb200_last_kernel_ms": (C.c_int, [vp, vp]),
        "sb200_sort_cost_matrix": (C.c_int, [i32, f32, f32, f32, f32, vp, i32, vp, vp, i32, vp, i32]),
        "sb200_visual_cost_matrix": (C.c_int, [i32, f32, vp, i32, vp, i32, i32, vp, i32]),
        "sb200_sort_voting": (C.c_int, [f32, vp, i32, i32, vp, i32]),
        "sb200_visual_voting": (C.c_int, [f32, i32, vp, vp, i32, i32, i32, vp, vp, i32]),
        "sb200_kalman_initiate": (C.c_int, [f32, f32, vp, i32, vp, i32]),
        "sb200_kalman_predict": (C.c_int, [f32, f32, vp, i32, vp, i32]),
        "sb200_kalman_update": (C.c_int, [f32, f32, vp, vp, i32, vp, i32]),
        "sb200_kalman_distance": (C.c_int, [f32, f32, vp, vp, i32, vp, i32]),
        "sb200_point_kalman_initiate": (C.c_int, [f32, f32, vp, i32, vp, i32]),
        "sb200_point_kalman_predict": (C.c_int, [f32, f32, vp, i32, vp, i32]),
        "sb200_point_kalman_update": (C.c_int, [f32, f32, vp, vp, i32, vp, i32]),
        "sb200_point_kalman_distance": (C.c_int, [f32, f32, vp, vp, i32, vp, i32]),
        "sb200_box_vertices": (C.c_int, [vp, i32, vp, i32]),
        "sb200_clip_polygons": (C.c_int, [vp, vp, i32, vp, vp, vp, i32]),
        "sb200_intersection_areas": (C.c_int, [vp, i32, vp, i32, vp, i32]),
        "sb200_nms": (i64, [vp, vp, i32, f32, f32, i32, vp, i32]),
        "sb200_nms_batch": (i64, [i32, vp, vp, vp, f32, f32, i32, vp, vp, vp, i32]),
        "sb200_nms_batch_device": (C.c_int, [i32, vp, vp, vp, f32, f32, i32, vp, vp, vp, i32, vp]),
        "sb200_own_area_shares": (C.c_int, [vp, i32, vp, i32]),
        "sb200_fstore_create": (C.c_int, [C.POINTER(FstoreOptions), C.POINTER(vp)]),
        "sb200_fstore_destroy": (None, [vp]),
        "sb200_fstore_add": (C.c_int, [vp, i32, vp, vp]),
        "sb200_fstore_search": (C.c_int, [vp, i32, vp, vp, vp, vp, vp, vp]),
        "sb200_fstore_associate": (C.c_int, [vp, i32, vp, vp, vp, vp, vp, vp, vp, vp]),
        "sb200_fstore_fetch": (i64, [vp, i32, vp, i32, vp, vp]),
        "sb200_fstore_size": (i64, [vp]),
        "sb200_fstore_ids": (i64, [vp, i64, vp]),
        "sb200_fstore_last_stage_ms": (C.c_int, [vp, vp]),
        "sb200_fstore_set_feature_type": (C.c_int, [vp, i32]),
        "sb200_fstore_get_options": (C.c_int, [vp, C.POINTER(FstoreOptions), C.POINTER(i32)]),
        "sb200_fstore_add_device": (C.c_int, [vp, i32, vp, vp, vp]),
        "sb200_fstore_search_device": (C.c_int, [vp, i32, vp, vp, vp, vp, vp, vp, vp]),
        "sb200_fstore_associate_device": (C.c_int, [vp, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp]),
        "sb200_fstore_save": (C.c_int, [vp, vp, u64, C.POINTER(u64)]),
        "sb200_fstore_load": (C.c_int, [vp, u64, i32, C.POINTER(vp)]),
        "sb200_fstore_search_owned": (C.c_int, [vp, i32, vp, i32, vp, vp, vp]),
        "sb200_fstore_merge_owned": (C.c_int, [vp, i32, vp, vp, i32]),
        "sb200_fstore_set_storage_type": (C.c_int, [vp, i32]),
        "sb200_fstore_set_gate": (C.c_int, [vp, i32]),
        "sb200_fstore_get_gate": (C.c_int, [vp, C.POINTER(i32)]),
        "sb200_fstore_set_voting": (C.c_int, [vp, i32]),
        "sb200_fstore_get_voting": (C.c_int, [vp, C.POINTER(i32)]),
        "sb200_fstore_add_attr": (C.c_int, [vp, i32, vp, C.POINTER(FstoreAttrs), vp, vp, vp]),
        "sb200_fstore_search_attr": (C.c_int, [vp, i32, vp, vp, C.POINTER(FstoreAttrs), vp, vp, vp, vp, vp, vp]),
        "sb200_fstore_associate_attr": (C.c_int, [vp, i32, vp, vp, C.POINTER(FstoreAttrs), vp, vp, vp, vp, vp, vp, vp,
                                                  vp]),
        "sb200_fstore_fetch_attr": (i64, [vp, i32, vp, vp, vp, vp]),
        "sb200_fstore_set_retention": (C.c_int, [vp, i32, i32, C.c_float]),
        "sb200_fstore_get_retention": (C.c_int, [vp, C.POINTER(i32), C.POINTER(i32), C.POINTER(C.c_float)]),
        "sb200_fstore_add_quality": (C.c_int, [vp, i32, vp, vp, C.POINTER(FstoreAttrs), vp, vp, vp]),
        "sb200_fstore_search_quality": (C.c_int, [vp, i32, vp, vp, vp, C.POINTER(FstoreAttrs), vp, vp, vp, vp, vp, vp]),
        "sb200_fstore_associate_quality": (C.c_int, [vp, i32, vp, vp, vp, C.POINTER(FstoreAttrs), vp, vp, vp, vp, vp,
                                                     vp, vp, vp]),
        "sb200_fstore_fetch_quality": (i64, [vp, i32, vp, i32, vp, vp, vp]),
        "sb200_fstore_merge_history": (i64, [vp, i32, vp, vp, i64, vp]),
        "sb200_fstore_find_baked": (i64, [vp, i64, i64, i64, vp]),
        "sb200_fstore_associate_store": (C.c_int, [vp, vp, i32, vp, i32, vp, vp, vp, vp, vp]),
        "sb200_fstore_set_classes": (C.c_int, [vp, i32, vp, vp]),
        "sb200_fstore_get_classes": (i32, [vp, i32, vp, vp]),
        "sb200_fstore_use_class": (C.c_int, [vp, u64]),
        "sb200_fstore_class_counts": (i64, [vp, i32, vp, vp]),
        "sb200_fstore_get_storage_type": (C.c_int, [vp, C.POINTER(i32)]),
        "sb200_fstore_associate_wasted": (i64, [vp, vp, i64, u64, vp, vp, vp, vp, vp, vp, i32, vp, vp, vp, vp, vp, vp, vp,
                                                vp, vp, vp]),
        "sb200_scene_observations": (i64, [vp, u64, i64, vp, vp, vp, vp, vp]),
        "sb200_fstore_search_tracks": (C.c_int, [vp, vp, i32, vp, vp, u64, C.POINTER(FstoreAttrs), vp, vp, vp, vp, vp,
                                                 vp]),
        "sb200_host_alloc": (vp, [C.c_size_t]),
        "sb200_host_free": (None, [vp]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(L, name)
        fn.restype = res
        fn.argtypes = args
    _lib = L
    return L


def check(rc):
    """Raises Sb200Error carrying sb200_last_error() when rc is a negative status."""
    if rc < 0:
        msg = lib().sb200_last_error()
        raise Sb200Error(f"sb200 status {rc}: {msg.decode() if msg else ''}")
    return rc


def ptr(a):
    """void* of a contiguous numpy array (or None)."""
    if a is None:
        return None
    return a.ctypes.data_as(C.c_void_p)


def default_options(**kw) -> Options:
    o = Options()
    lib().sb200_options_default(C.byref(o))
    constraints = kw.pop("constraints", None)
    if constraints:
        if len(constraints) > MAX_CONSTRAINTS:
            raise Sb200Error(f"at most {MAX_CONSTRAINTS} spatio-temporal constraints")
        o.n_constraints = len(constraints)
        for i, (e, d) in enumerate(constraints):
            o.constraint_epochs[i] = int(e)
            o.constraint_max_dist[i] = float(d)
    for k, v in kw.items():
        if not hasattr(o, k):
            raise AttributeError(k)
        setattr(o, k, v)
    return o


class _PinnedBuf:
    """Owns one sb200_host_alloc() block and exposes it through the array interface."""

    def __init__(self, nbytes):
        self.n = max(int(nbytes), 1)
        self.p = lib().sb200_host_alloc(self.n)
        if not self.p:
            raise Sb200Error("sb200_host_alloc failed")

    @property
    def __array_interface__(self):
        return {"shape": (self.n,), "typestr": "|u1", "data": (self.p, False), "version": 3}

    def __del__(self):
        try:
            if self.p and _lib is not None:
                _lib.sb200_host_free(self.p)
                self.p = None
        except Exception:
            pass


def pinned_empty(shape, dtype):
    """numpy array backed by pinned (page-locked) host memory from sb200_host_alloc."""
    dtype = np.dtype(dtype)
    count = int(np.prod(shape))
    raw = np.asarray(_PinnedBuf(count * dtype.itemsize))  # keeps the buffer alive as .base
    return raw[: count * dtype.itemsize].view(dtype).reshape(shape)
