"""CPU oracle for Similari's cost-matrix + assignment hot path -- TEST INFRASTRUCTURE ONLY.

ctypes binding of ``oracle/liboracle.so`` (built from ``similari_oracle.cpp`` by ``make -C oracle``).
Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s cpu_baseline / ``--impl reference``
legs may import this package; the product package ``similari_b200`` never does.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "liboracle.so")

NONE_ID = -(2**63)
POS_MAHA, POS_IOU = 0, 1
VIS_EUCLIDEAN, VIS_COSINE = 0, 1
KIND_SORT, KIND_BATCH_SORT, KIND_VISUAL_SORT, KIND_BATCH_VISUAL_SORT = 0, 1, 2, 3
VOTING_VISUAL, VOTING_POSITIONAL = 0, 1
MAX_CONSTRAINTS = 8


def build(force: bool = False) -> str:
    """Compile liboracle.so if missing or stale (g++ only, no GPU needed)."""
    src = os.path.join(_HERE, "similari_oracle.cpp")
    hdr = os.path.join(_HERE, "similari_oracle.h")
    stale = (
        force
        or not os.path.exists(_LIB_PATH)
        or (os.path.exists(src) and os.path.getmtime(_LIB_PATH) < max(os.path.getmtime(src), os.path.getmtime(hdr)))
    )
    if stale:
        subprocess.check_call(["make", "-C", _HERE, "-B", "liboracle.so"], stdout=subprocess.DEVNULL)
    return _LIB_PATH


class Options(C.Structure):
    """Field-for-field mirror of orc_options / sb200_options."""

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


def make_options(**kw) -> Options:
    """Options with the reference's defaults (sort/simple_api.rs:461-470, visual metric/builder.rs:26-42)."""
    o = Options()
    o.kind = KIND_SORT
    o.positional_kind = POS_MAHA
    o.iou_threshold = 0.3
    o.min_confidence = 0.05
    o.max_idle_epochs = 5
    o.history_length = 1
    o.kalman_position_weight = 1.0 / 20.0
    o.kalman_velocity_weight = 1.0 / 160.0
    o.n_constraints = 0
    o.visual_kind = VIS_EUCLIDEAN
    o.visual_threshold = np.finfo(np.float32).max
    o.feature_dim = 0
    o.visual_max_observations = 5
    o.visual_min_votes = 1
    o.visual_minimal_track_length = 3
    o.visual_minimal_area = 0.0
    o.visual_minimal_quality_use = 0.0
    o.visual_minimal_quality_collect = 0.0
    o.visual_minimal_own_area_percentage_use = 0.0
    o.visual_minimal_own_area_percentage_collect = 0.0
    o.max_scenes_hint = 0
    o.max_tracks_per_scene_hint = 0
    o.max_dets_per_scene_hint = 0
    o.device = 0
    constraints = kw.pop("constraints", None)
    if constraints:
        o.n_constraints = len(constraints)
        for i, (e, d) in enumerate(constraints):
            o.constraint_epochs[i] = int(e)
            o.constraint_max_dist[i] = float(d)
    for k, v in kw.items():
        if not hasattr(o, k):
            raise AttributeError(k)
        setattr(o, k, v)
    return o


_lib = None


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t)) if a is not None else None


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB_PATH)
        f32p, f64p, u64p, i64p, i32p, u32p, u8p = (
            C.POINTER(C.c_float), C.POINTER(C.c_double), C.POINTER(C.c_uint64), C.POINTER(C.c_int64),
            C.POINTER(C.c_int32), C.POINTER(C.c_uint32), C.POINTER(C.c_uint8))
        sig = {
            "orc_radius": (C.c_float, [f32p]),
            "orc_too_far": (C.c_int, [f32p, f32p]),
            "orc_dist_in_2r": (C.c_float, [f32p, f32p]),
            "orc_vertices": (None, [f32p, f64p]),
            "orc_sutherland_hodgman_clip": (C.c_int, [f64p, C.c_int, f64p, C.c_int, f64p]),
            "orc_polygon_area": (C.c_double, [f64p, C.c_int]),
            "orc_intersection": (C.c_double, [f32p, f32p]),
            "orc_iou": (C.c_int, [f32p, f32p, f32p]),
            "orc_kalman_initiate": (None, [C.c_float, C.c_float, f32p, f32p]),
            "orc_kalman_predict": (None, [C.c_float, C.c_float, f32p, f32p]),
            "orc_kalman_update": (None, [C.c_float, C.c_float, f32p, f32p, f32p]),
            "orc_kalman_distance": (C.c_float, [C.c_float, C.c_float, f32p, f32p]),
            "orc_kalman_calculate_cost": (C.c_float, [C.c_float, C.c_int]),
            "orc_kalman_state_box": (None, [f32p, f32p]),
            "orc_euclidean": (C.c_float, [f32p, f32p, C.c_int]),
            "orc_cosine": (C.c_float, [f32p, f32p, C.c_int]),
            "orc_sort_cost_matrix": (None, [C.c_int, C.c_float, C.c_float, C.c_float, C.c_float, f32p, C.c_int, f32p,
                                            f32p, C.c_int, f32p, C.c_int]),
            "orc_visual_cost_matrix": (None, [C.c_int, C.c_float, f32p, C.c_int, f32p, C.c_int, C.c_int, f32p, C.c_int]),
            "orc_kuhn_munkres": (C.c_int64, [i64p, C.c_int, C.c_int, i32p]),
            "orc_sort_voting": (C.c_int, [C.c_float, C.c_int, C.c_int, C.c_int, u64p, u64p, f32p, u64p, u64p]),
            "orc_bestfit_voting": (C.c_int, [C.c_float, C.c_int, C.c_int, u64p, u64p, f32p, u64p, u64p, f64p]),
            "orc_visual_voting": (C.c_int, [C.c_float, C.c_float, C.c_int, C.c_int, u64p, u64p, f32p, f32p, u64p, u64p, i32p]),
            "orc_nms": (C.c_int, [f32p, f32p, C.c_int, C.c_float, C.c_float, C.c_int, i32p]),
            "orc_tracker_create": (C.c_void_p, [C.POINTER(Options)]),
            "orc_tracker_destroy": (None, [C.c_void_p]),
            "orc_tracker_set_threads": (None, [C.c_void_p, C.c_int]),
            "orc_tracker_predict_batch": (C.c_int, [C.c_void_p, C.c_int, u64p, i32p, f32p, f32p, u8p, f32p, i64p, f32p,
                                                    u64p, u32p, u32p, u8p, f32p, f32p]),
            "orc_tracker_skip_epochs": (None, [C.c_void_p, C.c_uint64, C.c_int]),
            "orc_tracker_current_epoch": (C.c_int64, [C.c_void_p, C.c_uint64]),
            "orc_tracker_active_tracks": (C.c_int, [C.c_void_p]),
            "orc_tracker_wasted": (C.c_int, [C.c_void_p, C.c_int, u64p, u64p, u32p, u32p, f32p, f32p]),
            "orc_tracker_idle_tracks": (C.c_int, [C.c_void_p, C.c_uint64, C.c_int, u64p, u32p, u32p, f32p, f32p]),
            "orc_tracker_clear_wasted": (None, [C.c_void_p]),
            "orc_tracker_scene_tracks": (C.c_int, [C.c_void_p, C.c_uint64, C.c_int, u64p, f32p, f32p, i32p]),
            "orc_tracker_scene_observations": (C.c_int, [C.c_void_p, C.c_uint64, C.c_int, C.c_int, C.c_int, i32p, u8p,
                                                         f32p, f32p, f32p]),
            "orc_tracker_last_costs": (C.c_int, [C.c_void_p, C.c_uint64, C.c_int, f32p, i32p, i32p]),
        }
        for name, (res, args) in sig.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


# --------------------------------------------------------------------------- helpers
NAN = float("nan")


def box(xc, yc, angle, aspect, height, conf=1.0):
    """Universal2DBox as 6 floats; angle=None -> NaN."""
    return np.array([xc, yc, NAN if angle is None else angle, aspect, height, conf], dtype=np.float32)


def ltwh(left, top, width, height, conf=1.0):
    """From<&BoundingBox> for Universal2DBox (src/utils/bbox.rs:246-258), in f32 like the reference."""
    f = np.float32
    left, top, width, height = f(left), f(top), f(width), f(height)
    return np.array([left + width / f(2.0), top + height / f(2.0), NAN, width / height, height, conf], dtype=np.float32)


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def radius(b):
    return float(lib().orc_radius(_p(_f32(b), C.c_float)))


def too_far(l, r):
    return bool(lib().orc_too_far(_p(_f32(l), C.c_float), _p(_f32(r), C.c_float)))


def dist_in_2r(l, r):
    return float(lib().orc_dist_in_2r(_p(_f32(l), C.c_float), _p(_f32(r), C.c_float)))


def vertices(b):
    out = np.zeros(8, dtype=np.float64)
    lib().orc_vertices(_p(_f32(b), C.c_float), _p(out, C.c_double))
    return out.reshape(4, 2)


def sh_clip(subject, clip):
    s = np.ascontiguousarray(subject, dtype=np.float64)
    c = np.ascontiguousarray(clip, dtype=np.float64)
    out = np.zeros(64, dtype=np.float64)
    n = lib().orc_sutherland_hodgman_clip(_p(s, C.c_double), len(s), _p(c, C.c_double), len(c), _p(out, C.c_double))
    return out[: 2 * n].reshape(n, 2)


def polygon_area(poly):
    p = np.ascontiguousarray(poly, dtype=np.float64)
    return float(lib().orc_polygon_area(_p(p, C.c_double), len(p)))


def intersection(l, r):
    return float(lib().orc_intersection(_p(_f32(l), C.c_float), _p(_f32(r), C.c_float)))


def iou(l, r):
    out = C.c_float(0)
    ok = lib().orc_iou(_p(_f32(l), C.c_float), _p(_f32(r), C.c_float), C.byref(out))
    return float(out.value) if ok else None


def kalman_initiate(b, pw=1 / 20, vw=1 / 160):
    st = np.zeros(110, dtype=np.float32)
    lib().orc_kalman_initiate(pw, vw, _p(_f32(b), C.c_float), _p(st, C.c_float))
    return st


def kalman_predict(st, pw=1 / 20, vw=1 / 160):
    out = np.zeros(110, dtype=np.float32)
    lib().orc_kalman_predict(pw, vw, _p(_f32(st), C.c_float), _p(out, C.c_float))
    return out


def kalman_update(st, b, pw=1 / 20, vw=1 / 160):
    out = np.zeros(110, dtype=np.float32)
    lib().orc_kalman_update(pw, vw, _p(_f32(st), C.c_float), _p(_f32(b), C.c_float), _p(out, C.c_float))
    return out


def kalman_distance(st, b, pw=1 / 20, vw=1 / 160):
    return float(lib().orc_kalman_distance(pw, vw, _p(_f32(st), C.c_float), _p(_f32(b), C.c_float)))


def kalman_calculate_cost(d, inverted):
    return float(lib().orc_kalman_calculate_cost(d, int(inverted)))


def kalman_state_box(st):
    out = np.zeros(6, dtype=np.float32)
    lib().orc_kalman_state_box(_p(_f32(st), C.c_float), _p(out, C.c_float))
    return out


def euclidean(a, b):
    a, b = _f32(a), _f32(b)
    return float(lib().orc_euclidean(_p(a, C.c_float), _p(b, C.c_float), len(a)))


def cosine(a, b):
    a, b = _f32(a), _f32(b)
    return float(lib().orc_cosine(_p(a, C.c_float), _p(b, C.c_float), len(a)))


def sort_cost_matrix(positional_kind, cand_boxes, track_boxes, track_states=None, iou_threshold=0.3,
                     min_confidence=0.05, pw=1 / 20, vw=1 / 160, threads=1):
    cb, tb = _f32(cand_boxes).reshape(-1, 6), _f32(track_boxes).reshape(-1, 6)
    ts = _f32(track_states).reshape(-1, 110) if track_states is not None else None
    out = np.empty((len(cb), len(tb)), dtype=np.float32)
    lib().orc_sort_cost_matrix(positional_kind, iou_threshold, min_confidence, pw, vw, _p(cb, C.c_float), len(cb),
                               _p(tb, C.c_float), _p(ts, C.c_float), len(tb), _p(out, C.c_float), threads)
    return out


def visual_cost_matrix(visual_kind, threshold, cand_feats, track_feats, threads=1):
    cf, tf = _f32(cand_feats), _f32(track_feats)
    out = np.empty((len(cf), len(tf)), dtype=np.float32)
    lib().orc_visual_cost_matrix(visual_kind, threshold, _p(cf, C.c_float), len(cf), _p(tf, C.c_float), len(tf),
                                 cf.shape[1], _p(out, C.c_float), threads)
    return out


def kuhn_munkres(w):
    w = np.ascontiguousarray(w, dtype=np.int64)
    out = np.zeros(w.shape[0], dtype=np.int32)
    total = lib().orc_kuhn_munkres(_p(w, C.c_int64), w.shape[0], w.shape[1], _p(out, C.c_int32))
    return int(total), out


def _ents(ents):
    """ents: list of (from, to, attr|None, feat|None)."""
    fr = np.array([e[0] for e in ents], dtype=np.uint64)
    to = np.array([e[1] for e in ents], dtype=np.uint64)
    at = np.array([NAN if e[2] is None else e[2] for e in ents], dtype=np.float32)
    fe = np.array([NAN if e[3] is None else e[3] for e in ents], dtype=np.float32)
    return fr, to, at, fe


def sort_voting(threshold, candidates_num, tracks_num, ents):
    fr, to, at, _ = _ents(ents)
    of, ot = np.zeros(max(1, candidates_num), dtype=np.uint64), np.zeros(max(1, candidates_num), dtype=np.uint64)
    n = lib().orc_sort_voting(threshold, candidates_num, tracks_num, len(fr), _p(fr, C.c_uint64), _p(to, C.c_uint64),
                              _p(at, C.c_float), _p(of, C.c_uint64), _p(ot, C.c_uint64))
    return {int(of[i]): [int(ot[i])] for i in range(n)}


def bestfit_voting(max_distance, min_votes, ents):
    fr, to, _, fe = _ents(ents)
    cap = max(1, len(fr))
    q, w, wt = np.zeros(cap, dtype=np.uint64), np.zeros(cap, dtype=np.uint64), np.zeros(cap, dtype=np.float64)
    n = lib().orc_bestfit_voting(max_distance, min_votes, len(fr), _p(fr, C.c_uint64), _p(to, C.c_uint64),
                                 _p(fe, C.c_float), _p(q, C.c_uint64), _p(w, C.c_uint64), _p(wt, C.c_double))
    res = {}
    for i in range(n):
        res.setdefault(int(q[i]), []).append((int(w[i]), float(wt[i])))
    return res


def visual_voting(positional_threshold, max_allowed_feature_distance, min_votes, ents):
    fr, to, at, fe = _ents(ents)
    cap = max(1, len(fr))
    of, ot, ty = np.zeros(cap, dtype=np.uint64), np.zeros(cap, dtype=np.uint64), np.zeros(cap, dtype=np.int32)
    n = lib().orc_visual_voting(positional_threshold, max_allowed_feature_distance, min_votes, len(fr),
                                _p(fr, C.c_uint64), _p(to, C.c_uint64), _p(at, C.c_float), _p(fe, C.c_float),
                                _p(of, C.c_uint64), _p(ot, C.c_uint64), _p(ty, C.c_int32))
    return {int(of[i]): [(int(ot[i]), int(ty[i]))] for i in range(n)}


def own_area_shares(boxes):
    """exclusively_owned_areas_normalized_shares of one scene's boxes (src/utils/clipping/bbox_own_areas.rs:8-46)."""
    b = _f32(boxes).reshape(-1, 6)
    out = np.zeros(len(b), dtype=np.float32)
    lib().orc_own_area_shares(_p(b, C.c_float), len(b), _p(out, C.c_float))
    return out


def nms(boxes, scores, nms_threshold, score_threshold=None):
    b = _f32(boxes).reshape(-1, 6)
    s = _f32(scores) if scores is not None else None
    out = np.zeros(max(1, len(b)), dtype=np.int32)
    n = lib().orc_nms(_p(b, C.c_float), _p(s, C.c_float), len(b), nms_threshold,
                      0.0 if score_threshold is None else score_threshold, int(score_threshold is not None),
                      _p(out, C.c_int32))
    return out[:n].copy()


class Tracker:
    """Sort / BatchSort / VisualSort / BatchVisualSort semantics on the CPU (reference execution order)."""

    def __init__(self, opts: Options, threads: int = 1):
        self._L = lib()
        self.opts = opts
        self._h = self._L.orc_tracker_create(C.byref(opts))
        self._L.orc_tracker_set_threads(self._h, threads)

    def __del__(self):
        if getattr(self, "_h", None):
            self._L.orc_tracker_destroy(self._h)
            self._h = None

    def predict_batch(self, scene_ids, det_offsets, boxes, features=None, has_feature=None, quality=None,
                      custom_ids=None, own_area=None, want_boxes=True):
        scene_ids = np.ascontiguousarray(scene_ids, dtype=np.uint64)
        det_offsets = np.ascontiguousarray(det_offsets, dtype=np.int32)
        boxes = _f32(boxes).reshape(-1, 6)
        total = int(det_offsets[-1])
        assert len(boxes) == total
        features = _f32(features) if features is not None else None
        has_feature = np.ascontiguousarray(has_feature, dtype=np.uint8) if has_feature is not None else None
        quality = _f32(quality) if quality is not None else None
        custom_ids = np.ascontiguousarray(custom_ids, dtype=np.int64) if custom_ids is not None else None
        own_area = _f32(own_area) if own_area is not None else None
        out = {
            "ids": np.zeros(total, dtype=np.uint64),
            "epochs": np.zeros(total, dtype=np.uint32),
            "lengths": np.zeros(total, dtype=np.uint32),
            "voting_types": np.zeros(total, dtype=np.uint8),
            "predicted": np.zeros((total, 6), dtype=np.float32) if want_boxes else None,
            "observed": np.zeros((total, 6), dtype=np.float32) if want_boxes else None,
        }
        rc = self._L.orc_tracker_predict_batch(
            self._h, len(scene_ids), _p(scene_ids, C.c_uint64), _p(det_offsets, C.c_int32), _p(boxes, C.c_float),
            _p(features, C.c_float), _p(has_feature, C.c_uint8), _p(quality, C.c_float), _p(custom_ids, C.c_int64),
            _p(own_area, C.c_float), _p(out["ids"], C.c_uint64), _p(out["epochs"], C.c_uint32),
            _p(out["lengths"], C.c_uint32), _p(out["voting_types"], C.c_uint8), _p(out["predicted"], C.c_float),
            _p(out["observed"], C.c_float))
        assert rc == 0
        return out

    def skip_epochs(self, n, scene_id=0):
        self._L.orc_tracker_skip_epochs(self._h, scene_id, n)

    def current_epoch(self, scene_id=0):
        return int(self._L.orc_tracker_current_epoch(self._h, scene_id))

    def active_tracks(self):
        return int(self._L.orc_tracker_active_tracks(self._h))

    def _tracks(self, fn, cap, *pre, with_scene=True):
        ids, sc = np.zeros(cap, dtype=np.uint64), np.zeros(cap, dtype=np.uint64)
        ep, ln = np.zeros(cap, dtype=np.uint32), np.zeros(cap, dtype=np.uint32)
        pr, ob = np.zeros((cap, 6), dtype=np.float32), np.zeros((cap, 6), dtype=np.float32)
        if with_scene:
            n = fn(self._h, *pre, cap, _p(ids, C.c_uint64), _p(sc, C.c_uint64), _p(ep, C.c_uint32), _p(ln, C.c_uint32),
                   _p(pr, C.c_float), _p(ob, C.c_float))
        else:
            n = fn(self._h, *pre, cap, _p(ids, C.c_uint64), _p(ep, C.c_uint32), _p(ln, C.c_uint32), _p(pr, C.c_float),
                   _p(ob, C.c_float))
        return {"ids": ids[:n], "scene_ids": sc[:n], "epochs": ep[:n], "lengths": ln[:n], "predicted": pr[:n],
                "observed": ob[:n]}

    def wasted(self, cap=1 << 16):
        return self._tracks(self._L.orc_tracker_wasted, cap)

    def idle_tracks(self, scene_id=0, cap=1 << 16):
        return self._tracks(self._L.orc_tracker_idle_tracks, cap, scene_id, with_scene=False)

    def clear_wasted(self):
        self._L.orc_tracker_clear_wasted(self._h)

    def scene_tracks(self, scene_id=0, cap=1 << 14):
        ids = np.zeros(cap, dtype=np.uint64)
        bx = np.zeros((cap, 6), dtype=np.float32)
        st = np.zeros((cap, 110), dtype=np.float32)
        fc = np.zeros(cap, dtype=np.int32)
        n = self._L.orc_tracker_scene_tracks(self._h, scene_id, cap, _p(ids, C.c_uint64), _p(bx, C.c_float),
                                             _p(st, C.c_float), _p(fc, C.c_int32))
        return {"ids": ids[:n], "boxes": bx[:n], "states": st[:n], "feat_counts": fc[:n]}

    def scene_observations(self, scene_id=0):
        """Track::obs of every track of the scene, in store order: n_obs [n], and per observation [n, K] has_feat,
        quality, the feature zero-padded to d8 ([n, K, d8]) and its squared norm.  Entries past n_obs are zero."""
        K = max(1, int(self.opts.visual_max_observations))
        d8 = (int(self.opts.feature_dim) + 7) // 8 * 8
        cap = max(1, self.active_tracks())
        n_obs = np.zeros(cap, dtype=np.int32)
        hf = np.zeros((cap, K), dtype=np.uint8)
        q = np.zeros((cap, K), dtype=np.float32)
        feats = np.zeros((cap, K, d8), dtype=np.float32)
        n2 = np.zeros((cap, K), dtype=np.float32)
        n = self._L.orc_tracker_scene_observations(self._h, scene_id, cap, K, d8, _p(n_obs, C.c_int32),
                                                   _p(hf, C.c_uint8), _p(q, C.c_float), _p(feats, C.c_float),
                                                   _p(n2, C.c_float))
        return {"n_obs": n_obs[:n], "has_feat": hf[:n], "quality": q[:n], "feats": feats[:n], "norm2": n2[:n]}

    def last_costs(self, scene_id=0, cap=1 << 22):
        out = np.zeros(cap, dtype=np.float32)
        m, n = C.c_int32(0), C.c_int32(0)
        cnt = self._L.orc_tracker_last_costs(self._h, scene_id, cap, _p(out, C.c_float), C.byref(m), C.byref(n))
        return out[:cnt].reshape(m.value, n.value) if cnt else np.zeros((0, 0), dtype=np.float32)
