"""Array-level Python interface of the engine: numpy in, numpy out, one C-ABI call per frame.

This is the zero-glue path the benchmark and the parity tests use; `similari_b200.api` layers the reference's
PyO3 class names (Sort, BatchSort, VisualSort, BatchVisualSort, ...) on top of it.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib
from ._lib import Options, PredictOut, check, check_int32, default_options, lib, ptr

F32MAX = float(np.finfo(np.float32).max)


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


# element types of the features column (sb200_set_feature_type)
FEATURE_TYPES = {"f32": _lib.FEATURE_F32, "f16": _lib.FEATURE_F16, "bf16": _lib.FEATURE_BF16}


def _raw16(a, feature_type):
    """C-contiguous array of 2-byte elements passed as the feature column of type `feature_type` without conversion."""
    if feature_type not in FEATURE_TYPES:
        raise ValueError(f"feature_type must be one of {sorted(FEATURE_TYPES)}")
    a = np.ascontiguousarray(a)
    if a.dtype.itemsize != 2:
        raise ValueError(f"feature_type={feature_type!r} needs an array of 2-byte elements, got {a.dtype}")
    return a


class Tracker:
    """Device-resident Sort / BatchSort / VisualSort / BatchVisualSort (selected by opts.kind)."""

    def __init__(self, opts: Options):
        self.opts = opts
        self._L = lib()
        h = C.c_void_p()
        check(self._L.sb200_tracker_create(C.byref(opts), C.byref(h)))
        self._h = h

    def close(self):
        if getattr(self, "_h", None):
            self._L.sb200_tracker_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_stream(self, cuda_stream: int, join_per_call: bool = True):
        """Orders every call after what `cuda_stream` holds at that moment; with join_per_call the stream also waits for
        each call's frame (else use stream_join / sync before consuming device-resident outputs)."""
        check(self._L.sb200_tracker_set_stream(self._h, C.c_void_p(cuda_stream)))
        check(self._L.sb200_set_stream_join(self._h, 1 if join_per_call else 0))

    def stream_join(self, cuda_stream: int):
        """sb200_stream_join: `cuda_stream` waits on the device for every frame enqueued so far."""
        check(self._L.sb200_stream_join(self._h, C.c_void_p(cuda_stream)))

    def predict_batch(self, scene_ids, det_offsets, boxes, features=None, has_feature=None, quality=None,
                      custom_ids=None, own_area=None, want=("ids", "epochs", "lengths", "voting_types", "predicted",
                                                            "observed"), out=None, wait=True, feature_type=None):
        """Host-pointer call (sb200_predict_batch).  Returns a dict of numpy arrays (the SortTrack columns).
        wait=False: sb200_predict_batch_async -- the arrays (pass pinned ones in `out`) are defined after sync().
        Features: a float16 array is sent as it is; any other dtype is widened to float32.  feature_type="bf16" (or
        "f16") sends a 2-byte array (e.g. the uint16 bits of bfloat16 values) as it is, with that element type."""
        scene_ids = np.ascontiguousarray(scene_ids, dtype=np.uint64)
        det_offsets = np.ascontiguousarray(det_offsets, dtype=np.int32)
        total = int(det_offsets[-1]) if len(det_offsets) else 0
        boxes = _f32(boxes).reshape(-1, 6)
        if len(boxes) != total:
            raise ValueError("boxes rows != det_offsets[-1]")
        if features is not None:
            # float16 rows go to the device as they are (the kernels widen them exactly); anything else is widened here
            if feature_type not in (None, "f32"):
                features = _raw16(features, feature_type)
                self._use_feature_type(feature_type)
            elif feature_type is None and isinstance(features, np.ndarray) and features.dtype == np.float16:
                features = np.ascontiguousarray(features)
                self._use_feature_type("f16")
            else:
                features = _f32(features)
                self._use_feature_type("f32")
        has_feature = np.ascontiguousarray(has_feature, dtype=np.uint8) if has_feature is not None else None
        quality = _f32(quality) if quality is not None else None
        custom_ids = np.ascontiguousarray(custom_ids, dtype=np.int64) if custom_ids is not None else None
        own_area = _f32(own_area) if own_area is not None else None
        if out is None:
            out = {}
            if "ids" in want:
                out["ids"] = np.zeros(total, dtype=np.uint64)
            if "epochs" in want:
                out["epochs"] = np.zeros(total, dtype=np.uint32)
            if "lengths" in want:
                out["lengths"] = np.zeros(total, dtype=np.uint32)
            if "voting_types" in want:
                out["voting_types"] = np.zeros(total, dtype=np.uint8)
            if "predicted" in want:
                out["predicted"] = np.zeros((total, 6), dtype=np.float32)
            if "observed" in want:
                out["observed"] = np.zeros((total, 6), dtype=np.float32)
        po = PredictOut(ptr(out.get("ids")), ptr(out.get("epochs")), ptr(out.get("lengths")),
                        ptr(out.get("voting_types")), ptr(out.get("predicted")), ptr(out.get("observed")))
        fn = self._L.sb200_predict_batch if wait else self._L.sb200_predict_batch_async
        check(fn(self._h, len(scene_ids), ptr(scene_ids), ptr(det_offsets), ptr(boxes), ptr(features), ptr(has_feature),
                 ptr(quality), ptr(custom_ids), ptr(own_area), C.byref(po)))
        if not wait:   # the caller's arrays must outlive the frame
            self._keep = getattr(self, "_keep", [])[-16:] + [(boxes, features, has_feature, quality, custom_ids, own_area, out)]
        return out

    def set_feature_type(self, feature_type):
        """sb200_set_feature_type: element type ("f32", "f16" or "bf16") of the features column of the calls that follow.
        Frames already enqueued keep theirs.  A new or loaded tracker reads "f32"."""
        if feature_type not in FEATURE_TYPES:
            raise ValueError(f"feature_type must be one of {sorted(FEATURE_TYPES)}")
        check(self._L.sb200_set_feature_type(self._h, FEATURE_TYPES[feature_type]))
        self._feature_type = feature_type

    @property
    def feature_type(self):
        return getattr(self, "_feature_type", "f32")

    def _use_feature_type(self, feature_type):
        # (Sort / BatchSort ignore the features column, so their type never needs setting)
        visual = self.opts.kind in (_lib.KIND_VISUAL_SORT, _lib.KIND_BATCH_VISUAL_SORT)
        if visual and feature_type != self.feature_type:
            self.set_feature_type(feature_type)

    def set_feature_dim(self, dim):
        """sb200_set_feature_dim: fixes the feature length of a visual tracker that has not stored a feature yet."""
        check(self._L.sb200_set_feature_dim(self._h, int(dim)))
        self.opts.feature_dim = int(dim)

    def sync(self):
        """sb200_sync: waits for every frame in flight; raises the first error an asynchronous frame produced."""
        check(self._L.sb200_sync(self._h))

    def frames_in_flight(self):
        return int(check(self._L.sb200_frames_in_flight(self._h)))

    def work_counters(self):
        """Cumulative work of the completed frames (waits for the frames in flight)."""
        c = np.zeros(4, np.uint64)
        ms = np.zeros(8, np.float64)
        check(self._L.sb200_work_counters(self._h, ptr(c), ptr(ms)))
        return {"pair_associations": int(c[0]), "visual_dot_products": int(c[1]), "frames": int(c[2]), "dense_fallback_scenes": int(c[3]),
                "stage_ms": dict(zip(("prep", "positional_cost", "visual_cost", "voting", "apply"), map(float, ms[:5]))),
                "vis_screen_ms": float(ms[5]), "vis_refine_ms": float(ms[6]), "tc_frames": int(ms[7])}

    def screen_counters(self):
        """sb200_screen_counters: frames screened on e4m3 and on BF16 operands, survivors of those screens that were
        refined, and survivors the exact test cut (cumulative; waits for the frames in flight)."""
        c = np.zeros(4, np.uint64)
        check(self._L.sb200_screen_counters(self._h, ptr(c)))
        return {"fp8_frames": int(c[0]), "bf16_frames": int(c[1]), "survivors": int(c[2]), "cut": int(c[3])}

    def host_counters(self):
        """sb200_host_counters: calls of the predict entry points, wall ms inside them, ms of that blocked on the device."""
        o = np.zeros(3, np.float64)
        check(self._L.sb200_host_counters(self._h, ptr(o)))
        return {"calls": int(o[0]), "ms_total": float(o[1]), "ms_blocked": float(o[2])}

    def prefetch_inputs(self, boxes, features=None, has_feature=None, quality=None, custom_ids=None, own_area=None,
                        feature_type=None):
        """sb200_prefetch_inputs: start the H2D copy of a future request.  The arrays must be the very objects later
        passed to predict_batch (same memory) and C-contiguous with the right dtype (no conversion copies).  Features
        may be float32 or float16; the tracker's feature type follows them, and the later predict_batch must pass the
        same array (a predict under another type copies the columns again)."""
        if feature_type is None:
            feature_type = "f16" if isinstance(features, np.ndarray) and features.dtype == np.float16 else "f32"
        if feature_type not in FEATURE_TYPES:
            raise ValueError(f"feature_type must be one of {sorted(FEATURE_TYPES)}")
        fdt = np.float32 if feature_type == "f32" else (features.dtype if isinstance(features, np.ndarray) else np.float16)
        if fdt != np.float32 and np.dtype(fdt).itemsize != 2:
            raise ValueError("f16 / bf16 features need an array of 2-byte elements")
        for a, dt in ((boxes, np.float32), (features, fdt), (has_feature, np.uint8), (quality, np.float32),
                      (custom_ids, np.int64), (own_area, np.float32)):
            if a is not None and not (isinstance(a, np.ndarray) and a.dtype == dt and a.flags["C_CONTIGUOUS"]):
                raise ValueError("prefetch_inputs needs C-contiguous numpy arrays of the exact dtype")
        if features is not None:
            self._use_feature_type(feature_type)
        total = int(np.prod(boxes.shape)) // 6
        check(self._L.sb200_prefetch_inputs(self._h, total, ptr(boxes), ptr(features), ptr(has_feature), ptr(quality),
                                            ptr(custom_ids), ptr(own_area)))

    def predict_batch_device(self, scene_ids, det_offsets, d_boxes, d_features=0, d_has_feature=0, d_quality=0,
                             d_custom_ids=0, d_own_area=0, d_ids=0, d_epochs=0, d_lengths=0, d_voting_types=0,
                             d_predicted=0, d_observed=0, feature_type="f32"):
        """Device-pointer call (sb200_predict_batch_device); d_* are raw device addresses (0 == NULL).  Stream-ordered:
        returns as soon as the frame is enqueued.  feature_type: element type of d_features ("f32", "f16" or "bf16",
        e.g. the data_ptr() of a torch float16 / bfloat16 CUDA tensor)."""
        if d_features:
            if feature_type not in FEATURE_TYPES:
                raise ValueError(f"feature_type must be one of {sorted(FEATURE_TYPES)}")
            self._use_feature_type(feature_type)
        scene_ids = np.ascontiguousarray(scene_ids, dtype=np.uint64)
        det_offsets = np.ascontiguousarray(det_offsets, dtype=np.int32)
        vp = lambda a: C.c_void_p(a) if a else None  # noqa: E731
        po = PredictOut(vp(d_ids), vp(d_epochs), vp(d_lengths), vp(d_voting_types), vp(d_predicted), vp(d_observed))
        check(self._L.sb200_predict_batch_device(self._h, len(scene_ids), ptr(scene_ids), ptr(det_offsets), vp(d_boxes),
                                                 vp(d_features), vp(d_has_feature), vp(d_quality), vp(d_custom_ids),
                                                 vp(d_own_area), C.byref(po)))

    def skip_epochs(self, n, scene_id=0):
        check_int32(n, "skip_epochs count")   # ctypes would pass it on modulo 2^32
        check(self._L.sb200_skip_epochs(self._h, scene_id, n))

    def current_epoch(self, scene_id=0):
        return int(check(self._L.sb200_current_epoch(self._h, scene_id)))

    def active_tracks(self):
        return int(check(self._L.sb200_active_tracks(self._h)))

    def scene_track_counts(self, scene_ids):
        scene_ids = np.ascontiguousarray(scene_ids, dtype=np.uint64)
        out = np.zeros(len(scene_ids), np.int32)
        check(self._L.sb200_scene_track_counts(self._h, len(scene_ids), ptr(scene_ids), ptr(out)))
        return out

    def scene_live_counts(self, scene_ids):
        """(live tracks, feature blocks) per scene: what the device store holds / the visual cost kernel scans."""
        scene_ids = np.ascontiguousarray(scene_ids, dtype=np.uint64)
        live = np.zeros(len(scene_ids), np.int32)
        blocks = np.zeros(len(scene_ids), np.int32)
        check(self._L.sb200_scene_live_counts(self._h, len(scene_ids), ptr(scene_ids), ptr(live), ptr(blocks)))
        return live, blocks

    def set_auto_waste(self, periodicity):
        check(self._L.sb200_set_auto_waste(self._h, periodicity))

    def clear_wasted(self):
        check(self._L.sb200_clear_wasted(self._h))

    def wasted(self, cap=1 << 16):
        ids, sc = np.zeros(cap, np.uint64), np.zeros(cap, np.uint64)
        ep, ln = np.zeros(cap, np.uint32), np.zeros(cap, np.uint32)
        pr, ob = np.zeros((cap, 6), np.float32), np.zeros((cap, 6), np.float32)
        n = check(self._L.sb200_wasted(self._h, cap, ptr(ids), ptr(sc), ptr(ep), ptr(ln), ptr(pr), ptr(ob)))
        return {"ids": ids[:n], "scene_ids": sc[:n], "epochs": ep[:n], "lengths": ln[:n], "predicted": pr[:n],
                "observed": ob[:n]}

    def wasted_history(self, cap=1 << 14, history_cap=None):
        """wasted() plus the box history of every wasted track (oldest first): predicted_history / observed_history are
        lists of [count][6] arrays."""
        H = int(history_cap if history_cap is not None else max(1, min(64, self.opts.history_length or 64)))
        ids, sc = np.zeros(cap, np.uint64), np.zeros(cap, np.uint64)
        ep, ln = np.zeros(cap, np.uint32), np.zeros(cap, np.uint32)
        pr, ob = np.zeros((cap, 6), np.float32), np.zeros((cap, 6), np.float32)
        hp, ho = np.zeros((cap, H, 6), np.float32), np.zeros((cap, H, 6), np.float32)
        hc = np.zeros(cap, np.int32)
        n = check(self._L.sb200_wasted_history(self._h, cap, ptr(ids), ptr(sc), ptr(ep), ptr(ln), ptr(pr), ptr(ob), H,
                                               ptr(hp), ptr(ho), ptr(hc)))
        return {"ids": ids[:n], "scene_ids": sc[:n], "epochs": ep[:n], "lengths": ln[:n], "predicted": pr[:n],
                "observed": ob[:n], "predicted_history": [hp[i, : hc[i]].copy() for i in range(n)],
                "observed_history": [ho[i, : hc[i]].copy() for i in range(n)]}

    def set_feature_history(self, on=True):
        """sb200_set_feature_history: keep the feature of each of a visual track's last history_length observations for
        wasted_visual().  Only before the first predict."""
        check(self._L.sb200_set_feature_history(self._h, 1 if on else 0))

    def feature_history_pool(self):
        """sb200_feature_history_pool: {"capacity", "handed_out", "free"} blocks of the feature-history pool."""
        o = np.zeros(3, np.int64)
        check(self._L.sb200_feature_history_pool(self._h, ptr(o)))
        return {"capacity": int(o[0]), "handed_out": int(o[1]), "free": int(o[2])}

    def wasted_visual(self, history_cap=None, chunk_bytes=64 << 20):
        """wasted_history() of every wasted record plus its feature history: `features` is a list of [count][d8]
        float32 arrays (oldest first, zero-padded to 8 lanes), `feature_present` a list of [count] bool arrays (False: that
        observation had no feature; its row is zero).  The records are drained in chunks of about `chunk_bytes` of
        features each."""
        if history_cap is None:
            history_cap = max(1, min(64, self.opts.history_length or 64))
        H = int(history_cap)
        if H < 0:
            raise ValueError("history_cap must be >= 0")
        d8 = (int(self.opts.feature_dim) + 7) // 8 * 8
        cap = max(1, min(1 << 14, int(chunk_bytes) // max(1, H * d8 * 4)))
        res = {k: [] for k in ("ids", "scene_ids", "epochs", "lengths", "predicted", "observed", "predicted_history",
                               "observed_history", "features", "feature_present")}
        while True:
            ids, sc = np.zeros(cap, np.uint64), np.zeros(cap, np.uint64)
            ep, ln = np.zeros(cap, np.uint32), np.zeros(cap, np.uint32)
            pr, ob = np.zeros((cap, 6), np.float32), np.zeros((cap, 6), np.float32)
            hp, ho = np.zeros((cap, H, 6), np.float32), np.zeros((cap, H, 6), np.float32)
            hc = np.zeros(cap, np.int32)
            ft, fp = np.zeros((cap, H, d8), np.float32), np.zeros((cap, H), np.uint8)
            n = check(self._L.sb200_wasted_visual(self._h, cap, ptr(ids), ptr(sc), ptr(ep), ptr(ln), ptr(pr), ptr(ob), H,
                                                  ptr(hp), ptr(ho), ptr(hc), ptr(ft), ptr(fp)))
            for k, a in (("ids", ids), ("scene_ids", sc), ("epochs", ep), ("lengths", ln), ("predicted", pr), ("observed", ob)):
                res[k].append(a[:n])
            for i in range(n):
                c = hc[i]
                res["predicted_history"].append(hp[i, :c].copy())
                res["observed_history"].append(ho[i, :c].copy())
                res["features"].append(ft[i, :c].copy())
                res["feature_present"].append(fp[i, :c].astype(bool))
            if n < cap:
                break
        for k in ("ids", "scene_ids", "epochs", "lengths", "predicted", "observed"):
            res[k] = np.concatenate(res[k])
        return res

    def idle_tracks(self, scene_id=0, cap=1 << 16):
        ids = np.zeros(cap, np.uint64)
        ep, ln = np.zeros(cap, np.uint32), np.zeros(cap, np.uint32)
        pr, ob = np.zeros((cap, 6), np.float32), np.zeros((cap, 6), np.float32)
        n = check(self._L.sb200_idle_tracks(self._h, scene_id, cap, ptr(ids), ptr(ep), ptr(ln), ptr(pr), ptr(ob)))
        return {"ids": ids[:n], "epochs": ep[:n], "lengths": ln[:n], "predicted": pr[:n], "observed": ob[:n]}

    def scene_tracks(self, scene_id=0, cap=1 << 14):
        ids = np.zeros(cap, np.uint64)
        bx, st = np.zeros((cap, 6), np.float32), np.zeros((cap, 30), np.float32)
        fc = np.zeros(cap, np.int32)
        n = check(self._L.sb200_scene_tracks(self._h, scene_id, cap, ptr(ids), ptr(bx), ptr(st), ptr(fc)))
        return {"ids": ids[:n], "boxes": bx[:n], "states": st[:n], "feat_counts": fc[:n]}

    def scene_observations(self, scene_id=0):
        """sb200_scene_observations: Track::obs of every live track of the scene, in store order (the tracks
        scene_tracks lists), gathered on the device from the tracker's arena: ids [n], n_obs [n], and per logical
        observation has_feat [n, K], quality [n, K] and feats [n, K, feature_dim] (float32; zeros where the observation has
        no feature and past n_obs).  K = visual_max_observations.  An unknown scene gives n = 0."""
        K = max(1, int(self.opts.visual_max_observations))
        D = int(self.opts.feature_dim)
        cap = int(self.scene_track_counts([scene_id])[0])
        ids, n_obs = np.zeros(max(1, cap), np.uint64), np.zeros(max(1, cap), np.int32)
        hf, q = np.zeros((max(1, cap), K), np.uint8), np.zeros((max(1, cap), K), np.float32)
        feats = np.zeros((max(1, cap), K, D), np.float32)
        n = int(check(self._L.sb200_scene_observations(self._h, int(scene_id), cap, ptr(ids), ptr(n_obs), ptr(hf), ptr(q),
                                                        ptr(feats))))
        return {"ids": ids[:n], "n_obs": n_obs[:n], "has_feat": hf[:n], "quality": q[:n], "feats": feats[:n]}

    def last_costs(self, scene_id=0, cap=1 << 22):
        out = np.zeros(cap, np.float32)
        m, n = C.c_int32(0), C.c_int32(0)
        cnt = check(self._L.sb200_last_costs(self._h, scene_id, cap, ptr(out), C.byref(m), C.byref(n)))
        return out[:cnt].reshape(m.value, n.value) if cnt else np.zeros((m.value, n.value), np.float32)

    def last_stage_ms(self):
        out = np.zeros(5, np.float32)
        check(self._L.sb200_last_stage_ms(self._h, ptr(out)))
        return dict(zip(("prep", "positional_cost", "visual_cost", "voting", "apply"), map(float, out)))


    def last_kernel_ms(self):
        out = np.zeros(2, np.float32)
        check(self._L.sb200_last_kernel_ms(self._h, ptr(out)))
        return {"vis_screen": float(out[0]), "vis_refine": float(out[1])}

    # ---- state blob: save / restore the whole tracker, move scenes between trackers and GPUs
    def feature_dim_fixed(self):
        """True once a request has carried feature rows (set_feature_dim then refuses a change)."""
        o, fixed = Options(), C.c_int32(0)
        check(self._L.sb200_tracker_options(self._h, C.byref(o), C.byref(fixed)))
        return bool(fixed.value)

    def save(self):
        """sb200_tracker_save into host memory: the whole tracker as a uint8 array."""
        return _host_blob(lambda p, cap, n: self._L.sb200_tracker_save(self._h, p, cap, n))

    def save_device(self, d_ptr, cap):
        """sb200_tracker_save into device memory (any device) at raw address `d_ptr` of `cap` bytes; returns the bytes
        written.  d_ptr == 0 returns the size the blob needs and writes nothing."""
        return _device_blob(lambda p, c, n: self._L.sb200_tracker_save(self._h, p, c, n), d_ptr, cap)

    @classmethod
    def load(cls, blob_or_ptr, nbytes=None, device=0):
        """sb200_tracker_load: a new tracker on `device` from a blob of save() (a uint8 array / bytes) or at a raw device
        address `blob_or_ptr` of `nbytes` bytes.  The options are the blob's."""
        p, n, keep = _blob_src(blob_or_ptr, nbytes)
        L = lib()
        h = C.c_void_p()
        check(L.sb200_tracker_load(p, n, int(device), C.byref(h)))
        del keep
        self = cls.__new__(cls)
        self._L, self._h = L, h
        self.opts = Options()
        check(L.sb200_tracker_options(h, C.byref(self.opts), None))
        return self

    def export_scenes(self, scene_ids, remove=False, d_ptr=None, cap=None):
        """sb200_scenes_export: the live tracks and epochs of `scene_ids` as a uint8 array, or, with `d_ptr` (a raw
        device address of `cap` bytes), into device memory, returning the bytes written (d_ptr == 0: the size needed).
        remove=True takes the scenes out of this tracker."""
        sc = np.ascontiguousarray(scene_ids, dtype=np.uint64)
        fn = lambda p, c, n: self._L.sb200_scenes_export(self._h, len(sc), ptr(sc), 1 if remove else 0, p, c, n)  # noqa: E731
        if d_ptr is None:
            return _host_blob(fn)
        return _device_blob(fn, d_ptr, cap)

    def import_scenes(self, blob_or_ptr, nbytes=None):
        """sb200_scenes_import of a blob of export_scenes() (uint8 array / bytes, or a raw device address and size)."""
        p, n, keep = _blob_src(blob_or_ptr, nbytes)
        check(self._L.sb200_scenes_import(self._h, p, n))
        del keep


_ERR_CAPACITY = -3


def _host_blob(call, size_t=C.c_size_t):
    """Size query, then the blob into a uint8 array."""
    n = size_t(0)
    rc = call(None, 0, C.byref(n))
    if rc != _ERR_CAPACITY:
        check(rc)
    out = np.empty(n.value, np.uint8)
    check(call(ptr(out), n.value, C.byref(n)))
    return out[: n.value]


def _device_blob(call, d_ptr, cap, size_t=C.c_size_t):
    n = size_t(0)
    if not d_ptr:
        rc = call(None, 0, C.byref(n))
        if rc != _ERR_CAPACITY:
            check(rc)
        return int(n.value)
    check(call(C.c_void_p(d_ptr), int(cap), C.byref(n)))
    return int(n.value)


def _blob_src(blob_or_ptr, nbytes):
    """(void*, size, object to keep alive) of a host blob or a raw device address."""
    if isinstance(blob_or_ptr, (int, np.integer)):
        if nbytes is None:
            raise ValueError("a device blob needs its size (nbytes)")
        return C.c_void_p(int(blob_or_ptr)), int(nbytes), None
    a = np.frombuffer(blob_or_ptr, dtype=np.uint8) if isinstance(blob_or_ptr, (bytes, bytearray)) else \
        np.ascontiguousarray(blob_or_ptr).view(np.uint8).reshape(-1)
    n = len(a) if nbytes is None else int(nbytes)
    return ptr(a), n, a


def blob_options(blob) -> Options:
    """The tracker options embedded in a host state blob (save() / export_scenes()); no device call."""
    a = np.ascontiguousarray(blob).view(np.uint8).reshape(-1)
    off = 24   # magic, version, type, section count, total size
    if len(a) < off + C.sizeof(Options):
        raise _lib.Sb200Error("the blob is truncated")
    return Options.from_buffer_copy(a[off: off + C.sizeof(Options)].tobytes())


class Comm:
    """NCCL communicator of the scene-sharded path (sb200_comm_*): scatter a request from an ingest rank to the ranks that
    own its scenes, gather the assigned track records back.  All pointers are raw device addresses."""

    def __init__(self, rank, world, unique_id: bytes, device):
        self._L = lib()
        h = C.c_void_p()
        buf = C.create_string_buffer(unique_id, 128)
        check(self._L.sb200_comm_create(rank, world, buf, device, C.byref(h)))
        self._h, self.rank, self.world = h, rank, world

    @staticmethod
    def unique_id() -> bytes:
        buf = C.create_string_buffer(128)
        check(lib().sb200_comm_unique_id(buf))
        return buf.raw

    def close(self):
        if getattr(self, "_h", None):
            self._L.sb200_comm_destroy(self._h)
            self._h = None

    def scatter(self, root, det_range, feature_dim, all_boxes, all_features, my_boxes, my_features, stream):
        det_range = np.ascontiguousarray(det_range, dtype=np.int32)
        vp = lambda a: C.c_void_p(a) if a else None  # noqa: E731
        check(self._L.sb200_shard_scatter(self._h, root, ptr(det_range), feature_dim, vp(all_boxes), vp(all_features), None,
                                          None, None, vp(my_boxes), vp(my_features), None, None, None, C.c_void_p(stream)))

    def gather(self, root, det_range, mine: dict, all_: dict, stream):
        """mine / all_: {"ids": addr, "epochs": addr, "lengths": addr, "voting_types": addr} (device addresses)."""
        det_range = np.ascontiguousarray(det_range, dtype=np.int32)
        vp = lambda a: C.c_void_p(a) if a else None  # noqa: E731
        keys = ("ids", "epochs", "lengths", "voting_types", "predicted", "observed")
        pm = PredictOut(*[vp(mine.get(k, 0)) for k in keys])
        pa = PredictOut(*[vp((all_ or {}).get(k, 0)) for k in keys])
        check(self._L.sb200_shard_gather(self._h, root, ptr(det_range), C.byref(pm), C.byref(pa) if all_ else None,
                                         C.c_void_p(stream)))


def launch_count():
    """Kernels launched by libsimilari_b200.so since it was loaded."""
    return int(lib().sb200_launch_count())


# ------------------------------------------------------------------------------------------------ stateless operators
def sort_cost_matrix(positional_kind, cand_boxes, track_boxes, track_states30=None, iou_threshold=0.3,
                     min_confidence=0.05, pos_weight=1 / 20, vel_weight=1 / 160, device=0):
    cb, tb = _f32(cand_boxes).reshape(-1, 6), _f32(track_boxes).reshape(-1, 6)
    ts = _f32(track_states30).reshape(-1, 30) if track_states30 is not None else None
    out = np.empty((len(cb), len(tb)), np.float32)
    check(lib().sb200_sort_cost_matrix(positional_kind, iou_threshold, min_confidence, pos_weight, vel_weight, ptr(cb),
                                       len(cb), ptr(tb), ptr(ts), len(tb), ptr(out), device))
    return out


def visual_cost_matrix(visual_kind, threshold, cand_features, track_features, device=0):
    cf, tf = _f32(cand_features), _f32(track_features)
    out = np.empty((len(cf), len(tf)), np.float32)
    check(lib().sb200_visual_cost_matrix(visual_kind, threshold, ptr(cf), len(cf), ptr(tf), len(tf), cf.shape[1],
                                         ptr(out), device))
    return out


def sort_voting(threshold, cost_mn, device=0):
    c = _f32(cost_mn)
    w = np.full(c.shape[0], -1, np.int32)
    check(lib().sb200_sort_voting(threshold, ptr(c), c.shape[0], c.shape[1], ptr(w), device))
    return w


def visual_voting(positional_threshold, min_votes, pos_mn, vis_mnk, device=0):
    p, v = _f32(pos_mn), _f32(vis_mnk)
    m, n, k = v.shape
    w, vt = np.full(m, -1, np.int32), np.zeros(m, np.uint8)
    check(lib().sb200_visual_voting(positional_threshold, min_votes, ptr(p), ptr(v), m, n, k, ptr(w), ptr(vt), device))
    return w, vt


def kalman_initiate(boxes, pw=1 / 20, vw=1 / 160, device=0):
    b = _f32(boxes).reshape(-1, 6)
    out = np.empty((len(b), 30), np.float32)
    check(lib().sb200_kalman_initiate(pw, vw, ptr(b), len(b), ptr(out), device))
    return out


def kalman_predict(states30, pw=1 / 20, vw=1 / 160, device=0):
    s = _f32(states30).reshape(-1, 30)
    out = np.empty_like(s)
    check(lib().sb200_kalman_predict(pw, vw, ptr(s), len(s), ptr(out), device))
    return out


def kalman_update(states30, boxes, pw=1 / 20, vw=1 / 160, device=0):
    s, b = _f32(states30).reshape(-1, 30), _f32(boxes).reshape(-1, 6)
    out = np.empty_like(s)
    check(lib().sb200_kalman_update(pw, vw, ptr(s), ptr(b), len(s), ptr(out), device))
    return out


def kalman_distance(states30, boxes, pw=1 / 20, vw=1 / 160, device=0):
    """sb200_kalman_distance: squared Mahalanobis distance of boxes[i] ([n][6]) from states30[i] ([n][30])."""
    s, b = _f32(states30).reshape(-1, 30), _f32(boxes).reshape(-1, 6)
    if len(s) != len(b):
        raise ValueError("states and boxes differ in length")
    out = np.empty(len(s), np.float32)
    check(lib().sb200_kalman_distance(pw, vw, ptr(s), ptr(b), len(s), ptr(out), device))
    return out


def point_kalman_initiate(points, pw=1 / 20, vw=1 / 160, device=0):
    """sb200_point_kalman_initiate: points [n][2] -> packed states [n][12] (mean x, y, vx, vy; then the x and y blocks
    P[i][i], P[i][i+2], P[i+2][i], P[i+2][i+2])."""
    p = _f32(points).reshape(-1, 2)
    out = np.empty((len(p), 12), np.float32)
    check(lib().sb200_point_kalman_initiate(pw, vw, ptr(p), len(p), ptr(out), device))
    return out


def point_kalman_predict(states12, pw=1 / 20, vw=1 / 160, device=0):
    s = _f32(states12).reshape(-1, 12)
    out = np.empty_like(s)
    check(lib().sb200_point_kalman_predict(pw, vw, ptr(s), len(s), ptr(out), device))
    return out


def point_kalman_update(states12, points, pw=1 / 20, vw=1 / 160, device=0):
    s, p = _f32(states12).reshape(-1, 12), _f32(points).reshape(-1, 2)
    if len(s) != len(p):
        raise ValueError("states and points differ in length")
    out = np.empty_like(s)
    check(lib().sb200_point_kalman_update(pw, vw, ptr(s), ptr(p), len(s), ptr(out), device))
    return out


def point_kalman_distance(states12, points, pw=1 / 20, vw=1 / 160, device=0):
    s, p = _f32(states12).reshape(-1, 12), _f32(points).reshape(-1, 2)
    if len(s) != len(p):
        raise ValueError("states and points differ in length")
    out = np.empty(len(s), np.float32)
    check(lib().sb200_point_kalman_distance(pw, vw, ptr(s), ptr(p), len(s), ptr(out), device))
    return out


def box_vertices(boxes, device=0):
    """sb200_box_vertices: boxes [n][6] -> vertices [n][4][2] (f64)."""
    b = _f32(boxes).reshape(-1, 6)
    out = np.empty((len(b), 4, 2), np.float64)
    check(lib().sb200_box_vertices(ptr(b), len(b), ptr(out), device))
    return out


def clip_polygons(subjects, clippings, device=0):
    """sb200_clip_polygons: Sutherland-Hodgman clip of subjects[i] by clippings[i] ([n][6] each).  Returns
    (vertices [n][16][2] f64, counts [n] int32, areas [n] f64); ring i is vertices[i, :counts[i]] (not closed)."""
    s, c = _f32(subjects).reshape(-1, 6), _f32(clippings).reshape(-1, 6)
    if len(s) != len(c):
        raise ValueError("subjects and clippings differ in length")
    v = np.empty((len(s), 16, 2), np.float64)
    n = np.empty(len(s), np.int32)
    a = np.empty(len(s), np.float64)
    check(lib().sb200_clip_polygons(ptr(s), ptr(c), len(s), ptr(v), ptr(n), ptr(a), device))
    return v, n, a


def intersection_areas(a, b, device=0):
    """sb200_intersection_areas: [m][n] f64 matrix of the clipped areas of every (a[i], b[j]) box pair."""
    a, b = _f32(a).reshape(-1, 6), _f32(b).reshape(-1, 6)
    out = np.zeros((len(a), len(b)), np.float64)
    check(lib().sb200_intersection_areas(ptr(a), len(a), ptr(b), len(b), ptr(out), device))
    return out


def own_area_shares(boxes, device=0):
    """exclusively_owned_areas_normalized_shares of ONE scene's boxes ([n][6]) on the GPU."""
    b = _f32(boxes).reshape(-1, 6)
    out = np.zeros(len(b), np.float32)
    check(lib().sb200_own_area_shares(ptr(b), len(b), ptr(out), device))
    return out


def nms_indices(boxes, scores, nms_threshold, score_threshold=None, device=0):
    b = _f32(boxes).reshape(-1, 6)
    s = _f32(scores) if scores is not None else None
    out = np.zeros(max(1, len(b)), np.int32)
    n = check(lib().sb200_nms(ptr(b), ptr(s), len(b), nms_threshold, 0.0 if score_threshold is None else score_threshold,
                              int(score_threshold is not None), ptr(out), device))
    return out[:n].copy()


def nms_batch(boxes, scores, offsets, nms_threshold, score_threshold=None, device=0):
    """sb200_nms_batch: nms of every set s = rows [offsets[s], offsets[s+1]) of `boxes` in one call.  Returns one int32
    array per set: the kept indices relative to the set, in rank order (what nms_indices returns for the set alone)."""
    b = _f32(boxes).reshape(-1, 6)
    offs = np.ascontiguousarray(offsets, dtype=np.int32)
    if offs.ndim != 1 or len(offs) == 0 or int(offs[-1]) != len(b):
        raise ValueError("offsets needs n_sets + 1 entries ending at the number of boxes")
    s = _f32(scores) if scores is not None else None
    if s is not None and len(s) != len(b):
        raise ValueError("scores and boxes differ in length")
    n_sets = len(offs) - 1
    idx = np.empty(max(1, len(b)), np.int32)
    counts = np.zeros(max(1, n_sets), np.int32)
    check(lib().sb200_nms_batch(n_sets, ptr(offs), ptr(b), ptr(s), nms_threshold,
                                0.0 if score_threshold is None else score_threshold, int(score_threshold is not None),
                                ptr(idx), ptr(counts), None, device))
    return [idx[offs[i]: offs[i] + counts[i]].copy() for i in range(n_sets)]


def nms_batch_device(offsets, d_boxes, d_scores, nms_threshold, score_threshold, d_keep_idx, d_keep_counts, d_keep_mask=0,
                     stream=0, device=0):
    """sb200_nms_batch_device: d_* are raw device addresses (0 == NULL), `stream` a cudaStream_t (0: the legacy default
    stream).  Stream-ordered: returns as soon as the work is enqueued on `stream`."""
    offs = np.ascontiguousarray(offsets, dtype=np.int32)
    vp = lambda a: C.c_void_p(a) if a else None  # noqa: E731
    check(lib().sb200_nms_batch_device(len(offs) - 1, ptr(offs), vp(d_boxes), vp(d_scores), nms_threshold,
                                       0.0 if score_threshold is None else score_threshold,
                                       int(score_threshold is not None), vp(d_keep_idx), vp(d_keep_counts),
                                       vp(d_keep_mask), device, vp(stream)))


METRICS = {"euclidean": _lib.VIS_EUCLIDEAN, "cosine": _lib.VIS_COSINE}
# track attribute rules of the feature store (sb200_fstore_set_gate)
GATES = {None: _lib.FSTORE_GATE_NONE, "same_source": _lib.FSTORE_GATE_SAME_SOURCE,
         "any_source": _lib.FSTORE_GATE_ANY_SOURCE}
# retention rules of the feature store (sb200_fstore_set_retention)
RETENTIONS = {"newest": _lib.FSTORE_KEEP_NEWEST, "quality": _lib.FSTORE_KEEP_BEST_QUALITY}
# voting rules of the feature store (sb200_fstore_set_voting)
VOTINGS = {"topn": _lib.FSTORE_VOTING_TOPN, "best_fit": _lib.FSTORE_VOTING_BEST_FIT}


class FeatureStore:
    """Device-resident feature track store: the reference's TrackStore for feature-only tracks (one feature class, no
    track attributes) with TopNVoting(topn, max_distance, min_votes) (or BestFitVoting, voting=) on top
    (sb200_fstore_*).  Each track keeps its newest `max_observations` observations.  Queries are given in CSR form: ids[q] with the feature rows
    features[offsets[q]:offsets[q + 1]], oldest first.  numpy in, numpy out.

    Features: a float16 array is sent as it is; any other dtype is widened to float32.  After set_feature_type("bf16")
    (or "f16") a 2-byte array (e.g. the uint16 bits of bfloat16 values) is sent as it is, with that element type.  The
    *_device calls take the raw address of a column on the store's device, in the type set by set_feature_type, and a
    cudaStream_t (0: the legacy default stream) whose pending work the call waits for.  Results never depend on the
    type or on where the column lives: they are those of the widened float32 request.

    Storage: `storage` ("f32", "f16" or "bf16") is the element type of the stored rows (sb200_fstore_set_storage_type).
    A 2-byte store takes half the device memory and half the blob; each row is rounded to it once, when it is stored,
    and queries are never rounded.  Fed features of its own type, a 2-byte store returns exactly what an f32 store
    returns; fetch() returns the stored values as float32.

    Gate: with gate="same_source" or "any_source" every track carries a source id and a [t_start, t_end] window (the
    CamTrackingAttributes of the reference's examples/track_merging.rs), and a query and a track are compared, and
    merged, only when their windows are disjoint (touching counts as disjoint) and, for "same_source", their sources are
    equal.  add / search / associate and their _device forms then need sources=, t_start= and t_end= (one per row or
    query); attributes(ids) returns the stored ones.  gate=None (the default) is the store without attributes.

    Retention: retention="quality" keeps each track's best observations by quality, as the reference's
    examples/track_merging.rs does, instead of its newest ones: every row carries an f32 quality (quality=, one per row,
    required on such a store and refused on a newest one), every track a merge history (merge_history(ids)), and a track
    of history length h holds at most min(max_observations, int(initial_capacity * merge_extension ** h)) rows, best
    first; fetch_quality(ids) returns them with their qualities.  A query takes part with its best
    int(initial_capacity * merge_extension) rows.  associate_wasted is refused on such a store.

    Feature classes: classes={class_id: feature_dim, ...} declares several feature classes (the reference's
    feature_class), each with its own dim; None is {0: feature_dim}.  add, search, associate, their _device forms,
    search_owned, fetch, fetch_quality, associate_wasted and associate_store take feature_class= (None: the first
    declared class) and work on that class's rows alone; a stored track without rows of the class takes no part in a
    search of it.  merge_owned and associate_store move every class a track holds.  classes() and class_counts(ids)
    report the classes and each track's rows in each.  A store of the single class 0 saves as before; any other
    declaration saves as blob version 4, which carries the class table.

    Voting: voting="topn" (the default) ranks each query on its own, so several queries of one associate call can merge
    into the same track.  voting="best_fit" is the reference's BestFitVoting (the rule of its VisualVoting): over all the
    queries of a call, each stored track goes to the query whose group weighs most for it (the lower query index on
    ties), a reported winner that another query took is replaced by the query's own id, and associate merges a query
    only into a track it took, else adds it as a new track.  search_owned(each=True) is unchanged by it.  set_voting()
    changes the rule at any time; it is not saved in the blob, and load() takes voting= (default "topn")."""

    def __init__(self, metric="euclidean", distance_filter=100.0, max_observations=3, feature_dim=256, topn=1,
                 max_distance=100.0, min_votes=1, device=0, storage="f32", gate=None, retention="newest",
                 initial_capacity=4, merge_extension=1.5, classes=None, voting="topn"):
        if metric not in METRICS:
            raise ValueError(f"metric must be one of {sorted(METRICS)}")
        if storage not in FEATURE_TYPES:
            raise ValueError(f"storage must be one of {sorted(FEATURE_TYPES)}")
        if gate not in GATES:
            raise ValueError(f"gate must be one of {list(GATES)}")
        if retention not in RETENTIONS:
            raise ValueError(f"retention must be one of {list(RETENTIONS)}")
        self._L = lib()
        o = _lib.FstoreOptions(METRICS[metric], distance_filter, max_observations, feature_dim, topn, max_distance,
                               min_votes, device)
        h = C.c_void_p()
        check(self._L.sb200_fstore_create(C.byref(o), C.byref(h)))
        self._h = h
        self.K, self.D, self.topn = int(max_observations), int(feature_dim), int(topn)
        self._explicit_type = None
        check(self._L.sb200_fstore_set_storage_type(h, FEATURE_TYPES[storage]))
        check(self._L.sb200_fstore_set_gate(h, GATES[gate]))
        self.gate = gate
        check(self._L.sb200_fstore_set_retention(h, RETENTIONS[retention], int(initial_capacity),
                                                 float(merge_extension)))
        self._keep = retention
        if classes is not None:
            cls = {int(k): int(v) for k, v in dict(classes).items()}
            ids, dims = np.array(list(cls), np.uint64), np.array(list(cls.values()), np.int32)
            check(self._L.sb200_fstore_set_classes(h, len(ids), ptr(ids), ptr(dims)))
        self._read_classes()
        self.set_voting(voting)

    def set_voting(self, voting):
        """sb200_fstore_set_voting: "topn" or "best_fit", the rule of every later search, associate (every form,
        associate_wasted and associate_store included) and search_owned."""
        if voting not in VOTINGS:
            raise ValueError(f"voting must be one of {list(VOTINGS)}")
        check(self._L.sb200_fstore_set_voting(self._h, VOTINGS[voting]))

    def voting(self):
        """The voting rule, "topn" or "best_fit"."""
        v = C.c_int32(0)
        check(self._L.sb200_fstore_get_voting(self._h, C.byref(v)))
        return {k: n for n, k in VOTINGS.items()}[v.value]

    def _read_classes(self):
        n = int(check(self._L.sb200_fstore_get_classes(self._h, 0, None, None)))
        ids, dims = np.zeros(n, np.uint64), np.zeros(n, np.int32)
        check(self._L.sb200_fstore_get_classes(self._h, n, ptr(ids), ptr(dims)))
        self._classes = {int(k): int(d) for k, d in zip(ids, dims)}
        self._use(None)

    def _use(self, feature_class):
        """Selects the class of the next call (None: the first declared one); its dim becomes the row length D."""
        c = next(iter(self._classes)) if feature_class is None else int(feature_class)
        if c not in self._classes:
            raise ValueError(f"feature_class {c} is not one of the store's classes {list(self._classes)}")
        check(self._L.sb200_fstore_use_class(self._h, c))
        self.D = self._classes[c]

    def classes(self):
        """The declared classes, {class_id: feature_dim}, in declared order."""
        return dict(self._classes)

    def class_counts(self, ids):
        """counts[n][len(classes())]: each track's rows in each class, in declared order (0 where an id is not
        stored); the reference's get_feature_classes with their lengths."""
        ids = np.ascontiguousarray(ids, dtype=np.uint64)
        out = np.zeros((len(ids), len(self._classes)), np.int32)
        check(self._L.sb200_fstore_class_counts(self._h, len(ids), ptr(ids), ptr(out)))
        return out

    def retention(self):
        """(rule, initial_capacity, merge_extension): rule "newest" or "quality"."""
        r, i, e = C.c_int32(0), C.c_int32(0), C.c_float(0.0)
        check(self._L.sb200_fstore_get_retention(self._h, C.byref(r), C.byref(i), C.byref(e)))
        return {v: k for k, v in RETENTIONS.items()}[r.value], int(i.value), float(e.value)

    def _quality(self, n, quality):
        """The quality column of a call (n values), or None for a newest store: required on a quality store and
        refused on a newest one, as the gate keywords are."""
        if self._keep == "newest":
            if quality is not None:
                raise ValueError("quality= needs a quality store (FeatureStore(retention='quality'))")
            return None
        if quality is None:
            raise ValueError("a quality store needs quality=, one value per feature row")
        q = np.ascontiguousarray(quality, dtype=np.float32)
        if q.shape != (n,):
            raise ValueError("quality needs one value per feature row")
        return q

    def _attrs(self, n, sources, t_start, t_end):
        """The sb200_fstore_attrs of a call (and the arrays it points into), or None for an ungated store.  The three
        keywords are required on a gated store and refused on an ungated one."""
        given = [a is not None for a in (sources, t_start, t_end)]
        if self.gate is None:
            if any(given):
                raise ValueError("sources / t_start / t_end need a gated store (FeatureStore(gate=...))")
            return None
        if not all(given):
            raise ValueError(f"a gated store (gate={self.gate!r}) needs sources, t_start and t_end")
        cols = (np.ascontiguousarray(sources, dtype=np.uint64), np.ascontiguousarray(t_start, dtype=np.int64),
                np.ascontiguousarray(t_end, dtype=np.int64))
        if any(c.shape != (n,) for c in cols):
            raise ValueError("sources / t_start / t_end need one entry per row (add) or query (search / associate)")
        return _lib.FstoreAttrs(*(c.ctypes.data for c in cols)), cols

    def close(self):
        if getattr(self, "_h", None):
            self._L.sb200_fstore_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_feature_type(self, feature_type):
        """sb200_fstore_set_feature_type: "f32", "f16" or "bf16".  With a 2-byte type, host arrays of 2-byte elements are
        sent as they are; with "f32" (the default) the host calls pick float16 arrays up by their dtype."""
        if feature_type not in FEATURE_TYPES:
            raise ValueError(f"feature_type must be one of {sorted(FEATURE_TYPES)}")
        check(self._L.sb200_fstore_set_feature_type(self._h, FEATURE_TYPES[feature_type]))
        self._explicit_type = None if feature_type == "f32" else feature_type

    def feature_type(self):
        """The element type now set in the library."""
        t = C.c_int32(0)
        check(self._L.sb200_fstore_get_options(self._h, None, C.byref(t)))
        return {v: k for k, v in FEATURE_TYPES.items()}[t.value]

    def storage_type(self):
        """The element type of the stored rows: "f32", "f16" or "bf16" (a loaded store has its blob's)."""
        t = C.c_int32(0)
        check(self._L.sb200_fstore_get_storage_type(self._h, C.byref(t)))
        return {v: k for k, v in FEATURE_TYPES.items()}[t.value]

    def _use_declared_type(self):
        """Device columns and blobs go by the type set_feature_type declared, not by the dtype of the last host array."""
        check(self._L.sb200_fstore_set_feature_type(self._h, FEATURE_TYPES[self._explicit_type or "f32"]))

    def _column(self, features):
        """The host column as the library will read it, with the library's element type set to match."""
        if self._explicit_type is not None:
            return _raw16(features, self._explicit_type).reshape(-1, self.D)
        if isinstance(features, np.ndarray) and features.dtype == np.float16:
            check(self._L.sb200_fstore_set_feature_type(self._h, _lib.FEATURE_F16))
            return np.ascontiguousarray(features).reshape(-1, self.D)
        check(self._L.sb200_fstore_set_feature_type(self._h, _lib.FEATURE_F32))
        return _f32(features).reshape(-1, self.D)

    def add(self, ids, features, sources=None, t_start=None, t_end=None, quality=None, feature_class=None):
        """TrackStore::add for each (ids[i], features[i]) in order (a gated store: with sources[i] and the window
        [t_start[i], t_end[i]]; a quality store: with quality[i]), into class feature_class."""
        self._use(feature_class)
        ids = np.ascontiguousarray(ids, dtype=np.uint64)
        a = self._attrs(len(ids), sources, t_start, t_end)
        q = self._quality(len(ids), quality)
        f = self._column(features)
        if len(f) != len(ids):
            raise ValueError("features needs one row per id")
        self._call("add", a, (len(ids), ptr(ids)), f, q=q)

    def add_device(self, ids, d_features, stream=0, sources=None, t_start=None, t_end=None, quality=None,
                   feature_class=None):
        """sb200_fstore_add_device: `d_features` is the raw device address of [len(ids)][feature_dim] elements of the
        type set by set_feature_type (e.g. the data_ptr() of a torch CUDA tensor)."""
        self._use(feature_class)
        ids = np.ascontiguousarray(ids, dtype=np.uint64)
        a = self._attrs(len(ids), sources, t_start, t_end)
        q = self._quality(len(ids), quality)
        self._use_declared_type()
        self._call("add", a, (len(ids), ptr(ids)), None, d_features, stream, q=q)

    def _call(self, op, a, lead, f, d_features=None, stream=0, out=None, q=None):
        """sb200_fstore_{op} with the host column f, or sb200_fstore_{op}_device with the device column d_features and
        the caller's stream (f is None); on a gated store (a from _attrs) sb200_fstore_{op}_attr, which takes either;
        on a quality store (q: the qualities) sb200_fstore_{op}_quality, which takes either and a's attributes or NULL.
        lead: the arguments before the attributes and features; out: the output arrays, in the call's order."""
        res = [ptr(v) for v in out.values()] if out else []
        if f is None:
            col, st = (None, C.c_void_p(d_features or None)), C.c_void_p(stream or None)
        else:
            col, st = (ptr(f), None), None
        if q is not None:
            attrs = C.byref(a[0]) if a is not None else None
            check(getattr(self._L, f"sb200_fstore_{op}_quality")(self._h, *lead, ptr(q), attrs, *col, *res, st))
        elif a is not None:
            check(getattr(self._L, f"sb200_fstore_{op}_attr")(self._h, *lead, C.byref(a[0]), *col, *res, st))
        elif f is None:
            check(getattr(self._L, f"sb200_fstore_{op}_device")(self._h, *lead, col[1], *res, st))
        else:
            check(getattr(self._L, f"sb200_fstore_{op}")(self._h, *lead, col[0], *res))

    def _queries(self, ids, offsets, features, assoc=False):
        ids = np.ascontiguousarray(ids, dtype=np.uint64)
        offs = np.ascontiguousarray(offsets, dtype=np.int32)
        if len(offs) != len(ids) + 1:
            raise ValueError("offsets must have len(ids) + 1 entries")
        f = None
        if features is not None:   # None: a device column, which the caller sized
            f = self._column(features)
            if len(ids) and int(offs[-1]) > len(f):
                raise ValueError("offsets[-1] exceeds the feature rows")
        q = len(ids)
        out = {"counts": np.zeros(q, np.int32), "winners": np.zeros((q, self.topn), np.uint64),
               "weights": np.zeros((q, self.topn), np.float64)}
        if assoc:
            out["track_ids"] = np.zeros(q, np.uint64)
            out["merged"] = np.zeros(q, np.uint8)
        return ids, offs, f, out

    def search(self, ids, offsets, features, sources=None, t_start=None, t_end=None, quality=None, feature_class=None):
        """foreign_track_distances + TopNVoting::winners: counts[q], winners[q][topn] (track ids), weights[q][topn].  A
        gated store takes one source and window per query; incompatible pairs neither vote nor count toward max_dist.
        A quality store takes one quality per feature row.  feature_class: the class searched; a stored track without
        rows of it gives no entries."""
        self._use(feature_class)
        a = self._attrs(len(ids), sources, t_start, t_end)
        ids, offs, f, out = self._queries(ids, offsets, features)
        q = self._quality(int(offs[-1]) if len(ids) else 0, quality)
        self._call("search", a, (len(ids), ptr(ids), ptr(offs)), f, out=out, q=q)
        return out

    def associate(self, ids, offsets, features, sources=None, t_start=None, t_end=None, quality=None,
                  feature_class=None):
        """search, then merge each query with a result into its first winner and add the others as new tracks.  Adds
        track_ids[q] (where the query ended up) and merged[q] to the search outputs.  A gated store merges a query only
        if it is compatible with its first winner's window as the queries merged into it earlier in the call extended it;
        otherwise the query becomes a new track.  A merged query extends its winner's class feature_class; a new track
        holds that class alone."""
        self._use(feature_class)
        a = self._attrs(len(ids), sources, t_start, t_end)
        ids, offs, f, out = self._queries(ids, offsets, features, assoc=True)
        q = self._quality(int(offs[-1]) if len(ids) else 0, quality)
        self._call("associate", a, (len(ids), ptr(ids), ptr(offs)), f, out=out, q=q)
        return out

    def search_device(self, ids, offsets, d_features, stream=0, sources=None, t_start=None, t_end=None, quality=None,
                      feature_class=None):
        """sb200_fstore_search_device: search with the feature rows at the raw device address `d_features`."""
        self._use(feature_class)
        a = self._attrs(len(ids), sources, t_start, t_end)
        ids, offs, _, out = self._queries(ids, offsets, None)
        q = self._quality(int(offs[-1]) if len(ids) else 0, quality)
        self._use_declared_type()
        self._call("search", a, (len(ids), ptr(ids), ptr(offs)), None, d_features, stream, out, q=q)
        return out

    def associate_device(self, ids, offsets, d_features, stream=0, sources=None, t_start=None, t_end=None,
                         quality=None, feature_class=None):
        """sb200_fstore_associate_device: associate with the feature rows at the raw device address `d_features`."""
        self._use(feature_class)
        a = self._attrs(len(ids), sources, t_start, t_end)
        ids, offs, _, out = self._queries(ids, offsets, None, assoc=True)
        q = self._quality(int(offs[-1]) if len(ids) else 0, quality)
        self._use_declared_type()
        self._call("associate", a, (len(ids), ptr(ids), ptr(offs)), None, d_features, stream, out, q=q)
        return out

    def search_owned(self, ids, each=False, feature_class=None):
        """sb200_fstore_search_owned: owned_track_distances + TopNVoting::winners with stored tracks as the queries, on
        the device.  each=False: one group, whose members are not candidates of each other and share max_dist;
        each=True: every id on its own (excluding only itself), as one call per id; a whole store may be passed.
        Returns the search dict; an id that is not stored, or without rows of feature_class, gets count 0."""
        self._use(feature_class)
        ids = np.ascontiguousarray(ids, dtype=np.uint64)
        q = len(ids)
        out = {"counts": np.zeros(q, np.int32), "winners": np.zeros((q, self.topn), np.uint64),
               "weights": np.zeros((q, self.topn), np.float64)}
        check(self._L.sb200_fstore_search_owned(self._h, q, ptr(ids), int(bool(each)), ptr(out["counts"]),
                                                ptr(out["winners"]), ptr(out["weights"])))
        return out

    def merge_owned(self, dest_ids, src_ids, remove=True):
        """sb200_fstore_merge_owned: for each pair in order, extend dest_ids[i] by the observations of src_ids[i] and
        keep the newest max_observations; remove=True then takes every source out of the store.  Every class a source
        holds is merged, in ascending class id."""
        d = np.ascontiguousarray(dest_ids, dtype=np.uint64)
        s = np.ascontiguousarray(src_ids, dtype=np.uint64)
        if len(d) != len(s):
            raise ValueError("dest_ids and src_ids must have the same length")
        check(self._L.sb200_fstore_merge_owned(self._h, len(d), ptr(d), ptr(s), int(bool(remove))))

    def associate_wasted(self, tracker, cap=None, id_offset=0, history_cap=None, feature_class=None):
        """sb200_fstore_associate_wasted: collects up to `cap` wasted records of the visual `tracker` (None: every record,
        in one call) as tracker.wasted_history(cap, history_cap) does, and associates each record's present history
        features (oldest first) with this store under the id ids[i] + id_offset, as one associate() call would; the
        features never leave the device.  Returns the wasted_history() dict plus, per record, feature_counts,
        queried (bool) and the associate outputs counts / winners / weights / track_ids / merged (0 where not
        queried).  The tracker needs its feature history on (set_feature_history), and feature_class a dim equal to
        the tracker's."""
        if not isinstance(tracker, Tracker):
            raise TypeError("tracker must be an engine.Tracker")
        id_offset = int(id_offset)
        if not 0 <= id_offset < 1 << 64:
            raise ValueError("id_offset must lie in [0, 2^64)")
        H = int(history_cap if history_cap is not None else max(1, min(64, tracker.opts.history_length or 64)))
        if H < 0:
            raise ValueError("history_cap must be >= 0")
        if cap is None:
            cap = self._wasted_pending(tracker)
        cap = int(cap)
        if cap < 0:
            raise ValueError("cap must be >= 0")
        n_out, t = max(1, cap), self.topn
        ids, sc = np.zeros(n_out, np.uint64), np.zeros(n_out, np.uint64)
        ep, ln = np.zeros(n_out, np.uint32), np.zeros(n_out, np.uint32)
        pr, ob = np.zeros((n_out, 6), np.float32), np.zeros((n_out, 6), np.float32)
        hp, ho = np.zeros((n_out, max(1, H), 6), np.float32), np.zeros((n_out, max(1, H), 6), np.float32)
        hc, fc, qd = np.zeros(n_out, np.int32), np.zeros(n_out, np.int32), np.zeros(n_out, np.uint8)
        cn, wn, wt = np.zeros(n_out, np.int32), np.zeros((n_out, t), np.uint64), np.zeros((n_out, t), np.float64)
        ti, mg = np.zeros(n_out, np.uint64), np.zeros(n_out, np.uint8)
        self._use(feature_class)
        n = check(self._L.sb200_fstore_associate_wasted(
            self._h, tracker._h, cap, id_offset, ptr(ids), ptr(sc), ptr(ep), ptr(ln), ptr(pr), ptr(ob), H, ptr(hp),
            ptr(ho), ptr(hc), ptr(fc), ptr(qd), ptr(cn), ptr(wn), ptr(wt), ptr(ti), ptr(mg)))
        return {"ids": ids[:n], "scene_ids": sc[:n], "epochs": ep[:n], "lengths": ln[:n], "predicted": pr[:n],
                "observed": ob[:n], "predicted_history": [hp[i, : hc[i]].copy() for i in range(n)],
                "observed_history": [ho[i, : hc[i]].copy() for i in range(n)], "feature_counts": fc[:n],
                "queried": qd[:n].astype(bool), "counts": cn[:n], "winners": wn[:n], "weights": wt[:n],
                "track_ids": ti[:n], "merged": mg[:n]}

    def search_tracks(self, tracker, scene_ids, track_ids, id_offset=0, sources=None, t_start=None, t_end=None,
                      feature_class=None):
        """sb200_fstore_search_tracks: the live tracks (scene_ids[i], track_ids[i]) of the visual `tracker` as the
        queries of one search of this store, their present observations (Track::obs order, as
        tracker.scene_observations gives them) read on the device under the id track_ids[i] + id_offset.  The store's
        query rule picks the rows (a newest store keeps the last max_observations, which drops the newest observation
        first; a quality store the best ones, with the qualities the tracker keeps).  A gated store takes one source
        and window per pair.  Returns per pair found (bool: the track is live), feature_counts, queried (bool) and the
        search outputs counts / winners / weights (0 where not queried).  Changes neither the tracker nor the store."""
        if not isinstance(tracker, Tracker):
            raise TypeError("tracker must be an engine.Tracker")
        id_offset = int(id_offset)
        if not 0 <= id_offset < 1 << 64:
            raise ValueError("id_offset must lie in [0, 2^64)")
        sc = np.ascontiguousarray(scene_ids, dtype=np.uint64)
        ti = np.ascontiguousarray(track_ids, dtype=np.uint64)
        if sc.shape != ti.shape or sc.ndim != 1:
            raise ValueError("scene_ids and track_ids must be 1-d and of the same length")
        n, t = len(ti), self.topn
        a = self._attrs(n, sources, t_start, t_end)
        self._use(feature_class)
        fd, fc, qd = np.zeros(max(1, n), np.uint8), np.zeros(max(1, n), np.int32), np.zeros(max(1, n), np.uint8)
        cn, wn, wt = np.zeros(max(1, n), np.int32), np.zeros((max(1, n), t), np.uint64), np.zeros((max(1, n), t), np.float64)
        check(self._L.sb200_fstore_search_tracks(
            self._h, tracker._h, n, ptr(sc), ptr(ti), id_offset, C.byref(a[0]) if a is not None else None, ptr(fd), ptr(fc), ptr(qd),
            ptr(cn), ptr(wn), ptr(wt)))
        return {"found": fd[:n].astype(bool), "feature_counts": fc[:n], "queried": qd[:n].astype(bool), "counts": cn[:n],
                "winners": wn[:n], "weights": wt[:n]}

    def find_baked(self, now, baked_period=0):
        """sb200_fstore_find_baked: TrackStore::find_usable with the `baked` rule of the reference's
        examples/track_merging.rs on a gated store: the ids (uint64 array, store order) of the tracks with
        now > t_end + baked_period, compared exactly for every int64 now / baked_period.  Selected on the device."""
        now, period = int(now), int(baked_period)
        if not all(-(1 << 63) <= v < 1 << 63 for v in (now, period)):
            raise ValueError("now and baked_period must fit in int64")
        n = self.size()
        out = np.zeros(max(1, n), np.uint64)
        total = int(check(self._L.sb200_fstore_find_baked(self._h, now, period, n, ptr(out))))
        return out[:min(total, n)]

    def associate_store(self, src, ids, remove=True, feature_class=None):
        """sb200_fstore_associate_store: fetch_tracks(ids) from the FeatureStore `src`, then associate them with this
        store as one associate() call whose queries are those tracks (their kept rows, qualities, windows and merge
        histories), each merged into its winner or added whole; remove=True then takes them out of `src`.  The rows
        never leave the device.  Returns the associate dict.  The search runs on feature_class; a merged track then
        brings its other classes too, and a track without rows of feature_class is added whole."""
        if not isinstance(src, FeatureStore):
            raise TypeError("src must be an engine.FeatureStore")
        self._use(feature_class)
        ids = np.ascontiguousarray(ids, dtype=np.uint64)
        q = len(ids)
        out = {"counts": np.zeros(q, np.int32), "winners": np.zeros((q, self.topn), np.uint64),
               "weights": np.zeros((q, self.topn), np.float64), "track_ids": np.zeros(q, np.uint64),
               "merged": np.zeros(q, np.uint8)}
        check(self._L.sb200_fstore_associate_store(self._h, src._h, q, ptr(ids), int(bool(remove)),
                                                   *(ptr(v) for v in out.values())))
        return out

    @staticmethod
    def _wasted_pending(tracker):
        """An upper bound of the records the next collection of `tracker` can return: every live track and every
        uncollected wasted record holds one block of the feature-history pool."""
        pool = tracker.feature_history_pool()
        return pool["handed_out"] - pool["free"]

    def fetch(self, ids, remove=False, feature_class=None):
        """(counts[n], features[n][max_observations][feature_dim]) of the tracks `ids`, oldest observation first (count 0:
        not stored, or no rows of feature_class); remove=True takes them out of the store (fetch_tracks), every class
        with them."""
        self._use(feature_class)
        ids = np.ascontiguousarray(ids, dtype=np.uint64)
        counts = np.zeros(len(ids), np.int32)
        feats = np.zeros((len(ids), self.K, self.D), np.float32)
        check(self._L.sb200_fstore_fetch(self._h, len(ids), ptr(ids), int(bool(remove)), ptr(counts), ptr(feats)))
        return counts, feats

    def fetch_quality(self, ids, remove=False, feature_class=None):
        """(counts, features, qualities) of a quality store: fetch() plus qualities[n][max_observations], the quality of
        each returned row (0 past a count); rows in the track's order, best first."""
        self._use(feature_class)
        ids = np.ascontiguousarray(ids, dtype=np.uint64)
        counts = np.zeros(len(ids), np.int32)
        feats = np.zeros((len(ids), self.K, self.D), np.float32)
        qual = np.zeros((len(ids), self.K), np.float32)
        check(self._L.sb200_fstore_fetch_quality(self._h, len(ids), ptr(ids), int(bool(remove)), ptr(counts), ptr(feats),
                                                 ptr(qual)))
        return counts, feats, qual

    def merge_history(self, ids):
        """Track::get_merge_history of each of the tracks `ids` of a quality store: a uint64 array per id, starting with
        the track's own id (empty where an id is not stored)."""
        ids = np.ascontiguousarray(ids, dtype=np.uint64)
        lens = np.zeros(max(1, len(ids)), np.int32)
        total = int(check(self._L.sb200_fstore_merge_history(self._h, len(ids), ptr(ids), ptr(lens), 0, None)))
        out = np.zeros(max(1, total), np.uint64)
        check(self._L.sb200_fstore_merge_history(self._h, len(ids), ptr(ids), ptr(lens), total, ptr(out)))
        offs = np.concatenate([[0], np.cumsum(lens[:len(ids)])])
        return [out[offs[i]: offs[i + 1]].copy() for i in range(len(ids))]

    def attributes(self, ids):
        """(sources, t_start, t_end) of the tracks `ids` of a gated store, each an array with one entry per id (0 where
        an id is not stored)."""
        if self.gate is None:
            raise ValueError("attributes() needs a gated store (FeatureStore(gate=...))")
        ids = np.ascontiguousarray(ids, dtype=np.uint64)
        n = len(ids)
        src, t0, t1 = np.zeros(n, np.uint64), np.zeros(n, np.int64), np.zeros(n, np.int64)
        check(self._L.sb200_fstore_fetch_attr(self._h, n, ptr(ids), ptr(src), ptr(t0), ptr(t1)))
        return src, t0, t1

    def size(self):
        return int(check(self._L.sb200_fstore_size(self._h)))

    def ids(self):
        """Stored track ids in store order."""
        n = self.size()
        out = np.zeros(max(1, n), np.uint64)
        check(self._L.sb200_fstore_ids(self._h, n, ptr(out)))
        return out[:n]

    def last_stage_ms(self):
        """Device times (ms) of the last call: distances, voting (TopN, plus the claims under BestFit), apply."""
        out = np.zeros(3, np.float32)
        check(self._L.sb200_fstore_last_stage_ms(self._h, ptr(out)))
        return out

    # ---- the store blob
    def save(self):
        """sb200_fstore_save into host memory: the whole store as a uint8 array."""
        self._use_declared_type()
        return _host_blob(lambda p, cap, n: self._L.sb200_fstore_save(self._h, p, cap, n), C.c_uint64)

    def save_device(self, d_ptr, cap):
        """sb200_fstore_save into device memory (any device) at raw address `d_ptr` of `cap` bytes; returns the bytes
        written.  d_ptr == 0 returns the size the blob needs and writes nothing."""
        self._use_declared_type()
        return _device_blob(lambda p, c, n: self._L.sb200_fstore_save(self._h, p, c, n), d_ptr, cap, C.c_uint64)

    @classmethod
    def load(cls, blob_or_ptr, nbytes=None, device=0, voting="topn"):
        """sb200_fstore_load: a new store on `device` from a blob of save() (a uint8 array / bytes) or at a raw device
        address `blob_or_ptr` of `nbytes` bytes.  The options, and the feature type set, are the blob's; the voting rule,
        which the blob does not hold, is `voting`."""
        if voting not in VOTINGS:
            raise ValueError(f"voting must be one of {list(VOTINGS)}")
        p, n, keep = _blob_src(blob_or_ptr, nbytes)
        L = lib()
        h = C.c_void_p()
        check(L.sb200_fstore_load(p, n, int(device), C.byref(h)))
        del keep
        self = cls.__new__(cls)
        self._L, self._h = L, h
        o, t = _lib.FstoreOptions(), C.c_int32(0)
        check(L.sb200_fstore_get_options(h, C.byref(o), C.byref(t)))
        self.K, self.D, self.topn = int(o.max_observations), int(o.feature_dim), int(o.topn)
        name = {v: k for k, v in FEATURE_TYPES.items()}[t.value]
        self._explicit_type = None if name == "f32" else name
        g = C.c_int32(0)
        check(L.sb200_fstore_get_gate(h, C.byref(g)))
        self.gate = {v: k for k, v in GATES.items()}[g.value]
        self._keep = self.retention()[0]
        self._read_classes()
        self.set_voting(voting)
        return self
