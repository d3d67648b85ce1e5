"""The reference's Python surface (PyO3 module `similari`, src/lib.rs:117-161) over the H100 engine.

Class names, constructor defaults and method names follow the reference so that `import similari_b200.api as similari`
is a drop-in for scripts using the cost-matrix + assignment trackers.  Each class cites the PyO3 definition it mirrors.
Objects here are thin: all state lives on the GPU inside `engine.Tracker`.
"""
from __future__ import annotations

import math
from collections.abc import Sequence
from typing import List, Optional, Tuple

import numpy as np

from . import _lib, engine
from ._lib import NONE_ID, default_options

F32 = np.float32


class BoundingBox:
    """src/utils/bbox.rs `PyBoundingBox` (left, top, width, height, confidence)."""

    def __init__(self, left, top, width, height):
        self.left, self.top, self.width, self.height, self.confidence = F32(left), F32(top), F32(width), F32(height), F32(1.0)

    @staticmethod
    def new_with_confidence(left, top, width, height, confidence):
        assert 0.0 <= confidence <= 1.0, "Confidence must lay between 0.0 and 1.0"
        b = BoundingBox(left, top, width, height)
        b.confidence = F32(confidence)
        return b

    def as_xyaah(self) -> "Universal2DBox":
        # From<&BoundingBox> for Universal2DBox, src/utils/bbox.rs:246-258 (f32 arithmetic)
        return Universal2DBox.new_with_confidence(self.left + self.width / F32(2.0), self.top + self.height / F32(2.0),
                                                  None, self.width / self.height, self.height, self.confidence)

    def __repr__(self):
        return f"BoundingBox(left={self.left}, top={self.top}, width={self.width}, height={self.height}, confidence={self.confidence})"


class Universal2DBox:
    """src/utils/bbox.rs `PyUniversal2DBox` (xc, yc, angle, aspect, height, confidence)."""

    def __init__(self, xc, yc, angle, aspect, height):
        self.xc, self.yc, self.aspect, self.height = F32(xc), F32(yc), F32(aspect), F32(height)
        self.angle = None if angle is None else F32(angle)
        self.confidence = F32(1.0)

    @staticmethod
    def new_with_confidence(xc, yc, angle, aspect, height, confidence):
        assert 0.0 <= confidence <= 1.0, "Confidence must lay between 0.0 and 1.0"
        b = Universal2DBox(xc, yc, angle, aspect, height)
        b.confidence = F32(confidence)
        return b

    @staticmethod
    def ltwh(left, top, width, height):
        return BoundingBox(left, top, width, height).as_xyaah()

    @staticmethod
    def ltwh_with_confidence(left, top, width, height, confidence):
        return BoundingBox.new_with_confidence(left, top, width, height, confidence).as_xyaah()

    def as_ltwh(self) -> BoundingBox:
        if self.angle is not None:
            raise AttributeError("Generic BBox cannot be converted to a requested type")
        w = self.height * self.aspect
        return BoundingBox.new_with_confidence(self.xc - w / F32(2.0), self.yc - self.height / F32(2.0), w, self.height,
                                               self.confidence)

    def get_radius(self):
        hw, hh = self.aspect * self.height / F32(2.0), self.height / F32(2.0)
        return float(np.sqrt(hw * hw + hh * hh))

    def area(self):
        return float(self.height * self.aspect * self.height)

    def rotate(self, angle):
        self.angle = F32(angle)

    def gen_vertices(self):
        """Accepted for compatibility: the reference fills a vertex cache that no Python-visible result depends on."""

    def get_vertices(self) -> "Polygon":
        """src/utils/bbox.rs:685-687: the four vertices (angle None == 0) as a closed Polygon."""
        return Polygon._from_ring(engine.box_vertices(np.array([self._row()], dtype=np.float32))[0])

    def _row(self):
        return [self.xc, self.yc, math.nan if self.angle is None else self.angle, self.aspect, self.height, self.confidence]

    @staticmethod
    def _from_row(r) -> "Universal2DBox":
        return Universal2DBox.new_with_confidence(r[0], r[1], None if np.isnan(r[2]) else r[2], r[3], r[4], r[5])

    def __repr__(self):
        return (f"Universal2DBox(xc={self.xc}, yc={self.yc}, angle={self.angle}, aspect={self.aspect}, "
                f"height={self.height}, confidence={self.confidence})")


class PositionalMetricType:
    """src/trackers/sort.rs `PyPositionalMetricType`."""

    def __init__(self, kind, threshold=0.3):
        self.kind, self.threshold = kind, float(threshold)

    @staticmethod
    def maha():
        return PositionalMetricType(_lib.POS_MAHA)

    @staticmethod
    def iou(threshold):
        assert 0.0 < threshold < 1.0, "Threshold must lay between (0.0 and 1.0)"
        return PositionalMetricType(_lib.POS_IOU, threshold)


class VisualSortMetricType:
    """src/trackers/visual_sort/metric.rs `PyVisualSortMetricType`."""

    def __init__(self, kind, threshold):
        self.kind, self.threshold = kind, float(threshold)

    @staticmethod
    def euclidean(threshold):
        assert threshold > 0.0, "Threshold must be a positive number"
        return VisualSortMetricType(_lib.VIS_EUCLIDEAN, threshold)

    @staticmethod
    def cosine(threshold):
        assert -1.0 <= threshold <= 1.0, "Threshold must lay within [-1.0:1:0]"
        return VisualSortMetricType(_lib.VIS_COSINE, threshold)


class SpatioTemporalConstraints:
    """src/trackers/spatio_temporal_constraints.rs `PySpatioTemporalConstraints`."""

    def __init__(self):
        self.constraints: List[Tuple[int, float]] = []

    def add_constraints(self, constraints):
        for d, m in constraints:
            assert m > 0.0, "The distance is expected to be a positive float"
            self.constraints.append((int(d), float(m)))
        self.constraints.sort(key=lambda c: c[0])  # stable; dedup keeps the first
        out = []
        for c in self.constraints:
            if not out or out[-1][0] != c[0]:
                out.append(c)
        self.constraints = out

    def validate(self, epoch_delta, dist):
        assert dist >= 0.0, "The distance is expected to be a positive float"
        for d, m in self.constraints:
            if d >= epoch_delta:
                return dist <= m
        return True


class VotingType:
    Visual, Positional = _lib.VOTING_VISUAL, _lib.VOTING_POSITIONAL


class SortTrack:
    """src/trackers/sort.rs:286-311 `PySortTrack`."""

    __slots__ = ("id", "epoch", "predicted_bbox", "observed_bbox", "scene_id", "length", "voting_type", "custom_object_id")

    def __init__(self, id, epoch, predicted_bbox, observed_bbox, scene_id, length, voting_type, custom_object_id):
        self.id, self.epoch, self.predicted_bbox, self.observed_bbox = int(id), int(epoch), predicted_bbox, observed_bbox
        self.scene_id, self.length, self.voting_type, self.custom_object_id = int(scene_id), int(length), voting_type, custom_object_id

    def __repr__(self):
        return (f"SortTrack(id={self.id}, epoch={self.epoch}, scene_id={self.scene_id}, length={self.length}, "
                f"voting_type={self.voting_type}, custom_object_id={self.custom_object_id})")


class WastedSortTrack:
    """src/trackers/sort.rs:316-341 `PyWastedSortTrack`: predicted_boxes / observed_boxes hold the last bbox_history boxes."""

    __slots__ = ("id", "epoch", "predicted_bbox", "observed_bbox", "scene_id", "length", "predicted_boxes", "observed_boxes")

    def __init__(self, id, epoch, predicted_bbox, observed_bbox, scene_id, length, predicted_boxes=None, observed_boxes=None):
        self.id, self.epoch, self.scene_id, self.length = int(id), int(epoch), int(scene_id), int(length)
        self.predicted_bbox, self.observed_bbox = predicted_bbox, observed_bbox
        self.predicted_boxes = predicted_boxes if predicted_boxes is not None else [predicted_bbox]
        self.observed_boxes = observed_boxes if observed_boxes is not None else [observed_bbox]


class WastedVisualSortTrack(WastedSortTrack):
    """src/trackers/visual_sort.rs:195-224 `PyWastedVisualSortTrack`: a WastedSortTrack plus observed_features, the feature
    of each of the track's last kept_history_length observations (oldest first; None for an observation without one).
    Each feature is its f32 values zero-padded to a multiple of 8 (Vec::from_vec(&Feature), src/track/utils.rs:25-33)."""

    __slots__ = ("_feat_rows", "_feat_present", "_observed_features")

    def __init__(self, id, epoch, predicted_bbox, observed_bbox, scene_id, length, predicted_boxes=None,
                 observed_boxes=None, feature_rows=None, feature_present=None):
        super().__init__(id, epoch, predicted_bbox, observed_bbox, scene_id, length, predicted_boxes, observed_boxes)
        self._feat_rows = np.zeros((0, 8), np.float32) if feature_rows is None else feature_rows
        self._feat_present = np.zeros(len(self._feat_rows), bool) if feature_present is None else feature_present
        self._observed_features = None

    @property
    def observed_features(self) -> List[Optional[List[float]]]:
        # built from the packed [count][d8] rows when first read: most users of wasted() never look at it
        if self._observed_features is None:
            self._observed_features = [row.tolist() if p else None for row, p in zip(self._feat_rows, self._feat_present)]
        return self._observed_features


def _tracks_from(out, scene_id, custom_ids=None) -> List[SortTrack]:
    res = []
    for i in range(len(out["ids"])):
        cid = None
        if custom_ids is not None and custom_ids[i] != NONE_ID:
            cid = int(custom_ids[i])
        res.append(SortTrack(out["ids"][i], out["epochs"][i], Universal2DBox._from_row(out["predicted"][i]),
                             Universal2DBox._from_row(out["observed"][i]), scene_id, out["lengths"][i],
                             int(out["voting_types"][i]), cid))
    return res


class _TrackerBase:
    _t: engine.Tracker

    def skip_epochs(self, n):
        assert n > 0
        self._t.skip_epochs(int(n), 0)

    def skip_epochs_for_scene(self, scene_id, n):
        assert n > 0 and scene_id >= 0
        self._t.skip_epochs(int(n), int(scene_id))

    def shard_stats(self):
        return [self._t.active_tracks()]

    def current_epoch(self):
        return self._t.current_epoch(0)

    def current_epoch_with_scene(self, scene_id):
        assert scene_id >= 0
        return self._t.current_epoch(int(scene_id))

    def wasted(self):
        w = self._t.wasted_history()
        return [WastedSortTrack(w["ids"][i], w["epochs"][i], Universal2DBox._from_row(w["predicted"][i]),
                                Universal2DBox._from_row(w["observed"][i]), w["scene_ids"][i], w["lengths"][i],
                                [Universal2DBox._from_row(r) for r in w["predicted_history"][i]],
                                [Universal2DBox._from_row(r) for r in w["observed_history"][i]])
                for i in range(len(w["ids"]))]

    def clear_wasted(self):
        self._t.clear_wasted()

    def _idle(self, scene_id):
        w = self._t.idle_tracks(int(scene_id))
        return [SortTrack(w["ids"][i], w["epochs"][i], Universal2DBox._from_row(w["predicted"][i]),
                          Universal2DBox._from_row(w["observed"][i]), scene_id, w["lengths"][i], VotingType.Positional, None)
                for i in range(len(w["ids"]))]

    def save_state(self) -> np.ndarray:
        """The whole tracker as a uint8 array (sb200_tracker_save); `load_state` continues it exactly.  An extension with
        no PyO3 counterpart in the reference."""
        return self._t.save()


class _SceneTransfer:
    def export_scenes(self, scene_ids, remove=False) -> np.ndarray:
        """The live tracks and epochs of `scene_ids` as a uint8 array (sb200_scenes_export); remove=True takes the
        scenes out of this tracker.  An extension with no PyO3 counterpart in the reference."""
        return self._t.export_scenes([int(s) for s in scene_ids], remove=remove)

    def import_scenes(self, blob):
        """Adds the scenes of an export_scenes() blob of a tracker with the same options (sb200_scenes_import).  An
        extension with no PyO3 counterpart in the reference."""
        self._t.import_scenes(blob)


def _sort_options(kind, bbox_history, max_idle_epochs, method, min_confidence, constraints, pw, vw):
    method = method or PositionalMetricType.maha()
    assert bbox_history > 0
    return default_options(kind=kind, positional_kind=method.kind, iou_threshold=method.threshold,
                           min_confidence=min_confidence, max_idle_epochs=int(max_idle_epochs),
                           history_length=int(bbox_history), kalman_position_weight=pw, kalman_velocity_weight=vw,
                           constraints=constraints.constraints if constraints else None)


class Sort(_TrackerBase):
    """src/trackers/sort/simple_api.rs `PySort` (defaults :461-470).  `shards` is accepted and ignored: the GPU engine
    has no shard threads."""

    def __init__(self, shards=4, bbox_history=1, max_idle_epochs=5, method=None, min_confidence=0.05,
                 spatio_temporal_constraints=None, kalman_position_weight=1.0 / 20.0, kalman_velocity_weight=1.0 / 160.0):
        self._t = engine.Tracker(_sort_options(_lib.KIND_SORT, bbox_history, max_idle_epochs, method, min_confidence,
                                               spatio_temporal_constraints, kalman_position_weight, kalman_velocity_weight))

    def predict(self, bboxes):
        return self.predict_with_scene(0, bboxes)

    def predict_with_scene(self, scene_id, bboxes):
        assert scene_id >= 0
        boxes = np.array([b._row() for b, _ in bboxes], dtype=np.float32).reshape(-1, 6)
        custom = np.array([NONE_ID if c is None else c for _, c in bboxes], dtype=np.int64)
        out = self._t.predict_batch([scene_id], [0, len(bboxes)], boxes, custom_ids=custom)
        return _tracks_from(out, scene_id, custom)

    def idle_tracks(self):
        return self._idle(0)

    def idle_tracks_with_scene(self, scene_id):
        return self._idle(scene_id)


class PredictionBatchResult:
    """src/trackers/batch.rs `PyPredictionBatchResult`: per-scene results of one batch predict."""

    def __init__(self, items):
        self._items = list(items)
        self._size = len(self._items)

    def ready(self):
        return bool(self._items)

    def get(self):
        return self._items.pop(0)

    def batch_size(self):
        return self._size


class SortPredictionBatchRequest:
    """src/trackers/sort/batch_api.rs `PySortPredictionBatchRequest`."""

    def __init__(self):
        self.batch = {}

    def add(self, scene_id, bbox, custom_object_id=None):
        self.batch.setdefault(int(scene_id), []).append((bbox, custom_object_id))

    def prediction(self):
        return None


class BatchSort(_SceneTransfer, _TrackerBase):
    """src/trackers/sort/batch_api.rs `PyBatchSort` (defaults :391-401)."""

    def __init__(self, distance_shards=4, voting_shards=4, bbox_history=1, max_idle_epochs=5, method=None,
                 min_confidence=0.05, spatio_temporal_constraints=None, kalman_position_weight=1.0 / 20.0,
                 kalman_velocity_weight=1.0 / 160.0):
        self._t = engine.Tracker(_sort_options(_lib.KIND_BATCH_SORT, bbox_history, max_idle_epochs, method, min_confidence,
                                               spatio_temporal_constraints, kalman_position_weight, kalman_velocity_weight))

    def predict(self, batch: SortPredictionBatchRequest) -> PredictionBatchResult:
        scenes = list(batch.batch.keys())
        offs, boxes, custom = [0], [], []
        for s in scenes:
            for b, c in batch.batch[s]:
                boxes.append(b._row())
                custom.append(NONE_ID if c is None else c)
            offs.append(len(custom))
        custom = np.array(custom, dtype=np.int64)
        out = self._t.predict_batch(scenes, offs, np.array(boxes, dtype=np.float32).reshape(-1, 6), custom_ids=custom)
        items = []
        for i, s in enumerate(scenes):
            sl = slice(offs[i], offs[i + 1])
            items.append((s, _tracks_from({k: v[sl] for k, v in out.items()}, s, custom[sl])))
        return PredictionBatchResult(items)

    def idle_tracks(self, scene_id):
        return self._idle(scene_id)


class VisualSortOptions:
    """src/trackers/visual_sort/options.rs `PyVisualSortOptions` (defaults :194-205 + metric/builder.rs:26-42)."""

    def __init__(self):
        self._kw = dict(max_idle_epochs=2, history_length=10, visual_kind=_lib.VIS_EUCLIDEAN,
                        visual_threshold=float(np.finfo(np.float32).max), positional_kind=_lib.POS_IOU, iou_threshold=0.3,
                        visual_minimal_track_length=3, visual_minimal_area=0.0, visual_minimal_quality_use=0.0,
                        visual_minimal_quality_collect=0.0, visual_max_observations=5, visual_min_votes=1,
                        visual_minimal_own_area_percentage_use=0.0, visual_minimal_own_area_percentage_collect=0.0,
                        min_confidence=0.1, kalman_position_weight=1.0 / 20.0, kalman_velocity_weight=1.0 / 160.0)
        self._constraints = None

    def max_idle_epochs(self, n):
        self._kw["max_idle_epochs"] = int(n)

    def kept_history_length(self, n):
        assert n > 0, "History length must be a positive number"
        self._kw["history_length"] = int(n)

    def visual_min_votes(self, n):
        self._kw["visual_min_votes"] = int(n)

    def visual_metric(self, metric: VisualSortMetricType):
        self._kw["visual_kind"], self._kw["visual_threshold"] = metric.kind, metric.threshold

    def spatio_temporal_constraints(self, constraints: SpatioTemporalConstraints):
        self._constraints = constraints.constraints

    def positional_metric(self, metric: PositionalMetricType):
        self._kw["positional_kind"], self._kw["iou_threshold"] = metric.kind, metric.threshold

    def visual_minimal_track_length(self, length):
        assert length > 0
        self._kw["visual_minimal_track_length"] = int(length)

    def visual_minimal_area(self, area):
        assert area >= 0.0
        self._kw["visual_minimal_area"] = float(area)

    def visual_minimal_quality_use(self, q):
        self._kw["visual_minimal_quality_use"] = float(q)

    def positional_min_confidence(self, conf):
        self._kw["min_confidence"] = float(conf)

    def visual_max_observations(self, n):
        assert n > 0
        self._kw["visual_max_observations"] = int(n)

    def visual_minimal_quality_collect(self, q):
        self._kw["visual_minimal_quality_collect"] = float(q)

    def visual_minimal_own_area_percentage_use(self, area):
        assert 0.0 <= area <= 1.0
        self._kw["visual_minimal_own_area_percentage_use"] = float(area)

    def visual_minimal_own_area_percentage_collect(self, area):
        assert 0.0 <= area <= 1.0
        self._kw["visual_minimal_own_area_percentage_collect"] = float(area)

    def kalman_position_weight(self, weight):
        self._kw["kalman_position_weight"] = float(weight)

    def kalman_velocity_weight(self, weight):
        self._kw["kalman_velocity_weight"] = float(weight)

    def _build(self, kind, feature_dim):
        return default_options(kind=kind, feature_dim=feature_dim, constraints=self._constraints, **self._kw)


class VisualSortObservation:
    """src/trackers/visual_sort.rs `PyVisualSortObservation`."""

    def __init__(self, feature: Optional[List[float]], feature_quality: Optional[float], bounding_box: Universal2DBox,
                 custom_object_id: Optional[int]):
        self.feature = None if feature is None else np.asarray(feature, dtype=np.float32)
        self.feature_quality, self.bounding_box, self.custom_object_id = feature_quality, bounding_box, custom_object_id


class VisualSortObservationSet:
    """src/trackers/visual_sort.rs `PyVisualSortObservationSet`."""

    def __init__(self):
        self.inner: List[VisualSortObservation] = []

    def add(self, observation):
        self.inner.append(observation)


class VisualSortPredictionBatchRequest:
    """src/trackers/visual_sort/batch_api.rs `PyVisualSortPredictionBatchRequest`."""

    def __init__(self):
        self.batch = {}

    def add(self, scene_id, elt: VisualSortObservation):
        self.batch.setdefault(int(scene_id), []).append(elt)

    def prediction(self):
        return None


class _VisualBase(_TrackerBase):
    _dim_provisional = False

    def _ensure(self, kind, observations):
        dim = next((len(o.feature) for o in observations if o.feature is not None), 0)
        if self._t is None:
            if dim == 0:
                dim = 8  # no feature seen yet (feature is an Option in the reference): provisional until one arrives
                self._dim_provisional = True
            self._t = engine.Tracker(self._opts._build(kind, dim))
            self._t.set_feature_history(True)   # the reference always keeps it (kept_history_length is its memory knob)
            self._dim = dim
        elif self._dim_provisional and dim > 0:
            # first featured observation: the tracker keeps its tracks, ids, epochs and Kalman state, only the (still
            # empty) feature arena is re-created for the real feature length
            self._t.set_feature_dim(dim)
            self._dim = dim
            self._dim_provisional = False

    def _flatten(self, observations):
        n = len(observations)
        boxes = np.array([o.bounding_box._row() for o in observations], dtype=np.float32).reshape(-1, 6)
        has = np.zeros(n, dtype=np.uint8)
        if all(o.feature is None for o in observations):
            feats = None    # a frame without features: the request carries no feature column at all
            has = None
        else:
            if self._dim_provisional:
                self._dim_provisional = False
            feats = np.zeros((n, self._dim), dtype=np.float32)
            for i, o in enumerate(observations):
                if o.feature is not None:
                    if len(o.feature) != self._dim:
                        raise ValueError("all features of a tracker must have the same dimension")
                    feats[i], has[i] = o.feature, 1
        q = np.array([1.0 if o.feature_quality is None else o.feature_quality for o in observations], dtype=np.float32)
        custom = np.array([NONE_ID if o.custom_object_id is None else o.custom_object_id for o in observations], dtype=np.int64)
        return boxes, feats, has, q, custom

    def _kind(self):
        return _lib.KIND_BATCH_VISUAL_SORT if isinstance(self, BatchVisualSort) else _lib.KIND_VISUAL_SORT

    def save_state(self) -> np.ndarray:
        """See _TrackerBase.save_state; a tracker that has seen no observation yet saves an empty state."""
        if self._t is None:
            self._ensure(self._kind(), [])
        return self._t.save()

    def wasted(self) -> List[WastedVisualSortTrack]:
        if self._t is None:
            return []
        w = self._t.wasted_visual()
        return [WastedVisualSortTrack(w["ids"][i], w["epochs"][i], Universal2DBox._from_row(w["predicted"][i]),
                                      Universal2DBox._from_row(w["observed"][i]), w["scene_ids"][i], w["lengths"][i],
                                      [Universal2DBox._from_row(r) for r in w["predicted_history"][i]],
                                      [Universal2DBox._from_row(r) for r in w["observed_history"][i]],
                                      w["features"][i], w["feature_present"][i])
                for i in range(len(w["ids"]))]

    def wasted_to_store(self, store: engine.FeatureStore, id_offset=0,
                        feature_class=None) -> List[Tuple[WastedSortTrack, Optional[int]]]:
        """Collects the wasted tracks as wasted() does and associates each one's observed features (the present ones,
        oldest first) with the feature track `store` under the id track.id + id_offset, as one
        FeatureStore.associate call would (under the store's voting rule: with "best_fit" no two tracks of one
        collection merge into one stored track), without the features leaving the device (the TrackStore side of the
        reference's examples/track_merging.rs).  Returns [(track, where it went in the store)], the store track id
        being None for a track without a feature; the box histories are those wasted() reports.  feature_class: the
        store's class the features go to (None: its first declared class).  An extension with no PyO3 counterpart in the
        reference."""
        if self._t is None:
            return []
        w = store.associate_wasted(self._t, id_offset=id_offset, feature_class=feature_class)
        return [(WastedSortTrack(w["ids"][i], w["epochs"][i], Universal2DBox._from_row(w["predicted"][i]),
                                 Universal2DBox._from_row(w["observed"][i]), w["scene_ids"][i], w["lengths"][i],
                                 [Universal2DBox._from_row(r) for r in w["predicted_history"][i]],
                                 [Universal2DBox._from_row(r) for r in w["observed_history"][i]]),
                 int(w["track_ids"][i]) if w["queried"][i] else None)
                for i in range(len(w["ids"]))]

    def search_store(self, store: engine.FeatureStore, tracks: List[SortTrack], id_offset=0, sources=None, t_start=None,
                     t_end=None, feature_class=None) -> List[Tuple[SortTrack, Optional[List[Tuple[int, float]]]]]:
        """Re-identification: looks the live `tracks` (the SortTracks a predict returned, by scene_id and id) up in the
        feature track `store` with one FeatureStore.search_tracks call, their observed features read where the tracker
        keeps them.  Returns [(track, [(store track id, weight), ...])], the list being None for a track that is no
        longer live or holds no feature.  A gated store takes sources / t_start / t_end, one per track.  An extension
        with no PyO3 counterpart in the reference."""
        tracks = list(tracks)
        if self._t is None:
            return [(tr, None) for tr in tracks]
        r = store.search_tracks(self._t, [tr.scene_id for tr in tracks], [tr.id for tr in tracks], id_offset=id_offset,
                                sources=sources, t_start=t_start, t_end=t_end, feature_class=feature_class)
        return [(tr, [(int(r["winners"][i, e]), float(r["weights"][i, e])) for e in range(int(r["counts"][i]))]
                 if r["queried"][i] else None)
                for i, tr in enumerate(tracks)]


class VisualSort(_VisualBase):
    """src/trackers/visual_sort/simple_api.rs `PyVisualSort`."""

    def __init__(self, shards: int, opts: VisualSortOptions):
        self._opts, self._t = opts, None

    def predict(self, observation_set: VisualSortObservationSet):
        return self.predict_with_scene(0, observation_set)

    def predict_with_scene(self, scene_id, observation_set: VisualSortObservationSet):
        obs = observation_set.inner
        self._ensure(_lib.KIND_VISUAL_SORT, obs)
        boxes, feats, has, q, custom = self._flatten(obs)
        out = self._t.predict_batch([scene_id], [0, len(obs)], boxes, features=feats, has_feature=has, quality=q,
                                    custom_ids=custom)
        return _tracks_from(out, scene_id, custom)

    def idle_tracks(self):
        return self._idle(0)

    def idle_tracks_with_scene(self, scene_id):
        return self._idle(scene_id)


class BatchVisualSort(_SceneTransfer, _VisualBase):
    """src/trackers/visual_sort/batch_api.rs `PyBatchVisualSort`."""

    def __init__(self, distance_shards: int, voting_shards: int, opts: VisualSortOptions):
        self._opts, self._t = opts, None

    def predict(self, py_batch: VisualSortPredictionBatchRequest) -> PredictionBatchResult:
        scenes = list(py_batch.batch.keys())
        allobs = [o for s in scenes for o in py_batch.batch[s]]
        self._ensure(_lib.KIND_BATCH_VISUAL_SORT, allobs)
        offs = [0]
        for s in scenes:
            offs.append(offs[-1] + len(py_batch.batch[s]))
        boxes, feats, has, q, custom = self._flatten(allobs)
        out = self._t.predict_batch(scenes, offs, boxes, features=feats, has_feature=has, quality=q, custom_ids=custom)
        items = []
        for i, s in enumerate(scenes):
            sl = slice(offs[i], offs[i + 1])
            items.append((s, _tracks_from({k: v[sl] for k, v in out.items()}, s, custom[sl])))
        return PredictionBatchResult(items)

    def idle_tracks(self, scene_id):
        return self._idle(scene_id)

    def export_scenes(self, scene_ids, remove=False) -> np.ndarray:
        if self._t is None:
            self._ensure(self._kind(), [])
        return _SceneTransfer.export_scenes(self, scene_ids, remove)

    def import_scenes(self, blob):
        if self._t is None:
            # the engine tracker is created with the blob's feature length (the options must match anyway)
            dim = int(engine.blob_options(blob).feature_dim)
            self._t = engine.Tracker(self._opts._build(self._kind(), dim))
            self._t.set_feature_history(True)
            self._dim = dim
        self._t.import_scenes(blob)
        # the source's dimension may still have been provisional (no feature seen): then so is this one
        self._dim_provisional = not self._t.feature_dim_fixed()


def load_state(blob, device=0):
    """A Sort / BatchSort / VisualSort / BatchVisualSort restored from a save_state() blob on `device`, options
    included; it continues exactly where the saved tracker stood.  An extension with no PyO3 counterpart in the
    reference."""
    t = engine.Tracker.load(blob, device=device)
    o = t.opts
    cls = {_lib.KIND_SORT: Sort, _lib.KIND_BATCH_SORT: BatchSort, _lib.KIND_VISUAL_SORT: VisualSort,
           _lib.KIND_BATCH_VISUAL_SORT: BatchVisualSort}[int(o.kind)]
    obj = cls.__new__(cls)
    obj._t = t
    if cls in (VisualSort, BatchVisualSort):
        opts = VisualSortOptions()
        for k in opts._kw:
            opts._kw[k] = getattr(o, k)
        n = int(o.n_constraints)
        opts._constraints = [(int(o.constraint_epochs[i]), float(o.constraint_max_dist[i])) for i in range(n)] or None
        obj._opts, obj._dim = opts, int(o.feature_dim)
        obj._dim_provisional = not t.feature_dim_fixed()
    return obj


def nms(detections, nms_threshold, score_threshold):
    """src/utils/nms/nms_py.rs `nms(detections, nms_threshold, score_threshold)` -> kept boxes in rank order."""
    boxes = np.array([b._row() for b, _ in detections], dtype=np.float32).reshape(-1, 6)
    scores = np.array([math.nan if s is None else s for _, s in detections], dtype=np.float32)
    idx = engine.nms_indices(boxes, scores, nms_threshold, score_threshold)
    return [detections[i][0] for i in idx]


def nms_batch(detections_by_scene, nms_threshold, score_threshold):
    """`nms` of every scene in one GPU call: {scene_id: [(Universal2DBox, score or None), ...]} -> {scene_id: kept boxes
    in rank order}.  An extension with no PyO3 counterpart in the reference; for each scene the result equals
    nms(detections_by_scene[scene_id], nms_threshold, score_threshold)."""
    scenes = list(detections_by_scene.keys())
    dets = [d for s in scenes for d in detections_by_scene[s]]
    offsets = np.cumsum([0] + [len(detections_by_scene[s]) for s in scenes])
    boxes = np.array([b._row() for b, _ in dets], dtype=np.float32).reshape(-1, 6)
    scores = np.array([math.nan if s is None else s for _, s in dets], dtype=np.float32)
    kept = engine.nms_batch(boxes, scores, offsets, nms_threshold, score_threshold)
    return {s: [detections_by_scene[s][i][0] for i in k] for s, k in zip(scenes, kept)}


class Polygon:
    """src/utils/clipping/clipping_py.rs:5-27 `PyPolygon` (a geo::Polygon<f64> without interiors)."""

    def __init__(self, points):
        self._points = [(float(x), float(y)) for x, y in points]

    @staticmethod
    def _from_ring(xy) -> "Polygon":
        # geo::Polygon::new closes the exterior ring: the first coordinate is repeated unless the last already equals it
        pts = [(float(x), float(y)) for x, y in xy]
        if pts and pts[0] != pts[-1]:
            pts.append(pts[0])
        return Polygon(pts)

    def get_points(self) -> List[Tuple[float, float]]:
        return list(self._points)

    def __repr__(self):
        coords = ", ".join(f"Coord {{ x: {x!r}, y: {y!r} }}" for x, y in self._points)
        return f"PyPolygon(Polygon {{ exterior: LineString([{coords}]), interiors: [] }})"


def _clip_one(subject: Universal2DBox, clipping: Universal2DBox):
    v, n, a = engine.clip_polygons(np.array([subject._row()], dtype=np.float32),
                                   np.array([clipping._row()], dtype=np.float32))
    return v[0, : n[0]], float(a[0])


def sutherland_hodgman_clip(subject: Universal2DBox, clipping: Universal2DBox) -> Polygon:
    """src/utils/clipping/clipping_py.rs:29-39 (Universal2DBox::sutherland_hodgman_clip, src/utils/bbox.rs:216-238: a
    None angle is 0)."""
    return Polygon._from_ring(_clip_one(subject, clipping)[0])


def intersection_area(subject: Universal2DBox, clipping: Universal2DBox) -> float:
    """src/utils/clipping/clipping_py.rs:41-46: unsigned area of sutherland_hodgman_clip(subject, clipping)."""
    return _clip_one(subject, clipping)[1]


def intersection_areas(subjects, clippings) -> np.ndarray:
    """intersection_area of every (subjects[i], clippings[j]) pair in one GPU call: an [m][n] float64 matrix.  An
    extension with no PyO3 counterpart in the reference; element (i, j) equals intersection_area(subjects[i],
    clippings[j])."""
    a = np.array([b._row() for b in subjects], dtype=np.float32).reshape(-1, 6)
    b = np.array([c._row() for c in clippings], dtype=np.float32).reshape(-1, 6)
    return engine.intersection_areas(a, b)


# CHI2INV95 and CHI2_UPPER_BOUND, src/utils/kalman.rs:16-20
_CHI2INV95 = np.array([3.8415, 5.9915, 7.8147, 9.4877, 11.070, 12.592, 14.067, 15.507, 16.919], dtype=np.float32)
_CHI2_UPPER = F32(100.0)


def _cost(distance, inverted, plain_index):
    """calculate_cost of the Kalman filters in f32: the non-inverted branch compares with CHI2INV95[plain_index] (4 for
    the box filter, kalman_2d_box.rs:172-184; 1 for the point filter, kalman_2d_point.rs:139-151), the inverted one
    with CHI2INV95[4] in both."""
    d = F32(distance)
    if not inverted:
        return float(_CHI2_UPPER if d > _CHI2INV95[plain_index] else d)
    return float(F32(0.0) if d > _CHI2INV95[4] else _CHI2_UPPER - d)


class Universal2DBoxKalmanFilterState:
    """src/utils/kalman/kalman_2d_box.rs:267-284 `PyUniversal2DBoxKalmanFilterState`.  Holds the packed 30-float state
    (mean[10], then five 2x2 covariance blocks; DESIGN.md)."""

    __slots__ = ("_st",)

    def __init__(self, st):
        self._st = st

    def universal_bbox(self) -> Universal2DBox:
        # TryFrom<KalmanState> for Universal2DBox, src/utils/kalman.rs:72-92: angle None when mean[2] == 0, confidence 1
        m = self._st
        return Universal2DBox(m[0], m[1], None if m[2] == 0.0 else m[2], m[3], m[4])

    def bbox(self) -> BoundingBox:
        return self.universal_bbox().as_ltwh()


class Universal2DBoxKalmanFilter:
    """src/utils/kalman/kalman_2d_box.rs:260-265,286-338 `PyUniversal2DBoxKalmanFilter`.  Each call is one GPU call over one
    state; for many states use engine.kalman_* on packed arrays."""

    def __init__(self, position_weight=0.05, velocity_weight=0.00625):
        self._pw, self._vw = float(F32(position_weight)), float(F32(velocity_weight))

    def initiate(self, bbox: Universal2DBox) -> Universal2DBoxKalmanFilterState:
        return Universal2DBoxKalmanFilterState(engine.kalman_initiate([bbox._row()], self._pw, self._vw)[0])

    def predict(self, state: Universal2DBoxKalmanFilterState) -> Universal2DBoxKalmanFilterState:
        return Universal2DBoxKalmanFilterState(engine.kalman_predict(state._st, self._pw, self._vw)[0])

    def update(self, state: Universal2DBoxKalmanFilterState, bbox: Universal2DBox) -> Universal2DBoxKalmanFilterState:
        return Universal2DBoxKalmanFilterState(engine.kalman_update(state._st, [bbox._row()], self._pw, self._vw)[0])

    def distance(self, state: Universal2DBoxKalmanFilterState, bbox: Universal2DBox) -> float:
        return float(engine.kalman_distance(state._st, [bbox._row()], self._pw, self._vw)[0])

    @staticmethod
    def calculate_cost(distance, inverted) -> float:
        return _cost(distance, inverted, 4)


class Point2DKalmanFilterState:
    """src/utils/kalman/kalman_2d_point.rs:237-264 `PyPoint2DKalmanFilterState`.  Holds the packed 12-float state
    (x, y, vx, vy, then the x and y covariance blocks; DESIGN.md)."""

    __slots__ = ("_st",)

    def __init__(self, st):
        self._st = st

    def x(self) -> float:
        return float(self._st[0])

    def y(self) -> float:
        return float(self._st[1])


class Point2DKalmanFilter:
    """src/utils/kalman/kalman_2d_point.rs:230-234,266-312 `PyPoint2DKalmanFilter`.  Each call is one GPU call over one state."""

    def __init__(self, position_weight=0.05, velocity_weight=0.00625):
        self._pw, self._vw = float(F32(position_weight)), float(F32(velocity_weight))

    def initiate(self, x, y) -> Point2DKalmanFilterState:
        return Point2DKalmanFilterState(engine.point_kalman_initiate([[x, y]], self._pw, self._vw)[0])

    def predict(self, state: Point2DKalmanFilterState) -> Point2DKalmanFilterState:
        return Point2DKalmanFilterState(engine.point_kalman_predict(state._st, self._pw, self._vw)[0])

    def update(self, state: Point2DKalmanFilterState, x, y) -> Point2DKalmanFilterState:
        return Point2DKalmanFilterState(engine.point_kalman_update(state._st, [[x, y]], self._pw, self._vw)[0])

    def distance(self, state: Point2DKalmanFilterState, x, y) -> float:
        return float(engine.point_kalman_distance(state._st, [[x, y]], self._pw, self._vw)[0])

    @staticmethod
    def calculate_cost(distance, inverted) -> float:
        return _cost(distance, inverted, 1)


class Point2DKalmanFilterStates(Sequence):
    """What Vec2DKalmanFilter.initiate / predict / update return: a read-only sequence of Point2DKalmanFilterState over
    one packed [n][12] array.  The reference returns a list; indexing, len() and iteration behave the same, and passing
    the sequence back to Vec2DKalmanFilter hands the packed array to the GPU without touching the elements."""

    __slots__ = ("_a",)

    def __init__(self, a):
        self._a = a

    def __len__(self):
        return len(self._a)

    def __getitem__(self, i):
        if isinstance(i, slice):
            return Point2DKalmanFilterStates(self._a[i])
        return Point2DKalmanFilterState(self._a[i])


def _pack_points(states) -> np.ndarray:
    if isinstance(states, Point2DKalmanFilterStates):
        return states._a
    return np.array([s._st for s in states], dtype=np.float32).reshape(-1, 12)


def _xy(points) -> np.ndarray:
    return np.array(points, dtype=np.float32).reshape(-1, 2)


class Vec2DKalmanFilter:
    """src/utils/kalman/kalman_2d_point_vec.rs:86-166 `PyVec2DKalmanFilter`: every call is one GPU launch over the whole
    list of states."""

    def __init__(self, position_weight=0.05, velocity_weight=0.00625):
        self._pw, self._vw = float(F32(position_weight)), float(F32(velocity_weight))

    def initiate(self, points) -> Point2DKalmanFilterStates:
        return Point2DKalmanFilterStates(engine.point_kalman_initiate(_xy(points), self._pw, self._vw))

    def predict(self, state) -> Point2DKalmanFilterStates:
        return Point2DKalmanFilterStates(engine.point_kalman_predict(_pack_points(state), self._pw, self._vw))

    def update(self, state, points) -> Point2DKalmanFilterStates:
        assert len(state) == len(points), "Lengths of state and points must match"
        return Point2DKalmanFilterStates(engine.point_kalman_update(_pack_points(state), _xy(points), self._pw, self._vw))

    def distance(self, state, points) -> List[float]:
        assert len(state) == len(points), "Lengths of state and points must match"
        return engine.point_kalman_distance(_pack_points(state), _xy(points), self._pw, self._vw).tolist()

    @staticmethod
    def calculate_cost(distances, inverted) -> List[float]:
        return [_cost(d, inverted, 1) for d in distances]


def version():
    return "0.26.12-b200"
