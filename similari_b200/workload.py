"""Seeded synthetic workloads for the BASELINE.json configs (SURVEY.md section 8d), shared by tests and bench.py.

Every scene holds `n_objects` ground-truth objects on a canvas; each frame every object random-walks a little,
~5 % of the objects are missed by the "detector" and ~5 % are replaced by fresh identities, and the surviving
detections are emitted in random order -- so the match / new-track / idle branches of the trackers all fire.
ReID features are unit vectors around a per-identity centroid.
"""
from __future__ import annotations

import dataclasses

import numpy as np


@dataclasses.dataclass
class WorkloadConfig:
    name: str
    n_scenes: int
    n_objects: int
    oriented: bool
    feature_dim: int = 0
    canvas: tuple = (1920.0, 1080.0)
    drop_frac: float = 0.05
    fresh_frac: float = 0.05
    pos_jitter: float = 2.0
    size_jitter: float = 0.02
    angle_jitter: float = 0.02
    feat_noise: float = 0.02
    seed: int = 0x5EED0000


# BASELINE.json configs (index == position in `configs`)
CONFIGS = {
    "cfg1": WorkloadConfig("Sort IoU 1x100x100", 1, 100, False, seed=0x5EED0001),
    "cfg2": WorkloadConfig("BatchSort IoU 64 scenes x 256x256", 64, 256, False, seed=0x5EED0002),
    "cfg3": WorkloadConfig("VisualSort cosine 1 scene 1024x1024 D=512", 1, 1024, False, 512, (3840.0, 2160.0), seed=0x5EED0003),
    "cfg4": WorkloadConfig("BatchSort Mahalanobis oriented 128 scenes x 512x512", 128, 512, True, 0, (3840.0, 2160.0), seed=0x5EED0004),
    "cfg5": WorkloadConfig("BatchVisualSort 256 scenes x 512x512 D=512", 256, 512, True, 512, (3840.0, 2160.0), seed=0x5EED0005),
}


class Workload:
    """Frame generator.  `next_frame()` returns the flat request of sb200_predict_batch."""

    def __init__(self, cfg: WorkloadConfig, scene_base: int = 0):
        self.cfg = cfg
        self.rng = np.random.default_rng(cfg.seed)
        S, N = cfg.n_scenes, cfg.n_objects
        W, H = cfg.canvas
        r = self.rng
        self.scene_ids = np.arange(scene_base, scene_base + S, dtype=np.uint64)
        self.xc = r.uniform(0, W, (S, N)).astype(np.float32)
        self.yc = r.uniform(0, H, (S, N)).astype(np.float32)
        self.h = r.uniform(40, 160, (S, N)).astype(np.float32)
        self.a = r.uniform(0.3, 0.8, (S, N)).astype(np.float32)
        self.ang = r.uniform(-np.pi / 2, np.pi / 2, (S, N)).astype(np.float32)
        self.conf = r.uniform(0.3, 1.0, (S, N)).astype(np.float32)
        if cfg.feature_dim:
            self.cent = self._unit(r.standard_normal((S, N, cfg.feature_dim), dtype=np.float32))
        self.frame_no = 0

    @staticmethod
    def _unit(v):
        return v / np.linalg.norm(v, axis=-1, keepdims=True)

    def _refresh(self, mask):
        """Replaces the masked objects by fresh identities."""
        cfg, r = self.cfg, self.rng
        k = int(mask.sum())
        if k == 0:
            return
        W, H = cfg.canvas
        self.xc[mask] = r.uniform(0, W, k).astype(np.float32)
        self.yc[mask] = r.uniform(0, H, k).astype(np.float32)
        self.h[mask] = r.uniform(40, 160, k).astype(np.float32)
        self.a[mask] = r.uniform(0.3, 0.8, k).astype(np.float32)
        self.ang[mask] = r.uniform(-np.pi / 2, np.pi / 2, k).astype(np.float32)
        self.conf[mask] = r.uniform(0.3, 1.0, k).astype(np.float32)
        if cfg.feature_dim:
            self.cent[mask] = self._unit(r.standard_normal((k, cfg.feature_dim), dtype=np.float32))

    def next_frame(self):
        cfg, r = self.cfg, self.rng
        S, N = cfg.n_scenes, cfg.n_objects
        if self.frame_no > 0:
            self.xc += r.normal(0, cfg.pos_jitter, (S, N)).astype(np.float32)
            self.yc += r.normal(0, cfg.pos_jitter, (S, N)).astype(np.float32)
            self.h *= r.uniform(1 - cfg.size_jitter, 1 + cfg.size_jitter, (S, N)).astype(np.float32)
            self.a *= r.uniform(1 - cfg.size_jitter, 1 + cfg.size_jitter, (S, N)).astype(np.float32)
            if cfg.oriented:
                self.ang += r.normal(0, cfg.angle_jitter, (S, N)).astype(np.float32)
            self._refresh(r.random((S, N)) < cfg.fresh_frac)
        keep = r.random((S, N)) >= (cfg.drop_frac if self.frame_no > 0 else 0.0)
        boxes_l, feats_l, offs = [], [], [0]
        for s in range(S):
            idx = np.flatnonzero(keep[s])
            r.shuffle(idx)
            b = np.empty((len(idx), 6), np.float32)
            b[:, 0] = self.xc[s, idx]
            b[:, 1] = self.yc[s, idx]
            b[:, 2] = self.ang[s, idx] if cfg.oriented else np.nan
            b[:, 3] = self.a[s, idx]
            b[:, 4] = self.h[s, idx]
            b[:, 5] = self.conf[s, idx]
            boxes_l.append(b)
            if cfg.feature_dim:
                f = self.cent[s, idx] + cfg.feat_noise * r.standard_normal((len(idx), cfg.feature_dim), dtype=np.float32)
                feats_l.append(self._unit(f).astype(np.float32))
            offs.append(offs[-1] + len(idx))
        self.frame_no += 1
        frame = {
            "scene_ids": self.scene_ids.copy(),
            "det_offsets": np.asarray(offs, dtype=np.int32),
            "boxes": np.concatenate(boxes_l, axis=0) if boxes_l else np.zeros((0, 6), np.float32),
            "features": np.concatenate(feats_l, axis=0) if cfg.feature_dim else None,
        }
        return frame

    def pair_associations(self, frame, n_tracks_per_scene):
        """sum over scenes of N_s * M_s (the BASELINE metric's unit of work)."""
        m = np.diff(frame["det_offsets"]).astype(np.int64)
        return int((m * np.asarray(n_tracks_per_scene, dtype=np.int64)).sum())


def tracker_options_for(name: str, make_options, **over):
    """Tracker options matching the BASELINE configs (SURVEY.md section 8d).  `make_options` is either
    similari_b200._lib.default_options or oracle.make_options (same field names)."""
    from ._lib import (KIND_BATCH_SORT, KIND_BATCH_VISUAL_SORT, KIND_SORT, KIND_VISUAL_SORT, POS_IOU, POS_MAHA,
                       VIS_COSINE, VIS_EUCLIDEAN)

    if name == "cfg1":
        kw = dict(kind=KIND_SORT, positional_kind=POS_IOU, iou_threshold=0.3, max_idle_epochs=1, history_length=10,
                  constraints=[(1, 1.0)])
    elif name == "cfg2":
        kw = dict(kind=KIND_BATCH_SORT, positional_kind=POS_IOU, iou_threshold=0.3, max_idle_epochs=5)
    elif name == "cfg3":
        kw = dict(kind=KIND_VISUAL_SORT, positional_kind=POS_IOU, iou_threshold=0.3, max_idle_epochs=5,
                  visual_kind=VIS_COSINE, visual_threshold=0.2, feature_dim=512, visual_max_observations=3,
                  visual_min_votes=2, visual_minimal_track_length=1, min_confidence=0.1)
    elif name == "cfg4":
        kw = dict(kind=KIND_BATCH_SORT, positional_kind=POS_MAHA, max_idle_epochs=5)
    elif name == "cfg5":
        kw = dict(kind=KIND_BATCH_VISUAL_SORT, positional_kind=POS_IOU, iou_threshold=0.3, max_idle_epochs=5,
                  visual_kind=VIS_EUCLIDEAN, visual_threshold=0.7, feature_dim=512, visual_max_observations=3,
                  visual_min_votes=2, visual_minimal_track_length=1, min_confidence=0.1)
    else:
        raise KeyError(name)
    kw.update(over)
    return make_options(**kw)


class FeatGen:
    """Seeded counterpart of the reference's FeatGen (src/examples.rs:266-293), which benches/feature_tracker.rs feeds
    its store with: every call returns a `dim`-long row x + U(-drift, drift), f32."""

    def __init__(self, x: float, dim: int, drift: float, seed: int):
        self.x, self.dim, self.drift = np.float32(x), int(dim), float(drift)
        self.rng = np.random.default_rng(seed)

    def next(self) -> np.ndarray:
        u = self.rng.uniform(-self.drift, self.drift, self.dim).astype(np.float32)
        return self.x + u
