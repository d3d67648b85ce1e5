"""BASELINE.json configs at (or near) their full per-scene sizes: GPU engine vs the oracle, plus size-independent
properties where the oracle would take too long."""
import dataclasses

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    import similari_b200.engine as e
    from similari_b200._lib import lib

    if lib().sb200_device_count() <= 0:
        pytest.fail("no CUDA device: the gpu-marked tests must run on an H100")
    return e


def _threads():
    import os

    try:
        return max(4, min(24, len(os.sched_getaffinity(0))))
    except Exception:
        return 16


def _run(eng, oracle, name, n_scenes, frames, threads=None, opts_over=None, **cfg_over):
    from similari_b200._lib import default_options
    from similari_b200.workload import CONFIGS, Workload, tracker_options_for

    cfg = dataclasses.replace(CONFIGS[name], n_scenes=n_scenes, **cfg_over)
    g = eng.Tracker(tracker_options_for(name, default_options, **(opts_over or {})))
    o = oracle.Tracker(tracker_options_for(name, oracle.make_options, **(opts_over or {})), threads=threads or _threads())
    wl = Workload(cfg)
    for fr in range(frames):
        f = wl.next_frame()
        rg = g.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=f["features"])
        ro = o.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=f["features"])
        for key in ("ids", "epochs", "lengths", "voting_types"):
            assert np.array_equal(rg[key], ro[key]), (name, fr, key, int((rg[key] != ro[key]).sum()))
    return g, o


def test_cfg1_sort_iou_100x100_sparse_bench_workload(eng, oracle):
    """benches/simple_sort_iou_tracker.rs: 100 objects 1000 px apart, constraints (1, 1.0), Sort IoU(0.3)."""
    from similari_b200._lib import default_options
    from similari_b200.workload import tracker_options_for

    g = eng.Tracker(tracker_options_for("cfg1", default_options))
    o = oracle.Tracker(tracker_options_for("cfg1", oracle.make_options))
    rng = np.random.default_rng(1)
    x = 1000.0 * np.arange(100, dtype=np.float32)
    y = x.copy()
    w = np.full(100, 50.0, np.float32)
    h = np.full(100, 50.0, np.float32)
    for it in range(12):
        x += rng.uniform(-1, 1, 100).astype(np.float32)
        y += rng.uniform(-1, 1, 100).astype(np.float32)
        w = np.maximum(w + rng.uniform(-0.001, 0.001, 100).astype(np.float32), 1.0)
        h = np.maximum(h + rng.uniform(-0.001, 0.001, 100).astype(np.float32), 1.0)
        boxes = np.stack([x + w / 2, y + h / 2, np.full(100, np.nan, np.float32), w / h, h, np.ones(100, np.float32)], 1)
        rg = g.predict_batch([0], [0, 100], boxes)
        ro = o.predict_batch([0], [0, 100], boxes)
        assert np.array_equal(rg["ids"], ro["ids"]) and np.array_equal(rg["lengths"], ro["lengths"])
    assert g.active_tracks() == 100 and np.all(rg["lengths"] == 12)      # the bench's own assertions
    g.skip_epochs(2)
    assert len(g.wasted()["ids"]) == 100


def test_cfg2_batchsort_iou_64x256x256_matches_oracle(eng, oracle):
    _run(eng, oracle, "cfg2", 64, 5)


def test_cfg3_visualsort_cosine_1024x1024x512_matches_oracle(eng, oracle):
    _run(eng, oracle, "cfg3", 1, 4)


def test_cfg4_batchsort_maha_oriented_512x512_matches_oracle(eng, oracle):
    _run(eng, oracle, "cfg4", 16, 5)


def test_cfg5_batchvisualsort_512x512x512_matches_oracle(eng, oracle):
    _run(eng, oracle, "cfg5", 8, 5)


def test_cfg4_full_128_scenes_matches_oracle(eng, oracle):
    """BASELINE cfg4 at its full size -- 128 scenes x 512 x 512, oriented boxes, Mahalanobis -- against the oracle, frame
    by frame (the request the bench times: its own list-base / offset arithmetic included)."""
    _run(eng, oracle, "cfg4", 128, 5)


def test_cfg5_full_256_scenes_matches_oracle(eng, oracle):
    """BASELINE cfg5 at its full size -- 256 scenes x 512 x 512 x 512-d -- against the oracle for five frames: every id,
    epoch, length and voting type of ~124 k detections per frame.  This is the exact batch bench.py times (tile list,
    column offsets and list bases of 256 scenes)."""
    g, o = _run(eng, oracle, "cfg5", 256, 5)
    assert g.active_tracks() == o.active_tracks()


def test_cfg5_scene_with_degenerate_features_overflows_its_list_mid_batch(eng, oracle):
    """List overflow at BASELINE size: in one scene of the batch every feature is (almost) the same vector, so every
    (candidate, observation) pair passes the threshold -- ~512 x 1500 survivors against a list of 16 k -- and that scene
    alone falls back to the dense exact kernels on the device while the others stay on the sparse path.  Assignments must
    be the oracle's for every scene."""
    from similari_b200._lib import default_options
    from similari_b200.workload import CONFIGS, Workload, tracker_options_for

    cfg = dataclasses.replace(CONFIGS["cfg5"], n_scenes=6)
    g = eng.Tracker(tracker_options_for("cfg5", default_options))
    o = oracle.Tracker(tracker_options_for("cfg5", oracle.make_options), threads=_threads())
    wl = Workload(cfg)
    rng = np.random.default_rng(77)
    common = rng.standard_normal(512).astype(np.float32)
    common /= np.linalg.norm(common)
    for fr in range(5):
        f = wl.next_frame()
        offs = f["det_offsets"]
        feats = f["features"].copy()
        # scene 2: one shared vector plus a little noise (distances ~0.05 << 0.7)
        n2 = offs[3] - offs[2]
        v = common[None, :] + 0.002 * rng.standard_normal((n2, 512)).astype(np.float32)
        feats[offs[2]:offs[3]] = v / np.linalg.norm(v, axis=1, keepdims=True)
        rg = g.predict_batch(f["scene_ids"], offs, f["boxes"], features=feats)
        ro = o.predict_batch(f["scene_ids"], offs, f["boxes"], features=feats)
        for key in ("ids", "epochs", "lengths", "voting_types"):
            assert np.array_equal(rg[key], ro[key]), (fr, key, int((rg[key] != ro[key]).sum()))


@pytest.mark.parametrize("gate", ["quality", "area", "has_feature", "own_area"])
def test_visual_gates_on_the_tensor_core_path_at_baseline_size(eng, oracle, gate, monkeypatch):
    """The gates of VisualMetric::metric (src/trackers/visual_sort/metric.rs:227-249, 280-290) -- candidate quality,
    minimal box area, feature present, own-area share -- at 512 x 512 x 512-d with the tensor-core path forced: candidates the
    gate rejects must not vote visually (row mask of the screen), tracks below the minimal feature count must not be
    scored (column mask), and rejected features must not be collected."""
    from similari_b200._lib import default_options
    from similari_b200.workload import CONFIGS, Workload, tracker_options_for

    monkeypatch.setenv("SB200_VIS_KERNEL", "tc")
    over = {}
    if gate == "quality":
        over = dict(visual_minimal_quality_use=0.5, visual_minimal_quality_collect=0.7)
    elif gate == "area":
        over = dict(visual_minimal_area=5000.0)
    elif gate == "own_area":
        over = dict(visual_minimal_own_area_percentage_use=0.6, visual_minimal_own_area_percentage_collect=0.8)
    over["visual_minimal_track_length"] = 2
    cfg = dataclasses.replace(CONFIGS["cfg5"], n_scenes=3, canvas=(2600.0, 1500.0) if gate == "own_area" else (3840.0, 2160.0))
    g = eng.Tracker(tracker_options_for("cfg5", default_options, **over))
    o = oracle.Tracker(tracker_options_for("cfg5", oracle.make_options, **over), threads=_threads())
    wl = Workload(cfg)
    rng = np.random.default_rng(9)
    vis_votes = 0
    for fr in range(6):
        f = wl.next_frame()
        total = len(f["boxes"])
        quality = rng.uniform(0.2, 1.0, total).astype(np.float32) if gate == "quality" else None
        hasf = (rng.random(total) > 0.3).astype(np.uint8) if gate == "has_feature" else None
        kw = dict(features=f["features"], quality=quality, has_feature=hasf)
        rg = g.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], **kw)
        ro = o.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], **kw)
        for key in ("ids", "epochs", "lengths", "voting_types"):
            assert np.array_equal(rg[key], ro[key]), (gate, fr, key, int((rg[key] != ro[key]).sum()))
        vis_votes += int((ro["voting_types"] == 0).sum())
        for sid in f["scene_ids"]:
            assert np.array_equal(g.scene_tracks(int(sid))["feat_counts"], o.scene_tracks(int(sid))["feat_counts"]), (gate, fr)
    assert vis_votes > 100     # the visual path did decide candidates; the gate did not switch it off altogether
    n_pos = int((ro["voting_types"] == 1).sum())
    assert n_pos > 20          # and the gate did send candidates to the positional stage


def test_cfg5_full_size_properties(eng):
    """256 scenes x 512 x 512 x 512-d: properties that do not need the oracle."""
    from similari_b200._lib import default_options
    from similari_b200.workload import CONFIGS, Workload, tracker_options_for

    cfg = CONFIGS["cfg5"]
    t = eng.Tracker(tracker_options_for("cfg5", default_options, max_scenes_hint=cfg.n_scenes,
                                        max_tracks_per_scene_hint=1200, max_dets_per_scene_hint=cfg.n_objects))
    wl = Workload(cfg)
    prev = None
    seen = np.empty(0, np.uint64)
    for fr in range(4):
        f = wl.next_frame()
        r = t.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=f["features"],
                            want=("ids", "epochs", "lengths", "voting_types"))
        offs = f["det_offsets"]
        assert np.all(r["epochs"] == fr + 1)
        # a track id is handed out at most once per frame (python/bugfixes/bug_vs_1: "ids unique per frame")
        assert len(np.unique(r["ids"])) == len(r["ids"])
        if prev is not None:
            cont = np.isin(r["ids"], prev)
            assert cont.mean() > 0.85                       # ~90 % of the detections continue a track
            assert np.all(r["lengths"][~np.isin(r["ids"], seen)] == 1)   # never-seen ids start at length 1
            if fr >= 2:
                assert (r["voting_types"][cont] == 0).mean() > 0.9   # with >= 2 stored features the match is Visual
        prev = r["ids"].copy()
        seen = np.union1d(seen, prev)
    assert t.active_tracks() == sum(int(x) for x in t.scene_track_counts(f["scene_ids"]))


def test_nms_10k_oriented_boxes_matches_oracle(eng, oracle):
    """cfg5's NMS part: 2000 clusters x 5 near-duplicates on 3840 x 2160, threshold 0.8."""
    rng = np.random.default_rng(5)
    base = np.empty((2000, 6), np.float32)
    base[:, 0] = rng.uniform(0, 3840, 2000)
    base[:, 1] = rng.uniform(0, 2160, 2000)
    base[:, 2] = rng.uniform(-1.5, 1.5, 2000)
    base[:, 3] = rng.uniform(0.3, 0.8, 2000)
    base[:, 4] = rng.uniform(40, 160, 2000)
    base[:, 5] = 1.0
    boxes = np.repeat(base, 5, axis=0)
    boxes[:, :2] += rng.normal(0, 3, (10000, 2)).astype(np.float32)
    boxes[:, 2] += rng.normal(0, 0.03, 10000).astype(np.float32)
    scores = rng.uniform(0, 1, 10000).astype(np.float32)
    ref = oracle.nms(boxes, scores, 0.8)
    got = eng.nms_indices(boxes, scores, 0.8)
    assert list(ref) == list(got) and 2000 <= len(got) < 10000


def test_cfg5_default_visual_metric_dense_path_matches_oracle(eng, oracle):
    """BASELINE cfg5 with the reference's DEFAULT visual metric, Euclidean(f32::MAX)
    (src/trackers/visual_sort/metric/builder.rs:26-42): every distance is an entry, BestFit decides every candidate that
    carries a feature.  32 scenes x 512 x 512 x 512-d on the dense tensor-core path against the oracle."""
    g, o = _run(eng, oracle, "cfg5", 32, 5, opts_over=dict(visual_threshold=float(np.finfo(np.float32).max)))
    wc = g.work_counters()
    assert wc["tc_frames"] >= 3 and wc["dense_fallback_scenes"] == 0


def test_cfg5_published_bench_metric_euclidean_10_matches_oracle(eng, oracle):
    """The published VisualSORT bench's metric, Euclidean(10.0) on unit vectors (benches/simple_visual_sort_tracker.rs:111),
    at cfg5's per-scene size: screen first (lists overflow), then the dense path."""
    g, o = _run(eng, oracle, "cfg5", 8, 7, opts_over=dict(visual_threshold=10.0))
    assert g.work_counters()["tc_frames"] >= 5
