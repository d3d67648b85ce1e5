"""Visual trackers that keep 9 to 32 observations per track (visual_max_observations above kMaxObs = 8), against the
oracle: the apply stage's warp-per-merge observation lists, the sweep's row compaction of the observation columns and
the dense path's warp-per-block metadata and selection.  The reference's VisualSORT examples ask for 25."""
import numpy as np
import pytest

from test_gpu_track_observations import ObservationWorkload, below, both, check_outputs, check_state, predict_both, set_path

pytestmark = pytest.mark.gpu

F32MAX = float(np.finfo(np.float32).max)
WIDE_KS = [9, 16, 25, 32]
D_OF_K = {9: 64, 16: 60, 25: 128, 32: 64}
PATHS = ["simt", "tc16", "tc8", "dense", "dense-generic"]


@pytest.fixture(scope="module")
def eng():
    import similari_b200.engine as e
    from similari_b200._lib import lib

    if lib().sb200_device_count() <= 0:
        pytest.fail("no CUDA device: the gpu-marked tests must run on an H100")
    return e


class ManyObservations(ObservationWorkload):
    """ObservationWorkload with most detections carrying a collectable feature, so that observation lists fill up to K
    (and the drop of the lowest quality runs) within a few dozen frames.  Quality ties and the values one ulp below the
    thresholds stay."""

    def __init__(self, n_scenes, n_objects, d, seed):
        super().__init__(n_scenes, n_objects, d, seed)
        self.qset = np.array([0.5, 0.8, 0.8, 1.0, 1.0, 1.0, 0.9, 0.6, below(self.Q_COLLECT), below(self.Q_USE), 0.3],
                             np.float32)

    def next_frame(self):
        f = self.wl.next_frame()
        n = len(f["boxes"])
        f["quality"] = self.rng.choice(self.qset, n).astype(np.float32)
        f["has_feature"] = (self.rng.random(n) >= 0.08).astype(np.uint8)
        return f


def _case(K, kind, path, **over):
    d = D_OF_K[K]
    vis = (K + kind) % 2
    opts = ObservationWorkload.options(kind, K, d, vis, path, max_idle=2, min_track_length=3)
    opts.update(over)
    wl = ManyObservations(1 if kind == 2 else 3, 90 if kind == 2 else 40, d, 0x5EED9000 + 97 * K + 13 * kind)
    return opts, wl


def _run(eng, oracle, K, kind, path, frames, **over):
    opts, wl = _case(K, kind, path, **over)
    g, o = both(eng, oracle, **opts)
    full = 0
    for fr in range(frames):
        f = wl.next_frame()
        rg, ro = predict_both(g, o, f)
        check_outputs(rg, ro, fr)
        if fr < 6 or fr % 3 == 2 or fr == frames - 1:
            st = check_state(g, o, opts, f["scene_ids"], fr)
            full = max(full, max(int(s["obs_n"].max(initial=0)) for s in st.values()))
    return g, full


CASES = [(K, kind, path) for K in WIDE_KS for kind in (2, 3) for path in PATHS]


@pytest.mark.parametrize("K,kind,path", CASES, ids=[f"K{c[0]}-k{c[1]}-{c[2]}" for c in CASES])
def test_track_state_matches_oracle(eng, oracle, K, kind, path, monkeypatch):
    """Frame after frame: the SortTrack columns, and the device store (Kalman states, observation lists in order with
    their flags and qualities, arena rows, norms, BF16 copies, block bookkeeping) against the oracle.  Some track's list
    reaches K observations, so the drop of the last one after the quality sort runs too."""
    set_path(monkeypatch, path)
    frames = 3 * K + 8
    g, full = _run(eng, oracle, K, kind, path, frames)
    assert full == K
    wc, sc = g.work_counters(), g.screen_counters()
    if path != "simt":
        assert wc["tc_frames"] >= frames - 2, wc
    if path == "tc8":
        assert sc["fp8_frames"] >= frames - 2, sc
    if path == "tc16":
        assert sc["bf16_frames"] >= frames - 2, sc


@pytest.mark.parametrize("path", ["simt", "tc16", "dense"])
def test_min_votes_equal_to_k(eng, oracle, path, monkeypatch):
    """visual_min_votes = K = 25: only tracks with 25 valid observations vote."""
    set_path(monkeypatch, path)
    _, full = _run(eng, oracle, 25, 3, path, 83, visual_min_votes=25)
    assert full == 25


# ------------------------------------------------------------------------------------------- the bound constructions
@pytest.mark.parametrize("path", ["simt", "tc", "dense"])
@pytest.mark.parametrize("vis", [0, 1])
@pytest.mark.parametrize("kobs", [9, 32])
def test_column_tie_matches_oracle(eng, oracle, path, vis, kobs, monkeypatch):
    """The column near-tie of test_gpu_visual_bounds.tie_scene_frames with 9 and 32 observations per track, in four
    scenes, on every visual path."""
    from test_gpu_visual_bounds import VIS_KW, _drive, _frame, _tie_scenes

    monkeypatch.setenv("SB200_VIS_KERNEL", path)
    d, n = 128, 60
    per_scene = _tie_scenes(d, n, kobs, 300 + kobs + vis, [(None, None)] * 4)
    frames = [_frame([sc[fr] for sc in per_scene]) for fr in range(kobs + 1)]
    if path == "dense":
        thr = F32MAX if vis == 0 else -1.0
    else:
        thr = 1.2 if vis == 0 else 0.1
    g = _drive(eng, oracle, dict(kind=3, visual_kind=vis, visual_threshold=thr, feature_dim=d,
                                 visual_max_observations=kobs, visual_min_votes=2, **VIS_KW), frames)
    wc = g.work_counters()
    if path != "simt":
        assert wc["tc_frames"] >= kobs
    if path == "dense":   # the selection decided most scene-frames itself
        assert wc["dense_fallback_scenes"] < 4 * (kobs + 1) // 2, wc


@pytest.mark.parametrize("path", ["simt", "tc", "dense"])
@pytest.mark.parametrize("vis", [0, 1])
@pytest.mark.parametrize("kobs", [9, 32])
def test_row_tie_matches_oracle(eng, oracle, path, vis, kobs, monkeypatch):
    """The row near-tie of test_gpu_visual_bounds.row_tie_features with 9 and 32 identical observations of t1 and t2:
    the reference gives q nothing visual, a selection that dropped (q, t1) would give it t2."""
    from test_gpu_visual_bounds import ROW_TIE_SEEDS, VIS_KW, _drive, _far_box, _frame, _grid_boxes, row_tie_features, unit

    monkeypatch.setenv("SB200_VIS_KERNEL", path)
    d, n = 128, 40
    q, t1, t2 = row_tie_features(ROW_TIE_SEEDS[vis], d)
    rng = np.random.default_rng(7)
    base = np.stack([unit(rng, d) for _ in range(n)]).astype(np.float32) * np.float32(np.linalg.norm(q))
    base[0], base[1] = t1, t2
    frames = []
    for fr in range(kobs + 1):
        scenes = []
        for s in range(3):
            boxes, feats = _grid_boxes(n), base.copy()
            if fr == kobs:
                feats[1] = q
                boxes[1] = _far_box(0)
            scenes.append((boxes, feats))
        frames.append(_frame(scenes))
    if path == "dense":
        thr = F32MAX if vis == 0 else -1.0
    else:
        thr = 1.2 if vis == 0 else 0.1
    g = _drive(eng, oracle, dict(kind=3, visual_kind=vis, visual_threshold=thr, feature_dim=d,
                                 visual_max_observations=kobs, visual_min_votes=2, **VIS_KW), frames)
    if path == "dense":
        wc = g.work_counters()
        assert wc["tc_frames"] >= kobs and wc["dense_fallback_scenes"] == 0, wc


# ------------------------------------------------------------------------------------------- layers above the kernels
def test_api_batch_visual_sort_script_with_25_observations(eng, oracle):
    """The calls of the reference's python/visual_sort/batch_visual_sort.py (6 objects, 2 scenes; 30 frames, so
    that the lists fill) with its own visual_max_observations(25), through api.BatchVisualSort, against the oracle fed the same requests; then every
    track is wasted and its observed_features are the features it was fed, newest 25."""
    import similari_b200.api as sim
    from similari_b200._lib import KIND_BATCH_VISUAL_SORT

    constraints = sim.SpatioTemporalConstraints()
    constraints.add_constraints([(1, 1.0)])
    opts = sim.VisualSortOptions()
    opts.spatio_temporal_constraints(constraints)
    opts.max_idle_epochs(15)
    opts.kept_history_length(25)
    opts.visual_metric(sim.VisualSortMetricType.euclidean(0.7))
    opts.positional_metric(sim.PositionalMetricType.maha())
    opts.visual_minimal_track_length(7)
    opts.visual_minimal_area(5.0)
    opts.visual_minimal_quality_use(0.45)
    opts.visual_minimal_quality_collect(0.5)
    opts.visual_max_observations(25)
    opts.visual_min_votes(5)
    tracker = sim.BatchVisualSort(distance_shards=1, voting_shards=1, opts=opts)
    o = oracle.Tracker(oracle.make_options(kind=KIND_BATCH_VISUAL_SORT, feature_dim=128, constraints=opts._constraints,
                                           **opts._kw))
    objs = np.random.default_rng(3).random((6, 4 + 128 + 1))
    seen = {}
    for fr in range(30):
        req = sim.VisualSortPredictionBatchRequest()
        allobs = []
        for batch_i, batch_objs in enumerate(np.split(objs, 2)):
            for obj in batch_objs:
                ob = sim.VisualSortObservation(feature=obj[4:132], feature_quality=obj[132],
                                               bounding_box=sim.BoundingBox(*obj[:4]).as_xyaah(), custom_object_id=None)
                req.add(batch_i, ob)
                allobs.append(ob)
        result = tracker.predict(req)
        got = {}
        for _ in range(result.batch_size()):
            scene_id, tracks = result.get()
            got[scene_id] = [t.id for t in tracks]
            for k, track in enumerate(tracks):
                seen.setdefault(track.id, []).append(objs[scene_id * 3 + k, 4:132].astype(np.float32).tolist())
        boxes = np.array([ob.bounding_box._row() for ob in allobs], np.float32)
        feats = np.array([ob.feature for ob in allobs], np.float32)
        qual = np.array([ob.feature_quality for ob in allobs], np.float32)
        ro = o.predict_batch(np.array([0, 1], np.uint64), np.array([0, 3, 6], np.int32), boxes, features=feats,
                             quality=qual)
        assert got[0] + got[1] == [int(i) for i in ro["ids"]], fr
    tracker.skip_epochs_for_scene(0, 20)
    tracker.skip_epochs_for_scene(1, 20)
    wasted = tracker.wasted()
    assert {w.id for w in wasted} == set(seen)
    for w in wasted:
        assert len(w.observed_features) == len(w.observed_boxes) == min(25, w.length)
        assert w.observed_features == seen[w.id][-25:]


def _same_frames(ra, rb, where):
    for key in ("ids", "epochs", "lengths", "voting_types"):
        assert np.array_equal(ra[key], rb[key]), (where, key)


@pytest.mark.parametrize("kind", [2, 3])
def test_save_load_and_export_import_at_25(eng, oracle, kind, monkeypatch):
    """K = 25: a tracker restored from save() and one that imported every scene continue exactly as the tracker that
    never stopped, frame by frame and in the store they end with; save -> load -> save and export -> import -> export
    give the same blobs."""
    set_path(monkeypatch, "tc16")
    opts, wl = _case(25, kind, "tc16")
    from similari_b200._lib import default_options

    R = eng.Tracker(default_options(**opts))
    T = eng.Tracker(default_options(**opts))
    frames = [wl.next_frame() for _ in range(48)]
    args = lambda f: ((f["scene_ids"], f["det_offsets"], f["boxes"]),
                      dict(features=f["features"], has_feature=f["has_feature"], quality=f["quality"]))
    for f in frames[:30]:
        a, kw = args(f)
        R.predict_batch(*a, **kw)
        T.predict_batch(*a, **kw)
    blob = R.save()
    L = eng.Tracker.load(blob)
    assert np.array_equal(L.save(), blob)
    scenes = sorted(int(s) for s in frames[0]["scene_ids"])
    moved = T.export_scenes(scenes, remove=True)
    I = eng.Tracker(default_options(**opts))
    I.import_scenes(moved)
    assert np.array_equal(I.export_scenes(scenes), moved)
    for i, f in enumerate(frames[30:]):
        a, kw = args(f)
        rr = R.predict_batch(*a, **kw)
        _same_frames(rr, L.predict_batch(*a, **kw), ("load", i))
        _same_frames(rr, I.predict_batch(*a, **kw), ("import", i))
    want = _live_state(R)
    assert _live_state(L) == want and _live_state(I) == want


def _live_state(t):
    """The tracker's store as read_state reads it, with each track's observation columns cut at its observation count
    (the slots past it were never written for the track that holds the row now)."""
    from test_gpu_track_observations import read_state

    out = {}
    for sid, sc in read_state(t.save()).items():
        cols = {}
        for name, v in sc.items():
            if name in ("obs_phys", "obs_hasf", "obs_q"):
                cols[name] = [row[:n].tobytes() for row, n in zip(v, sc["obs_n"])]
            else:
                cols[name] = np.asarray(v).tobytes()
        out[sid] = cols
    return out


def test_wasted_to_store_at_25(eng):
    """associate_wasted from a K = 25 tracker with feature history equals its host composition (wasted_visual, the
    present rows, one associate), and leaves the same tracker and store state."""
    from test_gpu_wasted_store import HIST, Driver, _collect, _prefill, _store, _tracker

    dim, hist = 64, 10
    ta = _tracker(eng, 3, hist, dim, visual_max_observations=25)
    sa, sb = _store(eng, dim, K=25), _store(eng, dim, K=25)
    _prefill([sa, sb], dim, 50, 25)
    d = Driver(3, 40, dim, 0x5EED0125)
    collected = 0
    for fr in range(40):
        d.frame([ta])
        if fr % 8 == 7:
            collected += len(_collect(eng, ta, None, sa, sb, HIST[hist])["ids"])
    ta.skip_epochs(5, 0)
    _collect(eng, ta, None, sa, sb, HIST[hist])
    assert collected > 20


@pytest.mark.parametrize("kernel", ["dense", "sparse", "prepass"])
def test_stateless_visual_voting_k32(eng, oracle, monkeypatch, kernel):
    """sb200_visual_voting with k = 32 observations per track, min_votes 1, 16 and 32."""
    from test_gpu_voting import _visual_scene, check_visual

    rng = np.random.default_rng(1032)
    pos, vis = _visual_scene(rng, 40, 30, 32)
    for mv in (1, 16, 32):
        check_visual(eng, oracle, monkeypatch, kernel, 0.3, mv, pos, vis)


def test_33_observations_are_refused(eng):
    """K = 33: the tracker and the stateless voting refuse it before anything is created; the message names 32."""
    import similari_b200.api as sim
    from similari_b200._lib import Sb200Error, default_options, lib

    before = lib().sb200_device_count()
    with pytest.raises(Sb200Error, match=r"status -3: .*\[1, 32\]"):
        eng.Tracker(default_options(kind=3, feature_dim=16, visual_max_observations=33))
    opts = sim.VisualSortOptions()
    opts.visual_max_observations(33)
    t = sim.VisualSort(shards=1, opts=opts)
    obs = sim.VisualSortObservationSet()
    obs.add(sim.VisualSortObservation(feature=np.ones(16), feature_quality=1.0,
                                      bounding_box=sim.BoundingBox(0, 0, 10, 20).as_xyaah(), custom_object_id=None))
    with pytest.raises(Sb200Error, match=r"\[1, 32\]"):
        t.predict(obs)
    assert t._t is None
    pos = np.zeros((2, 2), np.float32)
    with pytest.raises(Sb200Error):
        eng.visual_voting(0.3, 1, pos, np.zeros((2, 2, 33), np.float32))
    assert lib().sb200_device_count() == before
