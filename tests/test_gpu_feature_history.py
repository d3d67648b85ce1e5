"""Feature history of the visual trackers (WastedVisualSortTrack.observed_features, src/trackers/visual_sort.rs:117-119,
210-213): every observation pushes its input feature (or None) before the collect gate (VisualMetric::optimize,
visual_sort/metric.rs:319-336), the last history_length of them are kept, oldest first, zero-padded to 8 lanes.

Expected histories are rebuilt from the per-frame SortTrack ids the tracker itself returned and the inputs; every
comparison is bit-exact through uint32 views."""
import dataclasses

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

F32 = np.float32


@pytest.fixture(scope="module")
def eng():
    import similari_b200.engine as e
    from similari_b200._lib import lib

    if lib().sb200_device_count() <= 0:
        pytest.fail("no CUDA device: the gpu-marked tests must run on an H100")
    return e


def _cfg(n_scenes, n_objects, dim, seed=0x5EED0F00):
    from similari_b200.workload import CONFIGS

    return dataclasses.replace(CONFIGS["cfg5"], n_scenes=n_scenes, n_objects=n_objects, feature_dim=dim,
                               canvas=(900.0, 600.0), drop_frac=0.25, fresh_frac=0.15, seed=seed)


def _opts(kind, hist, dim, **over):
    from similari_b200._lib import default_options

    kw = dict(kind=kind, positional_kind=0, max_idle_epochs=1, history_length=hist, visual_kind=0, visual_threshold=0.7,
              feature_dim=dim, visual_max_observations=3, visual_min_votes=1, visual_minimal_track_length=1)
    kw.update(over)
    return default_options(**kw)


def _pad(row, d8):
    out = np.zeros(d8, F32)
    out[: len(row)] = row
    return out


class History:
    """Expected feature history per track id: (present, row padded to d8) per observation."""

    def __init__(self, d8):
        self.d8, self.seen = d8, {}

    def add(self, ids, feats, hasf):
        for i, tid in enumerate(ids):
            ok = feats is not None and (hasf is None or hasf[i] != 0)
            self.seen.setdefault(int(tid), []).append(_pad(feats[i], self.d8) if ok else None)

    def check(self, w, H):
        for i, tid in enumerate(w["ids"]):
            exp = self.seen[int(tid)][-H:]
            assert int(w["lengths"][i]) == len(self.seen[int(tid)])
            rows, pres = w["features"][i], w["feature_present"][i]
            assert len(rows) == len(pres) == len(exp) == len(w["observed_history"][i])
            for e, r, p in zip(exp, rows, pres):
                assert bool(p) == (e is not None)
                if e is not None:
                    assert np.array_equal(e.view(np.uint32), r.view(np.uint32))
                else:
                    assert not r.any()
        return len(w["ids"])


def _special(feats, rng):
    """NaN payloads, -0.0 and +-inf in some rows."""
    f = feats.copy()
    u = f.view(np.uint32)
    n = len(f)
    for i in rng.choice(n, size=max(1, n // 10), replace=False):
        j = int(rng.integers(0, f.shape[1]))
        kind = int(rng.integers(0, 4))
        if kind == 0:
            u[i, j] = 0x7FC00000 | int(rng.integers(1, 1 << 22))   # quiet NaN with a payload
        elif kind == 1:
            u[i, j] = 0x80000000   # -0.0
        elif kind == 2:
            f[i, j] = np.inf
        else:
            f[i, j] = -np.inf
    return f


@pytest.mark.parametrize("kind", [2, 3])
@pytest.mark.parametrize("hist", [1, 3, 10, 64, 100])
@pytest.mark.parametrize("dim", [30, 64, 512])
def test_wasted_tracks_carry_their_feature_history(eng, kind, hist, dim):
    from similari_b200.workload import Workload

    wl = Workload(_cfg(3 if kind == 3 else 1, 40, dim))
    g = eng.Tracker(_opts(kind, hist, dim))
    g.set_feature_history(True)
    H = min(hist, 64)
    exp = History((dim + 7) // 8 * 8)
    rng = np.random.default_rng(hist * 1000 + dim)
    checked = 0
    for fr in range(16):
        f = wl.next_frame()
        feats, hasf = _special(f["features"], rng), None
        if fr % 5 == 2:
            feats = None   # a frame without a feature column
        elif fr % 3 == 1:
            hasf = (rng.random(len(feats)) > 0.3).astype(np.uint8)
        r = g.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=feats, has_feature=hasf)
        exp.add(r["ids"], feats, hasf)
        if fr % 4 == 3:
            checked += exp.check(g.wasted_visual(), H)
    g.skip_epochs(5, 0)
    checked += exp.check(g.wasted_visual(), H)
    assert checked > 20


@pytest.mark.parametrize("gate", ["quality", "own_area"])
def test_features_the_collect_gate_drops_are_in_the_history(eng, gate):
    """A merge whose feature fails the collect thresholds keeps it out of the metric's observations (feat_counts stays at
    the creating observation's 1) but not out of the history."""
    from similari_b200.workload import Workload

    dim = 32
    over = {"quality": dict(visual_minimal_quality_collect=0.5),
            "own_area": dict(visual_minimal_own_area_percentage_collect=0.5)}[gate]
    wl = Workload(_cfg(1, 30, dim))
    g = eng.Tracker(_opts(2, 8, dim, max_idle_epochs=3, **over))
    g.set_feature_history(True)
    exp = History(dim)
    for fr in range(10):
        f = wl.next_frame()
        q = np.full(len(f["boxes"]), 0.9 if fr == 0 else 0.2, F32) if gate == "quality" else None
        own = np.full(len(f["boxes"]), 0.1, F32) if gate == "own_area" else None
        r = g.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=f["features"], quality=q, own_area=own)
        exp.add(r["ids"], f["features"], None)
    st = g.scene_tracks(0)
    assert len(st["ids"]) > 10 and int(st["feat_counts"].max()) == 1
    g.skip_epochs(10, 0)
    w = g.wasted_visual()
    assert exp.check(w, 8) > 10
    assert max(int(p.sum()) for p in w["feature_present"]) >= 5   # dropped merges are in the history


def test_minimal_area_gate(eng):
    """visual_minimal_area also gates collection: merges of boxes below it stay out of the metric, not the history."""
    from similari_b200.workload import Workload

    dim = 16
    wl = Workload(_cfg(1, 20, dim, seed=0x5EED0F01))
    g = eng.Tracker(_opts(2, 6, dim, max_idle_epochs=3, visual_minimal_area=500.0, positional_kind=1,
                          iou_threshold=0.05))
    g.set_feature_history(True)
    exp = History(dim)
    f0 = wl.next_frame()
    boxes = f0["boxes"].copy()
    boxes[:, 4] = F32(10.0)   # area = aspect * 10 * 10 < 500
    for fr in range(6):
        b = boxes.copy()
        b[:, 0] += F32(fr * 0.5)
        r = g.predict_batch(f0["scene_ids"], f0["det_offsets"], b, features=f0["features"])
        exp.add(r["ids"], f0["features"], None)
    st = g.scene_tracks(0)
    assert len(st["ids"]) == 20 and int(st["feat_counts"].max()) == 1
    g.skip_epochs(10, 0)
    w = g.wasted_visual()
    assert exp.check(w, 6) == 20 and all(int(p.sum()) == 6 for p in w["feature_present"])


@pytest.mark.parametrize("kind", [2, 3])
def test_history_on_and_off_compute_the_same(eng, kind):
    from similari_b200.workload import Workload

    dim = 64
    trk = []
    for on in (False, True):
        t = eng.Tracker(_opts(kind, 5, dim))
        if on:
            t.set_feature_history(True)
        trk.append(t)
    wl = Workload(_cfg(3 if kind == 3 else 1, 60, dim))
    for fr in range(20):
        f = wl.next_frame()
        outs, launches = [], []
        for t in trk:
            l0 = eng.launch_count()
            outs.append(t.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=f["features"]))
            launches.append(eng.launch_count() - l0)
        assert launches[0] == launches[1]
        for k in outs[0]:
            assert np.array_equal(outs[0][k].view(np.uint8), outs[1][k].view(np.uint8)), k
        assert trk[0].active_tracks() == trk[1].active_tracks()
        sc = f["scene_ids"]
        assert np.array_equal(trk[0].scene_track_counts(sc), trk[1].scene_track_counts(sc))
        for s in sc:
            a, b = trk[0].idle_tracks(int(s)), trk[1].idle_tracks(int(s))
            assert np.array_equal(a["ids"], b["ids"]) and np.array_equal(a["lengths"], b["lengths"])
        if fr % 6 == 5:
            # the scenes' sweeps append their records concurrently: compare record sets keyed by id
            a, b = trk[0].wasted_history(), trk[1].wasted_visual()
            ia, ib = np.argsort(a["ids"]), np.argsort(b["ids"])
            assert np.array_equal(a["ids"][ia], b["ids"][ib]) and np.array_equal(a["lengths"][ia], b["lengths"][ib])
            for i, j in zip(ia, ib):
                for k in ("observed_history", "predicted_history"):
                    assert np.array_equal(a[k][i].view(np.uint32), b[k][j].view(np.uint32))


def test_collection_points_and_block_reuse(eng):
    """skip_epochs, wasted(), the auto-waste tick and clear_wasted() all release blocks; records swept early stay hidden
    and keep their blocks until collected.  Each block is freed once: many cycles do not grow the pool."""
    from similari_b200.workload import Workload

    dim = 24
    g = eng.Tracker(_opts(3, 4, dim, max_idle_epochs=1))
    g.set_feature_history(True)
    wl = Workload(_cfg(2, 30, dim))
    exp = History(dim)   # 24: already a multiple of 8
    sizes = []
    for cycle in range(12):
        for fr in range(4):
            f = wl.next_frame()
            r = g.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=f["features"])
            exp.add(r["ids"], f["features"], None)
        point = cycle % 4
        if point == 0:
            exp.check(g.wasted_visual(), 4)
        elif point == 1:
            g.skip_epochs(3, 0)
            g.skip_epochs(3, 1)
            exp.check(g.wasted_visual(), 4)
        elif point == 2:
            g.set_auto_waste(1)   # the next predict is a collection point
            f = wl.next_frame()
            r = g.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=f["features"])
            exp.add(r["ids"], f["features"], None)
            g.clear_wasted()
        else:
            g.skip_epochs(5, 0)
            g.skip_epochs(5, 1)
            g.clear_wasted()
        pool = g.feature_history_pool()
        assert 0 <= pool["free"] <= pool["handed_out"] <= pool["capacity"]
        sizes.append(pool["handed_out"])
    # after the first cycles every new track reuses a block that a collected record gave back
    assert sizes[-1] <= 2 * sizes[3], sizes


def test_growth_of_pool_wasted_buffer_and_store(eng):
    """A burst of new scenes mid-run grows the pool, the wasted buffer and the store; histories stay intact."""
    from similari_b200.workload import Workload

    dim = 40
    g = eng.Tracker(_opts(3, 6, dim, max_idle_epochs=2))
    g.set_feature_history(True)
    small, big = Workload(_cfg(2, 20, dim)), Workload(_cfg(40, 90, dim, seed=0x5EED0F02), scene_base=100)
    exp = History(40)
    cap0 = None
    for fr in range(14):
        f = (big if 4 <= fr < 8 else small).next_frame()
        r = g.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=f["features"])
        exp.add(r["ids"], f["features"], None)
        if fr == 2:
            cap0 = g.feature_history_pool()["capacity"]
    assert g.feature_history_pool()["capacity"] > cap0
    for s in list(range(2)) + list(range(100, 140)):
        g.skip_epochs(5, s)
    assert exp.check(g.wasted_visual(), 6) > 1000


def test_device_inputs_async_and_stream_join(eng):
    """predict_batch_device on resident inputs, the async host path with frames in flight, set_stream_join(False)."""
    import torch

    from similari_b200._lib import pinned_empty
    from similari_b200.workload import Workload

    dim = 64
    exp = {m: History(dim) for m in ("device", "async", "nojoin")}
    trk = {}
    for m in exp:
        t = eng.Tracker(_opts(3, 5, dim, max_idle_epochs=1))
        t.set_feature_history(True)
        trk[m] = t
    stream = torch.cuda.Stream()
    trk["nojoin"].set_stream(stream.cuda_stream, join_per_call=False)
    wl = Workload(_cfg(3, 50, dim))
    frames = [wl.next_frame() for _ in range(12)]
    pend = []
    for fr, f in enumerate(frames):
        total = int(f["det_offsets"][-1])
        for m in ("device", "nojoin"):
            db = torch.from_numpy(f["boxes"]).cuda()
            dfe = torch.from_numpy(f["features"]).cuda()
            ids = torch.zeros(total, dtype=torch.int64, device="cuda")
            torch.cuda.synchronize()
            trk[m].predict_batch_device(f["scene_ids"], f["det_offsets"], db.data_ptr(), dfe.data_ptr(),
                                        d_ids=ids.data_ptr())
            if m == "nojoin":
                trk[m].stream_join(torch.cuda.current_stream().cuda_stream)
            trk[m].sync()
            exp[m].add(ids.cpu().numpy().view(np.uint64), f["features"], None)
        out = {"ids": pinned_empty(total, np.uint64)}
        trk["async"].predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=f["features"], out=out,
                                   wait=False)
        pend.append((out, f))
        if fr % 3 == 2:
            trk["async"].sync()
            for o, ff in pend:
                exp["async"].add(o["ids"], ff["features"], None)
            pend = []
            exp["async"].check(trk["async"].wasted_visual(), 5)
        if fr % 4 == 3:
            for m in ("device", "nojoin"):
                exp[m].check(trk[m].wasted_visual(), 5)
    trk["async"].sync()
    for o, ff in pend:
        exp["async"].add(o["ids"], ff["features"], None)
    for m, t in trk.items():
        for s in f["scene_ids"]:
            t.skip_epochs(5, int(s))
        assert exp[m].check(t.wasted_visual(), 5) > 0


@pytest.mark.parametrize("path", ["calls", "device_chunks"])
def test_chunked_drain(eng, path):
    """wasted_visual drains in chunks: many C calls of a few records each (small chunk_bytes), or one call whose records
    the device gathers in several 64 MB staging chunks (H = 64, D = 512: 512 records per chunk)."""
    from similari_b200.workload import Workload

    dim, hist = 512, 64
    g = eng.Tracker(_opts(3, hist, dim, max_idle_epochs=1))
    g.set_feature_history(True)
    wl = Workload(_cfg(3, 300 if path == "device_chunks" else 40, dim))
    exp = History(dim)
    rng = np.random.default_rng(11)
    for fr in range(6):
        f = wl.next_frame()
        hasf = (rng.random(len(f["boxes"])) > 0.2).astype(np.uint8)
        r = g.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=f["features"], has_feature=hasf)
        exp.add(r["ids"], f["features"], hasf)
    for s in f["scene_ids"]:
        g.skip_epochs(5, int(s))
    row_bytes = hist * dim * 4
    chunk = 7 * row_bytes if path == "calls" else 2048 * row_bytes
    w = g.wasted_visual(chunk_bytes=chunk)
    n = exp.check(w, hist)
    assert n == len(exp.seen)
    assert n > (7 * 5 if path == "calls" else 2 * 512)
    assert g.wasted_visual()["ids"].size == 0


def test_c_abi_writes_every_row(eng):
    """sb200_wasted_visual writes zero rows for entries without a feature and past a record's count, whatever the
    caller's buffers held."""
    import ctypes as C

    from similari_b200._lib import ptr

    dim, H = 16, 4
    g = eng.Tracker(_opts(2, H, dim, max_idle_epochs=1))
    g.set_feature_history(True)
    boxes = np.array([[100, 100, 0.0, 0.5, 40, 0.9], [400, 300, 0.0, 0.5, 40, 0.9]], F32)
    feats = np.arange(2 * dim, dtype=F32).reshape(2, dim) + F32(1)
    for fr in range(2):   # track 0: featured then feature-less; track 1: feature-less twice
        hasf = np.array([1 if fr == 0 else 0, 0], np.uint8)
        g.predict_batch([0], [0, 2], boxes, features=feats, has_feature=hasf)
    g.skip_epochs(5, 0)
    cap = 4
    ids, sc = np.zeros(cap, np.uint64), np.zeros(cap, np.uint64)
    ep, ln = np.zeros(cap, np.uint32), np.zeros(cap, np.uint32)
    pr, ob = np.zeros((cap, 6), F32), np.zeros((cap, 6), F32)
    hp, ho, hc = np.zeros((cap, H, 6), F32), np.zeros((cap, H, 6), F32), np.zeros(cap, np.int32)
    ft = np.full((cap, H, dim), np.nan, F32)
    fp = np.full((cap, H), 0xEE, np.uint8)
    n = g._L.sb200_wasted_visual(g._h, cap, ptr(ids), ptr(sc), ptr(ep), ptr(ln), ptr(pr), ptr(ob), C.c_int32(H), ptr(hp),
                                 ptr(ho), ptr(hc), ptr(ft), ptr(fp))
    assert n == 2 and list(hc[:2]) == [2, 2]
    for i in range(2):
        first = int(ids[i]) == int(min(ids[:2]))
        want = [1, 0, 0, 0] if first else [0, 0, 0, 0]
        assert list(fp[i]) == want
        for c in range(H):
            if want[c]:
                assert np.array_equal(ft[i, c].view(np.uint32), feats[0].view(np.uint32))
            else:
                assert not ft[i, c].view(np.uint32).any()
    assert np.isnan(ft[2:]).all() and (fp[2:] == 0xEE).all()   # nothing past the returned records


def test_wasted_visual_needs_the_history(eng):
    from similari_b200._lib import Sb200Error

    g = eng.Tracker(_opts(2, 4, 8))
    with pytest.raises(Sb200Error):
        g.wasted_visual()
    g.predict_batch([0], [0, 1], np.array([[10, 10, 0.0, 0.5, 50, 0.9]], F32), features=np.ones((1, 8), F32))
    with pytest.raises(Sb200Error):
        g.set_feature_history(True)   # only before the first predict
    s = eng.Tracker(_opts(0, 4, 8))
    with pytest.raises(Sb200Error):
        s.set_feature_history(True)


# ----------------------------------------------------------------------------------------------------------- API
def test_api_visual_sort_script(eng):
    """The calls of the reference's python/visual_sort.py, restated."""
    import similari_b200.api as sim

    constraints = sim.SpatioTemporalConstraints()
    constraints.add_constraints([(1, 1.0)])
    opts = sim.VisualSortOptions()
    opts.spatio_temporal_constraints(constraints)
    opts.max_idle_epochs(3)
    opts.kept_history_length(10)
    opts.visual_metric(sim.VisualSortMetricType.euclidean(1.0))
    opts.positional_metric(sim.PositionalMetricType.maha())
    opts.visual_minimal_track_length(3)
    opts.visual_minimal_area(5.0)
    opts.visual_minimal_quality_use(0.45)
    opts.visual_minimal_quality_collect(0.5)
    opts.visual_max_observations(5)
    opts.visual_min_votes(2)
    tracker = sim.VisualSort(shards=4, opts=opts)
    observation_set = sim.VisualSortObservationSet()
    observation_set.add(sim.VisualSortObservation(feature=np.array([0.1, 0.1]), feature_quality=0.96,
                                                  bounding_box=sim.BoundingBox(0, 0, 5, 10).as_xyaah(),
                                                  custom_object_id=10))
    tracks = tracker.predict(observation_set)
    assert len(tracks) == 1
    tracker.skip_epochs(10)
    wasted = tracker.wasted()
    assert len(wasted) == 1 and isinstance(wasted[0], sim.WastedSortTrack)
    assert isinstance(wasted[0], sim.WastedVisualSortTrack)
    assert wasted[0].observed_features == [[F32(0.1), F32(0.1), 0, 0, 0, 0, 0, 0]]
    assert len(wasted[0].observed_features) == len(wasted[0].observed_boxes)
    tracker.clear_wasted()
    assert tracker.wasted() == []


def test_api_batch_visual_sort_script(eng):
    """The calls of the reference's python/visual_sort/batch_visual_sort.py (10 frames, 6 objects, 2 scenes), restated;
    then every track is wasted and its observed_features are the features it was fed, newest 25."""
    import similari_b200.api as sim

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
    opts.visual_max_observations(8)   # the script asks for 25; the device keeps at most 8 (kMaxObs, DESIGN section 7)
    opts.visual_min_votes(5)
    tracker = sim.BatchVisualSort(distance_shards=1, voting_shards=1, opts=opts)
    objs = np.random.default_rng(3).random((6, 4 + 128 + 1))
    seen = {}
    for _ in range(10):
        req = sim.VisualSortPredictionBatchRequest()
        for batch_i, batch_objs in enumerate(np.split(objs, 2)):
            for obj in batch_objs:
                req.add(batch_i, sim.VisualSortObservation(feature=obj[4:132], feature_quality=obj[132],
                                                           bounding_box=sim.BoundingBox(*obj[:4]).as_xyaah(),
                                                           custom_object_id=None))
        result = tracker.predict(req)
        for _ in range(result.batch_size()):
            scene_id, tracks = result.get()
            for k, track in enumerate(tracks):   # tracks come back in the scene's observation order
                feat = objs[scene_id * 3 + k, 4:132].astype(F32)
                seen.setdefault(track.id, []).append(feat.tolist())
    tracker.skip_epochs_for_scene(0, 20)
    tracker.skip_epochs_for_scene(1, 20)
    wasted = tracker.wasted()
    assert {w.id for w in wasted} == set(seen)
    for w in wasted:
        assert len(w.observed_features) == len(w.observed_boxes) == min(25, w.length)
        assert w.observed_features == seen[w.id][-25:]


def test_api_provisional_dimension_and_batch(eng):
    """Feature-less first frames (provisional dimension), then featured ones; BatchVisualSort over several scenes."""
    import similari_b200.api as sim

    opts = sim.VisualSortOptions()
    opts.kept_history_length(4)
    opts.max_idle_epochs(1)
    t = sim.BatchVisualSort(4, 4, opts)
    rng = np.random.default_rng(7)
    n_scenes, n_obj, dim = 3, 5, 12
    cx = rng.uniform(50, 800, (n_scenes, n_obj))
    seen = {}
    for fr in range(7):
        req = sim.VisualSortPredictionBatchRequest()
        feats = {}
        for s in range(n_scenes):
            for k in range(n_obj):
                feat = None if fr < 2 or (fr + k) % 4 == 0 else rng.standard_normal(dim).astype(F32).tolist()
                feats[(s, k)] = feat
                box = sim.Universal2DBox.new_with_confidence(cx[s, k] + fr, 100.0 + 40 * k, None, 0.5, 30.0, 0.9)
                req.add(s, sim.VisualSortObservation(feat, 0.9, box, k))
        res = t.predict(req)
        for _ in range(res.batch_size()):
            s, tracks = res.get()
            for tr in tracks:
                f = feats[(s, tr.custom_object_id)]
                seen.setdefault(tr.id, []).append(None if f is None else [float(F32(x)) for x in f] + [0.0] * 4)
    for s in range(n_scenes):
        t.skip_epochs_for_scene(s, 5)
    wasted = t.wasted()
    assert len(wasted) >= n_scenes * n_obj
    for w in wasted:
        assert isinstance(w, sim.WastedVisualSortTrack)
        assert len(w.observed_features) == len(w.observed_boxes)
        assert w.observed_features == seen[w.id][-4:]
