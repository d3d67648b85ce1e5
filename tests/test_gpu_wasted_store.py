"""sb200_fstore_associate_wasted: the wasted records of a visual tracker associated with a feature track store on the
device.  Every case compares the call with its host composition (sb200_wasted_visual, the present rows of each record's
history, one sb200_fstore_associate) on a twin tracker and a twin store in the same state: records, box histories and
store outputs bit for bit (f64 weights through uint64 views), then both store blobs and both tracker blobs byte for
byte.

The twin tracker is a clone (sb200_tracker_load of the tracker's blob) taken right before the call.  Two trackers fed the
same frames keep the same records, but a multi-scene frame appends its scenes' records to the wasted buffer in the
order their blocks finish, so their collection order can differ between the two; a clone has the tracker's own order.
Single-scene twins fed identically are used where the call must meet frames still in flight."""
import dataclasses

import numpy as np
import pytest

from fstore_checks import same_results, same_store, store_pair

pytestmark = pytest.mark.gpu

F32 = np.float32
HIST = {1: 1, 10: 10, 64: 64, 0: 64}   # history_length -> kept entries H


@pytest.fixture(scope="module")
def eng():
    import similari_b200.engine as e
    from similari_b200._lib import lib

    if lib().sb200_device_count() <= 0:
        pytest.fail("no CUDA device: the gpu-marked tests must run on an H100")
    return e


def _cfg(n_scenes, n_objects, dim, seed):
    from similari_b200.workload import CONFIGS

    return dataclasses.replace(CONFIGS["cfg5"], n_scenes=n_scenes, n_objects=n_objects, feature_dim=dim,
                               canvas=(900.0, 600.0), drop_frac=0.3, fresh_frac=0.1, seed=seed)


def _opts(kind, hist, dim, **over):
    from similari_b200._lib import default_options

    kw = dict(kind=kind, positional_kind=0, max_idle_epochs=1, history_length=hist, visual_kind=0, visual_threshold=0.7,
              feature_dim=dim, visual_max_observations=3, visual_min_votes=1, visual_minimal_track_length=1)
    kw.update(over)
    return default_options(**kw)


def _tracker(eng, kind, hist, dim, **over):
    t = eng.Tracker(_opts(kind, hist, dim, **over))
    t.set_feature_history(True)
    return t


def _store(eng, dim, metric="euclidean", storage="f32", K=3, topn=2, **over):
    kw = dict(distance_filter=1.0 if metric == "euclidean" else 0.5, max_observations=K, feature_dim=dim, topn=topn,
              max_distance=1.0 if metric == "euclidean" else 0.5, min_votes=1, storage=storage)
    kw.update(over)
    return eng.FeatureStore(metric=metric, **kw)


def _special(feats, rng):
    """NaN payloads, -0.0 and +-inf in some rows."""
    f = feats.copy()
    u = f.view(np.uint32)
    for i in rng.choice(len(f), size=max(1, len(f) // 12), replace=False):
        j = int(rng.integers(0, f.shape[1]))
        u[i, j] = [0x7FC00000 | int(rng.integers(1, 1 << 22)), 0x80000000, 0x7F800000, 0xFF800000][int(rng.integers(0, 4))]
    return f


def _typed(feats, ftype):
    """The column as the tracker is fed it: f32, float16, or the uint16 bits of bfloat16 (round to nearest even)."""
    if feats is None or ftype == "f32":
        return feats, None
    if ftype == "f16":
        return feats.astype(np.float16), None
    u = feats.view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)
    r = np.where(np.isnan(feats), (u >> 16).astype(np.uint16) | 0x40, r)
    return r, "bf16"


class Driver:
    """Feeds the same seeded frames to every tracker given: feature gaps, frames without a feature column, special
    values."""

    def __init__(self, n_scenes, n_objects, dim, seed, ftype="f32", gaps=True):
        from similari_b200.workload import Workload

        self.wl, self.rng, self.ftype, self.gaps = Workload(_cfg(n_scenes, n_objects, dim, seed)), np.random.default_rng(seed), ftype, gaps
        self.fr = 0

    def frame(self, trackers, wait=True):
        f = self.wl.next_frame()
        feats, hasf = _special(f["features"], self.rng), None
        if self.gaps and self.fr % 5 == 2:
            feats = None
        elif self.gaps and self.fr % 3 == 1:
            hasf = (self.rng.random(len(feats)) > 0.3).astype(np.uint8)
        col, ft = _typed(feats, self.ftype)
        self.fr += 1
        return [t.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=col, has_feature=hasf,
                                feature_type=ft, wait=wait) for t in trackers]


def _wasted_visual(eng, t, cap, H):
    """One sb200_wasted_visual call of `cap` records with every kept history entry."""
    from similari_b200._lib import check, ptr

    d8 = (int(t.opts.feature_dim) + 7) // 8 * 8
    c = max(cap, 1)
    o = {"ids": np.zeros(c, np.uint64), "scene_ids": np.zeros(c, np.uint64), "epochs": np.zeros(c, np.uint32),
         "lengths": np.zeros(c, np.uint32), "predicted": np.zeros((c, 6), F32), "observed": np.zeros((c, 6), F32),
         "hp": np.zeros((c, H, 6), F32), "ho": np.zeros((c, H, 6), F32), "hc": np.zeros(c, np.int32),
         "ft": np.zeros((c, H, d8), F32), "fp": np.zeros((c, H), np.uint8)}
    n = check(t._L.sb200_wasted_visual(t._h, cap, *(ptr(o[k]) for k in ("ids", "scene_ids", "epochs", "lengths",
                                                                        "predicted", "observed")),
                                       H, ptr(o["hp"]), ptr(o["ho"]), ptr(o["hc"]), ptr(o["ft"]), ptr(o["fp"])))
    return {k: v[:n] for k, v in o.items()}


def _compose(eng, t, s, cap, H, id_offset=0, history_cap=None):
    """The host composition the call must equal: wasted_visual, present rows, one associate."""
    hcap = H if history_cap is None else history_cap
    w = _wasted_visual(eng, t, cap, H)
    n, D, topn = len(w["ids"]), s.D, s.topn
    rows, offs, qi = [], [0], []
    for i in range(n):
        p = w["fp"][i, : w["hc"][i]].astype(bool)
        if p.any():
            rows.append(w["ft"][i, : w["hc"][i]][p][:, :D])
            offs.append(offs[-1] + int(p.sum()))
            qi.append(i)
    qid = w["ids"][qi] + np.uint64(id_offset)
    res = {"ids": w["ids"], "scene_ids": w["scene_ids"], "epochs": w["epochs"], "lengths": w["lengths"],
           "predicted": w["predicted"], "observed": w["observed"],
           "predicted_history": [w["hp"][i, max(0, w["hc"][i] - hcap): w["hc"][i]] for i in range(n)],
           "observed_history": [w["ho"][i, max(0, w["hc"][i] - hcap): w["hc"][i]] for i in range(n)],
           "feature_counts": w["fp"].sum(axis=1).astype(np.int32), "queried": w["fp"].any(axis=1),
           "counts": np.zeros(n, np.int32), "winners": np.zeros((n, topn), np.uint64),
           "weights": np.zeros((n, topn), np.float64), "track_ids": np.zeros(n, np.uint64),
           "merged": np.zeros(n, np.uint8)}
    if hcap == 0:
        res["predicted_history"] = [np.zeros((0, 6), F32)] * n
        res["observed_history"] = [np.zeros((0, 6), F32)] * n
    if qi:
        r = s.associate(qid, offs, np.concatenate(rows))
        for k in ("counts", "winners", "weights", "track_ids", "merged"):
            res[k][qi] = r[k]
    return res


def _same_state(ta, tb, sa, sb):
    same_store(sa, sb)
    assert np.array_equal(sa.save(), sb.save())
    assert np.array_equal(ta.save(), tb.save())


def _collect(eng, ta, tb, sa, sb, H, cap=None, id_offset=0, history_cap=None):
    """tb None: the twin tracker is a clone of ta taken now."""
    if tb is None:
        tb = eng.Tracker.load(ta.save())
    a = sa.associate_wasted(ta, cap=cap, id_offset=id_offset, history_cap=history_cap)
    b = _compose(eng, tb, sb, len(a["ids"]) if cap is None else cap, H, id_offset, history_cap)
    same_results(a, b)
    _same_state(ta, tb, sa, sb)
    return a


def _prefill(s_list, dim, n, seed):
    rng = np.random.default_rng(seed)
    rows = rng.standard_normal((n, dim)).astype(F32)
    rows /= np.linalg.norm(rows, axis=1, keepdims=True)
    ids = np.arange(1 << 40, (1 << 40) + n, dtype=np.uint64)
    for s in s_list:
        s.add(ids, rows)


CASES = [
    # kind, hist, dim, tracker feature type, metric, storage, K
    (3, 10, 64, "f32", "euclidean", "f32", 3),
    (3, 10, 64, "f32", "cosine", "f32", 3),
    (3, 10, 64, "f32", "euclidean", "f16", 3),
    (3, 10, 64, "f32", "cosine", "bf16", 64),
    (3, 10, 30, "f16", "euclidean", "f32", 3),
    (3, 10, 64, "bf16", "euclidean", "bf16", 3),
    (3, 10, 64, "f16", "cosine", "f16", 64),
    (2, 10, 64, "f32", "euclidean", "f32", 3),
    (3, 1, 64, "f32", "euclidean", "f32", 3),
    (3, 64, 40, "f32", "euclidean", "f32", 64),
    (3, 0, 64, "bf16", "cosine", "f32", 3),
    (2, 64, 512, "f32", "euclidean", "f16", 3),
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "-".join(map(str, c)))
def test_equals_the_host_composition(eng, case):
    kind, hist, dim, ftype, metric, storage, K = case
    H = HIST[hist]
    n_scenes = 1 if kind == 2 else 3
    ta = _tracker(eng, kind, hist, dim)
    sa, sb = _store(eng, dim, metric, storage, K), _store(eng, dim, metric, storage, K)
    _prefill([sa, sb], dim, 50, dim + K)
    d = Driver(n_scenes, 40, dim, 0x5EED0100 + dim + hist, ftype)
    merged = new = collected = 0
    for fr in range(24):
        d.frame([ta])
        if fr % 4 == 3:
            a = _collect(eng, ta, None, sa, sb, H)
            merged += int(a["merged"].sum())
            new += int((a["queried"] & (a["merged"] == 0)).sum())
            collected += len(a["ids"])
    ta.skip_epochs(5, 0)
    _collect(eng, ta, None, sa, sb, H)
    assert collected > 20 and new > 0
    if metric == "euclidean":
        assert merged > 0


def test_cap_id_offset_and_history_cap(eng):
    """A cap below the wasted count (the rest comes with a second call), an id offset that wraps past 2^64, and a
    history_cap below the kept history (it bounds only the box histories)."""
    dim, H = 48, 10
    ta = _tracker(eng, 3, H, dim)
    sa, sb = _store(eng, dim, K=4), _store(eng, dim, K=4)
    d = Driver(3, 50, dim, 0x5EED0200)
    off = (1 << 64) - 5
    for fr in range(16):
        d.frame([ta])
        if fr % 5 == 4:
            a = _collect(eng, ta, None, sa, sb, H, cap=7, id_offset=off, history_cap=3)
            assert len(a["ids"]) == 7
            _collect(eng, ta, None, sa, sb, H, id_offset=off, history_cap=3)
    ta.skip_epochs(4, 0)
    a = _collect(eng, ta, None, sa, sb, H, cap=1, id_offset=off, history_cap=0)
    assert len(a["ids"]) == 1
    _collect(eng, ta, None, sa, sb, H, id_offset=off)
    assert sa.size() > 0


def test_frames_in_flight_and_restored_trackers(eng):
    """Frames still in flight from predict_batch_async are absorbed by the call's collection point (single-scene twins
    fed the same frames); trackers restored with load and with import_scenes continue exactly."""
    dim, H = 64, 10
    ta, tb = _tracker(eng, 2, H, dim), _tracker(eng, 2, H, dim)
    sa, sb = _store(eng, dim), _store(eng, dim)
    d = Driver(1, 60, dim, 0x5EED0300)
    for fr in range(10):
        d.frame([ta, tb], wait=fr % 2 == 1)
        if fr % 4 == 2:   # the frame just enqueued is still in flight
            _collect(eng, ta, tb, sa, sb, H)
    ta, tb = eng.Tracker.load(ta.save()), eng.Tracker.load(tb.save())
    for fr in range(6):
        d.frame([ta, tb])
    _collect(eng, ta, tb, sa, sb, H)
    scenes = np.arange(1, dtype=np.uint64)
    ia, ib = _tracker(eng, 2, H, dim), _tracker(eng, 2, H, dim)
    ia.import_scenes(ta.export_scenes(scenes, remove=True))
    ib.import_scenes(tb.export_scenes(scenes, remove=True))
    _collect(eng, ta, tb, sa, sb, H)   # the old trackers: what they had collected before the export
    for fr in range(8):
        d.frame([ia, ib], wait=fr != 7)
    _collect(eng, ia, ib, sa, sb, H)


def test_freed_blocks_reused_by_the_next_frame(eng):
    """The frame right after the call takes the history blocks the call freed; the rows a later call stores are the
    tracks' own features, checked against the inputs (every record becomes a new track: min_votes is out of reach)."""
    dim, H, K = 24, 6, 64
    t = _tracker(eng, 3, H, dim)
    s = _store(eng, dim, K=K, min_votes=1 << 30)
    d = Driver(2, 30, dim, 0x5EED0400)
    seen = {}

    def feed():
        f = d.wl.next_frame()
        feats = _special(f["features"], d.rng)
        hasf = (d.rng.random(len(feats)) > 0.25).astype(np.uint8)
        r = t.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=feats, has_feature=hasf)
        for i, tid in enumerate(r["ids"]):
            seen.setdefault(int(tid), []).append(feats[i] if hasf[i] else None)

    checked = 0
    for cycle in range(6):
        for _ in range(3):
            feed()
        before = t.feature_history_pool()
        a = s.associate_wasted(t, id_offset=cycle << 32)
        after = t.feature_history_pool()
        assert after["free"] == before["free"] + len(a["ids"])
        feed()   # new tracks take the freed blocks first
        assert t.feature_history_pool()["free"] <= after["free"]
        for i, tid in enumerate(a["ids"]):
            exp = [r for r in seen[int(tid)][-H:] if r is not None]
            assert int(a["feature_counts"][i]) == len(exp)
            if not exp:
                assert not a["queried"][i]
                continue
            cnt, rows = s.fetch(np.array([int(tid) + (cycle << 32)], np.uint64))
            assert cnt[0] == len(exp)
            assert np.array_equal(rows[0, : len(exp)].view(np.uint32), np.stack(exp).view(np.uint32))
            checked += 1
    assert checked > 30


def test_matches_the_oracle_directly(eng):
    """The composed rows through fstore_oracle's ofs_associate: winners and f64 weights match the call exactly."""
    dim, H = 32, 10
    t = _tracker(eng, 3, H, dim)
    s, o = store_pair(distance_filter=1.0, max_observations=3, feature_dim=dim, topn=3, max_distance=1.0)
    d = Driver(2, 40, dim, 0x5EED0500, gaps=True)
    merged = 0
    for fr in range(16):
        d.frame([t])
        if fr % 4 == 3:
            tb = eng.Tracker.load(t.save())
            a = s.associate_wasted(t)
            w = _wasted_visual(eng, tb, len(a["ids"]), H)
            rows, offs, qi = [], [0], []
            for i in range(len(w["ids"])):
                p = w["fp"][i, : w["hc"][i]].astype(bool)
                if p.any():
                    rows.append(w["ft"][i, : w["hc"][i]][p][:, :dim])
                    offs.append(offs[-1] + int(p.sum()))
                    qi.append(i)
            if not qi:
                continue
            r = o.associate(w["ids"][qi], offs, np.concatenate(rows))
            same_results({k: a[k][qi] for k in ("counts", "winners", "weights", "merged")},
                         {k: r[k] for k in ("counts", "winners", "weights", "merged")})
            merged += int(r["merged"].sum())
    assert merged > 0


# ---------------------------------------------------------------------------------------------------------- refusals
def _refused(eng, s, t, code, words, **kw):
    from similari_b200._lib import Sb200Error

    with pytest.raises(Sb200Error) as e:
        s.associate_wasted(t, **kw)
    assert f"status {code}:" in str(e.value), str(e.value)
    for w in words:
        assert w in str(e.value), str(e.value)


def _fed_pair(eng, dim, frames=6, kind=3, hist=5):
    """A tracker holding wasted records, and its clone."""
    ta = _tracker(eng, kind, hist, dim)
    d = Driver(2, 30, dim, 0x5EED0600, gaps=False)
    for _ in range(frames):
        d.frame([ta])
    ta.skip_epochs(3, 0)
    return ta, eng.Tracker.load(ta.save())


def _nothing_moved(eng, ta, tb, s, blob, H=5):
    """After a refusal the records are all still there (a wasted_visual of each twin returns the same) and the store
    blob is unchanged."""
    assert np.array_equal(s.save(), blob)
    a, b = _wasted_visual(eng, ta, 1 << 14, H), _wasted_visual(eng, tb, 1 << 14, H)
    assert len(a["ids"]) > 0
    same_results(a, b)


def test_refusals_before_anything_happens(eng):
    dim = 16
    s = _store(eng, dim)
    blob = s.save()
    sort = eng.Tracker(_opts(1, 5, dim))
    _refused(eng, s, sort, -1, ["not a visual tracker"], cap=4)
    off = eng.Tracker(_opts(3, 5, dim))
    _refused(eng, s, off, -1, ["feature history is off"], cap=4)
    ta, tb = _fed_pair(eng, 24)
    _refused(eng, s, ta, -1, ["feature_dim differs", "24", "16"], cap=1 << 10)
    _nothing_moved(eng, ta, tb, s, blob)
    with pytest.raises(ValueError):
        s.associate_wasted(ta, cap=-1)
    with pytest.raises(ValueError):
        s.associate_wasted(ta, history_cap=-1)
    L = s._L
    assert L.sb200_fstore_associate_wasted(s._h, ta._h, -1, 0, *([None] * 6), 0, *([None] * 10)) == -1
    assert L.sb200_fstore_associate_wasted(s._h, ta._h, 1, 0, *([None] * 6), -1, *([None] * 10)) == -1
    assert L.sb200_fstore_associate_wasted(None, ta._h, 1, 0, *([None] * 6), 1, *([None] * 10)) == -1
    with pytest.raises(TypeError):
        s.associate_wasted(ta._h)


def test_refusal_on_another_device(eng):
    from similari_b200._lib import lib

    if lib().sb200_device_count() < 2:
        pytest.skip("needs two CUDA devices")
    dim = 16
    s = _store(eng, dim, device=1)
    blob = s.save()
    ta, tb = _fed_pair(eng, dim)
    _refused(eng, s, ta, -1, ["device 0", "device 1"])
    _nothing_moved(eng, ta, tb, s, blob)


def test_refusal_of_a_stored_query_id(eng):
    dim = 16
    ta, tb = _fed_pair(eng, dim)
    w = _wasted_visual(eng, eng.Tracker.load(tb.save()), 1 << 14, 5)
    i = int(np.flatnonzero(w["fp"].any(axis=1))[-1])
    s = _store(eng, dim)
    s.add(np.array([w["ids"][i] + np.uint64(9)], np.uint64), np.ones((1, dim), F32))
    blob = s.save()
    _refused(eng, s, ta, -1, ["already stored", str(int(w["ids"][i]) + 9)], id_offset=9)
    _nothing_moved(eng, ta, tb, s, blob)


def test_refusal_at_the_pair_bound(eng):
    """K = 1, d = 8: 2^20 stored tracks x 1,200 one-row queries is past 2^30 pairs; the 4 GB matrix is never made."""
    dim = 8
    ta = _tracker(eng, 3, 5, dim)
    d = Driver(4, 300, dim, 0x5EED0700, gaps=False)
    d.frame([ta])
    for sc in range(4):
        ta.skip_epochs(3, sc)
    tb = eng.Tracker.load(ta.save())
    s = _store(eng, dim, K=1, topn=1)
    n = 1 << 20
    s.add(np.arange(1 << 40, (1 << 40) + n, dtype=np.uint64), np.ones((n, dim), F32))
    blob = s.save()
    _refused(eng, s, ta, -3, ["2^30"])
    _nothing_moved(eng, ta, tb, s, blob)


# ---------------------------------------------------------------------------------------------------------- empty calls
def _launches(eng):
    return int(eng.launch_count())


def test_empty_buffer_and_featureless_records_launch_no_store_kernel(eng):
    dim = 16
    ta = _tracker(eng, 3, 5, dim)
    s = _store(eng, dim)
    _prefill([s], dim, 10, 1)
    blob = s.save()
    d = Driver(2, 20, dim, 0x5EED0800, gaps=False)
    d.frame([ta])
    # nothing wasted yet: the same launches as a wasted_history of a clone
    tb = eng.Tracker.load(ta.save())
    l0 = _launches(eng)
    a = s.associate_wasted(ta)
    l1 = _launches(eng)
    tb.wasted_history()
    l2 = _launches(eng)
    assert len(a["ids"]) == 0 and l1 - l0 == l2 - l1
    # records without any feature: only the count kernel beyond the twin's collection
    f = d.wl.next_frame()
    ta.skip_epochs(3, 0)
    ta.skip_epochs(3, 1)
    ta.clear_wasted()
    ta.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=None)
    ta.skip_epochs(3, 0)
    ta.skip_epochs(3, 1)
    tb = eng.Tracker.load(ta.save())
    l0 = _launches(eng)
    a = s.associate_wasted(ta)
    l1 = _launches(eng)
    b = tb.wasted_history()
    l2 = _launches(eng)
    assert len(a["ids"]) == len(b["ids"]) > 0
    assert not a["queried"].any() and not a["feature_counts"].any() and not a["track_ids"].any()
    assert l1 - l0 == l2 - l1 + 1
    assert np.array_equal(s.save(), blob)
    assert np.array_equal(ta.save(), tb.save())


def test_tracker_without_a_fixed_dimension(eng):
    """A tracker that has never seen a feature is not held to the store's dimension: it has no present rows."""
    t = _tracker(eng, 3, 5, 8)
    s = _store(eng, 64)
    f = Driver(1, 10, 8, 0x5EED0900).wl.next_frame()
    t.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"])
    t.skip_epochs(3, 0)
    a = s.associate_wasted(t)
    assert len(a["ids"]) == 10 and not a["queried"].any() and s.size() == 0


# ---------------------------------------------------------------------------------------------------------- api
def test_api_wasted_to_store(eng):
    """VisualSort / BatchVisualSort.wasted_to_store equals wasted() of a twin tracker (load_state of the tracker's
    save_state) plus FeatureStore.associate."""
    from similari_b200 import api

    dim = 16
    rng = np.random.default_rng(7)

    def opts():
        o = api.VisualSortOptions()
        o.max_idle_epochs(1)
        o.kept_history_length(4)
        o.visual_metric(api.VisualSortMetricType.euclidean(0.7))
        o.visual_minimal_track_length(1)
        return o

    for batch in (False, True):
        a = api.BatchVisualSort(1, 1, opts()) if batch else api.VisualSort(1, opts())
        sa, sb = _store(eng, dim, K=3), _store(eng, dim, K=3)
        cent = rng.standard_normal((12, dim)).astype(F32)
        for fr in range(12):
            keep = [i for i in range(12) if rng.random() > 0.3]
            obs = [api.VisualSortObservation(
                (cent[i] + 0.01 * rng.standard_normal(dim)).astype(F32).tolist() if rng.random() > 0.2 else None,
                None, api.Universal2DBox.new_with_confidence(10.0 + 40 * i, 20.0, 0.0, 0.5, 30.0, 0.9), None)
                for i in keep]
            if batch:
                req = api.VisualSortPredictionBatchRequest()
                for j, o in enumerate(obs):
                    req.add(j % 2, o)
                a.predict(req)
            else:
                s = api.VisualSortObservationSet()
                for o in obs:
                    s.add(o)
                a.predict(s)
            if fr % 3 == 2:
                b = api.load_state(a.save_state())
                got = a.wasted_to_store(sa, id_offset=100)
                ref = b.wasted()
                assert len(got) == len(ref)
                ids, offs, rows, where = [], [0], [], []
                for j, tr in enumerate(ref):
                    fs = [f for f in tr.observed_features if f is not None]
                    if fs:
                        ids.append(tr.id + 100)
                        rows.append(np.asarray(fs, F32)[:, :dim])
                        offs.append(offs[-1] + len(fs))
                        where.append(j)
                exp = [None] * len(ref)
                if ids:
                    r = sb.associate(np.asarray(ids, np.uint64), offs, np.concatenate(rows))
                    for j, tid in zip(where, r["track_ids"]):
                        exp[j] = int(tid)
                for (tr, tid), rt, e in zip(got, ref, exp):
                    assert (tr.id, tr.epoch, tr.scene_id, tr.length) == (rt.id, rt.epoch, rt.scene_id, rt.length)
                    assert [x._row() for x in tr.predicted_boxes] == [x._row() for x in rt.predicted_boxes]
                    assert [x._row() for x in tr.observed_boxes] == [x._row() for x in rt.observed_boxes]
                    assert tid == e
                assert np.array_equal(sa.save(), sb.save())
        assert sa.size() > 0
