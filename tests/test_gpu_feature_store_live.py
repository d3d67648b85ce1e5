"""sb200_scene_observations and sb200_fstore_search_tracks on the device.

Read-back: scene_observations equals the oracle tracker's dump of Track::obs bit for bit (K from 1 to 32, f32 / FP16 /
BF16 feature columns, frames in flight).  Search: search_tracks equals its host composition -- scene_observations, each
found track's present rows in Track::obs order (with their qualities on a quality store), one FeatureStore.search --
bit for bit (f64 weights through uint64 views), across metrics, store K around the tracker's, storage types, voting
rules, retention, gates, classes, id offsets and multi-scene calls, with ids that are not live among the pairs.  Both
blobs are byte-identical after every call, refused ones included, and the next frame equals a clone's that never made
the call."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

from fstore_checks import same_results, store_pair

pytestmark = pytest.mark.gpu

F32 = np.float32
SB200_ERR_INVALID, SB200_ERR_CAPACITY = -1, -3
Q_SET = np.array([0.3, 0.5, 0.5, 0.8, 0.8, 1.0, 1.0, np.nextafter(F32(0.5), F32(0))], F32)


@pytest.fixture(scope="module")
def eng():
    import similari_b200.engine as e
    from similari_b200._lib import lib

    if lib().sb200_device_count() <= 0:
        pytest.fail("no CUDA device: the gpu-marked tests must run on an H100")
    return e


def _kw(K, dim, kind=3, **over):
    kw = dict(kind=kind, positional_kind=1, iou_threshold=0.3, max_idle_epochs=1, visual_kind=0, visual_threshold=0.7,
              feature_dim=dim, visual_max_observations=K, visual_min_votes=1, visual_minimal_track_length=1,
              min_confidence=0.1, visual_minimal_quality_use=0.8, visual_minimal_quality_collect=0.5)
    kw.update(over)
    return kw


def _tracker(eng, K, dim, **over):
    from similari_b200._lib import default_options

    return eng.Tracker(default_options(**_kw(K, dim, **over)))


def _typed(feats, ftype):
    """The column as the tracker is fed it, and the f32 values it widens to (what the oracle is fed)."""
    if ftype == "f32":
        return feats, None, feats
    if ftype == "f16":
        h = feats.astype(np.float16)
        return h, None, h.astype(F32)
    u = feats.view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)
    return r, "bf16", (r.astype(np.uint32) << 16).view(F32)


class Driver:
    """Seeded frames with qualities from a set full of ties and the collect threshold, and a fifth of the detections
    without a feature."""

    def __init__(self, n_scenes, n_objects, dim, seed, ftype="f32"):
        from similari_b200.workload import CONFIGS, Workload

        cfg = dataclasses.replace(CONFIGS["cfg5"], n_scenes=n_scenes, n_objects=n_objects, feature_dim=dim,
                                  oriented=False, canvas=(1200.0, 800.0), drop_frac=0.2, fresh_frac=0.15, seed=seed)
        self.wl, self.rng, self.ftype = Workload(cfg), np.random.default_rng(seed), ftype

    def frame(self, trackers, oracles=(), wait=True):
        f = self.wl.next_frame()
        n = len(f["boxes"])
        q = self.rng.choice(Q_SET, n).astype(F32)
        hasf = (self.rng.random(n) >= 0.2).astype(np.uint8)
        col, ft, wide = _typed(f["features"], self.ftype)
        args = (f["scene_ids"], f["det_offsets"], f["boxes"])
        for t in trackers:
            t.predict_batch(*args, features=col, has_feature=hasf, quality=q, feature_type=ft, wait=wait)
        for o in oracles:
            o.predict_batch(*args, features=wide, has_feature=hasf, quality=q)
        return f


# ---------------------------------------------------------------------------------------------------------- read-back
def _oracle_live(o, sid, max_idle):
    """Positions of the oracle's tracks the device still holds (it sweeps expired tracks at the end of their frame, the
    oracle at its next collection point)."""
    cur = o.current_epoch(sid)
    ep = {int(i): int(e) for i, e in zip(*(o.idle_tracks(sid)[k] for k in ("ids", "epochs")))}
    ids = o.scene_tracks(sid)["ids"]
    return [j for j, i in enumerate(ids) if ep.get(int(i), cur) + max_idle >= cur]


def _check_against_oracle(g, o, scene_ids, dim, where):
    for sid in map(int, scene_ids):
        a = g.scene_observations(sid)
        live = _oracle_live(o, sid, 1)
        ob = o.scene_observations(sid)
        assert a["ids"].tolist() == o.scene_tracks(sid)["ids"][live].tolist(), (where, sid)
        assert a["ids"].tolist() == g.scene_tracks(sid)["ids"].tolist(), (where, sid)
        want = {"ids": a["ids"], "n_obs": ob["n_obs"][live], "has_feat": ob["has_feat"][live],
                "quality": ob["quality"][live], "feats": np.ascontiguousarray(ob["feats"][live][:, :, :dim])}
        same_results(a, want)


CASES = [(1, "f32"), (3, "f32"), (5, "f16"), (8, "bf16"), (25, "f32"), (32, "bf16")]


@pytest.mark.parametrize("K,ftype", CASES, ids=[f"K{k}-{t}" for k, t in CASES])
def test_scene_observations_match_the_oracle(eng, oracle, K, ftype):
    dim = 20 if K % 2 else 64
    g = _tracker(eng, K, dim)
    o = oracle.Tracker(oracle.make_options(**_kw(K, dim)))
    d = Driver(3, 40, dim, 0x0B5E0000 + K, ftype)
    seen = 0
    for fr in range(12):
        f = d.frame([g], [o])
        _check_against_oracle(g, o, f["scene_ids"], dim, fr)
        seen += int(g.scene_observations(int(f["scene_ids"][0]))["n_obs"].sum())
    assert seen > 0
    empty = g.scene_observations(987654321)
    assert len(empty["ids"]) == 0 and empty["feats"].shape == (0, K, dim)


def test_scene_observations_with_frames_in_flight(eng, oracle):
    K, dim = 5, 32
    g = _tracker(eng, K, dim)
    o = oracle.Tracker(oracle.make_options(**_kw(K, dim)))
    d = Driver(2, 50, dim, 0x0F1F)
    for fr in range(9):
        f = d.frame([g], [o], wait=False)
        if fr % 3 == 2:   # up to three frames still enqueued: the call drains them first
            _check_against_oracle(g, o, f["scene_ids"], dim, fr)


# ---------------------------------------------------------------------------------------------------------- search
def _compose(t, s, scene_ids, track_ids, id_offset=0, feature_class=None, attrs=None):
    """The host composition the call must equal."""
    n, topn = len(track_ids), s.topn
    obs = {int(sid): t.scene_observations(int(sid)) for sid in set(map(int, scene_ids))}
    res = {"found": np.zeros(n, bool), "feature_counts": np.zeros(n, np.int32), "queried": np.zeros(n, bool),
           "counts": np.zeros(n, np.int32), "winners": np.zeros((n, topn), np.uint64),
           "weights": np.zeros((n, topn), np.float64)}
    rows, qual, offs, qi = [], [], [0], []
    for i, (sid, tid) in enumerate(zip(map(int, scene_ids), map(int, track_ids))):
        ob = obs[sid]
        hit = np.flatnonzero(ob["ids"] == np.uint64(tid))
        if len(hit) == 0:
            continue
        j = int(hit[0])
        p = ob["has_feat"][j, : ob["n_obs"][j]].astype(bool)
        res["found"][i], res["feature_counts"][i] = True, int(p.sum())
        if p.any():
            rows.append(ob["feats"][j, : ob["n_obs"][j]][p])
            qual.append(ob["quality"][j, : ob["n_obs"][j]][p])
            offs.append(offs[-1] + int(p.sum()))
            qi.append(i)
    res["queried"][qi] = True
    if qi:
        qid = (np.asarray(track_ids, np.uint64)[qi] + np.uint64(id_offset)).astype(np.uint64)
        kw = {k: np.asarray(v)[qi] for k, v in (attrs or {}).items()}
        if s.retention()[0] == "quality":
            kw["quality"] = np.concatenate(qual)
        r = s.search(qid, offs, np.concatenate(rows), feature_class=feature_class, **kw)
        for k in ("counts", "winners", "weights"):
            res[k][qi] = r[k]
    return res


def _gallery(s, t, scene_ids, n_extra, seed, attrs_of=None, **kw):
    """Stores noisy copies of the tracker's present rows (so that searches find them) and random rows."""
    rng = np.random.default_rng(seed)
    rows = []
    for sid in scene_ids:
        ob = t.scene_observations(int(sid))
        rows += [ob["feats"][j, k] for j in range(len(ob["ids"])) for k in range(ob["n_obs"][j]) if ob["has_feat"][j, k]]
    D = int(t.opts.feature_dim)
    rows = np.array(rows, F32).reshape(-1, D)[:: 2]
    rows = rows + rng.standard_normal(rows.shape).astype(F32) * F32(0.02)
    rows = np.concatenate([rows, rng.standard_normal((n_extra, D)).astype(F32)])
    ids = np.arange(1 << 40, (1 << 40) + len(rows), dtype=np.uint64) // np.uint64(2)   # two rows per stored track
    extra = attrs_of(ids) if attrs_of else {}
    if s.retention()[0] == "quality":
        extra["quality"] = rng.choice(Q_SET, len(rows)).astype(F32)
    s.add(ids, rows, **extra, **kw)


def _pairs(t, scene_ids, gone, rng):
    """Every live track of the scenes, shuffled, plus ids that are not live: expired ones, unknown ones and an unknown
    scene."""
    sc, ti = [], []
    for sid in scene_ids:
        ids = t.scene_tracks(int(sid))["ids"]
        sc += [int(sid)] * len(ids)
        ti += list(map(int, ids))
    for i, (sid, tid) in enumerate(gone[:6]):
        sc.append(sid)
        ti.append(tid)
    sc += [int(scene_ids[0]), 424242]
    ti += [(1 << 63) + 5, int(ti[0]) if ti else 1]
    perm = rng.permutation(len(sc))
    return np.array(sc, np.uint64)[perm], np.array(ti, np.uint64)[perm]


def _store(eng, dim, metric="euclidean", K=3, storage="f32", topn=3, **kw):
    thr = 1.0 if metric == "euclidean" else 0.3
    return eng.FeatureStore(metric=metric, distance_filter=thr, max_observations=K, feature_dim=dim, topn=topn,
                            max_distance=thr, min_votes=1, storage=storage, **kw)


SEARCH = [
    dict(name="euclid-Kbelow", K=2),
    dict(name="euclid-Kequal", K=5),
    dict(name="euclid-Kabove", K=8),
    dict(name="cosine", metric="cosine", K=3),
    dict(name="fp16", storage="f16", K=4),
    dict(name="bf16-cosine", storage="bf16", metric="cosine", K=6),
    dict(name="bestfit", voting="best_fit", K=3, topn=2),
    dict(name="bestfit-cosine", voting="best_fit", metric="cosine", K=7),
    dict(name="quality", retention="quality", initial_capacity=2, merge_extension=1.5, K=6),
    dict(name="quality-bestfit", retention="quality", initial_capacity=4, merge_extension=1.0, voting="best_fit", K=4),
    dict(name="same-source", gate="same_source", K=3),
    dict(name="any-source-quality", gate="any_source", retention="quality", initial_capacity=3, K=5),
    dict(name="classes", classes={7: 16, 9: 40, 11: 8}, feature_class=9, K=3),
    dict(name="offset-wrap", id_offset=(1 << 64) - 3, K=3),
]


@pytest.mark.parametrize("case", SEARCH, ids=[c["name"] for c in SEARCH])
def test_search_tracks_equals_the_host_composition(eng, case):
    case = dict(case)
    name, fclass, off = case.pop("name"), case.pop("feature_class", None), case.pop("id_offset", 0)
    dim = 40
    t = _tracker(eng, 5, dim)
    s = _store(eng, dim if "classes" not in case else 16, **case)
    gated = "gate" in case
    rng = np.random.default_rng(sum(map(ord, name)))
    d = Driver(3, 60, dim, 0x5EA0 + sum(map(ord, name)))
    prev = {}
    gone = []
    for fr in range(8):
        f = d.frame([t])
        cur = {(int(sid), int(i)) for sid in f["scene_ids"] for i in t.scene_tracks(int(sid))["ids"]}
        gone += sorted(set(prev) - cur)
        prev = dict.fromkeys(cur)
    scenes = list(map(int, f["scene_ids"]))

    def attrs_of(ids):
        n = len(ids)
        return dict(sources=(ids % np.uint64(2)).astype(np.uint64), t_start=(np.arange(n) % 7).astype(np.int64),
                    t_end=(np.arange(n) % 7 + 3).astype(np.int64))

    _gallery(s, t, scenes, 200, 0x6A11, attrs_of if gated else None, feature_class=fclass)
    sc, ti = _pairs(t, scenes, gone, rng)
    assert len(gone) > 0
    attrs = None
    if gated:   # windows that miss some stored windows and touch others
        n = len(ti)
        attrs = dict(sources=rng.integers(0, 2, n).astype(np.uint64), t_start=rng.integers(0, 12, n).astype(np.int64))
        attrs["t_end"] = attrs["t_start"] + rng.integers(0, 3, n).astype(np.int64)
    tb, sb = t.save(), s.save()   # the tracker blob carries the wasted buffer and its count
    a = s.search_tracks(t, sc, ti, id_offset=off, feature_class=fclass, **(attrs or {}))
    assert np.array_equal(t.save(), tb) and np.array_equal(s.save(), sb)
    b = _compose(t, s, sc, ti, off, fclass, attrs)
    same_results(a, b)
    n_gone = min(len(gone), 6)
    assert a["found"].sum() == len(ti) - n_gone - 2   # every live track; no expired, unknown or unknown-scene pair
    assert (a["counts"] > 0).sum() > 0, "no query found a stored track: the case checks nothing"


def test_next_frames_equal_a_twin_that_never_searched(eng):
    """A clone taken before the call, fed the same frames after it, ends in the same blob.  One scene: a multi-scene
    frame appends its scenes' wasted records in the order their blocks finish, so two trackers' buffers may differ in
    order whatever this call does."""
    dim = 32
    t = _tracker(eng, 5, dim)
    s = _store(eng, dim, K=3)
    d = Driver(1, 80, dim, 0x7A1)
    for _ in range(5):
        f = d.frame([t])
    scenes = list(map(int, f["scene_ids"]))
    _gallery(s, t, scenes, 50, 3)
    twin = eng.Tracker.load(t.save())
    sc, ti = _pairs(t, scenes, [], np.random.default_rng(1))
    s.search_tracks(t, sc, ti)
    for _ in range(3):
        f = d.wl.next_frame()
        args = (f["scene_ids"], f["det_offsets"], f["boxes"])
        ra = t.predict_batch(*args, features=f["features"])
        rb = twin.predict_batch(*args, features=f["features"])
        for k in ("ids", "epochs", "lengths", "voting_types"):
            assert np.array_equal(np.asarray(ra[k]), np.asarray(rb[k])), k
        assert np.array_equal(t.save(), twin.save())


def test_matches_the_oracles_directly(eng, oracle):
    """The oracle tracker fed the same frames, its scene_observations' present rows through fstore_oracle's search."""
    K, dim = 5, 24
    g = _tracker(eng, K, dim)
    o = oracle.Tracker(oracle.make_options(**_kw(K, dim)))
    s, so = store_pair(distance_filter=1.0, max_observations=3, feature_dim=dim, topn=3, max_distance=1.0)
    d = Driver(2, 40, dim, 0x0AC1E)
    for _ in range(6):
        f = d.frame([g], [o])
    scenes = list(map(int, f["scene_ids"]))
    rng = np.random.default_rng(5)
    rows = np.concatenate([g.scene_observations(sid)["feats"].reshape(-1, dim) for sid in scenes])
    rows = rows[np.abs(rows).sum(axis=1) > 0][::3]
    rows = rows + rng.standard_normal(rows.shape).astype(F32) * F32(0.02)
    ids = np.arange(500, 500 + len(rows), dtype=np.uint64)
    s.add(ids, rows)
    so.add(ids, rows)
    sc, ti = _pairs(g, scenes, [], rng)
    a = s.search_tracks(g, sc, ti)
    qrows, offs, qi = [], [0], []
    for i, (sid, tid) in enumerate(zip(map(int, sc), map(int, ti))):
        if sid not in scenes:
            continue
        live = _oracle_live(o, sid, 1)
        ob = o.scene_observations(sid)
        ids_o = o.scene_tracks(sid)["ids"][live]
        hit = np.flatnonzero(ids_o == np.uint64(tid))
        if len(hit) == 0:
            continue
        j = live[int(hit[0])]
        p = ob["has_feat"][j, : ob["n_obs"][j]].astype(bool)
        if p.any():
            qrows.append(ob["feats"][j, : ob["n_obs"][j]][p][:, :dim])
            offs.append(offs[-1] + int(p.sum()))
            qi.append(i)
    assert np.flatnonzero(a["queried"]).tolist() == qi
    r = so.search(ti[qi], offs, np.concatenate(qrows))
    same_results({k: a[k][qi] for k in r}, r)
    assert r["counts"].sum() > 0


def test_api_search_store(eng):
    """VisualSort / BatchVisualSort.search_store: the SortTracks a predict returned, looked up in a store; the result is
    search_tracks' per pair."""
    from similari_b200 import api

    dim = 16
    rng = np.random.default_rng(9)
    cent = rng.standard_normal((6, dim)).astype(F32)

    def opts():
        o = api.VisualSortOptions()
        o.max_idle_epochs(2)
        o.visual_metric(api.VisualSortMetricType.euclidean(0.7))
        o.visual_minimal_track_length(1)
        o.visual_max_observations(4)
        return o

    for batch in (False, True):
        a = api.BatchVisualSort(1, 1, opts()) if batch else api.VisualSort(1, opts())
        store = _store(eng, dim, K=3, topn=2)
        assert a.search_store(store, []) == []
        store.add(np.array([11, 12], np.uint64), cent[:2])
        for fr in range(3):
            obs = [api.VisualSortObservation((cent[i] + 0.001 * rng.standard_normal(dim)).astype(F32).tolist()
                                             if i != 5 else None, 0.9,
                                             api.Universal2DBox.new_with_confidence(10.0 + 60 * i, 20.0, 0.0, 0.5, 30.0,
                                                                                    0.9), None) for i in range(6)]
            if batch:
                req = api.VisualSortPredictionBatchRequest()
                for j, o in enumerate(obs):
                    req.add(j % 2, o)
                res = a.predict(req)
                tracks = [t for _ in range(res.batch_size()) for t in res.get()[1]]
            else:
                s = api.VisualSortObservationSet()
                for o in obs:
                    s.add(o)
                tracks = a.predict(s)
        out = a.search_store(store, tracks)
        r = store.search_tracks(a._t, [t.scene_id for t in tracks], [t.id for t in tracks])
        assert [t for t, _ in out] == tracks
        for i, (t, got) in enumerate(out):
            if not r["queried"][i]:
                assert got is None
                continue
            assert got == [(int(r["winners"][i, e]), float(r["weights"][i, e])) for e in range(int(r["counts"][i]))]
        assert {w for _, got in out if got for w, _ in got} == {11, 12}
        assert sum(got is None for _, got in out) == 1   # the track without a feature


# ---------------------------------------------------------------------------------------------------------- refusals
def _refused(fn, code, words):
    from similari_b200._lib import Sb200Error

    with pytest.raises(Sb200Error) as e:
        fn()
    assert f"status {code}:" in str(e.value), str(e.value)
    assert words in str(e.value), str(e.value)


def test_refusals_change_nothing(eng):
    from similari_b200._lib import default_options

    dim = 16
    t = _tracker(eng, 5, dim)
    d = Driver(1, 60, dim, 0x4EF)
    for _ in range(4):
        f = d.frame([t])
    sid = int(f["scene_ids"][0])
    ids = t.scene_tracks(sid)["ids"]
    s = _store(eng, dim)
    s.add(np.arange(1, 9, dtype=np.uint64), np.random.default_rng(0).standard_normal((8, dim)).astype(F32))
    tb, sb = t.save(), s.save()

    def same():
        assert np.array_equal(t.save(), tb) and np.array_equal(s.save(), sb)

    _refused(lambda: s.search_tracks(t, [sid, sid], [ids[0], ids[0]]), SB200_ERR_INVALID, "twice")
    same()
    plain = eng.Tracker(default_options(kind=1, positional_kind=1))
    _refused(lambda: s.search_tracks(plain, [sid], [ids[0]]), SB200_ERR_INVALID, "not a visual")
    _refused(lambda: plain.scene_observations(0), SB200_ERR_INVALID, "not a visual")
    wide = _store(eng, dim + 8)
    _refused(lambda: wide.search_tracks(t, [sid], [ids[0]]), SB200_ERR_INVALID, "feature_dim")
    cls = _store(eng, dim, classes={1: dim, 2: dim + 1})
    _refused(lambda: cls.search_tracks(t, [sid], [ids[0]], feature_class=2), SB200_ERR_INVALID, "feature_dim")
    g = _store(eng, dim, gate="same_source")
    from similari_b200._lib import check, lib, ptr

    L = lib()
    one = np.array([sid], np.uint64), np.array([ids[0]], np.uint64)
    attrs, cols = g._attrs(1, [0], [0], [1])

    def raw(store, n=1, a=None):
        return lambda: check(L.sb200_fstore_search_tracks(store._h, t._h, n, ptr(one[0]), ptr(one[1]), 0,
                                                          C.byref(a) if a is not None else None, *([None] * 6)))

    _refused(raw(g), SB200_ERR_INVALID, "gated")
    _refused(raw(s, a=attrs), SB200_ERR_INVALID, "ungated")
    _refused(raw(s, n=-1), SB200_ERR_INVALID, "n < 0")
    _refused(lambda: g.search_tracks(t, [sid], [ids[0]], sources=[0], t_start=[5], t_end=[1]), SB200_ERR_INVALID,
             "t_start")
    same()
    # a NaN quality on a quality store: a track created from a detection of NaN quality keeps it
    tq = _tracker(eng, 3, dim)
    fq = d.wl.next_frame()
    q = np.full(len(fq["boxes"]), np.nan, F32)
    tq.predict_batch(fq["scene_ids"], fq["det_offsets"], fq["boxes"], features=fq["features"], quality=q)
    sq = int(fq["scene_ids"][0])
    obq = tq.scene_observations(sq)
    assert np.isnan(obq["quality"][obq["has_feat"].astype(bool)]).all() and obq["has_feat"].any()
    qs = _store(eng, dim, retention="quality")
    qb, tqb = qs.save(), tq.save()
    _refused(lambda: qs.search_tracks(tq, [sq], [obq["ids"][0]]), SB200_ERR_INVALID, "NaN")
    assert np.array_equal(qs.save(), qb) and np.array_equal(tq.save(), tqb)
    # the pair bound (request rows x stored tracks x max_observations > 2^30) on a store of small D
    R = int(s.search_tracks(t, [sid] * len(ids), ids)["feature_counts"].sum())   # every row kept: p <= 5 <= K
    Kb = 8
    live = (1 << 30) // (R * Kb) + 1
    big = eng.FeatureStore(metric="euclidean", distance_filter=1.0, max_observations=Kb, feature_dim=dim, topn=1,
                           max_distance=1.0, min_votes=1)
    big.add(np.arange(live, dtype=np.uint64), np.zeros((live, dim), F32))
    bb = big.save()
    _refused(lambda: big.search_tracks(t, [sid] * len(ids), ids), SB200_ERR_CAPACITY, "2^30")
    assert np.array_equal(big.save(), bb)
    same()


def test_no_pair_and_no_feature_launch_no_store_kernel(eng):
    from similari_b200._lib import lib

    L = lib()
    dim = 16
    t = _tracker(eng, 3, dim)
    s = _store(eng, dim)
    s.add(np.arange(4, dtype=np.uint64), np.ones((4, dim), F32))
    f = Driver(1, 20, dim, 0x11).wl.next_frame()
    t.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"])   # no feature column: no present observation
    sid = int(f["scene_ids"][0])
    ids = t.scene_tracks(sid)["ids"]
    t.sync()
    n0 = L.sb200_launch_count()
    r = s.search_tracks(t, [], [])
    assert L.sb200_launch_count() == n0 and len(r["found"]) == 0
    r = s.search_tracks(t, [sid] * len(ids), ids)
    assert L.sb200_launch_count() == n0 + 1   # the lookup alone
    assert r["found"].all() and not r["queried"].any() and not r["counts"].any()
