"""CPU checks of the live-track calls (sb200_scene_observations, sb200_fstore_search_tracks).

The query rule of search_tracks on the oracles alone: an oracle tracker is fed a scripted track (quality ties,
feature-less detections, a merge below the collect threshold), its scene_observations give Track::obs, and each track's
present rows in that order go to an fstore_oracle search.  A store keeps the last max_observations rows of a query, so
with the store's K below the tracker's present count the NEWEST observation is the one dropped (optimize swaps it to
the front); one case pins that by hand.  The entry points refuse NULL handles without touching a device."""
import ctypes as C

import numpy as np
import pytest

D = 12
Q_COLLECT = 0.4
# (quality, has_feature) of detection 0 (the new track) and of every merge after it
SCRIPT = [(0.5, True), (0.5, True), (0.9, True), (0.3, False), (0.5, True), (0.3, True), (0.9, True), (0.7, False),
          (0.5, True), (0.4, True), (np.nextafter(np.float32(0.4), np.float32(0)), True), (0.6, True)]


@pytest.fixture(scope="module")
def L():
    from similari_b200 import _build, _lib

    _build.build()
    return _lib.lib()


def _tracker(oracle, K):
    return oracle.Tracker(oracle.make_options(kind=oracle.KIND_VISUAL_SORT, positional_kind=oracle.POS_IOU,
                                              iou_threshold=0.3, max_idle_epochs=3, feature_dim=D,
                                              visual_max_observations=K, visual_minimal_track_length=1,
                                              visual_minimal_quality_collect=Q_COLLECT))


def _feed(oracle, o, steps, seed):
    """One track merged frame after frame by SCRIPT[:steps]; returns the features fed."""
    rng = np.random.default_rng(seed)
    box = oracle.box(100.0, 80.0, None, 0.5, 60.0, 0.9)
    feats = []
    for q, hf in SCRIPT[:steps]:
        f = rng.standard_normal(D).astype(np.float32)
        f /= np.linalg.norm(f)
        o.predict_batch([0], [0, 1], box[None], features=f[None], has_feature=[hf], quality=[np.float32(q)])
        feats.append(f)
    return feats


def _present(obs, i):
    """Track i's present rows in Track::obs order and their qualities."""
    p = obs["has_feat"][i, : obs["n_obs"][i]].astype(bool)
    return obs["feats"][i, : obs["n_obs"][i]][p][:, :D], obs["quality"][i, : obs["n_obs"][i]][p]


def _gallery(fo, rows, K, **kw):
    s = fo.FeatureStore(metric=fo.EUCLIDEAN, distance_filter=2.0, max_observations=K, feature_dim=D, topn=4,
                        max_distance=2.0, min_votes=1, **kw)
    ids = np.arange(100, 100 + len(rows), dtype=np.uint64)
    if kw.get("retention") == "quality":
        s.add(ids, rows, quality=np.ones(len(rows), np.float32))
    else:
        s.add(ids, rows)
    return s, ids


@pytest.mark.parametrize("K,Ks", [(5, 2), (5, 5), (5, 8), (3, 1), (8, 3), (1, 1)])
def test_store_keeps_the_last_rows_of_track_obs(oracle, K, Ks):
    """The composition (every present row, Track::obs order) searches as the last min(p, K_store) rows alone do."""
    import fstore_oracle as fo

    o = _tracker(oracle, K)
    feats = _feed(oracle, o, len(SCRIPT), 0x11FE + K)
    obs = o.scene_observations(0)
    rows, _ = _present(obs, 0)
    p = len(rows)
    assert p == int(o.scene_tracks(0)["feat_counts"][0]) and p >= 1
    noise = np.random.default_rng(K).standard_normal((len(feats), D)).astype(np.float32) * np.float32(0.05)
    s, _ = _gallery(fo, np.stack(feats) + noise, Ks)
    whole = s.search([7], [0, p], rows)
    big, _ = _gallery(fo, np.stack(feats) + noise, max(p, Ks))
    last = big.search([7], [0, min(p, Ks)], rows[p - min(p, Ks):])
    for k in ("counts", "winners"):
        assert np.array_equal(whole[k], last[k]), k
    assert np.array_equal(whole["weights"].view(np.uint64), last["weights"].view(np.uint64))


def test_a_smaller_store_drops_the_newest_observation(oracle):
    """Tracker K = 3 after the detections (0.5, f0), (0.9, f1), (0.5, f2): optimize leaves [f2, f0, f1] (the newest
    swapped to the front, the best at the end).  A store with K = 2 keeps [f0, f1]: the stored copy of f2 is not found;
    with K = 3 it is."""
    import fstore_oracle as fo

    o = _tracker(oracle, 3)
    rng = np.random.default_rng(0x2F)
    box = oracle.box(100.0, 80.0, None, 0.5, 60.0, 0.9)
    f = rng.standard_normal((3, D)).astype(np.float32) * np.float32(10.0)   # far apart: each row matches only itself
    for i, q in enumerate((0.5, 0.9, 0.5)):
        o.predict_batch([0], [0, 1], box[None], features=f[i][None], has_feature=[1], quality=[np.float32(q)])
    obs = o.scene_observations(0)
    rows, qual = _present(obs, 0)
    assert np.array_equal(rows, f[[2, 0, 1]]) and qual.tolist() == [np.float32(0.5), np.float32(0.5), np.float32(0.9)]
    got = {}
    for Ks in (2, 3):
        s, ids = _gallery(fo, f, Ks)
        r = s.search([7], [0, 3], rows)
        got[Ks] = set(r["winners"][0, : r["counts"][0]].tolist())
    assert got[2] == {100, 101} and got[3] == {100, 101, 102}


@pytest.mark.parametrize("K", [2, 5])
def test_quality_store_takes_the_best_rows_with_the_tracker_qualities(oracle, K):
    """On a quality store every row carries its observation's quality; the store keeps the best c(1) of them, stably,
    whatever their order in Track::obs."""
    import fstore_oracle as fo

    o = _tracker(oracle, K)
    feats = _feed(oracle, o, len(SCRIPT), 0x3C + K)
    rows, qual = _present(o.scene_observations(0), 0)
    s, _ = _gallery(fo, np.stack(feats), 8, retention="quality", initial_capacity=2, merge_extension=1.0)
    whole = s.search([7], [0, len(rows)], rows, quality=qual)
    keep = np.argsort(-qual, kind="stable")[:2]
    best = s.search([7], [0, len(keep)], rows[keep], quality=qual[keep])
    for k in ("counts", "winners"):
        assert np.array_equal(whole[k], best[k]), k
    assert np.array_equal(whole["weights"].view(np.uint64), best["weights"].view(np.uint64))


def test_featureless_tracks_are_not_queried(oracle):
    o = _tracker(oracle, 3)
    box = oracle.box(100.0, 80.0, None, 0.5, 60.0, 0.9)
    for _ in range(3):
        o.predict_batch([0], [0, 1], box[None], features=np.zeros((1, D), np.float32), has_feature=[0], quality=[1.0])
    obs = o.scene_observations(0)
    assert obs["n_obs"].tolist() == [1] and not obs["has_feat"].any()
    assert len(_present(obs, 0)[0]) == 0


def test_null_handles_without_a_device(L):
    fake = C.c_void_p(16)   # never dereferenced: the handles are checked first
    assert L.sb200_scene_observations(None, 0, 1, *([None] * 5)) == -1
    assert b"NULL" in L.sb200_last_error()
    for s, t in ((None, None), (None, fake), (fake, None)):
        assert L.sb200_fstore_search_tracks(s, t, 0, None, None, 0, *([None] * 7)) == -1
        assert b"NULL" in L.sb200_last_error()


def test_python_wrapper_validates_its_arguments():
    from similari_b200 import engine

    s = engine.FeatureStore.__new__(engine.FeatureStore)   # no device: never reaches the library
    s._h, s.topn, s.gate = None, 1, None
    t = engine.Tracker.__new__(engine.Tracker)
    t._h, t.opts = None, None
    with pytest.raises(TypeError):
        s.search_tracks(object(), [0], [1])
    for off in (-1, 1 << 64):
        with pytest.raises(ValueError):
            s.search_tracks(t, [0], [1], id_offset=off)
    with pytest.raises(ValueError):
        s.search_tracks(t, [0, 1], [1])
    with pytest.raises(ValueError):
        s.search_tracks(t, [0], [1], sources=[0], t_start=[0], t_end=[1])   # an ungated store takes no windows
