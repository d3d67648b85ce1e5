"""CPU checks of the feature track store: the oracle's TopN voting against the known answers of
src/track/voting/topn.rs, the oracle's store semantics on hand-built cases (keep-newest-K, same-id skip, the strict
distance filter, max_dist across the queries of a call, min_votes, the tie order)."""
import numpy as np
import pytest

import fstore_oracle as fo

TOPN_RS = [(0, 1, 0.2), (0, 1, 0.22), (0, 2, 0.21), (0, 2, 0.2), (0, 3, 0.22), (0, 3, 0.2)]


def _sorted(res):
    return {q: sorted(v) for q, v in res.items()}


def test_topn_default_voting():
    """default_voting (topn.rs:143-226), after the same sort by winner id."""
    v = lambda ents: _sorted(fo.topn_voting(5, 0.32, 1, ents))
    assert v([(0, 1, 0.2)]) == {0: [(1, 0.0)]}
    assert v([(0, 1, 0.2), (0, 1, 0.3)]) == {0: [(1, 0.10000000894069672)]}
    assert v([(0, 1, 0.2), (0, 1, 0.4)]) == {0: [(1, 0.20000000298023224)]}
    assert v([(0, 1, 0.2), (0, 2, 0.2)]) == {0: [(1, 0.0), (2, 0.0)]}
    ents = TOPN_RS + [(0, 4, 0.23), (0, 4, 0.3), (0, 5, 0.24), (0, 5, 0.3), (0, 6, 0.25), (0, 6, 0.5)]
    assert v(ents) == {0: [(1, 0.5800000131130219), (2, 0.5900000333786011), (3, 0.5800000131130219),
                           (4, 0.4699999690055847), (5, 0.4599999785423279)]}


def test_topn_two_query_vecs():
    """two_query_vecs (topn.rs:228-276): max_dist is shared by both queries."""
    ents = TOPN_RS + [(7, 4, 0.23), (7, 4, 0.3), (7, 5, 0.24), (7, 5, 0.3), (7, 6, 0.25), (7, 6, 0.5)]
    assert _sorted(fo.topn_voting(5, 0.32, 1, ents)) == {
        0: [(1, 0.5800000131130219), (2, 0.5900000333786011), (3, 0.5800000131130219)],
        7: [(4, 0.4699999690055847), (5, 0.4599999785423279), (6, 0.250)]}


def test_topn_none_distance_is_skipped():
    assert fo.topn_voting(5, 0.32, 1, [(0, 1, None), (0, 2, 0.3)]) == {0: [(2, 0.0)]}


def _store(**kw):
    base = dict(metric=fo.EUCLIDEAN, distance_filter=100.0, max_observations=2, feature_dim=1, topn=5,
                max_distance=100.0, min_votes=1)
    base.update(kw)
    return fo.FeatureStore(**base)


def _q(ids, rows_per_query):
    offs = np.cumsum([0] + [len(r) for r in rows_per_query]).astype(np.int32)
    feats = np.array([x for r in rows_per_query for x in r], np.float32).reshape(-1, 1)
    return np.array(ids, np.uint64), offs, feats


def test_keep_newest_on_add():
    s = _store()
    s.add([1, 2, 1, 1], np.array([[1.0], [5.0], [2.0], [3.0]], np.float32))
    assert list(s.ids()) == [1, 2]
    cnt, f = s.fetch([1, 2])
    assert list(cnt) == [2, 1]
    assert f[0, :, 0].tolist() == [2.0, 3.0] and f[1, 0, 0] == 5.0


def test_keep_newest_on_merge_and_new_tracks_in_query_order():
    s = _store(max_distance=1.5)
    s.add([1, 2], np.array([[0.0], [50.0]], np.float32))
    r = s.associate(*_q([10, 11, 12], [[1.0], [30.0], [0.5, 1.0]]))
    assert r["merged"].tolist() == [1, 0, 1]
    assert r["track_ids"].tolist() == [1, 11, 1]
    assert list(s.ids()) == [1, 2, 11]
    cnt, f = s.fetch([1])
    # track 1: 0.0, then query 10's 1.0, then query 12's 0.5, 1.0 -> newest two
    assert cnt[0] == 2 and f[0, :, 0].tolist() == [0.5, 1.0]


def test_query_keeps_only_its_newest_observations():
    s = _store(max_distance=1.0, max_observations=2)
    s.add([1], np.array([[0.0]], np.float32))
    # the oldest observation (0.0) would vote for track 1; with K = 2 it does not take part
    r = s.search(*_q([9], [[0.0, 40.0, 41.0]]))
    assert r["counts"].tolist() == [0]
    r = s.search(*_q([9], [[40.0, 0.0, 41.0]]))
    assert r["counts"].tolist() == [1] and r["winners"][0, 0] == 1


def test_same_id_is_skipped():
    s = _store()
    s.add([5, 6], np.array([[0.0], [1.0]], np.float32))
    r = s.search(*_q([5], [[0.0]]))
    assert r["counts"].tolist() == [1] and r["winners"][0, 0] == 6


def test_filter_is_strict_and_max_distance_inclusive():
    s = _store(distance_filter=3.0, max_distance=3.0)
    s.add([1], np.array([[0.0]], np.float32))
    assert s.search(*_q([9], [[3.0]]))["counts"].tolist() == [0]   # d == filter: dropped
    s = _store(distance_filter=3.5, max_distance=3.0)
    s.add([1], np.array([[0.0]], np.float32))
    r = s.search(*_q([9], [[3.0]]))
    assert r["counts"].tolist() == [1] and r["weights"][0, 0] == 0.0   # d == max_distance: kept, max_dist == d


def test_max_dist_is_taken_across_queries():
    s = _store(distance_filter=20.0, max_distance=2.0)
    s.add([1, 2], np.array([[0.0], [10.0]], np.float32))
    alone = s.search(*_q([9], [[1.0]]))
    both = s.search(*_q([9, 8], [[1.0], [15.0]]))
    assert alone["weights"][0, 0] == 8.0    # max_dist = 9 (q9 -> track 2)
    assert both["weights"][0, 0] == 14.0    # max_dist = 15 (q8 -> track 1, above max_distance, below the filter)
    assert both["counts"].tolist() == [1, 0]


def test_min_votes():
    s = _store(max_distance=1.0, min_votes=2)
    s.add([1, 1, 2], np.array([[0.0], [0.5], [0.2]], np.float32))
    r = s.search(*_q([9], [[0.1]]))
    assert r["counts"].tolist() == [1] and r["winners"][0, 0] == 1   # track 2 has one vote


def test_ties_go_to_the_lower_store_position():
    s = _store()
    s.add([11, 10, 12], np.array([[1.0], [1.0], [1.0]], np.float32))
    r = s.search(*_q([9], [[0.0]]))
    assert r["counts"].tolist() == [3] and r["winners"][0, :3].tolist() == [11, 10, 12]


def test_remove_then_add_appends():
    s = _store()
    s.add([1, 2, 3], np.array([[1.0], [2.0], [3.0]], np.float32))
    cnt, _ = s.fetch([2, 2], remove=True)
    assert cnt.tolist() == [1, 0]
    s.add([2], np.array([[7.0]], np.float32))
    assert list(s.ids()) == [1, 3, 2]


def test_rejected_requests():
    s = _store()
    s.add([1], np.array([[0.0]], np.float32))
    for ids, rows in (([9, 9], [[1.0], [2.0]]), ([9, 8], [[1.0], []])):
        with pytest.raises(ValueError):
            s.search(*_q(ids, rows))
    with pytest.raises(ValueError):
        s.associate(*_q([1], [[1.0]]))
    assert list(s.ids()) == [1]
