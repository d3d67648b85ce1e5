"""The CPU oracle's feature classes, pinned by hand: per-class rows and counts, a class search that skips the tracks
without rows of the class (max_dist and the f64 weights worked out), merges that walk the source's classes in
ascending id (a quality store's history step per class), new tracks that hold only the queried class, an
associate_store query without the searched class added whole, and every refusal."""
import numpy as np
import pytest

import fstore_oracle as fo


def _store(classes, **kw):
    o = dict(distance_filter=1e9, max_observations=3, feature_dim=2, topn=3, max_distance=1e9, min_votes=1)
    o.update(kw)
    return fo.FeatureStore(classes=classes, **o)


def test_two_classes_of_different_dims():
    s = _store({4: 2, 1: 5})
    s.add([1, 1, 2], np.arange(6, dtype=np.float32).reshape(3, 2), feature_class=4)
    s.add([2, 3], np.ones((2, 5), np.float32), feature_class=1)
    assert s.classes() == {4: 2, 1: 5}
    assert s.class_counts([1, 2, 3, 7]).tolist() == [[2, 0], [1, 1], [0, 1], [0, 0]]
    c, f = s.fetch([1, 2, 3], feature_class=1)
    assert c.tolist() == [0, 1, 1] and f.shape == (3, 3, 5)
    c, f = s.fetch([1], feature_class=4)
    assert c.tolist() == [2] and f[0, :2].tolist() == [[0, 1], [2, 3]]


def test_class_search_skips_tracks_without_the_class():
    """Track 1 holds class 0 alone, at distance 100 from the query: were it scored, max_dist would be 100.  Tracks 2
    and 3 hold class 1 at distances 5 and 0, so max_dist = 5 and the weights are 5 - 0 = 5 and 5 - 5 = 0."""
    s = _store({0: 2, 1: 2})
    s.add([1], [[100.0, 0.0]], feature_class=0)
    s.add([2, 3], [[3.0, 4.0], [0.0, 0.0]], feature_class=1)
    r = s.search([9], [0, 1], [[0.0, 0.0]], feature_class=1)
    assert r["counts"].tolist() == [2]
    assert r["winners"][0, :2].tolist() == [3, 2]
    assert r["weights"][0, :2].tolist() == [5.0, 0.0]
    r = s.search([9], [0, 1], [[0.0, 0.0]], feature_class=0)
    assert r["counts"].tolist() == [1] and r["winners"][0, 0] == 1 and r["weights"][0, 0] == 0.0


def test_quality_merge_steps_each_class_in_ascending_id():
    """initial_capacity 2, merge_extension 1.5: c(1) = 3, c(2) = 4, c(3) = 6.  Source 2 holds classes 5 and 0, so
    dest 1's history becomes [1, 2, 2]; class 0 goes first and is truncated at c(2) = 4, class 5 then at c(3) = 6."""
    s = _store({5: 2, 0: 2}, max_observations=8, retention="quality", initial_capacity=2, merge_extension=1.5)
    f = np.zeros((3, 2), np.float32)
    s.add([1, 1, 1], f, quality=[3, 2, 1], feature_class=0)
    s.add([2, 2, 2], f, quality=[9, 8, 7], feature_class=0)
    s.add([1, 1, 1], f, quality=[30, 20, 10], feature_class=5)
    s.add([2, 2, 2], f, quality=[90, 80, 70], feature_class=5)
    s.merge_owned([1], [2], remove=False)
    assert [h.tolist() for h in s.merge_history([1, 2])] == [[1, 2, 2], [2]]
    c, _, q = s.fetch_quality([1], feature_class=0)
    assert c.tolist() == [4] and q[0, :4].tolist() == [9, 8, 7, 3]
    c, _, q = s.fetch_quality([1], feature_class=5)
    assert c.tolist() == [6] and q[0, :6].tolist() == [90, 80, 70, 30, 20, 10]


def test_newest_merge_moves_both_classes():
    s = _store({0: 2, 1: 2}, max_observations=2)
    s.add([1], [[1.0, 1.0]], feature_class=0)
    s.add([1], [[2.0, 2.0]], feature_class=1)
    s.add([2, 2], [[3.0, 3.0], [4.0, 4.0]], feature_class=0)
    s.add([2], [[5.0, 5.0]], feature_class=1)
    s.merge_owned([1], [2])
    assert s.ids().tolist() == [1]
    c, f = s.fetch([1], feature_class=0)
    assert c.tolist() == [2] and f[0].tolist() == [[3, 3], [4, 4]]
    c, f = s.fetch([1], feature_class=1)
    assert c.tolist() == [2] and f[0].tolist() == [[2, 2], [5, 5]]


def test_new_track_holds_the_queried_class_alone():
    s = _store({0: 2, 1: 2})
    s.add([1], [[0.0, 0.0]], feature_class=0)
    out = s.associate([2], [0, 1], [[1.0, 1.0]], feature_class=1)
    assert out["merged"].tolist() == [0]
    assert s.class_counts([1, 2]).tolist() == [[1, 0], [0, 1]]
    out = s.associate([3], [0, 1], [[1.0, 1.0]], feature_class=0)
    assert out["merged"].tolist() == [1] and out["track_ids"].tolist() == [1]
    assert s.class_counts([1]).tolist() == [[2, 0]]


def test_associate_store_query_without_the_class_is_added_whole():
    dst, src = _store({0: 2, 1: 2}), _store({0: 2, 1: 2})
    dst.add([1], [[0.0, 0.0]], feature_class=0)
    src.add([7, 7], [[1.0, 1.0], [2.0, 2.0]], feature_class=1)
    src.add([8], [[0.5, 0.5]], feature_class=0)
    src.add([8], [[9.0, 9.0]], feature_class=1)
    out = dst.associate_store(src, [7, 8], feature_class=0)
    assert out["counts"].tolist() == [0, 1] and out["merged"].tolist() == [0, 1]
    assert out["track_ids"].tolist() == [7, 1]
    assert dst.ids().tolist() == [1, 7] and src.size() == 0
    assert dst.class_counts([1, 7]).tolist() == [[2, 1], [0, 2]]
    c, f = dst.fetch([1], feature_class=1)
    assert f[0, 0].tolist() == [9, 9]


def test_refusals():
    with pytest.raises(ValueError):
        _store({3: 2, 4: 0})
    with pytest.raises(ValueError):
        _store({3: 2, 4: 8193})
    with pytest.raises(ValueError):
        _store({k: 2 for k in range(17)})
    with pytest.raises(ValueError):
        _store({})
    s = _store({0: 2, 1: 2})
    s.add([1], [[0.0, 0.0]])
    L = fo.lib()
    ids, dims = np.array([0, 0], np.uint64), np.array([2, 2], np.int32)
    assert L.ofs_set_classes(s._h, 2, ids.ctypes.data, dims.ctypes.data) == -1   # repeated id
    ids = np.array([5], np.uint64)
    assert L.ofs_set_classes(s._h, 1, ids.ctypes.data, dims.ctypes.data) == -1   # the store holds tracks
    with pytest.raises(ValueError):
        s.search([9], [0, 1], [[0.0, 0.0]], feature_class=2)
    other = _store({0: 2, 1: 3})
    other.add([8], [[0.0, 0.0]])
    with pytest.raises(ValueError):
        s.associate_store(other, [8])
    assert s.classes() == {0: 2, 1: 2} and s.class_counts([1]).tolist() == [[1, 0]] and other.size() == 1
