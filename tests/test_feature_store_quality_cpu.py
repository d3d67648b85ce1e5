"""CPU checks of the oracle's quality retention (fstore_oracle, retention="quality"): the merge history of
src/track.rs:1107-1130, the capacity growth of examples/track_merging.rs:257-265 with its defaults, the stable order of
equal qualities, the sequential truncation of merges in one associate call, a query's best c(1) rows with a weight worked
out by hand, and every refusal.  The GPU store is held to this oracle by tests/test_gpu_feature_store_quality.py."""
import numpy as np
import pytest

import fstore_oracle as fo

D = 8


def _store(K=12, **kw):
    o = dict(distance_filter=1e9, max_observations=K, feature_dim=D, topn=3, max_distance=1e9, min_votes=1)
    o.update(kw)
    return fo.FeatureStore(retention="quality", **o)


def _rows(values):
    """One row per value: value * e0 (its euclidean norm is the value, exactly)."""
    f = np.zeros((len(values), D), np.float32)
    f[:, 0] = values
    return f


def test_merge_history_of_two_tracks():
    # src/track.rs:1107-1130: merging track 1 into track 0 with merge_history = true gives [0, 1]
    s = _store()
    s.add([0, 1], _rows([1, 2]), quality=[1, 1])
    s.merge_owned([0], [1], remove=False)
    h = s.merge_history([0, 1, 7])
    assert h[0].tolist() == [0, 1] and h[1].tolist() == [1] and h[2].tolist() == []
    s.merge_owned([1], [0], remove=True)   # a source's whole history is appended
    assert s.merge_history([1])[0].tolist() == [1, 0, 1]


def test_capacity_grows_with_the_merge_history():
    # defaults 4 / 1.5 with K = 12: c(1) = 6, c(2) = 9, c(3) = min(12, 13) = 12
    s = _store()
    assert s.retention() == ("quality", 4, 1.5)
    for t in range(3):
        s.add([t] * 10, _rows(np.arange(10) + 10 * t), quality=np.arange(10, dtype=np.float32))
    counts, _, q = s.fetch_quality([0, 1, 2])
    assert counts.tolist() == [6, 6, 6]
    assert q[0, :6].tolist() == [9, 8, 7, 6, 5, 4]   # the best, best first
    s.merge_owned([0], [1])
    assert s.fetch_quality([0])[0].tolist() == [9]
    s.merge_owned([0], [2])
    counts, f, q = s.fetch_quality([0])
    assert counts.tolist() == [12]
    assert q[0].tolist() == [9, 9, 9, 8, 8, 8, 7, 7, 7, 6, 6, 6]
    assert f[0, :3, 0].tolist() == [9, 19, 29]   # equal qualities: dest first, then the sources in merge order


def test_equal_qualities_keep_dest_then_source_order():
    s = _store()
    s.add([1, 1, 2, 2], _rows([1, 2, 3, 4]), quality=[0.5, -0.0, 0.5, 0.0])   # -0.0 == +0.0
    s.merge_owned([1], [2])
    counts, f, q = s.fetch_quality([1])
    assert counts.tolist() == [4]
    assert f[0, :4, 0].tolist() == [1, 3, 2, 4]
    s.add([1], _rows([5]), quality=[0.5])   # an appended row goes after its equals
    assert s.fetch_quality([1])[1][0, :5, 0].tolist() == [1, 3, 5, 2, 4]


def test_sequential_truncation_in_one_associate_call():
    # track 1 holds 6 rows of quality 5 (h = 1); three queries win it in one call.  Query 10 (4 rows of quality 3) makes
    # h = 2, c = 9: one of its rows is dropped.  Queries 11 and 12 (1 row each) make h = 3 and 4, c = 12: 11 rows.  One
    # sort of all 12 rows at the end would keep the dropped row.
    s = _store(topn=1)
    s.add([1] * 6, _rows([1] * 6), quality=[5] * 6)
    r = s.associate([10, 11, 12], [0, 4, 5, 6], _rows([2, 3, 4, 5, 6, 7]), quality=[3, 3, 3, 3, 1, 1])
    assert r["merged"].tolist() == [1, 1, 1] and r["track_ids"].tolist() == [1, 1, 1]
    counts, f, q = s.fetch_quality([1])
    assert counts.tolist() == [11]
    assert f[0, 6:9, 0].tolist() == [2, 3, 4]   # row 5 of query 10 is gone
    assert q[0, :11].tolist() == [5] * 6 + [3] * 3 + [1] * 2
    assert s.merge_history([1])[0].tolist() == [1, 10, 11, 12]


def test_a_query_takes_part_with_its_best_c1_rows():
    # one stored row at the origin; the query's 8 rows have norms 1..7 and 10, so d = the norm exactly.  c(1) = 6 rows
    # take part, in quality order; the two worst (norms 4 and 10) do not, so max_dist = 7, not 10.
    s = _store(topn=1)
    s.add([1], _rows([0]), quality=[0])
    norms = [1, 2, 3, 4, 5, 6, 7, 10]
    qual = [0.9, 0.8, 0.7, 0.1, 0.6, 0.5, 0.95, 0.05]
    r = s.search([9], [0, 8], _rows(norms), quality=qual)
    used = [7, 1, 2, 3, 5, 6]   # quality order: 0.95, 0.9, 0.8, 0.7, 0.6, 0.5
    w = 0.0
    for d in used:
        w += float(np.float32(7.0) - np.float32(d))
    assert r["counts"].tolist() == [1] and r["weights"][0, 0] == w == 18.0
    # associated, the query's 6 rows join track 1 (h = 2, c = 9) ahead of its row of quality 0
    r = s.associate([20], [0, 8], _rows(norms), quality=qual)
    assert r["merged"].tolist() == [1]
    counts, f, _ = s.fetch_quality([1])
    assert counts.tolist() == [7] and f[0, :7, 0].tolist() == [7, 1, 2, 3, 5, 6, 0]


def test_a_newest_store_is_unchanged_by_the_new_keywords():
    s = fo.FeatureStore(max_observations=2, feature_dim=D)
    s.add([1, 1, 1], _rows([1, 2, 3]))
    assert s.fetch([1])[1][0, :, 0].tolist() == [2, 3]
    with pytest.raises(ValueError):
        s.add([1], _rows([4]), quality=[1])
    with pytest.raises(ValueError):
        s.merge_history([1])
    with pytest.raises(ValueError):
        s.fetch_quality([1])


@pytest.mark.parametrize("init, ext", [(0, 1.5), (-1, 1.5), (4, float("nan")), (4, float("inf")), (4, 0.5),
                                       (1, 1.00001)])
def test_bad_parameters_are_refused(init, ext):
    with pytest.raises(ValueError):
        _store(K=64, initial_capacity=init, merge_extension=ext)


def test_constant_capacity_and_slow_growth_limits():
    s = _store(K=12, initial_capacity=3, merge_extension=1.0)   # c(h) = 3 for every h
    s.add([1] * 5 + [2] * 5, _rows(range(10)), quality=list(range(10)))
    s.merge_owned([1], [2])
    assert s.fetch_quality([1])[0].tolist() == [3]
    _store(K=12, initial_capacity=1, merge_extension=1.0001)   # reaches 12 before h = 65536


def test_quality_refusals_change_nothing():
    s = _store()
    s.add([1, 2], _rows([1, 2]), quality=[1, 2])
    before = (s.ids().tolist(), s.fetch_quality([1, 2])[2].tolist())
    with pytest.raises(ValueError):
        s.add([1], _rows([3]))   # no quality on a quality store
    for call in (lambda: s.add([1, 3], _rows([3, 4]), quality=[1, np.nan]),
                 lambda: s.search([9], [0, 2], _rows([3, 4]), quality=[np.nan, 1]),
                 lambda: s.associate([9], [0, 2], _rows([3, 4]), quality=[1, np.nan])):
        with pytest.raises(ValueError):
            call()
    assert (s.ids().tolist(), s.fetch_quality([1, 2])[2].tolist()) == before
    assert s._L.ofs_set_retention(s._h, 0, 4, 1.5) == -1   # fixed while the store holds tracks


def test_fetch_with_remove_and_a_repeated_id():
    # the second entry of an id the first entry removed returns nothing: count 0, zero rows, zero qualities
    s = _store()
    s.add([1, 1, 2], _rows([1, 2, 3]), quality=[0.5, 0.75, 1])
    counts, f, q = s.fetch_quality([1, 1, 2], remove=True)
    assert counts.tolist() == [2, 0, 1]
    assert q[0, :2].tolist() == [0.75, 0.5] and not q[1].any() and not f[1].any() and q[2, 0] == 1
    assert s.size() == 0
