"""CPU checks of the feature store's owned calls (search_owned, merge_owned): the oracle on hand-built 1-d stores with
weights worked out by hand, and the oracle's owned calls against compositions of its existing calls."""
import numpy as np
import pytest

import fstore_oracle as fo
from fstore_checks import same_results



def _store(**kw):
    base = dict(metric=fo.EUCLIDEAN, distance_filter=100.0, max_observations=2, feature_dim=1, topn=5,
                max_distance=100.0, min_votes=1)
    base.update(kw)
    return fo.FeatureStore(**base)


def _add(s, ids, vals):
    s.add(np.array(ids, np.uint64), np.array(vals, np.float32).reshape(-1, s.D))


def _rows(s, i):
    cnt, f = s.fetch([i])
    return f[0, :cnt[0], 0].tolist()


def _res(r, q):
    n = int(r["counts"][q])
    return list(zip(r["winners"][q, :n].tolist(), r["weights"][q, :n].tolist()))


def test_group_mode_never_scores_one_query_against_another():
    s = _store()
    _add(s, [1, 2, 3], [0.0, 1.0, 10.0])
    r = s.search_owned([1, 2])
    # candidates are {3} only: q1 -> 3 at 10, q2 -> 3 at 9; max_dist = 10 over the whole call
    assert _res(r, 0) == [(3, 0.0)]
    assert _res(r, 1) == [(3, 1.0)]


def test_each_mode_has_its_own_exclusion_and_max_dist():
    s = _store()
    _add(s, [1, 2, 3], [0.0, 1.0, 10.0])
    r = s.search_owned([1, 2], each=True)
    # q1: candidates {2, 3} at 1 and 10, max_dist 10; q2: candidates {1, 3} at 1 and 9, max_dist 9
    assert _res(r, 0) == [(2, 9.0), (3, 0.0)]
    assert _res(r, 1) == [(1, 8.0), (3, 0.0)]


def test_queries_use_their_stored_observations():
    s = _store(max_distance=1.5)
    _add(s, [1, 1, 1, 2], [0.0, 5.0, 6.0, 5.5])   # K = 2: track 1 holds 5, 6
    r = s.search_owned([1])
    # entries 5 -> 5.5 (0.5) and 6 -> 5.5 (0.5); max_dist 0.5; weight 0 + 0
    assert _res(r, 0) == [(2, 0.0)]
    r = s.search_owned([2])
    assert _res(r, 0) == [(1, 0.0)]


def test_unknown_id_gets_count_zero_and_duplicates_are_refused():
    s = _store()
    _add(s, [1, 2, 3], [0.0, 1.0, 10.0])
    for each in (False, True):
        r = s.search_owned([99, 1], each=each)
        assert r["counts"][0] == 0 and r["winners"][0].tolist() == [0] * 5
        assert r["counts"][1] > 0
        with pytest.raises(ValueError):
            s.search_owned([1, 2, 1], each=each)
    assert s.search_owned([])["counts"].shape == (0,)


def test_merge_chain_and_star():
    s = _store()
    _add(s, [1, 2, 3, 3], [1.0, 2.0, 3.0, 4.0])
    s.merge_owned([1, 3], [2, 1], remove=False)   # 1 <- 2, then 3 <- 1 (with 2's row)
    assert list(s.ids()) == [1, 2, 3]
    assert (_rows(s, 1), _rows(s, 2), _rows(s, 3)) == ([1.0, 2.0], [2.0], [1.0, 2.0])
    s = _store()
    _add(s, [1, 2, 3, 3], [1.0, 2.0, 3.0, 4.0])
    s.merge_owned([1, 3], [2, 1], remove=True)
    assert list(s.ids()) == [3] and _rows(s, 3) == [1.0, 2.0]
    s = _store(max_observations=3)
    _add(s, [1, 2, 3, 3, 4], [1.0, 2.0, 3.0, 4.0, 5.0])
    s.merge_owned([1, 1, 1], [2, 3, 4], remove=False)   # star: 1 <- 2, 1 <- 3, 1 <- 4
    assert _rows(s, 1) == [3.0, 4.0, 5.0] and list(s.ids()) == [1, 2, 3, 4]


def test_remove_src_keeps_the_order_of_the_rest():
    s = _store()
    _add(s, [5, 6, 7, 8], [1.0, 2.0, 3.0, 4.0])
    s.merge_owned([8, 5], [6, 7], remove=True)
    assert list(s.ids()) == [5, 8]
    assert _rows(s, 5) == [1.0, 3.0] and _rows(s, 8) == [4.0, 2.0]
    _add(s, [6], [9.0])   # a removed id comes back at the end
    assert list(s.ids()) == [5, 8, 6]


@pytest.mark.parametrize("pairs, remove", [
    (([1], [1]), False),          # dest == src
    (([9], [1]), False),          # dest not stored
    (([1], [9]), True),           # src not stored
    (([1, 3], [2, 2]), True),     # src removed by an earlier pair
    (([1, 2], [2, 3]), True),     # dest removed by an earlier pair
    (([1, 1], [2, 1]), False),    # the refused pair comes after a good one
])
def test_refused_merges_change_nothing(pairs, remove):
    s = _store()
    _add(s, [1, 2, 3, 3], [1.0, 2.0, 3.0, 4.0])
    before = [(i, _rows(s, i)) for i in s.ids()]
    with pytest.raises(ValueError):
        s.merge_owned(*pairs, remove=remove)
    assert [(i, _rows(s, i)) for i in s.ids()] == before
    with pytest.raises(ValueError):
        s.merge_owned([1, 2], [3])


def test_a_removed_track_may_be_named_without_remove():
    s = _store()
    _add(s, [1, 2, 3], [1.0, 2.0, 3.0])
    s.merge_owned([1, 3], [2, 2], remove=False)
    assert _rows(s, 1) == [1.0, 2.0] and _rows(s, 3) == [3.0, 2.0]


def _random_store(seed, metric, **kw):
    rng = np.random.default_rng(seed)
    opts = dict(metric=metric, max_observations=3, feature_dim=5, topn=4, distance_filter=3.0, max_distance=2.5,
                min_votes=1)
    opts.update(kw)
    ids = rng.integers(1, 30, 120).astype(np.uint64)
    feats = rng.standard_normal((120, 5)).astype(np.float32)

    def make():
        s = fo.FeatureStore(**opts)
        s.add(ids, feats)
        return s
    return make, rng


@pytest.mark.parametrize("metric", [fo.EUCLIDEAN, fo.COSINE])
def test_each_equals_one_search_of_the_fetched_rows_per_id(metric):
    make, rng = _random_store(1 + metric, metric)
    s = make()
    ids = s.ids()
    q = np.concatenate([ids[rng.permutation(len(ids))[:12]], [1000]]).astype(np.uint64)
    r = s.search_owned(q, each=True)
    for i, qid in enumerate(q):
        cnt, f = s.fetch([qid])
        if cnt[0] == 0:
            assert r["counts"][i] == 0
            continue
        one = s.search([qid], np.array([0, cnt[0]], np.int32), f[0, :cnt[0]])
        same_results({k: v[i:i + 1] for k, v in r.items()}, one)


@pytest.mark.parametrize("metric", [fo.EUCLIDEAN, fo.COSINE])
def test_group_equals_a_search_on_a_copy_without_the_queried_ids(metric):
    make, rng = _random_store(5 + metric, metric)
    s = make()
    q = s.ids()[rng.permutation(s.size())[:8]]
    r = s.search_owned(q)
    copy = make()
    cnt, f = copy.fetch(q, remove=True)
    offs = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int32)
    rows = np.concatenate([f[i, :cnt[i]] for i in range(len(q))])
    same_results(r, copy.search(q, offs, rows))
    assert np.array_equal(s.ids(), make().ids())   # the owned search leaves the store as it was


def test_merge_equals_fetch_and_add():
    make, rng = _random_store(9, fo.EUCLIDEAN)
    for remove in (False, True):
        s, e = make(), make()
        ids = list(s.ids())
        dest, src, gone = [], [], set()
        while len(dest) < 15:
            d, c = (int(x) for x in rng.choice(ids, 2, replace=False))
            if remove and (d in gone or c in gone):
                continue
            dest.append(d)
            src.append(c)
            if remove:
                gone.add(c)
        s.merge_owned(dest, src, remove=remove)
        for d, c in zip(dest, src):
            cnt, f = e.fetch([c])
            e.add(np.full(cnt[0], d, np.uint64), f[0, :cnt[0]])
            if remove:
                e.fetch([c], remove=True)
        assert np.array_equal(s.ids(), e.ids())
        cs, fs = s.fetch(s.ids())
        ce, fe = e.fetch(e.ids())
        assert np.array_equal(cs, ce) and np.array_equal(fs.view(np.uint32), fe.view(np.uint32))
