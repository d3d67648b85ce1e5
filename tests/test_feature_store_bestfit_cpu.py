"""The CPU oracle's BestFit voting, pinned by hand: a track goes to the heaviest group of the whole call (the lower
query index on ties), a group past a query's topn cut still claims its track, a reported element whose track another
query took names the query itself, and associate merges a query only into a track it took.  Also min_votes /
max_distance filtering, search_owned(each=True) equal to TopN, a quality store, a gated store whose gate changes
nothing, the unknown-rule refusal, and ofs_bestfit_voting against the tracker oracle's restatement of best.rs."""
import numpy as np
import pytest

import fstore_oracle as fo
import oracle


def _store(voting="best_fit", **kw):
    o = dict(distance_filter=1e9, max_observations=1, feature_dim=2, topn=2, max_distance=1e9, min_votes=1,
             voting=voting)
    o.update(kw)
    return fo.FeatureStore(**o)


def _rows(*xs):
    return np.array([[x, 0.0] for x in xs], np.float32)


def _one_row_queries(n):
    return np.arange(n + 1, dtype=np.int32)


def test_the_heavier_query_takes_the_shared_best_track():
    """Tracks 1 (x = 0) and 2 (x = 10); queries 100 (x = 1) and 101 (x = 2).  Distances 1, 9 and 2, 8, so
    max_dist = 9 and the elements, heaviest first, are (100, 1, 8), (101, 1, 7), (101, 2, 1), (100, 2, 0).  Query 100
    takes track 1; query 101 loses it and takes track 2; query 100's element on track 2 names 100 itself."""
    for voting in ("best_fit", "topn"):
        s = _store(voting)
        s.add([1, 2], _rows(0, 10))
        r = s.associate([100, 101], _one_row_queries(2), _rows(1, 2))
        assert r["counts"].tolist() == [2, 2]
        assert r["weights"].tolist() == [[8.0, 0.0], [7.0, 1.0]]
        if voting == "topn":
            assert r["winners"].tolist() == [[1, 2], [1, 2]]
            assert r["merged"].tolist() == [1, 1] and r["track_ids"].tolist() == [1, 1]
            continue
        assert r["winners"].tolist() == [[1, 100], [101, 2]]
        # 101's first element lost its track: a new track, although no other query took its second candidate
        assert r["merged"].tolist() == [1, 0] and r["track_ids"].tolist() == [1, 101]
        assert s.ids().tolist() == [1, 2, 101]


@pytest.mark.parametrize("order", [(100, 101), (101, 100)])
def test_equal_weights_go_to_the_lower_query_index(order):
    """Track 1 at x = 0 is at distance 1 from both queries (x = 1 and x = -1); track 2 at x = 5 sets max_dist = 6,
    so both groups on track 1 weigh 5.  The query first in the call takes it, whatever its id."""
    s = _store(topn=1)
    s.add([1, 2], _rows(0, 5))
    x = {100: 1.0, 101: -1.0}
    r = s.associate(list(order), _one_row_queries(2), _rows(*(x[q] for q in order)))
    assert r["weights"][:, 0].tolist() == [5.0, 5.0]
    assert r["winners"][:, 0].tolist() == [1, order[1]]
    assert r["merged"].tolist() == [1, 0]


def test_a_group_past_the_topn_cut_claims_its_track():
    """Tracks 1 (x = 0) and 2 (x = 3); query 100 at x = 6, query 101 at x = 1; topn = 1.  max_dist = 6; the elements
    are (101, 1, 5), (101, 2, 4), (100, 2, 3), (100, 1, 0).  Query 101 reports track 1 alone, but its unreported group on
    track 2 outweighs query 100's, so query 100's only reported element names 100 and it becomes a new track.  Claims
    read off the reported lists would have given track 2 to query 100."""
    s = _store(topn=1)
    s.add([1, 2], _rows(0, 3))
    r = s.associate([100, 101], _one_row_queries(2), _rows(6, 1))
    assert r["counts"].tolist() == [1, 1]
    assert r["winners"].tolist() == [[100], [1]] and r["weights"].tolist() == [[3.0], [5.0]]
    assert r["merged"].tolist() == [0, 1] and r["track_ids"].tolist() == [100, 1]
    t = _store("topn", topn=1)
    t.add([1, 2], _rows(0, 3))
    assert t.associate([100, 101], _one_row_queries(2), _rows(6, 1))["track_ids"].tolist() == [2, 1]


def test_min_votes_and_max_distance_filter_before_the_claims():
    """K = 2, min_votes = 2, max_distance = 5.  Track 1 holds x = 0, 1; track 2 holds x = 4, 30 (one vote at most: no
    element, no claim); track 3 holds x = 20, 21 (above max_distance: no votes).  Query 100 (x = 2) sees distances
    2, 1 | 2, 28 | 18, 19 and query 101 (x = 3) 3, 2 | 1, 27 | 17, 18.  max_dist = 28, taken over every entry, those
    above max_distance and those of groups short of min_votes included.  The groups on track 1 weigh
    (28 - 2) + (28 - 1) = 53 and (28 - 3) + (28 - 2) = 51."""
    s = _store(max_observations=2, min_votes=2, max_distance=5.0)
    s.add([1, 1, 2, 2, 3, 3], _rows(0, 1, 4, 30, 20, 21))
    r = s.search([100, 101], _one_row_queries(2), _rows(2, 3))
    assert r["counts"].tolist() == [1, 1]
    assert r["winners"][:, 0].tolist() == [1, 101]
    assert r["weights"][:, 0].tolist() == [53.0, 51.0]


def test_owned_each_equals_topn_and_owned_group_claims():
    ids = np.repeat(np.arange(1, 13, dtype=np.uint64), 3)
    f = np.random.default_rng(4).standard_normal((len(ids), 4)).astype(np.float32)
    stores = {}
    for voting in ("topn", "best_fit"):
        stores[voting] = _store(voting, max_observations=3, feature_dim=4, topn=3)
        stores[voting].add(ids, f)
    q = [3, 7, 1, 12, 5]
    a, b = stores["topn"].search_owned(q, each=True), stores["best_fit"].search_owned(q, each=True)
    for k in a:
        assert np.array_equal(a[k], b[k]), k
    a, b = stores["topn"].search_owned(q), stores["best_fit"].search_owned(q)
    assert np.array_equal(a["counts"], b["counts"]) and np.array_equal(a["weights"], b["weights"])
    # a track is reported as the winner of at most one query; the others name themselves
    named = [int(w) for i, qi in enumerate(q) for w in b["winners"][i, : b["counts"][i]] if w != qi]
    assert len(named) == len(set(named))
    assert not np.array_equal(a["winners"], b["winners"])


def test_quality_store_merges_the_winner_alone():
    """The two queries of the first test on quality stores: query 100 merges into track 1 (history [1, 100]), query
    101 becomes a track of its own (history [101]) with its one row."""
    s = _store(retention="quality", max_observations=4)
    s.add([1, 2], _rows(0, 10), quality=[0.5, 0.5])
    r = s.associate([100, 101], _one_row_queries(2), _rows(1, 2), quality=[0.9, 0.8])
    assert r["merged"].tolist() == [1, 0] and r["track_ids"].tolist() == [1, 101]
    assert [h.tolist() for h in s.merge_history([1, 2, 101])] == [[1, 100], [2], [101]]
    c, f, q = s.fetch_quality([1, 101])
    assert c.tolist() == [2, 1] and q[0, :2].tolist() == [np.float32(0.9), 0.5] and f[1, 0, 0] == 2.0


def test_gated_store_the_gate_changes_nothing():
    """Queries 100 and 101 have overlapping windows, both disjoint from track 1's.  TopN sends both to track 1 and the
    gate keeps the earlier one, 100.  BestFit gives track 1 to 101, the better match, and its destinations are what an
    ungated BestFit store gives: the gate keeps each of them."""
    out = {}
    for voting, gate in (("topn", "any_source"), ("best_fit", "any_source"), ("best_fit", None)):
        s = _store(voting, topn=1, gate=gate)
        kw = dict(sources=[0, 0], t_start=[0, 20], t_end=[10, 21]) if gate else {}
        s.add([1, 2], _rows(0, 10), **kw)
        kw = dict(sources=[0, 0], t_start=[30, 35], t_end=[40, 45]) if gate else {}
        r = s.associate([100, 101], _one_row_queries(2), _rows(4, 1), **kw)
        out[voting, gate] = r
        if gate:
            src, t0, t1 = s.attributes([1])
            assert (t0[0], t1[0]) == (0, 40 if voting == "topn" else 45)
    assert out["topn", "any_source"]["track_ids"].tolist() == [1, 101]
    assert out["best_fit", "any_source"]["track_ids"].tolist() == [100, 1]
    for k in ("counts", "winners", "weights", "track_ids", "merged"):
        assert np.array_equal(out["best_fit", "any_source"][k], out["best_fit", None][k]), k


def test_unknown_rule_is_refused_and_changes_nothing():
    s = _store()
    with pytest.raises(ValueError):
        s.set_voting("sort")
    assert s.voting() == "best_fit"
    assert fo.lib().ofs_set_voting(s._h, 2) == -1
    s.add([1, 2], _rows(0, 10))
    assert s.associate([100, 101], _one_row_queries(2), _rows(1, 2))["merged"].tolist() == [1, 0]
    with pytest.raises(ValueError):
        fo.FeatureStore(voting="best")


def test_entry_list_voting_matches_the_tracker_oracle():
    """ofs_bestfit_voting against oracle.bestfit_voting (best.rs, pinned by the VisualVoting tests) on random entry
    lists whose group weights are distinct, so that the reference's unpinned tie order cannot matter."""
    rng = np.random.default_rng(7)
    checked = 0
    for _ in range(200):
        n = int(rng.integers(1, 60))
        ents = [(int(rng.integers(1, 6)), int(rng.integers(10, 18)),
                 None if rng.random() < 0.1 else float(np.float32(rng.random() * 2))) for _ in range(n)]
        md, mv = float(rng.choice([0.5, 1.0, 3.0])), int(rng.integers(1, 3))
        mine = fo.bestfit_voting(1000, md, mv, ents)
        ws = [w for v in mine.values() for _, w in v]
        if len(set(ws)) != len(ws):
            continue
        ref = oracle.bestfit_voting(md, mv, [(a, b, None, d) for a, b, d in ents])
        assert mine == ref
        cut = fo.bestfit_voting(1, md, mv, ents)
        assert cut == {q: v[:1] for q, v in ref.items()}
        checked += 1
    assert checked > 100
