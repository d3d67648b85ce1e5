"""CPU checks of the feature store's track attributes and gate (sb200_fstore_set_gate, the _attr calls): the oracle on
hand-built 1-d stores with results worked out by hand, against the ungated oracle where no window conflicts, and the
layout of the version-2 blob header with the gate constants of the C header."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import fstore_oracle as fo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "similari_b200.h")


def _store(gate="same_source", **kw):
    base = dict(metric=fo.EUCLIDEAN, distance_filter=1000.0, max_observations=2, feature_dim=1, topn=5,
                max_distance=1000.0, min_votes=1, gate=gate)
    base.update(kw)
    return fo.FeatureStore(**base)


def _add(s, ids, vals, src=None, t0=None, t1=None):
    s.add(np.array(ids, np.uint64), np.array(vals, np.float32).reshape(-1, 1), sources=src, t_start=t0, t_end=t1)


def _one(vals):
    """CSR of one observation per query."""
    return np.arange(len(vals) + 1, dtype=np.int32), np.array(vals, np.float32).reshape(-1, 1)


def _res(r, q):
    n = int(r["counts"][q])
    return list(zip(r["winners"][q, :n].tolist(), r["weights"][q, :n].tolist()))


def _search(s, ids, vals, src, t0, t1):
    offs, f = _one(vals)
    return s.search(ids, offs, f, sources=src, t_start=t0, t_end=t1)


def test_touching_and_point_windows_are_compatible():
    s = _store()
    _add(s, [1], [0.0], [7], [0], [5])
    cases = {   # query window -> compatible with [0, 5] (>= / <= : touching counts as disjoint)
        (5, 8): True, (-3, 0): True, (5, 5): True, (0, 0): True, (3, 3): False, (4, 6): False, (-1, 1): False,
        (-10, 10): False,
    }
    for (a, b), ok in cases.items():
        r = _search(s, [9], [1.0], [7], [a], [b])
        assert (int(r["counts"][0]) == 1) == ok, (a, b)
    # two equal point windows touch: compatible
    p = _store()
    _add(p, [1], [0.0], [7], [2], [2])
    assert int(_search(p, [9], [1.0], [7], [2], [2])["counts"][0]) == 1


def test_same_source_rule_needs_equal_sources_and_any_source_does_not():
    for gate, want in (("same_source", 0), ("any_source", 1)):
        s = _store(gate)
        _add(s, [1], [0.0], [7], [0], [5])
        assert int(_search(s, [9], [1.0], [8], [10], [20])["counts"][0]) == want, gate
        assert int(_search(s, [9], [1.0], [7], [10], [20])["counts"][0]) == 1, gate   # equal sources: both rules
        assert int(_search(s, [9], [1.0], [7], [3], [20])["counts"][0]) == 0, gate    # overlap: neither rule


def test_a_gated_pair_neither_votes_nor_raises_max_dist():
    # track 2 (value 100) overlaps both queries in time: its entries are gone, so max_dist is 3, not 99
    kw = dict(max_distance=50.0)
    s, u = _store(**kw), _store(None, **kw)
    _add(s, [1, 2], [0.0, 100.0], [1, 1], [0, 20], [10, 30])
    _add(u, [1, 2], [0.0, 100.0])
    rs = _search(s, [11, 12], [1.0, 3.0], [1, 1], [25, 25], [26, 26])
    offs, f = _one([1.0, 3.0])
    ru = u.search([11, 12], offs, f)
    assert _res(rs, 0) == [(1, 2.0)] and _res(rs, 1) == [(1, 0.0)]
    assert _res(ru, 0) == [(1, 98.0)] and _res(ru, 1) == [(1, 96.0)]


def test_coexisting_queries_that_win_one_track_are_not_both_merged():
    s = _store()
    _add(s, [1], [0.0], [1], [0], [10])
    offs, f = _one([0.5, 0.6, 0.7])
    r = s.associate([11, 12, 13], offs, f, sources=[1, 1, 1], t_start=[20, 25, 30], t_end=[30, 35, 40])
    assert r["counts"].tolist() == [1, 1, 1] and r["winners"][:, 0].tolist() == [1, 1, 1]
    # 11 extends track 1 to [0, 30]; 12 overlaps that and becomes a new track; 13 touches it and is merged
    assert r["merged"].tolist() == [1, 0, 1]
    assert r["track_ids"].tolist() == [1, 12, 1]
    assert s.ids().tolist() == [1, 12]
    src, t0, t1 = s.attributes([1, 12, 11, 99])
    assert src.tolist() == [1, 1, 0, 0] and t0.tolist() == [0, 25, 0, 0] and t1.tolist() == [40, 35, 0, 0]
    cnt, feats = s.fetch([1, 12])
    assert cnt.tolist() == [2, 1] and feats[0, :, 0].tolist() == pytest.approx([0.5, 0.7])
    # without a gate both queries land in track 1
    u = _store(None)
    _add(u, [1], [0.0])
    assert u.associate([11, 12, 13], offs, f)["merged"].tolist() == [1, 1, 1]


def test_add_takes_the_hull_and_refuses_another_source():
    s = _store()
    _add(s, [1, 1, 2], [0.0, 1.0, 2.0], [5, 5, 6], [10, 0, 3], [12, 4, 3])
    src, t0, t1 = s.attributes([1, 2])
    assert src.tolist() == [5, 6] and t0.tolist() == [0, 3] and t1.tolist() == [12, 3]
    before = (s.ids().tolist(), s.fetch([1, 2])[1].tolist(), [a.tolist() for a in s.attributes([1, 2])])
    for ids, src in (([1], [6]), ([3, 3], [1, 2]), ([3, 1], [1, 4])):
        with pytest.raises(ValueError):
            _add(s, ids, [9.0] * len(ids), src, [0] * len(ids), [1] * len(ids))
    with pytest.raises(ValueError):   # t_start > t_end
        _add(s, [4], [9.0], [1], [2], [1])
    assert (s.ids().tolist(), s.fetch([1, 2])[1].tolist(), [a.tolist() for a in s.attributes([1, 2])]) == before


def test_a_merge_owned_chain_that_turns_incompatible_is_refused_whole():
    s = _store()
    _add(s, [1, 2, 3], [0.0, 1.0, 2.0], [1, 1, 1], [0, 10, 15], [10, 20, 18])
    snap = lambda: (s.ids().tolist(), s.fetch([1, 2, 3])[1].tolist(), [a.tolist() for a in s.attributes([1, 2, 3])])
    before = snap()
    # 3 ([15, 18]) is compatible with 1 as it is ([0, 10]), not with 1 after it absorbed 2 ([0, 20])
    with pytest.raises(ValueError):
        s.merge_owned([1, 1], [2, 3], remove=True)
    assert snap() == before
    s.merge_owned([1], [3], remove=False)
    src, t0, t1 = s.attributes([1, 3])
    assert t0.tolist() == [0, 15] and t1.tolist() == [18, 18]


def test_owned_search_gates_by_stored_attributes():
    s = _store()
    _add(s, [1, 2, 3], [0.0, 1.0, 2.0], [1, 1, 2], [0, 5, 20], [10, 8, 30])
    # 1 and 2 overlap; 3 has another source: under same_source, 1 finds nothing
    assert int(s.search_owned([1], each=True)["counts"][0]) == 0
    a = _store("any_source")
    _add(a, [1, 2, 3], [0.0, 1.0, 2.0], [1, 1, 2], [0, 5, 20], [10, 8, 30])
    assert _res(a.search_owned([1], each=True), 0) == [(3, 0.0)]


def test_the_rule_is_fixed_while_tracks_are_stored_and_calls_must_match_it():
    s = _store()
    _add(s, [1], [0.0], [1], [0], [1])
    assert s._L.ofs_set_gate(s._h, 2) == -1
    s.fetch([1], remove=True)
    assert s._L.ofs_set_gate(s._h, 2) == 0
    with pytest.raises(ValueError):
        _add(s, [1], [0.0])   # a gated store needs the attributes
    with pytest.raises(ValueError):
        _add(_store(None), [1], [0.0], [1], [0], [1])   # an ungated store takes none


@pytest.mark.parametrize("gate", ["same_source", "any_source"])
@pytest.mark.parametrize("metric", [fo.EUCLIDEAN, fo.COSINE])
def test_windows_that_never_conflict_give_the_ungated_results(gate, metric):
    rng = np.random.default_rng(3 + metric)
    kw = dict(metric=metric, max_observations=3, feature_dim=8, topn=4, distance_filter=1e9, max_distance=1e9)
    s, u = _store(gate, **kw), _store(None, **kw)
    n_tracks = 30
    ids = np.repeat(np.arange(1, n_tracks + 1, dtype=np.uint64), 1 + np.arange(n_tracks) % 4)
    rng.shuffle(ids)
    f = rng.standard_normal((len(ids), 8)).astype(np.float32)
    w0 = (ids.astype(np.int64) - 1) * 10   # track i lives in [10 (i - 1), 10 (i - 1) + 5]
    s.add(ids, f, sources=np.full(len(ids), 3, np.uint64), t_start=w0, t_end=w0 + 5)
    u.add(ids, f)
    offs = np.array([0, 2, 3, 6, 7], np.int32)
    qf = rng.standard_normal((7, 8)).astype(np.float32)
    q0 = 10_000 + np.arange(4, dtype=np.int64) * 10
    attrs = dict(sources=np.full(4, 3, np.uint64), t_start=q0, t_end=q0 + 5)
    rs, ru = s.search([101, 102, 103, 104], offs, qf, **attrs), u.search([101, 102, 103, 104], offs, qf)
    for k in ru:
        assert np.array_equal(rs[k], ru[k]), k
    for k in ("counts", "winners", "weights"):
        a, b = s.search_owned(s.ids(), each=True)[k], u.search_owned(u.ids(), each=True)[k]
        assert np.array_equal(a, b), k
    # later queries lie after earlier ones in time, so a track extended by one query still admits the next
    rs, ru = s.associate([101, 102, 103, 104], offs, qf, **attrs), u.associate([101, 102, 103, 104], offs, qf)
    for k in ru:
        assert np.array_equal(rs[k], ru[k]), k
    assert np.array_equal(s.ids(), u.ids())
    assert np.array_equal(s.fetch(s.ids())[1], u.fetch(u.ids())[1])


# ---- the C header
def test_version_2_header_mirror_repeats_version_1_through_live():
    from similari_b200 import _lib

    hdr = open(HEADER).read()
    for k, v in (("SB200_FSTORE_GATE_NONE", 0), ("SB200_FSTORE_GATE_SAME_SOURCE", 1), ("SB200_FSTORE_GATE_ANY_SOURCE", 2),
                 ("SB200_FSTORE_BLOB_VERSION_GATED", 2), ("SB200_FSTORE_BLOB_SECTIONS_V2", 7)):
        assert re.search(r"#define %s %du?\b" % (k, v), hdr), k

    v1, v2 = _lib.FstoreBlobHeader, _lib.FstoreBlobHeaderV2
    assert v1.live.offset == v2.live.offset == 56
    assert (v2.gate.offset, v2.sec_off.offset, v2.sec_bytes.offset, C.sizeof(v2)) == (64, 72, 128, 184)
    for name, *_ in v1._fields_[:-2]:
        assert getattr(v1, name).offset == getattr(v2, name).offset, name
