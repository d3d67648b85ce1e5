"""CPU checks of the oracle's store-to-store calls (fstore_oracle): find_baked, the `baked` rule of the reference's
examples/track_merging.rs:240-247 (now > t_end + baked_period, exact at its edge and at the int64 extremes), and
associate_store, that example's fetch_tracks + merge_external(.., true) / add_track (:371-481): a quality merge worked
out by hand (h + h_q, ties to the destination, the truncation at c(h), the history concatenation), a new track kept
whole, two sources winning one destination in one call, a gated query turned into a new track by a window the call
extended, and every refusal.  The GPU store is held to this oracle by tests/test_gpu_feature_store_promote.py."""
import ctypes as C

import numpy as np
import pytest

import fstore_oracle as fo

D = 8
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1


def _store(K=12, retention="quality", **kw):
    o = dict(distance_filter=1e9, max_observations=K, feature_dim=D, topn=1, max_distance=1e9, min_votes=1)
    o.update(kw)
    return fo.FeatureStore(retention=retention, **o)


def _rows(values):
    """One row per value: value * e0."""
    f = np.zeros((len(values), D), np.float32)
    f[:, 0] = values
    return f


def _win(n, t0, t1, src=1):
    return dict(sources=[src] * n, t_start=[t0] * n, t_end=[t1] * n)


def test_bake_rule_at_its_edge():
    s = _store(retention="newest", gate="same_source")
    s.add([1, 2], _rows([1, 2]), **dict(sources=[1, 1], t_start=[0, 0], t_end=[100, 101]))
    assert s.find_baked(105, 5).tolist() == []    # now == t_end + period: not baked
    assert s.find_baked(106, 5).tolist() == [1]   # one more: baked
    assert s.find_baked(107, 5).tolist() == [1, 2]
    assert s.find_baked(101).tolist() == [1]      # baked_period defaults to 0


def test_bake_rule_at_the_int64_extremes():
    ends = [I64_MIN, I64_MIN + 1, -1, 0, 1, I64_MAX - 1, I64_MAX]
    s = _store(retention="newest", gate="any_source")
    n = len(ends)
    s.add(np.arange(n), _rows(np.arange(n)), sources=[1] * n, t_start=[I64_MIN] * n, t_end=ends)
    for now in (I64_MIN, I64_MIN + 1, -1, 0, 1, I64_MAX - 1, I64_MAX):
        for period in (I64_MIN, I64_MIN + 1, -7, -1, 0, 1, 7, I64_MAX - 1, I64_MAX):
            want = [i for i, e in enumerate(ends) if now > e + period]   # Python integers: no wrap-around
            assert s.find_baked(now, period).tolist() == want, (now, period)


def test_quality_merge_adds_the_source_history():
    # defaults 4 / 1.5, K = 12: c(1) = 6, c(2) = 9, c(3) = min(12, 13) = 12.  The destination d (h = 1) holds 4 rows; the
    # source s holds 9 rows after absorbing s' (h = 2).  Merged: h = 3, 13 rows for 12 slots, so one row is dropped, and
    # every quality tie goes to the destination's row.
    dst, src = _store(), _store()
    dst.add([100] * 4, _rows([1, 2, 3, 4]), quality=[5, 4, 3, 2])
    src.add([7] * 6, _rows([11, 12, 13, 14, 15, 16]), quality=[6, 5, 4, 3, 2, 1])
    src.add([8] * 6, _rows([21, 22, 23, 24, 25, 26]), quality=[6, 5, 4, 3, 2, 1])
    src.merge_owned([7], [8])
    c, f, q = src.fetch_quality([7])
    assert c.tolist() == [9] and f[0, :9, 0].tolist() == [11, 21, 12, 22, 13, 23, 14, 24, 15]
    r = dst.associate_store(src, [7])
    assert r["merged"].tolist() == [1] and r["track_ids"].tolist() == [100] and r["counts"].tolist() == [1]
    c, f, q = dst.fetch_quality([100])
    assert c.tolist() == [12]
    assert f[0, :, 0].tolist() == [11, 21, 1, 12, 22, 2, 13, 23, 3, 14, 24, 4]   # 15 (quality 2, from s) is dropped
    assert q[0].tolist() == [6, 6, 5, 5, 5, 4, 4, 4, 3, 3, 3, 2]
    assert dst.merge_history([100])[0].tolist() == [100, 7, 8]
    assert src.size() == 0 and dst.ids().tolist() == [100]


def test_a_new_track_keeps_its_list_and_history():
    dst, src = _store(max_distance=0.5), _store()
    dst.add([100], _rows([50]), quality=[1])
    src.add([7] * 6, _rows([11, 12, 13, 14, 15, 16]), quality=[1, 2, 3, 4, 5, 6])
    src.add([8] * 3, _rows([21, 22, 23]), quality=[6, 0, 6])
    src.merge_owned([7], [8])   # h = 2, c(2) = 9: all 9 rows kept
    want = src.fetch_quality([7])
    r = dst.associate_store(src, [7], remove=False)
    assert r["merged"].tolist() == [0] and r["track_ids"].tolist() == [7] and r["counts"].tolist() == [0]
    got = dst.fetch_quality([7])
    for a, b in zip(got, want):
        assert np.array_equal(a, b)
    assert got[0].tolist() == [9]
    assert dst.merge_history([7])[0].tolist() == [7, 8]
    assert dst.ids().tolist() == [100, 7] and src.ids().tolist() == [7]   # remove=False leaves src as it was


def test_two_sources_win_one_destination_in_one_call():
    dst, src = _store(), _store()
    dst.add([100], _rows([1]), quality=[1])
    src.add([7, 8, 9], _rows([2, 3, 4]), quality=[2, 0.5, 3])
    src.merge_owned([7], [8])   # 7: h = 2, rows [2 (q 2), 3 (q 0.5)]
    r = dst.associate_store(src, [9, 7])
    assert r["merged"].tolist() == [1, 1] and r["track_ids"].tolist() == [100, 100]
    # item order: 9 (h 1 -> 2, c = 9), then 7 (h 2 -> 4, c = 12)
    c, f, q = dst.fetch_quality([100])
    assert c.tolist() == [4] and f[0, :4, 0].tolist() == [4, 2, 1, 3] and q[0, :4].tolist() == [3, 2, 1, 0.5]
    assert dst.merge_history([100])[0].tolist() == [100, 9, 7, 8]
    assert src.ids().tolist() == []


def test_gated_query_turned_new_by_the_window_the_call_extended():
    # d holds [0, 10].  Query 7 ([20, 30]) and query 8 ([25, 40]) are both compatible with d as stored and both win it;
    # 7 merges first and extends d to [0, 30], which 8 overlaps, so 8 becomes a new track with its own triple.
    for retention in ("newest", "quality"):
        dst = _store(retention=retention, gate="same_source", topn=1)
        src = _store(retention=retention, gate="same_source", topn=1)
        kw = lambda n: dict(quality=[1] * n) if retention == "quality" else {}
        dst.add([100], _rows([1]), **_win(1, 0, 10), **kw(1))
        src.add([7, 8], _rows([1, 1]), sources=[1, 1], t_start=[20, 25], t_end=[30, 40], **kw(2))
        r = dst.associate_store(src, [7, 8])
        assert r["counts"].tolist() == [1, 1]
        assert r["merged"].tolist() == [1, 0] and r["track_ids"].tolist() == [100, 8]
        s, t0, t1 = dst.attributes([100, 8])
        assert s.tolist() == [1, 1] and t0.tolist() == [0, 25] and t1.tolist() == [30, 40]
        assert src.size() == 0


def test_refusals_change_neither_store():
    L = fo.lib()
    dst, src = _store(gate="same_source"), _store(gate="same_source")
    dst.add([100], _rows([1]), quality=[1], **_win(1, 0, 1))
    src.add([7, 8], _rows([1, 2]), quality=[1, 1], sources=[1, 1], t_start=[5, 5], t_end=[6, 6])

    def state():
        return [(x.ids().tolist(), [a.tolist() for a in x.fetch_quality(x.ids())],
                 [h.tolist() for h in x.merge_history(x.ids())]) for x in (dst, src)]

    before = state()
    bad_stores = [_store(gate="same_source", feature_dim=16), _store(gate="same_source", K=6),
                  _store(gate="any_source"), _store(), _store(retention="newest", gate="same_source"),
                  _store(gate="same_source", initial_capacity=3), _store(gate="same_source", merge_extension=2.0)]
    for other in bad_stores:
        with pytest.raises(ValueError):
            dst.associate_store(other, [])
    for ids in ([7, 7], [9], [100], [7, 100]):
        with pytest.raises(ValueError):
            dst.associate_store(src, ids)
    with pytest.raises(ValueError):
        dst.associate_store(dst, [])
    out = [np.zeros(2, np.int32), np.zeros((2, 1), np.uint64), np.zeros((2, 1), np.float64), np.zeros(2, np.uint64),
           np.zeros(2, np.uint8)]
    ids = np.array([7, 8], np.uint64)
    p = [o.ctypes.data_as(C.c_void_p) for o in out]
    assert L.ofs_associate_store(dst._h, src._h, -1, ids.ctypes.data_as(C.c_void_p), 1, *p, 1) == -1
    assert L.ofs_associate_store(dst._h, src._h, 2, ids.ctypes.data_as(C.c_void_p), 2, *p, 1) == -1
    assert state() == before
    with pytest.raises(ValueError):
        _store().find_baked(0)   # an ungated store keeps no windows
    assert L.ofs_find_baked(dst._h, 0, 0, -1, None) == -1
    assert dst.associate_store(src, [])["counts"].tolist() == []
    assert state() == before
