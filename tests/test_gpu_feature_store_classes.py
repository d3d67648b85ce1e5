"""Feature classes of the feature store (sb200_fstore_set_classes / _use_class / _class_counts) on the GPU.

A class search is checked against single-class stores holding the same tracks' rows of that class, bit for bit
(counts, winner ids, f64 weights; a track without rows of the class takes no part, so it neither votes nor raises
max_dist); the rows kept by add, associate, merge_owned and associate_store against the retention rule restated on the
host from the rows fetched before each call; a store that declares its default class against one that never did,
blobs included; and every refusal against an unchanged store."""
import numpy as np
import pytest

from fstore_checks import gpu_store, same_results, same_store, store_pair

pytestmark = pytest.mark.gpu

METRICS = ("euclidean", "cosine")
TYPES = ("f32", "f16", "bf16")


def _rows(s, ids, c, quality=False):
    """{id: (rows, qualities)} of class c, as the store returns them"""
    if quality:
        cnt, f, q = s.fetch_quality(ids, feature_class=c)
    else:
        cnt, f = s.fetch(ids, feature_class=c)
        q = np.zeros(f.shape[:2], np.float32)
    return {int(i): (f[k, :cnt[k]].copy(), q[k, :cnt[k]].copy()) for k, i in enumerate(ids)}


def _fill(s, singles, rng, n, classes, K, storage_round=None):
    """n tracks; track t holds class c when (t + c) % 3 != 0 (so each class misses some tracks), with 1 .. 2K + 1 rows
    added in interleaved calls.  singles[c] gets the same rows of class c, so its tracks are in the same order."""
    order = []
    for t in range(1, n + 1):
        for c in classes:
            if (t + c) % 3 != 0:
                order.append((t, c))
    for part in np.array_split(np.arange(len(order)), 2):
        for c, d in classes.items():
            sel = [order[i][0] for i in part if order[i][1] == c]
            if not sel:
                continue
            ids = np.repeat(np.array(sel, np.uint64), [1 + (t * 5 + c) % (2 * K + 1) for t in sel])
            f = rng.standard_normal((len(ids), d)).astype(np.float32)
            s.add(ids, f, feature_class=c)
            if singles is not None:
                singles[c].add(ids, f)


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("storage", TYPES)
def test_class_search_is_a_single_class_search(metric, storage):
    rng = np.random.default_rng(7)
    classes = {3: 16, 1: 24}
    s = gpu_store(metric, storage, classes=classes)
    singles = {c: gpu_store(metric=metric, storage=storage, feature_dim=d) for c, d in classes.items()}
    _fill(s, singles, rng, 40, classes, 3)
    assert s.classes() == classes
    ids = np.arange(1, 41, dtype=np.uint64)
    cc = s.class_counts(np.append(ids, 999))
    for k, c in enumerate(classes):
        got = _rows(s, ids, c)
        want = _rows(singles[c], ids, None)
        for t in ids:
            assert len(got[int(t)][0]) == cc[int(t) - 1, k]
            assert np.array_equal(got[int(t)][0].view(np.uint32), want[int(t)][0].view(np.uint32))
    assert not cc[-1].any()
    for c, d in classes.items():
        q = rng.standard_normal((9, d)).astype(np.float32)
        qid, off = np.arange(500, 504, dtype=np.uint64), np.array([0, 2, 5, 6, 9], np.int32)
        same_results(s.search(qid, off, q, feature_class=c), singles[c].search(qid, off, q))
        same_results(s.search_owned(ids[:6], feature_class=c), singles[c].search_owned(ids[:6]))
        same_results(s.search_owned(ids[:6], each=True, feature_class=c), singles[c].search_owned(ids[:6], each=True))
        same_results(s.associate(qid, off, q, feature_class=c), singles[c].associate(qid, off, q))
        n = len(singles[c].ids())
        got = _rows(s, singles[c].ids(), c)
        want = _rows(singles[c], singles[c].ids(), None)
        for t in want:
            assert np.array_equal(got[t][0].view(np.uint32), want[t][0].view(np.uint32))
        assert n == len(want)


def test_new_track_holds_the_queried_class_alone():
    s = gpu_store(classes={0: 8, 9: 16})
    s.add([1], np.ones((1, 16), np.float32), feature_class=9)
    out = s.associate([2], [0, 1], np.full((1, 8), 5, np.float32), feature_class=0)
    assert out["merged"][0] == 0
    assert s.class_counts([1, 2]).tolist() == [[0, 1], [1, 0]]
    # a class-0 search does not see track 1, which has no class-0 rows
    r = s.search([3], [0, 1], np.zeros((1, 8), np.float32), feature_class=0)
    assert r["counts"][0] == 1 and r["winners"][0, 0] == 2
    s.add([2], np.zeros((1, 16), np.float32), feature_class=9)
    assert s.class_counts([2]).tolist() == [[1, 1]]
    c, f = s.fetch([1, 2], feature_class=0)
    assert c.tolist() == [0, 1]


def _newest(rows, extra, K):
    return np.concatenate([rows, extra])[-K:] if len(extra) else rows


@pytest.mark.parametrize("gate", [None, "any_source"])
@pytest.mark.parametrize("storage", TYPES)
def test_merge_owned_moves_every_class(gate, storage):
    rng = np.random.default_rng(11)
    classes = {4: 8, 2: 16}
    K = 3
    s = gpu_store(classes=classes, storage=storage, gate=gate, max_observations=K)
    kw = {}
    ids = np.arange(1, 13, dtype=np.uint64)
    for c, d in classes.items():
        sel = ids[(ids + c) % 3 != 0]
        rep = np.repeat(sel, (1 + sel % 4).astype(np.int64))
        if gate:
            kw = dict(sources=np.zeros(len(rep)), t_start=rep * 10, t_end=rep * 10 + 1)
        s.add(rep, rng.standard_normal((len(rep), d)).astype(np.float32), feature_class=c, **kw)
    before = {c: _rows(s, ids, c) for c in classes}
    order = s.ids()   # creation order: the class-4 tracks, then the tracks holding class 2 alone
    dest, src = [1, 2, 1, 7], [3, 4, 5, 8]
    s.merge_owned(dest, src, remove=True)
    want = {c: dict(before[c]) for c in classes}
    for d_, s_ in zip(dest, src):
        for c in classes:
            want[c][d_] = (_newest(want[c][d_][0], want[c][s_][0], K), None)
    kept = [t for t in order if t not in src]
    assert np.array_equal(s.ids(), np.array(kept, np.uint64))
    for c in classes:
        got = _rows(s, kept, c)
        for t in kept:
            assert np.array_equal(got[int(t)][0].view(np.uint32), want[c][int(t)][0].view(np.uint32)), (c, t)
    if gate:
        src_, t0, t1 = s.attributes([1])
        assert t0[0] == 10 and t1[0] == 51


def _quality_keep(rows, q, h, init, K):
    cap = min(K, init * 2 ** h)
    ix = np.argsort(-q, kind="stable")[:cap]
    return rows[ix], q[ix]


def test_quality_merge_owned_steps_each_class():
    """init 1, extension 2: c(h) = min(K, 2^h), exact.  A source holding two classes appends its history twice; the
    lower class id is truncated at c(h + 1), the higher at c(h + 2)."""
    K = 8
    s = gpu_store(classes={7: 8, 2: 8}, max_observations=K, retention="quality", initial_capacity=1,
                  merge_extension=2.0)
    rng = np.random.default_rng(3)
    f = rng.standard_normal((20, 8)).astype(np.float32)
    q = rng.permutation(20).astype(np.float32)
    # dest 1: h = 1, capacity 2; source 2 holds both classes
    s.add([1, 1, 1], f[:3], quality=q[:3], feature_class=2)
    s.add([1, 1], f[3:5], quality=q[3:5], feature_class=7)
    s.add([2, 2], f[5:7], quality=q[5:7], feature_class=2)
    s.add([2, 2], f[7:9], quality=q[7:9], feature_class=7)
    before = {c: _rows(s, [1, 2], c, quality=True) for c in (2, 7)}
    s.merge_owned([1], [2], remove=False)
    assert [h.tolist() for h in s.merge_history([1, 2])] == [[1, 2, 2], [2]]
    for c, h in ((2, 2), (7, 3)):   # ascending class id: class 2 first, at h = 2; class 7 at h = 3
        r = np.concatenate([before[c][1][0], before[c][2][0]])
        qq = np.concatenate([before[c][1][1], before[c][2][1]])
        wr, wq = _quality_keep(r, qq, h, 1, K)
        got = _rows(s, [1], c, quality=True)[1]
        assert np.array_equal(got[0].view(np.uint32), wr.view(np.uint32)), c
        assert np.array_equal(got[1], wq), c


@pytest.mark.parametrize("gate", [None, "same_source"])
def test_associate_store_brings_every_class(gate):
    rng = np.random.default_rng(5)
    classes = {0: 8, 1: 16}
    K = 4
    kw = dict(max_observations=K, gate=gate)
    dst, src = gpu_store(classes=classes, **kw), gpu_store(classes=classes, **kw)
    single_d, single_s = gpu_store(feature_dim=8, **kw), gpu_store(feature_dim=8, **kw)

    def add(stores, ids, c, t):
        f = rng.standard_normal((len(ids), classes[c])).astype(np.float32)
        a = dict(sources=np.zeros(len(ids)), t_start=np.full(len(ids), t), t_end=np.full(len(ids), t)) if gate else {}
        for st in stores:
            st.add(ids, f, feature_class=c, **a) if st in (dst, src) else st.add(ids, f, **a)

    add([dst, single_d], np.repeat(np.arange(1, 7, dtype=np.uint64), 2), 0, 1)
    add([dst], np.arange(2, 5, dtype=np.uint64), 1, 1)
    add([src, single_s], np.repeat(np.arange(10, 15, dtype=np.uint64), 2), 0, 5)
    add([src], np.array([11, 12, 16, 16], np.uint64), 1, 5)   # 16 holds class 1 alone
    q = np.array([10, 11, 12, 16], np.uint64)
    bd = {c: _rows(dst, np.arange(1, 7), c) for c in classes}
    bs = {c: _rows(src, q, c) for c in classes}
    out = dst.associate_store(src, q, remove=True, feature_class=0)
    ref = single_d.associate_store(single_s, q[:3], remove=True)
    same_results({k: v[:3] for k, v in out.items()}, ref)
    assert out["counts"][3] == 0 and out["merged"][3] == 0 and out["track_ids"][3] == 16
    assert src.ids().tolist() == [13, 14]
    cur = {c: {d: r[0] for d, r in bd[c].items()} for c in classes}
    for i, t in enumerate(q):   # the queries in order, each appended to where it went
        d = int(out["track_ids"][i])
        for c in classes:
            cur[c][d] = _newest(cur[c].get(d, np.zeros((0, classes[c]), np.float32)), bs[c][int(t)][0], K)
    for c in classes:
        for d, want in cur[c].items():
            got = _rows(dst, [d], c)[d][0]
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (d, c)
    assert dst.class_counts([16]).tolist() == [[0, 2]]


def test_default_class_declared_is_the_default():
    rng = np.random.default_rng(1)
    a, b = gpu_store(retention="quality"), gpu_store(classes={0: 16}, retention="quality")
    ids = np.repeat(np.arange(1, 9, dtype=np.uint64), 3)
    f, q = rng.standard_normal((len(ids), 16)).astype(np.float32), rng.random(len(ids)).astype(np.float32)
    for s in (a, b):
        s.add(ids, f, quality=q)
    qq = rng.standard_normal((4, 16)).astype(np.float32)
    same_results(a.associate([20, 21], [0, 2, 4], qq, quality=np.ones(4, np.float32)),
          b.associate([20, 21], [0, 2, 4], qq, quality=np.ones(4, np.float32)))
    a.merge_owned([1], [2])
    b.merge_owned([1], [2])
    assert np.array_equal(a.save(), b.save())
    import similari_b200.engine as eng

    c = eng.FeatureStore.load(b.save())
    assert c.classes() == {0: 16}
    assert np.array_equal(c.save(), a.save())


def test_large_gallery_class_search():
    """20,000 tracks, classes of 128 and 512 dims, K = 12: every track holds both, so each class search is the search
    of a single-class store of the same rows."""
    rng = np.random.default_rng(9)
    K, n = 12, 20000
    classes = {0: 128, 1: 512}
    s = gpu_store(classes=classes, max_observations=K, topn=5, storage="f16")
    singles = {c: gpu_store(max_observations=K, topn=5, feature_dim=d, storage="f16") for c, d in classes.items()}
    ids = np.repeat(np.arange(1, n + 1, dtype=np.uint64), 2)
    for c, d in classes.items():
        f = rng.standard_normal((len(ids), d)).astype(np.float16)
        s.add(ids, f, feature_class=c)
        singles[c].add(ids, f)
    for c, d in classes.items():
        q = rng.standard_normal((64, d)).astype(np.float16)
        off = np.arange(0, 65, 2, dtype=np.int32)
        same_results(s.search(np.arange(10**6, 10**6 + 32, dtype=np.uint64), off, q, feature_class=c),
              singles[c].search(np.arange(10**6, 10**6 + 32, dtype=np.uint64), off, q))


def _state(s):
    ids = s.ids()
    return ids, s.class_counts(ids), {c: s.fetch(ids, feature_class=c) for c in s.classes()}


def test_refusals_leave_the_store_unchanged():
    from similari_b200._lib import Sb200Error

    s = gpu_store(classes={0: 8, 1: 16})
    s.add([1, 2], np.ones((2, 8), np.float32), feature_class=0)
    s.add([2], np.ones((1, 16), np.float32), feature_class=1)
    before = _state(s)
    L, h = s._L, s._h
    ids16 = np.arange(17, dtype=np.uint64)
    dims16 = np.full(17, 8, np.int32)
    from similari_b200._lib import ptr

    for n, i, d in ((1, [5], [8]), (0, [0], [8])):
        assert L.sb200_fstore_set_classes(h, n, ptr(np.array(i, np.uint64)), ptr(np.array(d, np.int32))) != 0
    e = gpu_store()
    for n, i, d in ((0, ids16, dims16), (17, ids16, dims16), (2, np.array([3, 3], np.uint64), dims16),
                    (1, ids16, np.array([0], np.int32)), (1, ids16, np.array([8193], np.int32))):
        assert L.sb200_fstore_set_classes(e._h, n, ptr(i), ptr(d)) != 0
    e._read_classes()
    assert e.classes() == {0: 16} and e.save().tobytes() == gpu_store().save().tobytes()
    assert L.sb200_fstore_use_class(h, 5) != 0
    with pytest.raises(ValueError):
        s.search([9], [0, 1], np.ones((1, 8), np.float32), feature_class=5)
    other = gpu_store(classes={0: 8, 1: 24})
    other.add([7], np.ones((1, 8), np.float32))
    with pytest.raises(Sb200Error):
        s.associate_store(other, [7])
    same_results(_state(s), before)


# ---- against the CPU oracle (fstore_oracle), bit for bit
@pytest.mark.parametrize("device_cols", [False, True])
@pytest.mark.parametrize("gate,retention", [(None, "newest"), ("same_source", "newest"), (None, "quality"),
                                            ("any_source", "quality")])
@pytest.mark.parametrize("storage,metric", [("f32", "euclidean"), ("f16", "cosine"), ("bf16", "euclidean"),
                                            ("f32", "cosine")])
def test_mixed_sequence_matches_the_oracle(storage, metric, gate, retention, device_cols):
    """add into both classes (some tracks hold one), associate on one class, search the other, save and load halfway
    (the reloaded store re-saves byte for byte), merge_owned, search_owned, and associate_store from a second store."""
    import fstore_oracle as fo
    import similari_b200.engine as eng

    classes = {6: 16, 2: 24}
    qual = retention == "quality"
    kw = dict(gate=gate, retention=retention, initial_capacity=2, merge_extension=1.5, max_observations=4, topn=3)
    g, m = store_pair(metric, storage, classes=classes, **kw)
    rng = np.random.default_rng(21)

    def rows(n, d):
        return fo.round_rows(rng.standard_normal((n, d)).astype(np.float32), storage)

    def extra(n, t, ids=None):
        a = {}
        if gate:
            src = np.zeros(n, np.uint64) if ids is None else (np.asarray(ids) % 2).astype(np.uint64)
            a.update(sources=src, t_start=np.asarray(t, np.int64), t_end=np.asarray(t, np.int64) + 1)
        if qual:
            a["quality"] = rng.permutation(n).astype(np.float32)
        return a

    def both(call, *args, **k):
        ra = getattr(g, call)(*args, **k)
        rb = getattr(m, call)(*args, **k)
        if ra is not None:
            same_results(ra, rb)
        return ra

    for c, d in classes.items():
        tr = np.array([t for t in range(1, 25) if (t + c) % 5 != 0], np.uint64)
        ids = np.repeat(tr, (1 + tr % 3).astype(np.int64))
        both("add", ids, rows(len(ids), d), feature_class=c, **extra(len(ids), ids * 10, ids))

    def queries(c, base, nq):
        off = np.arange(0, 2 * nq + 1, 2, dtype=np.int32)
        qid = np.arange(base, base + nq, dtype=np.uint64)
        return qid, off, rows(2 * nq, classes[c]), extra(nq, (qid - base) * 10 - 5000, qid)

    qid, off, f, a = queries(2, 500, 6)
    if qual:
        a["quality"] = rng.permutation(len(f)).astype(np.float32)
    if device_cols:
        import torch

        t = torch.from_numpy(f).cuda()
        torch.cuda.synchronize()
        same_results(g.associate_device(qid, off, t.data_ptr(), feature_class=2, **a),
              m.associate(qid, off, f, feature_class=2, **a))
    else:
        both("associate", qid, off, f, feature_class=2, **a)
    qid, off, f, a = queries(6, 600, 5)
    if qual:
        a["quality"] = rng.permutation(len(f)).astype(np.float32)
    both("search", qid, off, f, feature_class=6, **a)
    same_store(g, m)

    blob = g.save()
    g = eng.FeatureStore.load(blob)
    assert g.classes() == classes
    assert np.array_equal(g.save(), blob)
    same_store(g, m)

    pairs_d, pairs_s = [], []   # pairs the gate allows, given the windows the associate left
    src_, t0, t1 = (dict(zip(m.ids().tolist(), v.tolist())) for v in m.attributes(m.ids())) if gate else ({}, {}, {})
    for d_, s_ in ((1, 3), (2, 4), (1, 5), (6, 8), (7, 9), (10, 12)):
        if gate:
            ok = (t0[d_] >= t1[s_] or t1[d_] <= t0[s_]) and (gate == "any_source" or src_[d_] == src_[s_])
            if not ok:
                continue
            t0[d_], t1[d_] = min(t0[d_], t0[s_]), max(t1[d_], t1[s_])
        pairs_d.append(d_)
        pairs_s.append(s_)
    assert len(pairs_d) >= 3
    both("merge_owned", pairs_d, pairs_s, remove=True)
    both("search_owned", m.ids()[:5], feature_class=6)
    both("search_owned", m.ids()[:5], each=True, feature_class=2)
    same_store(g, m)

    gs, ms = store_pair(metric, storage, classes=classes, **kw)
    for c, d in classes.items():
        tr = np.array([t for t in range(300, 310) if (t + c) % 3 != 0], np.uint64)
        ids = np.repeat(tr, 2)
        f = rows(len(ids), d)
        e = extra(len(ids), (ids - 300) * 10 + 2000, ids)
        gs.add(ids, f, feature_class=c, **e)
        ms.add(ids, f, feature_class=c, **e)
    q = np.arange(300, 310, dtype=np.uint64)
    same_results(g.associate_store(gs, q, feature_class=6), m.associate_store(ms, q, feature_class=6))
    same_store(g, m)
    same_store(gs, ms)
    blob = g.save()
    assert np.array_equal(eng.FeatureStore.load(blob).save(), blob)


def test_quality_associate_store_steps_each_class():
    """Two queries of history 1 merge into one destination of history 1 (init 2, ext 1.5: c(2) = 4, c(3) = 6,
    c(4) = 10 -> K = 8): the first brings classes 2 and 9 (steps at h = 2, 3), the second class 9 alone (h = 4)."""
    classes = {9: 8, 2: 8}
    kw = dict(retention="quality", initial_capacity=2, merge_extension=1.5, max_observations=8, topn=1)
    g, m = store_pair(classes=classes, **kw)
    gs, ms = store_pair(classes=classes, **kw)
    f = np.zeros((3, 8), np.float32)
    for s in (g, m):
        s.add([1, 1, 1], f, quality=[3, 2, 1], feature_class=2)
        s.add([1, 1, 1], f, quality=[30, 20, 10], feature_class=9)
    for s in (gs, ms):
        s.add([5, 5, 5], f, quality=[9, 8, 7], feature_class=2)
        s.add([5, 5, 5], f, quality=[90, 80, 70], feature_class=9)
        s.add([6, 6, 6], f, quality=[60, 50, 40], feature_class=9)
    same_results(g.associate_store(gs, [5, 6], feature_class=9), m.associate_store(ms, [5, 6], feature_class=9))
    same_store(g, m)
    assert [h.tolist() for h in g.merge_history([1])] == [[1, 5, 5, 6]]
    assert g.class_counts([1]).tolist() == [[8, 4]]


def test_version_4_blob_refusals():
    import similari_b200.engine as eng
    from similari_b200._lib import Sb200Error

    g = gpu_store(classes={0: 8, 3: 16})
    g.add([1, 2], np.ones((2, 8), np.float32))
    g.add([2], np.ones((1, 16), np.float32), feature_class=3)
    blob = g.save()
    assert int(blob[:8].view(np.uint32)[1]) == 4
    h = eng.FeatureStore.load(blob)
    assert h.classes() == {0: 8, 3: 16} and np.array_equal(h.save(), blob)
    import ctypes as C

    class V4(C.Structure):
        _fields_ = [("magic", C.c_uint32), ("version", C.c_uint32), ("total_bytes", C.c_uint64)] + \
                   [(n, C.c_int32 if n != "distance_filter" and n != "max_distance" else C.c_float) for n in
                    ("metric", "distance_filter", "max_observations", "feature_dim", "topn", "max_distance",
                     "min_votes", "d8", "feature_type", "storage_type")] + \
                   [("live", C.c_int64), ("gate", C.c_int32), ("retention", C.c_int32),
                    ("initial_capacity", C.c_int32), ("merge_extension", C.c_float), ("n_classes", C.c_int32),
                    ("reserved", C.c_int32), ("sec_off", C.c_uint64 * 72), ("sec_bytes", C.c_uint64 * 72)]

    hd = V4.from_buffer_copy(blob.tobytes()[:C.sizeof(V4)])

    def cnt_section(k):
        return int(hd.sec_off[8 + 4 * k]), int(hd.sec_off[9 + 4 * k])

    bad = []
    bad = []
    b = blob.copy(); V = V4.from_buffer(b); V.n_classes = 17; bad.append(b)
    b = blob.copy(); b[hd.sec_off[6] + 8: hd.sec_off[6] + 16] = b[hd.sec_off[6]: hd.sec_off[6] + 8]; bad.append(b)   # id twice
    b = blob.copy(); b[hd.sec_off[7] + 4: hd.sec_off[7] + 8] = np.array([9000], np.int32).view(np.uint8); bad.append(b)
    c0, _ = cnt_section(0)
    b = blob.copy(); b[c0: c0 + 4] = np.array([9], np.int32).view(np.uint8); bad.append(b)   # cnt above K
    b = blob.copy(); b[c0: c0 + 4] = np.array([0], np.int32).view(np.uint8); bad.append(b)   # track 1 without rows
    for b in bad:
        with pytest.raises(Sb200Error):
            eng.FeatureStore.load(b)
    assert np.array_equal(g.save(), blob)
