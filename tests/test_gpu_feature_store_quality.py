"""GPU checks of the feature store's quality retention (retention="quality") bit for bit against the CPU oracle: seeded
sequences of mixed add / search / associate (host and device columns) / search_owned / merge_owned / fetch calls over
every storage type, both metrics, gated and ungated, with a save and load in the middle that continues identically;
merge_owned chains and stars; a gallery-scale case; the version-3 blob (byte-equal twins, refusals); and every refusal
leaving the store (and, for associate_wasted, the tracker) as it was."""
import ctypes as C
import zlib

import numpy as np
import pytest

import fstore_oracle as fo
from fstore_checks import gpu_store, refused_blob, same_results, same_store, store_pair

pytestmark = pytest.mark.gpu

QUALITY = dict(retention="quality", max_observations=12)


def _feats(rng, n, dim, storage):
    """Rows the storage type holds exactly, so that a stored query row is the oracle's row."""
    return fo.round_rows(rng.standard_normal((n, dim)).astype(np.float32), storage)


def _quality(rng, n):
    """Qualities with many ties (and signed zeros), so the stable order is exercised."""
    q = rng.integers(-2, 4, n).astype(np.float32) * np.float32(0.25)
    q[rng.random(n) < 0.1] = -0.0
    return q


def _attrs(rng, n, gate, ids=None):
    if gate is None:
        return {}
    t0 = rng.integers(0, 2000, n).astype(np.int64)
    src = (ids % 2 + 1).astype(np.uint64) if ids is not None else rng.integers(1, 3, n).astype(np.uint64)
    return dict(sources=src, t_start=t0, t_end=t0 + rng.integers(0, 5, n).astype(np.int64))


def _device(x):
    import torch

    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _step(rng, g, o, it, dim, storage, gate, next_id):
    """One random call on both stores; returns the next free id."""
    import torch

    ids = o.ids()
    kind = rng.integers(0, 7)
    if kind <= 1 or len(ids) < 4:   # add: known and new ids
        n = int(rng.integers(1, 12))
        pool = np.concatenate([ids, np.arange(next_id, next_id + 4, dtype=np.uint64)])
        aid = rng.choice(pool, n).astype(np.uint64)
        f, q = _feats(rng, n, dim, storage), _quality(rng, n)
        at = _attrs(rng, n, gate, aid)
        if gate is not None:   # one source per track: the stored one, or the id's parity for a new track
            at["sources"] = (aid % 2 + 1).astype(np.uint64)
            if len(ids):
                known = o.attributes(aid)[0]
                at["sources"] = np.where(known > 0, known, at["sources"]).astype(np.uint64)
        o.add(aid, f, quality=q, **at)
        if it % 2:
            d = _device(f)
            g.add_device(aid, d.data_ptr(), quality=q, **at)
            torch.cuda.synchronize()
        else:
            g.add(aid, f, quality=q, **at)
        return next_id + 4
    if kind <= 3:   # search or associate of fresh queries, some longer than c(1)
        Q = int(rng.integers(1, 9))
        lens = 1 + rng.integers(0, 10, Q)
        offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
        qid = np.arange(next_id, next_id + Q, dtype=np.uint64)
        f, q = _feats(rng, int(offs[-1]), dim, storage), _quality(rng, int(offs[-1]))
        at = _attrs(rng, Q, gate)
        op = "associate" if kind == 3 else "search"
        ro = getattr(o, op)(qid, offs, f, quality=q, **at)
        if it % 3 == 1:
            d = _device(f)
            rg = getattr(g, op + "_device")(qid, offs, d.data_ptr(), quality=q, **at)
        else:
            rg = getattr(g, op)(qid, offs, f, quality=q, **at)
        same_results(rg, ro, op)
        return next_id + Q
    if kind == 4:   # owned search, both modes
        sel = rng.choice(ids, min(len(ids), int(rng.integers(1, 6))), replace=False).astype(np.uint64)
        each = bool(rng.integers(0, 2))
        same_results(g.search_owned(sel, each=each), o.search_owned(sel, each=each), "search_owned")
        return next_id
    if kind == 5:   # merge_owned: a chain or a star, with or without removal
        k = int(rng.integers(2, min(6, len(ids)) + 1))
        sel = rng.choice(ids, k, replace=False).astype(np.uint64)
        if rng.integers(0, 2):
            d, s = sel[1:], sel[:-1]      # chain: sel[1] <- sel[0], sel[2] <- sel[1], ...
        else:
            d, s = np.full(k - 1, sel[0], np.uint64), sel[1:]   # star into sel[0]
        remove = bool(rng.integers(0, 2)) and d is not None and not np.any(np.isin(d[1:], s[:-1]))
        try:
            o.merge_owned(d, s, remove=remove)
        except ValueError:   # the gate refused a pair: the GPU store must refuse the same call
            from similari_b200 import _lib

            with pytest.raises(_lib.Sb200Error):
                g.merge_owned(d, s, remove=remove)
            return next_id
        g.merge_owned(d, s, remove=remove)
        return next_id
    sel = rng.choice(ids, min(len(ids), 3), replace=False).astype(np.uint64)   # fetch, sometimes removing
    remove = bool(rng.integers(0, 4) == 0)
    same_results(g.fetch_quality(sel, remove=remove), o.fetch_quality(sel, remove=remove))
    return next_id


@pytest.mark.parametrize("storage", ["f32", "f16", "bf16"])
@pytest.mark.parametrize("metric", ["euclidean", "cosine"])
@pytest.mark.parametrize("gate", [None, "same_source"])
def test_mixed_sequences_match_the_oracle(storage, metric, gate):
    import similari_b200.engine as eng

    rng = np.random.default_rng(zlib.crc32(f"quality {storage} {metric} {gate}".encode()))
    dim = 24
    g, o = store_pair(metric, storage, gate, **QUALITY, feature_dim=dim)
    next_id = 1
    for it in range(240):
        next_id = _step(rng, g, o, it, dim, storage, gate, next_id)
        if it % 40 == 39:
            same_store(g, o)
        if it == 120:   # save and load in the middle: the loaded store continues identically
            blob = g.save()
            g = eng.FeatureStore.load(blob)
            assert g.retention() == ("quality", 4, 1.5) and g.gate == gate and g.storage_type() == storage
            assert np.array_equal(g.save(), blob)
    same_store(g, o)
    assert max(len(h) for h in o.merge_history(o.ids())) > 2   # merges happened


@pytest.mark.parametrize("remove", [False, True])
def test_merge_chains_and_stars(remove):
    rng = np.random.default_rng(3 + remove)
    g, o = store_pair(storage="bf16", retention="quality", max_observations=9, initial_capacity=2, merge_extension=2.0)
    n = 12
    aid = np.repeat(np.arange(1, n + 1, dtype=np.uint64), 7)
    f, q = _feats(rng, len(aid), 16, "bf16"), _quality(rng, len(aid))
    for s in (g, o):
        s.add(aid, f, quality=q)
    same_store(g, o)
    chain = (np.array([2, 3, 4, 5], np.uint64), np.array([1, 2, 3, 4], np.uint64))   # 2 <- 1, 3 <- 2, ...
    star = (np.array([6, 6, 6], np.uint64), np.array([7, 8, 9], np.uint64))
    for d, s in (chain, star):
        for x in (g, o):
            x.merge_owned(d, s, remove=remove)
        same_store(g, o)
    assert o.merge_history([5])[0].tolist() == [5, 4, 3, 2, 1]


def test_gallery_scale():
    rng = np.random.default_rng(20000)
    dim, n = 512, 20000
    g, o = store_pair("cosine", "f16", **QUALITY, feature_dim=dim, topn=5)
    aid = np.repeat(np.arange(1, n + 1, dtype=np.uint64), 8)
    rng.shuffle(aid)
    f, q = _feats(rng, len(aid), dim, "f16"), _quality(rng, len(aid))
    for s in (g, o):
        s.add(aid, f, quality=q)
    Q = 12
    lens = 1 + rng.integers(0, 10, Q)
    offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    qid = np.arange(10 ** 6, 10 ** 6 + Q, dtype=np.uint64)
    qf, qq = _feats(rng, int(offs[-1]), dim, "f16"), _quality(rng, int(offs[-1]))
    same_results(g.associate(qid, offs, qf, quality=qq), o.associate(qid, offs, qf, quality=qq), "associate")
    sel = o.ids()[::997]
    same_results(g.search_owned(sel), o.search_owned(sel), "search_owned")
    g.merge_owned(sel[1:], sel[:-1])
    o.merge_owned(sel[1:], sel[:-1])
    assert np.array_equal(g.ids(), o.ids())
    some = np.concatenate([sel[-1:], qid, o.ids()[::1009]])   # the merged track, the queries' tracks and a sample
    same_results(g.fetch_quality(some), o.fetch_quality(some))
    same_results(g.merge_history(some), o.merge_history(some))


def _rc(L, fn, *args):
    return fn(*args), L.sb200_last_error().decode()


def test_refusals_leave_the_store_unchanged():
    import similari_b200.engine as eng
    from similari_b200 import _lib

    L = _lib.lib()
    p = _lib.ptr
    g = gpu_store(**QUALITY, feature_dim=8)
    f = np.ones((3, 8), np.float32)
    g.add([1, 2, 1], f, quality=[1, 2, 3])
    blob = g.save()
    ids = np.array([9], np.uint64)
    offs = np.array([0, 1], np.int32)
    cnt, win, w = np.zeros(1, np.int32), np.zeros((1, 4), np.uint64), np.zeros((1, 4), np.float64)
    tid, mg = np.zeros(1, np.uint64), np.zeros(1, np.uint8)
    nan = np.array([np.nan], np.float32)
    d = _device(f)
    dp = C.c_void_p(d.data_ptr())
    checks = [
        (L.sb200_fstore_add, (g._h, 1, p(ids), p(f)), "_quality"),
        (L.sb200_fstore_search, (g._h, 1, p(ids), p(offs), p(f), p(cnt), p(win), p(w)), "_quality"),
        (L.sb200_fstore_associate, (g._h, 1, p(ids), p(offs), p(f), p(cnt), p(win), p(w), p(tid), p(mg)), "_quality"),
        (L.sb200_fstore_add_device, (g._h, 1, p(ids), dp, None), "_quality"),
        (L.sb200_fstore_search_device, (g._h, 1, p(ids), p(offs), dp, p(cnt), p(win), p(w), None), "_quality"),
        (L.sb200_fstore_associate_device, (g._h, 1, p(ids), p(offs), dp, p(cnt), p(win), p(w), p(tid), p(mg), None),
         "_quality"),
        (L.sb200_fstore_add_quality, (g._h, 1, p(ids), p(nan), None, p(f), None, None), "NaN"),
        (L.sb200_fstore_search_quality, (g._h, 1, p(ids), p(offs), p(nan), None, p(f), None, p(cnt), p(win), p(w),
                                         None), "NaN"),
        (L.sb200_fstore_associate_quality, (g._h, 1, p(ids), p(offs), p(nan), None, p(f), None, p(cnt), p(win), p(w),
                                            p(tid), p(mg), None), "NaN"),
        (L.sb200_fstore_add_quality, (g._h, 1, p(ids), None, None, p(f), None, None), "quality is NULL"),
        (L.sb200_fstore_set_retention, (g._h, 0, 4, 1.5), "holds tracks"),
        (L.sb200_fstore_set_retention, (g._h, 2, 4, 1.5), "unknown retention"),
    ]
    for fn, args, word in checks:
        rc, msg = _rc(L, fn, *args)
        assert rc == -1 and word in msg, (fn.__name__, rc, msg)
        assert np.array_equal(g.save(), blob), fn.__name__
    # associate_wasted: refused before the tracker or the store changes
    t = eng.Tracker(_lib.default_options())
    tb = t.save()
    with pytest.raises(_lib.Sb200Error):
        g.associate_wasted(t, cap=1)
    assert "quality" in L.sb200_last_error().decode()
    assert np.array_equal(g.save(), blob) and np.array_equal(t.save(), tb)
    # the _quality calls on a newest store, and bad parameters on an empty one
    u = gpu_store(max_observations=12, feature_dim=8)
    q1 = np.ones(1, np.float32)
    rc, msg = _rc(L, L.sb200_fstore_add_quality, u._h, 1, p(ids), p(q1), None, p(f), None, None)
    assert rc == -1 and "newest" in msg
    for init, ext, word in [(0, 1.5, "initial_capacity"), (4, float("nan"), "merge_extension"),
                            (4, 0.5, "merge_extension"), (1, 1.00001, "65536")]:
        rc, msg = _rc(L, L.sb200_fstore_set_retention, u._h, 1, init, ext)
        assert rc == -1 and word in msg, msg
    assert u.retention()[0] == "newest" and u.size() == 0
    with pytest.raises(ValueError):
        u.add([1], f[:1], quality=[1.0])


def test_quality_blob_twins_are_byte_equal_and_newest_blobs_unchanged():
    import similari_b200.engine as eng
    from similari_b200 import _lib

    rng = np.random.default_rng(31)
    for gate in (None, "any_source"):
        g1, o = store_pair(storage="f16", gate=gate, **QUALITY, feature_dim=20)
        g2 = gpu_store(storage="f16", gate=gate, **QUALITY, feature_dim=20)
        aid = np.repeat(np.arange(1, 21, dtype=np.uint64), 5)
        f, q = _feats(rng, len(aid), 20, "f16"), _quality(rng, len(aid))
        t0 = (aid.astype(np.int64) * 10)
        at = {} if gate is None else dict(sources=np.ones(len(aid), np.uint64), t_start=t0, t_end=t0 + 5)
        for s in (g1, g2, o):
            s.add(aid, f, quality=q, **at)
            s.merge_owned([1, 1], [2, 3], remove=True)
        b1, b2 = g1.save(), g2.save()
        assert np.array_equal(b1, b2)
        h = _lib.FstoreBlobHeaderV3.from_buffer_copy(b1[:C.sizeof(_lib.FstoreBlobHeaderV3)].tobytes())
        assert (h.version, h.retention, h.initial_capacity, h.merge_extension) == (3, 1, 4, 1.5)
        assert h.live == 18 and h.sec_bytes[8] == 4 * 18 and h.sec_bytes[9] == 8 * (18 + 2)
        assert (h.sec_bytes[4] == 0) == (gate is None)
        c = eng.FeatureStore.load(b1)
        assert np.array_equal(c.save(), b1)
        same_store(c, o)
    n = gpu_store(max_observations=12, feature_dim=8)
    n.add([1, 2], np.ones((2, 8), np.float32))
    hn = _lib.FstoreBlobHeader.from_buffer_copy(n.save()[:128].tobytes())
    assert hn.version == 1


def test_damaged_version_3_blobs_are_refused():
    import similari_b200.engine as eng
    from similari_b200 import _lib

    g = gpu_store(retention="quality", feature_dim=8, max_observations=4)
    g.add([1, 2, 3, 1], np.ones((4, 8), np.float32), quality=[1, 2, 3, 4])
    g.merge_owned([1], [2], remove=False)
    blob = g.save()
    V3 = _lib.FstoreBlobHeaderV3
    hdr = V3.from_buffer_copy(blob[:C.sizeof(V3)].tobytes())

    def damaged(edit):
        b = blob.copy()
        edit(b, V3.from_buffer(b))
        return b

    def column(b, sec, dtype):
        return b[hdr.sec_off[sec]: hdr.sec_off[sec] + hdr.sec_bytes[sec]].view(dtype)

    refused_blob(damaged(lambda b, h: setattr(h, "retention", 2)), "retention")
    refused_blob(damaged(lambda b, h: setattr(h, "initial_capacity", 0)), "initial_capacity")
    refused_blob(damaged(lambda b, h: setattr(h, "merge_extension", float("nan"))), "merge_extension")
    refused_blob(damaged(lambda b, h: column(b, 7, np.float32).__setitem__(4, np.nan)), "NaN")   # track 2's first slot
    refused_blob(damaged(lambda b, h: column(b, 8, np.int32).__setitem__(2, 0)), "length 0")
    refused_blob(damaged(lambda b, h: column(b, 9, np.uint64).__setitem__(2, 7)), "not with its id")
    refused_blob(damaged(lambda b, h: column(b, 8, np.int32).__setitem__(0, 3)), "history holds")
    refused_blob(damaged(lambda b, h: h.sec_bytes.__setitem__(7, h.sec_bytes[7] - 4)), "quality holds")
    # states the rule cannot produce: a list out of quality order, a ring start other than 0, a count above c(h)
    refused_blob(damaged(lambda b, h: column(b, 7, np.float32).__setitem__(1, 5.0)), "quality order")
    refused_blob(damaged(lambda b, h: column(b, 2, np.int32).__setitem__(1, 1)), "ring start")
    refused_blob(damaged(lambda b, h: setattr(h, "initial_capacity", 1)), "above its capacity")   # c(2) = 2 < 3 rows
    c = eng.FeatureStore.load(damaged(lambda b, h: column(b, 7, np.float32).__setitem__(7, np.nan)))   # empty slot
    assert np.array_equal(c.save(), blob)


def test_twins_reached_by_different_routes_save_byte_equal_blobs():
    """Two stores that hold the same lists and histories, reached differently (rows displaced by better ones, and a
    loaded blob with residue in its empty slots), save the same bytes."""
    import similari_b200.engine as eng
    from similari_b200 import _lib

    rng = np.random.default_rng(12)
    for storage in ("f32", "bf16"):
        ga, o = store_pair(storage=storage, **QUALITY, feature_dim=20)
        gb = gpu_store(storage=storage, **QUALITY, feature_dim=20)
        x, y, z = (_feats(rng, 6, 20, storage) for _ in range(3))
        one, two = np.ones(6, np.uint64), np.full(6, 2, np.uint64)
        ga.add(one, x, quality=np.full(6, 0.25, np.float32))   # displaced, row by row, by the six better rows of y
        ga.add(one, y, quality=np.ones(6, np.float32))
        ga.add(two, z, quality=np.arange(6, dtype=np.float32))
        gb.add(one, y, quality=np.ones(6, np.float32))
        gb.add(two, z[::-1], quality=np.arange(6, dtype=np.float32)[::-1])   # already in quality order
        for s in (o,):
            s.add(one, y, quality=np.ones(6, np.float32))
            s.add(two, z, quality=np.arange(6, dtype=np.float32))
        same_store(ga, o)
        same_store(gb, o)
        blob = gb.save()
        assert np.array_equal(ga.save(), blob)
        V3 = _lib.FstoreBlobHeaderV3
        h = V3.from_buffer_copy(blob[:C.sizeof(V3)].tobytes())
        res = blob.copy()   # residue in the empty slots 6 .. 11 of both tracks
        feat = res[h.sec_off[3]: h.sec_off[3] + h.sec_bytes[3]].reshape(2, 12, -1)
        feat[:, 6:] = 0x3C
        res[h.sec_off[7]: h.sec_off[7] + h.sec_bytes[7]].view(np.float32).reshape(2, 12)[:, 6:] = 3.0
        gc = eng.FeatureStore.load(res)
        assert np.array_equal(gc.save(), blob)
        # all three continue identically
        q = _quality(rng, 9)
        for s in (ga, gb, gc, o):
            s.add(np.array([1] * 4 + [2] * 5, np.uint64), _feats(np.random.default_rng(1), 9, 20, storage), quality=q)
        same_store(gc, o)
        assert np.array_equal(ga.save(), gb.save()) and np.array_equal(gb.save(), gc.save())


def test_fetch_with_remove_and_a_repeated_id():
    g, o = store_pair(**QUALITY, feature_dim=8)
    f = _feats(np.random.default_rng(4), 3, 8, "f32")
    for s in (g, o):
        s.add([1, 1, 2], f, quality=[0.5, 0.75, 1.0])
    rg, ro = g.fetch_quality([1, 1, 2, 3], remove=True), o.fetch_quality([1, 1, 2, 3], remove=True)
    same_results(rg, ro)
    assert rg[0].tolist() == [2, 0, 1, 0] and not rg[2][1].any()
    assert g.size() == o.size() == 0
