"""GPU checks of the store-to-store calls: find_baked and associate_store (the main loop of the reference's
examples/track_merging.rs).  On newest stores associate_store must leave both stores exactly as the host composition
src.fetch(ids, remove) (+ src.attributes(ids)) then dst.associate(rows) leaves twin stores, outputs and both blobs byte
for byte, for every pair of storage types, both metrics, gated and ungated, remove 0 and 1.  On quality stores it is
held to the CPU oracle bit for bit.  Also: a seeded collect / find_baked / promote pipeline with a save and load of both
stores in the middle, find_baked against Python integers, a gallery-scale case and every refusal."""
import itertools
import zlib

import numpy as np
import pytest

import fstore_oracle as fo
from fstore_checks import gpu_store, same_results, same_store, store_pair

pytestmark = pytest.mark.gpu

TYPES = ("f32", "f16", "bf16")
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
ERR_INVALID, ERR_CAPACITY = -1, -3
OPTS = dict(max_observations=4, feature_dim=20, topn=2, max_distance=3.0)


def _exact(x):
    """x as values every storage type holds exactly (bf16 values inside the f16 normal range), so that a store of any
    type holds the oracle's f32 row."""
    x = fo.round_rows(np.asarray(x, np.float32), "bf16")
    x[np.abs(x) < 1e-3] = 0.0
    assert np.array_equal(fo.round_rows(x, "f16"), x)
    return x


def _fill(stores, rng, ids, K, dim, centers=None, gate=None, quality=False, t_base=0):
    """Adds 1..K rows to each of `ids` in every store: near centers[i] when given, with a window per track (gated) and
    qualities with ties (quality)."""
    rows, rid, q, src, t0, t1 = [], [], [], [], [], []
    for i, t in enumerate(ids):
        n = int(rng.integers(1, K + 1))
        base = centers[i] if centers is not None else rng.standard_normal(dim)
        rows.append(base + 0.05 * rng.standard_normal((n, dim)))
        rid += [t] * n
        q += list(rng.integers(-2, 4, n) * 0.25)
        a = t_base + int(rng.integers(0, 1000))
        src += [int(t) % 2 + 1] * n
        t0 += [a] * n
        t1 += [a + int(rng.integers(0, 5))] * n
    f = _exact(np.concatenate(rows))
    kw = dict(sources=src, t_start=t0, t_end=t1) if gate else {}
    if quality:
        kw["quality"] = np.array(q, np.float32)
    for s in stores:
        s.add(np.array(rid, np.uint64), f, **kw)


def _compose(dst, src, ids, remove):
    """The host composition associate_store replaces: fetch (and the attributes) from src, associate into dst."""
    kw = {}
    if src.gate is not None:
        s, t0, t1 = src.attributes(ids)
        kw = dict(sources=s, t_start=t0, t_end=t1)
    counts, feats = src.fetch(ids, remove=remove)
    offs = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    rows = np.concatenate([feats[i, :counts[i]] for i in range(len(ids))]) if len(ids) else feats.reshape(0, dst.D)
    return dst.associate(ids, offs, rows, **kw)


@pytest.mark.parametrize("gate", [None, "same_source"])
@pytest.mark.parametrize("metric", ["euclidean", "cosine"])
def test_newest_stores_match_the_host_composition(metric, gate):
    merged = new = 0
    for st_d, st_s in itertools.product(TYPES, TYPES):
        for remove in (0, 1):
            rng = np.random.default_rng(zlib.crc32(repr((metric, gate, st_d, st_s, remove)).encode()))
            K, dim = 4, 20
            md = 3.0 if metric == "euclidean" else 0.5   # near pairs within, unrelated ones beyond
            da, db = (gpu_store(metric, st_d, gate=gate, **OPTS | dict(max_distance=md)) for _ in range(2))
            sa, sb = (gpu_store(metric, st_s, gate=gate, **OPTS | dict(topn=3)) for _ in range(2))
            centers = rng.standard_normal((30, dim))
            _fill([da, db], rng, np.arange(1, 31, dtype=np.uint64), K, dim, centers, gate)
            near = centers[rng.integers(0, 30, 40)] + 0.02
            near[30:] = rng.standard_normal((10, dim))   # a quarter of the source tracks resemble no stored track
            _fill([sa, sb], rng, np.arange(1000, 1040, dtype=np.uint64), K, dim, near, gate)
            for rnd in range(3):
                ids = rng.permutation(np.setdiff1d(sa.ids(), da.ids()))[: int(rng.integers(4, 14))]   # not in dst
                what = (metric, gate, st_d, st_s, remove, rnd)
                ra = da.associate_store(sa, ids, remove=bool(remove))
                rb = _compose(db, sb, ids, bool(remove))
                same_results(ra, rb, what)
                merged, new = merged + int(ra["merged"].sum()), new + int((ra["merged"] == 0).sum())
                assert np.array_equal(da.save(), db.save()), what
                assert np.array_equal(sa.save(), sb.save()), what
                assert sa.size() == (40 if not remove else sb.size())
    assert merged > 50 and new > 20, (merged, new)


def _quality_pair(metric, gate, st_d, st_s, rng, K=12, dim=24):
    kw = dict(max_observations=K, feature_dim=dim, topn=3, max_distance=4.0)
    dg, do = store_pair(metric, st_d, gate, "quality", **kw)
    sg, so = store_pair(metric, st_s, gate, "quality", **kw)
    centers = rng.standard_normal((24, dim))
    _fill([dg, do], rng, np.arange(1, 25, dtype=np.uint64), K, dim, centers, gate, quality=True)
    near = rng.integers(0, 24, 60)
    _fill([sg, so], rng, np.arange(1000, 1060, dtype=np.uint64), K, dim, centers[near] + 0.02, gate, quality=True,
          t_base=5000)
    # merge histories longer than 1 on both sides (merge_owned refuses incompatible windows: pick compatible pairs)
    for g, o, base in ((sg, so, 1000), (dg, do, 1)):
        pairs = [(base + 4 * i, base + 4 * i + 2) for i in range(6)]   # ids of one parity: one source
        if gate:
            src, t0, t1 = o.attributes([x for p in pairs for x in p])
            pairs = [p for i, p in enumerate(pairs) if src[2 * i] == src[2 * i + 1]
                     and (t0[2 * i] >= t1[2 * i + 1] or t1[2 * i] <= t0[2 * i + 1])]
        d = np.array([p[0] for p in pairs], np.uint64)
        s = np.array([p[1] for p in pairs], np.uint64)
        g.merge_owned(d, s)
        o.merge_owned(d, s)
    return dg, do, sg, so


@pytest.mark.parametrize("gate", [None, "same_source"])
@pytest.mark.parametrize("metric", ["euclidean", "cosine"])
@pytest.mark.parametrize("types", [("f32", "f32"), ("bf16", "f16"), ("f16", "f32")])
def test_quality_stores_match_the_oracle(types, metric, gate):
    rng = np.random.default_rng(zlib.crc32(repr((types, metric, gate)).encode()))
    dg, do, sg, so = _quality_pair(metric, gate, *types, rng)
    same_store(dg, do)
    same_store(sg, so)
    for rnd in range(4):
        ids = rng.permutation(np.setdiff1d(so.ids(), do.ids()))[: int(rng.integers(1, 16))]
        remove = rnd != 1
        rg = dg.associate_store(sg, ids, remove=remove)
        ro = do.associate_store(so, ids, remove=remove)
        same_results(rg, ro, (types, metric, gate, rnd))
        same_store(dg, do)
        same_store(sg, so)
    assert np.any([len(h) > 2 for h in dg.merge_history(dg.ids())])


@pytest.mark.parametrize("retention", ["newest", "quality"])
def test_pipeline_with_a_save_and_load_in_the_middle(retention):
    """Collect tracklets frame by frame in a gated store, promote the baked ones into a gallery every frame; halfway
    both stores are saved and reloaded, and the run continues exactly as the oracle's, which is never reloaded."""
    import similari_b200.engine as eng

    rng = np.random.default_rng(11 if retention == "newest" else 12)
    K, dim, period = 12, 32, 3
    kw = dict(max_observations=K, feature_dim=dim, topn=1, max_distance=2.5, min_votes=2)
    q = retention == "quality"
    col_g, col_o = store_pair("euclidean", "f16", "same_source", retention, **kw)
    gal_g, gal_o = store_pair("euclidean", "bf16", "same_source", retention, **kw)
    people = rng.standard_normal((20, dim)).astype(np.float32)
    active, next_id, promoted = {}, 1, 0
    for frame in range(60):
        if frame == 30:
            col_g = eng.FeatureStore.load(col_g.save())
            gal_g = eng.FeatureStore.load(gal_g.save())
        while len(active) < 12:   # tracklet id -> (person, camera, last frame)
            active[next_id] = (int(rng.integers(0, 20)), int(rng.integers(1, 4)), frame + int(rng.integers(3, 10)))
            next_id += 1
        ids = np.array(sorted(active), np.uint64)
        rows = _exact(0.0625 * rng.standard_normal((len(ids), dim)) + people[[active[int(t)][0] for t in ids]])
        a = dict(sources=[active[int(t)][1] for t in ids], t_start=[frame] * len(ids), t_end=[frame] * len(ids))
        if q:
            a["quality"] = rng.integers(0, 5, len(ids)).astype(np.float32)
        col_g.add(ids, rows, **a)
        col_o.add(ids, rows, **a)
        active = {t: v for t, v in active.items() if v[2] > frame}
        baked = col_o.find_baked(frame, period)
        assert np.array_equal(col_g.find_baked(frame, period), baked), frame
        rg = gal_g.associate_store(col_g, baked)
        ro = gal_o.associate_store(col_o, baked)
        same_results(rg, ro, frame)
        promoted += len(baked)
        assert np.array_equal(col_g.ids(), col_o.ids()) and np.array_equal(gal_g.ids(), gal_o.ids())
        if frame % 10 == 9:
            same_store(gal_g, gal_o)
            same_store(col_g, col_o)
    assert promoted > 40 and gal_o.size() < promoted   # tracklets were merged into identities


def test_find_baked_matches_python_integers():
    from similari_b200 import _lib

    rng = np.random.default_rng(5)
    extremes = [I64_MIN, I64_MIN + 1, -2, -1, 0, 1, 2, I64_MAX - 1, I64_MAX]
    n = 3000
    ends = rng.integers(-10**6, 10**6, n).astype(np.int64)
    ends[: len(extremes)] = extremes
    ends[rng.random(n) < 0.05] = rng.choice(extremes, 1)[0]
    g = gpu_store(gate="any_source", **OPTS | dict(max_observations=1, feature_dim=8))
    ids = rng.permutation(np.arange(1, n + 1, dtype=np.uint64) * 7)
    g.add(ids, np.zeros((n, 8), np.float32), sources=np.ones(n, np.uint64), t_start=np.full(n, I64_MIN, np.int64),
          t_end=ends)

    def check(store, tag):
        sid = store.ids()
        _, _, te = store.attributes(sid)
        for now in extremes + [int(x) for x in rng.integers(-10**6, 10**6, 6)]:
            for period in extremes + [int(x) for x in rng.integers(-10**6, 10**6, 3)]:
                want = [int(t) for t, e in zip(sid, te.tolist()) if now > e + period]
                assert store.find_baked(now, period).tolist() == want, (tag, now, period)

    check(g, "fresh")
    g.fetch(ids[rng.random(n) < 0.3], remove=True)   # removals: the compaction moves the windows
    check(g, "removed")
    h = type(g).load(g.save())
    check(h, "loaded")
    # cap truncation: the first min(cap, total) ids, the total returned
    L, p = _lib.lib(), _lib.ptr
    want = h.find_baked(0, 0)
    assert len(want) > 10
    for cap in (0, 1, 7, len(want), len(want) + 5):
        out = np.zeros(max(1, cap), np.uint64)
        total = L.sb200_fstore_find_baked(h._h, 0, 0, cap, p(out) if cap else None)
        assert total == len(want)
        assert np.array_equal(out[: min(cap, total)], want[:cap])


def test_gallery_scale():
    """20,000 tracks x K = 12 x 512-d gallery (gated, bf16), 256 collected tracks promoted at once, against the host
    composition on a twin loaded from the same blob."""
    import similari_b200.engine as eng

    rng = np.random.default_rng(7)
    K, dim, n = 12, 512, 20000
    kw = dict(max_observations=K, feature_dim=dim, topn=4, max_distance=12.0, min_votes=1)
    g = gpu_store("euclidean", "bf16", gate="same_source", **OPTS | kw)
    centers = rng.standard_normal((n, dim)).astype(np.float32)
    for a in range(0, n, 2000):
        ids = np.repeat(np.arange(a + 1, a + 2001, dtype=np.uint64), K)
        rows = np.repeat(centers[a:a + 2000], K, axis=0) + 0.05 * rng.standard_normal((2000 * K, dim), np.float32)
        t = np.repeat(np.arange(a, a + 2000, dtype=np.int64) * 10, K)
        g.add(ids, rows, sources=ids % 3 + 1, t_start=t, t_end=t + 5)
    blob = g.save()
    twin = eng.FeatureStore.load(blob)
    src_a, src_b = (gpu_store(gate="same_source", **OPTS | kw) for _ in range(2))
    pick = rng.integers(0, n, 256)
    _fill([src_a, src_b], rng, np.arange(10**6, 10**6 + 256, dtype=np.uint64), K, dim, centers[pick], "same_source",
          t_base=10**6)
    ids = src_a.ids()
    ra = g.associate_store(src_a, ids)
    rb = _compose(twin, src_b, ids, True)
    same_results(ra, rb, "gallery")
    assert ra["merged"].sum() > 40 and (ra["merged"] == 0).sum() > 40   # the source gate leaves about 1 in 3
    assert np.array_equal(g.save(), twin.save())
    assert src_a.size() == 0 and np.array_equal(src_a.save(), src_b.save())


def test_refusals_leave_both_stores_unchanged():
    from similari_b200 import _lib

    L, p = _lib.lib(), _lib.ptr
    kw = dict(max_observations=4, feature_dim=8)
    dst = gpu_store(gate="same_source", retention="quality", **OPTS | kw)
    src = gpu_store(storage="bf16", gate="same_source", retention="quality", **OPTS | kw)
    f = np.ones((3, 8), np.float32)
    dst.add([1], f[:1], sources=[1], t_start=[0], t_end=[1], quality=[1])
    src.add([7, 8], f[:2], sources=[1, 1], t_start=[5, 5], t_end=[6, 6], quality=[1, 1])
    blobs = (dst.save(), src.save())
    out = [np.zeros(2, np.int32), np.zeros((2, 2), np.uint64), np.zeros((2, 2), np.float64), np.zeros(2, np.uint64),
           np.zeros(2, np.uint8)]
    o = [p(x) for x in out]

    def refused(a, b, ids, word, n=None, remove=1, outs=o):
        ids = np.array(ids, np.uint64)
        rc = L.sb200_fstore_associate_store(a, b, len(ids) if n is None else n, p(ids), remove, *outs)
        msg = L.sb200_last_error().decode()
        assert rc == ERR_INVALID and word in msg, (word, rc, msg)
        assert np.array_equal(dst.save(), blobs[0]) and np.array_equal(src.save(), blobs[1]), word

    refused(dst._h, None, [7], "NULL")
    refused(None, src._h, [7], "NULL")
    refused(dst._h, dst._h, [1], "same store")
    for other, word in [(dict(gate="same_source", retention="quality", max_observations=4, feature_dim=16),
                         "feature_dim"),
                        (dict(gate="same_source", retention="quality", max_observations=6, feature_dim=8),
                         "max_observations"),
                        (dict(gate="any_source", retention="quality", **kw), "gate"),
                        (dict(retention="quality", **kw), "gate"),
                        (dict(gate="same_source", **kw), "retention"),
                        (dict(gate="same_source", retention="quality", initial_capacity=3, **kw), "retention"),
                        (dict(gate="same_source", retention="quality", merge_extension=2.0, **kw), "retention")]:
        other = gpu_store(**OPTS | other)
        refused(dst._h, other._h, [], word)
    refused(dst._h, src._h, [7], "n < 0", n=-1)
    refused(dst._h, src._h, [7], "remove", remove=2)
    refused(dst._h, src._h, [7, 7], "twice")
    refused(dst._h, src._h, [9], "not stored in src")
    refused(dst._h, src._h, [8, 1], "already stored")
    refused(dst._h, src._h, [7], "NULL", outs=[o[0], None, o[2], o[3], o[4]])
    # the pair bound: 65 x 64 queried rows against 4096 x 64 stored slots is just above 2^30 pairs
    big_d, big_s = (gpu_store(**OPTS | dict(max_observations=64, feature_dim=8)) for _ in range(2))
    big_d.add(np.repeat(np.arange(1, 4097, dtype=np.uint64), 64), np.zeros((4096 * 64, 8), np.float32))
    big_s.add(np.repeat(np.arange(10**6, 10**6 + 65, dtype=np.uint64), 64), np.zeros((65 * 64, 8), np.float32))
    bd, bs = big_d.save(), big_s.save()
    ids = big_s.ids()
    outs = [np.zeros(len(ids) * 4) for _ in range(5)]   # each holds any of the five outputs
    rc = L.sb200_fstore_associate_store(big_d._h, big_s._h, len(ids), p(ids), 1, *[p(x) for x in outs])
    assert rc == ERR_CAPACITY and "2^30" in L.sb200_last_error().decode()
    assert np.array_equal(big_d.save(), bd) and np.array_equal(big_s.save(), bs)
    # find_baked
    u = gpu_store(**OPTS | kw)
    assert L.sb200_fstore_find_baked(u._h, 0, 0, 0, None) < 0 and "gate" in L.sb200_last_error().decode()
    assert L.sb200_fstore_find_baked(dst._h, 0, 0, -1, None) < 0
    assert L.sb200_fstore_find_baked(dst._h, 0, 0, 1, None) < 0
    assert L.sb200_fstore_find_baked(dst._h, 10, 0, 0, None) == 1   # sizing call
    # n == 0 changes nothing
    assert dst.associate_store(src, [])["counts"].tolist() == []
    assert np.array_equal(dst.save(), blobs[0]) and np.array_equal(src.save(), blobs[1])
