"""GPU parity of the feature store's owned calls (sb200_fstore_search_owned / _merge_owned) with the CPU oracle: counts,
winner ids and f64 weights bit for bit, the stored rows after every merge, the blob of a merged store byte for byte
against the fetch + add emulation, and the chunked each-mode search against smaller calls."""
import numpy as np
import pytest

from fstore_checks import gpu_store, same_results, same_store, store_pair

pytestmark = pytest.mark.gpu


def _fill(stores, rng, n_tracks, dim, K, dup=0):
    """Tracks with 1 .. 2K + 1 observations (partial, full and wrapped rings), added in interleaved calls; the first
    `dup` tracks hold a copy of track 1's rows (equal weights)."""
    lens = 1 + (np.arange(n_tracks) * 7 + 3) % (2 * K + 1)
    ids = np.repeat(np.arange(1, n_tracks + 1, dtype=np.uint64), lens)
    rng.shuffle(ids)
    feats = rng.standard_normal((len(ids), dim)).astype(np.float32)
    for part in np.array_split(np.arange(len(ids)), 3):
        for s in stores:
            s.add(ids[part], feats[part])
    if dup:
        cnt, f = stores[-1].fetch([1])
        for t in range(n_tracks + 1, n_tracks + 1 + dup):
            for s in stores:
                s.add(np.full(cnt[0], t, np.uint64), f[0, :cnt[0]])


@pytest.mark.parametrize("metric", ["euclidean", "cosine"])
@pytest.mark.parametrize("K", [1, 3, 5])
@pytest.mark.parametrize("dim", [8, 250, 512])
def test_search_owned_matches_the_oracle(metric, K, dim):
    rng = np.random.default_rng(K * 1000 + dim)
    for topn, min_votes in ((1, 1), (5, 2)):
        g, o = store_pair(metric, max_observations=K, feature_dim=dim, topn=topn, min_votes=min_votes)
        _fill((g, o), rng, 40, dim, K, dup=2)
        ids = o.ids()
        q = np.concatenate([ids[rng.permutation(len(ids))[:9]], [777777]]).astype(np.uint64)
        for each in (False, True):
            same_results(g.search_owned(q, each=each), o.search_owned(q, each=each))
        same_results(g.search_owned(ids, each=True), o.search_owned(ids, each=True))
        same_store(g, o)
        assert np.all(g.last_stage_ms()[:2] >= 0)


@pytest.mark.parametrize("metric", ["euclidean", "cosine"])
def test_exact_thresholds_and_ties(metric):
    """max_distance and distance_filter placed on distances the oracle computes; duplicate rows tie on weight and go to
    the lower position."""
    rng = np.random.default_rng(17)
    g0, o0 = store_pair(metric, feature_dim=24, topn=5)
    _fill((g0, o0), rng, 30, 24, 3, dup=3)
    tie = o0.search_owned([5], each=True)
    same = [x for x in tie["winners"][0, :tie["counts"][0]].tolist() if x in (1, 31, 32, 33)]
    assert same == sorted(same)   # track 1 and its copies tie; the lower store position comes first
    same_results(g0.search_owned([5], each=True), tie)
    # distances from track 5's rows to every other stored row, as the oracle computes them
    import oracle
    cnt, f = o0.fetch([5])
    cs, fs = o0.fetch(o0.ids())
    dist = (lambda a, b: oracle.euclidean(a, b)) if metric == "euclidean" else \
        (lambda a, b: float(np.float32(1.0) - np.float32(oracle.cosine(a, b))))
    ds = sorted(dist(f[0, i], fs[t, j]) for i in range(cnt[0]) for t in range(len(cs)) for j in range(cs[t])
                if o0.ids()[t] != 5)
    for md, flt in ((ds[10], ds[30]), (ds[3], ds[10])):
        g, o = store_pair(metric, feature_dim=24, max_distance=md, distance_filter=flt, min_votes=2, topn=8)
        _fill((g, o), np.random.default_rng(17), 30, 24, 3, dup=3)
        for each in (False, True):
            q = np.array([5, 1, 31], np.uint64)
            same_results(g.search_owned(q, each=each), o.search_owned(q, each=each))


def test_search_owned_edges():
    g, o = store_pair(topn=5)
    for each in (False, True):
        same_results(g.search_owned([], each=each), o.search_owned([], each=each))
        same_results(g.search_owned([4, 5], each=each), o.search_owned([4, 5], each=each))   # empty store
    rng = np.random.default_rng(2)
    _fill((g, o), rng, 12, 16, 3)
    g.set_feature_type("f16")   # the rows are the stored f32 rows whatever the type
    for each in (False, True):
        same_results(g.search_owned(o.ids(), each=each), o.search_owned(o.ids(), each=each))
    import similari_b200._lib as L
    with pytest.raises(L.Sb200Error):
        g.search_owned([1, 1])
    same_store(g, o)


def _blob(s):
    return bytes(s.save())


def _emulate(e, dest, src, remove):
    for d, c in zip(dest, src):
        cnt, f = e.fetch([c])
        e.add(np.full(cnt[0], d, np.uint64), f[0, :cnt[0]])
        if remove:
            e.fetch([c], remove=True)


def _pairs(rng, ids, n, remove):
    """Random pairs with chains (a source that was a destination) and stars (one destination, many sources)."""
    ids = [int(x) for x in ids]
    dest, src, gone = [], [], set()
    hub = ids[0]
    while len(dest) < n and len(gone) < len(ids) - 2:
        kind = rng.integers(3)
        if kind == 0 and dest:   # chain: the last destination becomes a source
            c, d = dest[-1], int(rng.choice(ids))
        elif kind == 1:   # star into the hub
            d, c = hub, int(rng.choice(ids))
        else:
            d, c = (int(x) for x in rng.choice(ids, 2, replace=False))
        if d == c or d in gone or c in gone:
            continue
        dest.append(d)
        src.append(c)
        if remove:
            gone.add(c)
    return dest, src


@pytest.mark.parametrize("metric", ["euclidean", "cosine"])
@pytest.mark.parametrize("K", [1, 3, 5])
@pytest.mark.parametrize("remove", [False, True])
def test_merge_owned_matches_the_oracle_and_the_emulation(metric, K, remove):
    import similari_b200.engine as eng

    rng = np.random.default_rng(K * 10 + remove)
    g, o = store_pair(metric, max_observations=K, feature_dim=40, topn=5)
    e = gpu_store(metric, max_observations=K, feature_dim=40, topn=5)
    _fill((g, o, e), rng, 60, 40, K)
    for step in range(3):
        dest, src = _pairs(rng, o.ids(), 25, remove)
        g.merge_owned(dest, src, remove=remove)
        o.merge_owned(dest, src, remove=remove)
        _emulate(e, dest, src, remove)
        same_store(g, o)
        assert _blob(g) == _blob(e)
        assert g.last_stage_ms()[2] >= 0
        q = o.ids()[: 6]
        for each in (False, True):
            same_results(g.search_owned(q, each=each), o.search_owned(q, each=each))
        qid = np.arange(5000 + 10 * step, 5003 + 10 * step, dtype=np.uint64)
        offs = np.array([0, 1, 3, 4], np.int32)
        f = rng.standard_normal((4, 40)).astype(np.float32)
        same_results(g.search(qid, offs, f), o.search(qid, offs, f))
        same_results(g.associate(qid, offs, f), o.associate(qid, offs, f))
        e.associate(qid, offs, f)
        same_store(g, o)
    h = eng.FeatureStore.load(g.save())
    dest, src = _pairs(rng, o.ids(), 10, remove)
    for s in (g, h, o):
        s.merge_owned(dest, src, remove=remove)
    same_store(h, o)
    assert _blob(h) == _blob(g)


def test_star_of_many_sources_and_refusals():
    import similari_b200._lib as L

    rng = np.random.default_rng(5)
    g, o = store_pair(max_observations=4, feature_dim=8, topn=5)
    e = gpu_store(max_observations=4, feature_dim=8, topn=5)
    _fill((g, o, e), rng, 1200, 8, 4)
    src = [int(x) for x in o.ids()[1:1001]]
    dest = [int(o.ids()[0])] * len(src)
    before = _blob(g)
    for bad_dest, bad_src, rm in (([dest[0]], [dest[0]], False), ([99999], [src[0]], False),
                                  ([dest[0]], [99999], True), ([dest[0], src[0]], [src[0], src[1]], True),
                                  ([dest[0], dest[0]], [src[0], src[0]], True)):
        with pytest.raises(L.Sb200Error):
            g.merge_owned(bad_dest, bad_src, remove=rm)
        assert _blob(g) == before
    with pytest.raises(ValueError):
        g.merge_owned([1, 2], [3])
    g.merge_owned([], [], remove=True)
    assert _blob(g) == before
    for s in (g, o):
        s.merge_owned(dest, src, remove=True)
    _emulate(e, dest, src, True)
    same_store(g, o)
    assert _blob(g) == _blob(e)


def test_each_mode_chunks_a_whole_store():
    """40,000 single-observation 8-d tracks, all queried: 40,000 x 40,000 pairs need two chunks of 2^30."""
    rng = np.random.default_rng(40)
    n = 40000
    g, o = store_pair(max_observations=1, feature_dim=8, topn=3)
    ids = np.arange(1, n + 1, dtype=np.uint64)
    f = rng.standard_normal((n, 8)).astype(np.float32)
    g.add(ids, f)
    o.add(ids, f)
    whole = g.search_owned(ids, each=True)
    parts = [g.search_owned(ids[a:a + 9000], each=True) for a in range(0, n, 9000)]
    same_results(whole, {k: np.concatenate([p[k] for p in parts]) for k in whole})
    sample = rng.choice(n, 6, replace=False)
    ro = o.search_owned(ids[sample], each=True)
    same_results({k: v[sample] for k, v in whole.items()}, ro)
    import similari_b200._lib as L
    with pytest.raises(L.Sb200Error, match="-3|2\\^30"):
        g.search_owned(ids, each=False)
