"""GPU parity of the feature track store (sb200_fstore_*, kernels_fstore.cu) with the CPU oracle (fstore_oracle):
winner ids, f64 weights, merged flags and the stored observations after every call, bit for bit."""
import numpy as np
import pytest

from fstore_checks import same_results, same_store, store_pair
from similari_b200.workload import FeatGen

pytestmark = pytest.mark.gpu
# the options of benches/feature_tracker.rs (engine.FeatureStore's defaults)
BENCH = dict(distance_filter=100.0, feature_dim=256, topn=1, max_distance=100.0)


def _queries(rows_per_query, dim):
    offs = np.cumsum([0] + [len(r) for r in rows_per_query]).astype(np.int32)
    feats = np.concatenate([np.asarray(r, np.float32).reshape(-1, dim) for r in rows_per_query]) if rows_per_query \
        else np.zeros((0, dim), np.float32)
    return offs, feats


@pytest.mark.parametrize("metric", ["euclidean", "cosine"])
@pytest.mark.parametrize("objects", [10, 100, 500])
def test_feature_tracker_loop(metric, objects):
    """benches/feature_tracker.rs: every iteration one new single-observation track per object, associated with TopN(1,
    100.0, 1) under d < 100.0, K = 3, D = 256."""
    g, o = store_pair(metric, **BENCH)
    gens = [FeatGen(1000.0 * i, 256, 0.1, seed=1000 + i) for i in range(objects)]
    iteration = 0
    for _ in range(20):
        ids = np.arange(iteration + 1, iteration + 1 + objects, dtype=np.uint64)
        iteration += objects
        offs, feats = _queries([[gen.next()] for gen in gens], 256)
        same_results(g.associate(ids, offs, feats), o.associate(ids, offs, feats))
        same_store(g, o)
    assert g.size() >= objects
    assert np.all(g.last_stage_ms() >= 0)


@pytest.mark.parametrize("metric", ["euclidean", "cosine"])
def test_track_search_shape(metric):
    """benches/track_search.rs's shape: a 30-observation query against 100 tracks of 30 observations."""
    rng = np.random.default_rng(7)
    g, o = store_pair(metric, max_observations=30, feature_dim=128, topn=5)
    ids = np.repeat(np.arange(1, 101, dtype=np.uint64), 30)
    feats = rng.standard_normal((3000, 128)).astype(np.float32)
    g.add(ids, feats)
    o.add(ids, feats)
    same_store(g, o)
    offs, q = _queries([rng.standard_normal((30, 128))], 128)
    same_results(g.search(np.array([1000], np.uint64), offs, q), o.search(np.array([1000], np.uint64), offs, q))


@pytest.mark.parametrize("metric", ["euclidean", "cosine"])
@pytest.mark.parametrize("dim", [8, 250, 2048])
@pytest.mark.parametrize("topn", [1, 5, 64])
def test_dims_and_topn(metric, dim, topn):
    """D a multiple of 8, not one, and wide; topn 1, 5 and more than the store holds (40 tracks)."""
    rng = np.random.default_rng(dim * 100 + topn)
    g, o = store_pair(metric, feature_dim=dim, topn=topn, max_observations=4)
    for step in range(3):
        n = 40
        ids = rng.integers(1, 41, n).astype(np.uint64)
        f = rng.standard_normal((n, dim)).astype(np.float32)
        g.add(ids, f)
        o.add(ids, f)
        same_store(g, o)
        qid = np.arange(100, 108, dtype=np.uint64)
        offs, q = _queries([rng.standard_normal((k % 6 + 1, dim)) for k in range(8)], dim)
        same_results(g.search(qid, offs, q), o.search(qid, offs, q))
        qid = qid + 1000 * (step + 1)
        same_results(g.associate(qid, offs, q), o.associate(qid, offs, q))
        same_store(g, o)


@pytest.mark.parametrize("metric", ["euclidean", "cosine"])
def test_min_votes_and_exact_thresholds(metric):
    """min_votes 2 and 3, max_distance and distance_filter placed on distances the oracle computes."""
    import oracle

    rng = np.random.default_rng(11)
    dim = 24
    tracks = rng.standard_normal((60, dim)).astype(np.float32)
    ids = np.repeat(np.arange(1, 21, dtype=np.uint64), 3)
    queries = rng.standard_normal((4, dim)).astype(np.float32)
    dist = (lambda a, b: oracle.euclidean(a, b)) if metric == "euclidean" else \
        (lambda a, b: float(np.float32(1.0) - np.float32(oracle.cosine(a, b))))
    ds = sorted(dist(queries[0], t) for t in tracks)
    for min_votes in (2, 3):
        for md, flt in ((ds[20], ds[40]), (ds[5], ds[20])):
            g, o = store_pair(metric, feature_dim=dim, max_observations=3, topn=8, min_votes=min_votes, max_distance=md,
                              distance_filter=flt)
            g.add(ids, tracks)
            o.add(ids, tracks)
            offs, q = _queries([queries[:2], queries[2:]], dim)
            qid = np.array([500, 501], np.uint64)
            ro = o.search(qid, offs, q)
            same_results(g.search(qid, offs, q), ro)
            same_results(g.associate(qid, offs, q), o.associate(qid, offs, q))
            same_store(g, o)


@pytest.mark.parametrize("metric", ["euclidean", "cosine"])
def test_ties_empty_store_and_remove_then_add(metric):
    rng = np.random.default_rng(3)
    dim = 16
    g, o = store_pair(metric, feature_dim=dim, topn=6)
    offs, q = _queries([rng.standard_normal((2, dim))], dim)
    same_results(g.search(np.array([9], np.uint64), offs, q), o.search(np.array([9], np.uint64), offs, q))
    base = rng.standard_normal((1, dim)).astype(np.float32)
    dup = np.repeat(base, 5, axis=0)   # five identical tracks: equal weights, store order decides
    ids = np.array([30, 10, 50, 20, 40], np.uint64)
    for s in (g, o):
        s.add(ids, dup)
    same_results(g.search(np.array([9], np.uint64), offs, q), o.search(np.array([9], np.uint64), offs, q))
    r = g.search(np.array([9], np.uint64), offs, q)
    assert r["winners"][0, :5].tolist() == [30, 10, 50, 20, 40]
    for s in (g, o):
        s.fetch(np.array([10, 77, 10], np.uint64), remove=True)
        s.add(np.array([10, 60], np.uint64), dup[:2])
    same_store(g, o)
    same_results(g.search(np.array([9], np.uint64), offs, q), o.search(np.array([9], np.uint64), offs, q))
    cg = g.fetch(np.array([10, 77, 10], np.uint64))
    co = o.fetch(np.array([10, 77, 10], np.uint64))
    assert np.array_equal(cg[0], co[0]) and np.array_equal(cg[1], co[1])
    same_results(g.associate(np.array([9], np.uint64), offs, q), o.associate(np.array([9], np.uint64), offs, q))
    same_store(g, o)


@pytest.mark.parametrize("metric", ["euclidean", "cosine"])
def test_degenerate_features(metric):
    """NaN, inf and zero rows: their entries drop out (or not) exactly as in the oracle and leave max_dist alone."""
    rng = np.random.default_rng(5)
    dim = 16
    t = rng.standard_normal((8, dim)).astype(np.float32)
    t[1] = 0.0
    t[2, 3] = np.nan
    t[3, 0] = np.inf
    t[4] = 1e30
    t[5] = 1e-30
    g, o = store_pair(metric, feature_dim=dim, topn=8, distance_filter=50.0, max_distance=20.0)
    ids = np.arange(1, 9, dtype=np.uint64)
    g.add(ids, t)
    o.add(ids, t)
    q = rng.standard_normal((6, dim)).astype(np.float32)
    q[1] = 0.0
    q[2, 5] = np.nan
    q[3, 7] = -np.inf
    offs, qf = _queries([q[:2], q[2:4], q[4:]], dim)
    qid = np.array([100, 101, 102], np.uint64)
    same_results(g.search(qid, offs, qf), o.search(qid, offs, qf))
    same_results(g.associate(qid, offs, qf), o.associate(qid, offs, qf))
    same_store(g, o)


def test_growth_across_calls():
    rng = np.random.default_rng(9)
    g, o = store_pair("euclidean", feature_dim=32, max_observations=2, topn=3, distance_filter=9.0, max_distance=4.0)
    nid = 1
    for step in range(12):
        n = 50 * (step + 1)
        ids = np.arange(nid, nid + n, dtype=np.uint64)
        nid += n
        offs, q = _queries([rng.standard_normal((1 + i % 3, 32)) for i in range(n)], 32)
        same_results(g.associate(ids, offs, q), o.associate(ids, offs, q))
        same_store(g, o)
    assert g.size() > 2000


def test_rejected_calls_change_nothing():
    from similari_b200._lib import Sb200Error
    import similari_b200.engine as eng

    rng = np.random.default_rng(1)
    g, o = store_pair("euclidean", **BENCH | dict(feature_dim=8, max_observations=64, topn=2))
    ids = np.arange(1, 16385, dtype=np.uint64)
    f = rng.standard_normal((len(ids), 8)).astype(np.float32)
    g.add(ids, f)
    o.add(ids, f)
    before_ids = g.ids()
    before = g.fetch(before_ids)

    def unchanged():
        assert np.array_equal(g.ids(), before_ids)
        c, x = g.fetch(before_ids)
        assert np.array_equal(c, before[0]) and np.array_equal(x.view(np.uint32), before[1].view(np.uint32))

    q1 = rng.standard_normal((2, 8)).astype(np.float32)
    bad = [
        (np.array([70000, 70000], np.uint64), np.array([0, 1, 2], np.int32), q1),        # duplicate query id
        (np.array([70000, 70001], np.uint64), np.array([0, 2, 2], np.int32), q1),        # a query without observations
    ]
    for qid, offs, q in bad:
        for call in (g.search, g.associate):
            with pytest.raises(Sb200Error):
                call(qid, offs, q)
            unchanged()
    with pytest.raises(Sb200Error):   # a stored id as a query of associate
        g.associate(np.array([3], np.uint64), np.array([0, 1], np.int32), q1[:1])
    unchanged()
    # 1025 query rows x 16384 tracks x K = 64 slots > 2^30 observation pairs
    big = rng.standard_normal((1025, 8)).astype(np.float32)
    offs = np.arange(0, 1026, dtype=np.int32)
    for call in (g.search, g.associate):
        with pytest.raises(Sb200Error, match="-3"):
            call(np.arange(100000, 101025, dtype=np.uint64), offs, big)
        unchanged()
    same_store(g, o)
    for kw in (dict(topn=65), dict(max_observations=65), dict(feature_dim=8193), dict(topn=0)):
        opts = dict(feature_dim=8)
        opts.update(kw)
        with pytest.raises(Sb200Error, match="-1"):
            eng.FeatureStore(**opts)
