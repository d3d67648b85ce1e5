"""BestFit voting of the feature store (sb200_fstore_set_voting) on the GPU, bit for bit against the CPU oracle: counts,
winners (the query's own id where another query took the track), f64 weights (through uint64 views), track_ids and
merged, then the stored state (ids, rows, qualities, merge histories, windows).

Configurations: every storage type x both metrics x {ungated, same_source, any_source} x {newest, quality}; host f32,
f16 / bf16 and device columns; a two-class store.  Calls: associate, search, search_owned with each 0 and 1 (1 equal to
TopN), associate_store and associate_wasted (against the host composition on a twin BestFit store).  Contention:
thousands of queries on a handful of tracks, with exact ties from duplicated rows.  Rule switching between calls, a
TopN call after switching back equal to an untouched TopN twin byte for byte, and the same blob under both rules."""
import numpy as np
import pytest

import fstore_oracle as fo
from fstore_checks import gpu_store, same_results, same_store, store_pair

pytestmark = pytest.mark.gpu

F32 = np.float32
TYPES = ("f32", "f16", "bf16")
GATES = (None, "same_source", "any_source")
# thresholds per metric that take the near tracks in and leave the unrelated ones out
OPTS = {"euclidean": dict(max_observations=4, feature_dim=24, topn=3, distance_filter=8.0, max_distance=5.0),
        "cosine": dict(max_observations=4, feature_dim=24, topn=3, distance_filter=1.2, max_distance=0.5)}


@pytest.fixture(scope="module")
def eng():
    import similari_b200.engine as e
    from similari_b200._lib import lib

    if lib().sb200_device_count() <= 0:
        pytest.fail("no CUDA device: the gpu-marked tests must run on an H100")
    return e


def _distinct_merges(out):
    """BestFit destinations are exclusive: no two merged queries of one call name the same track."""
    t = out["track_ids"][out["merged"].astype(bool)]
    assert len(np.unique(t)) == len(t)


class World:
    """Seeded tracks around a few centres, and queries drawn near the tracks of the first centres, so that several
    queries of one call share their best track.  Every row is representable in the storage type, so that the oracle,
    which keeps f32 rows, holds what the store holds.  Windows: stored rows early, the queries of round k in one
    overlapping band after them (coexisting queries, compatible with every stored track)."""

    def __init__(self, seed, D, storage, gate, retention):
        self.rng, self.D, self.storage, self.gate, self.quality = np.random.default_rng(seed), D, storage, gate, \
            retention == "quality"
        self.centres = self.rng.standard_normal((8, D)).astype(F32) * 2.0

    def rows(self, centre_of):
        x = self.centres[centre_of] + 0.4 * self.rng.standard_normal((len(centre_of), self.D)).astype(F32)
        return fo.round_rows(x, self.storage)

    def add_kw(self, ids, t0):
        kw = {}
        if self.gate:
            kw.update(sources=ids % 2, t_start=t0 + ids, t_end=t0 + ids + 1)
        if self.quality:
            kw["quality"] = self.rng.integers(0, 8, len(ids)).astype(F32) / 4
        return kw

    def queries(self, first_id, n, band):
        cnt = self.rng.integers(1, 6, n)
        offs = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int32)
        ids = np.arange(first_id, first_id + n, dtype=np.uint64)
        rows = self.rows(np.repeat(self.rng.integers(0, 3, n), cnt))
        kw = {}
        if self.gate:
            start = band + np.arange(n, dtype=np.int64)
            kw.update(sources=ids % 2, t_start=start, t_end=start + 50)
        if self.quality:
            kw["quality"] = self.rng.integers(0, 8, len(rows)).astype(F32) / 4
        return ids, offs, rows, kw

    def fill(self, stores, first_id, n, t0):
        ids = np.repeat(np.arange(first_id, first_id + n, dtype=np.uint64), self.rng.integers(1, 7, n))
        self.rng.shuffle(ids)
        rows = self.rows((ids % 8).astype(np.int64))
        kw = self.add_kw(ids, t0)
        for s in stores:
            s.add(ids, rows, **kw)


@pytest.mark.parametrize("retention", ["newest", "quality"])
@pytest.mark.parametrize("gate", GATES)
@pytest.mark.parametrize("metric", ["euclidean", "cosine"])
@pytest.mark.parametrize("storage", TYPES)
def test_every_call_matches_the_oracle(eng, storage, metric, gate, retention):
    seed = TYPES.index(storage) * 100 + GATES.index(gate) * 10 + (metric == "cosine") * 2 + (retention == "quality")
    w = World(seed, 24, storage, gate, retention)
    g, r = store_pair(metric, storage, gate, retention, "best_fit", min_votes=1 + seed % 2, **OPTS[metric])
    w.fill([g, r], 1, 40, 0)
    merged = new_with_results = 0
    for k in range(3):
        ids, offs, rows, kw = w.queries(1000 + 100 * k, 60, 10_000 * (k + 1))
        same_results(g.search(ids, offs, rows, **kw), r.search(ids, offs, rows, **kw))
        a = g.associate(ids, offs, rows, **kw)
        same_results(a, r.associate(ids, offs, rows, **kw))
        _distinct_merges(a)
        merged += int(a["merged"].sum())
        new_with_results += int(((a["counts"] > 0) & (a["merged"] == 0)).sum())
        same_store(g, r)
    assert merged > 0 and new_with_results > 0
    owned = g.ids()[::3]
    same_results(g.search_owned(owned), r.search_owned(owned))
    each = g.search_owned(owned, each=True)
    same_results(each, r.search_owned(owned, each=True))
    g.set_voting("topn")
    same_results(each, g.search_owned(owned, each=True))
    g.set_voting("best_fit")
    # associate_store from a source store of the same configuration, with dst's BestFit rule
    gs, rs = store_pair(metric, storage, gate, retention, "best_fit", min_votes=1 + seed % 2, **OPTS[metric])
    gs.set_voting("topn")
    rs.set_voting("topn")
    w.fill([gs, rs], 5000, 30, 100_000)
    moved = gs.ids()[::2]
    a = g.associate_store(gs, moved, remove=True)
    same_results(a, r.associate_store(rs, moved, remove=True))
    _distinct_merges(a)
    same_store(g, r)
    same_store(gs, rs)
    blob = g.save()
    g.set_voting("topn")
    assert np.array_equal(g.save(), blob)
    back = eng.FeatureStore.load(blob)
    assert back.voting() == "topn" and eng.FeatureStore.load(blob, voting="best_fit").voting() == "best_fit"
    assert np.array_equal(back.save(), blob)


@pytest.mark.parametrize("ftype", ["f32", "f16", "bf16", "device"])
def test_column_types_and_device_columns(eng, ftype):
    import torch

    w = World(31, 40, "f16", None, "newest")
    g, r = store_pair("euclidean", "bf16", voting="best_fit", **OPTS["euclidean"] | dict(feature_dim=40))
    w.centres = fo.round_rows(fo.round_rows(w.centres, "f16"), "bf16")
    w.storage = "bf16"
    w.fill([g, r], 1, 50, 0)
    for k in range(2):
        ids, offs, rows, _ = w.queries(1000 + 100 * k, 80, 0)
        rows[np.abs(rows) < 1e-3] = 0.0   # bf16 values that f16 holds too (no f16 subnormals)
        if ftype == "f32":
            a = g.associate(ids, offs, rows)
        elif ftype == "device":
            d = torch.from_numpy(rows).cuda()
            a = g.associate_device(ids, offs, d.data_ptr())
        else:
            g.set_feature_type(ftype)
            col = rows.astype(np.float16) if ftype == "f16" else (rows.view(np.uint32) >> 16).astype(np.uint16)
            a = g.associate(ids, offs, col)
            g.set_feature_type("f32")
        same_results(a, r.associate(ids, offs, rows))
        _distinct_merges(a)
    same_store(g, r)


@pytest.mark.parametrize("retention", ["newest", "quality"])
def test_two_classes(eng, retention):
    classes = {7: 16, 2: 24}
    g, r = store_pair(retention=retention, voting="best_fit", classes=classes,
                      **OPTS["euclidean"] | dict(feature_dim=16))
    rng = np.random.default_rng(5)
    q = retention == "quality"
    cen = {c: rng.standard_normal((6, d)).astype(F32) * 2 for c, d in classes.items()}
    for c, d in classes.items():
        ids = np.repeat(np.arange(1, 31, dtype=np.uint64), 2)
        ids = ids[(ids + c) % 4 != 0]
        rows = cen[c][ids % 6] + 0.4 * rng.standard_normal((len(ids), d)).astype(F32)
        kw = dict(quality=rng.integers(0, 4, len(ids)).astype(F32)) if q else {}
        g.add(ids, rows, feature_class=c, **kw)
        r.add(ids, rows, feature_class=c, **kw)
    for c, d in classes.items():
        n = 40
        ids = np.arange(100 * (c + 1), 100 * (c + 1) + n, dtype=np.uint64)
        offs = np.arange(n + 1, dtype=np.int32) * 2
        rows = cen[c][np.repeat(rng.integers(0, 2, n), 2)] + 0.4 * rng.standard_normal((2 * n, d)).astype(F32)
        kw = dict(quality=rng.integers(0, 4, 2 * n).astype(F32)) if q else {}
        a = g.associate(ids, offs, rows, feature_class=c, **kw)
        same_results(a, r.associate(ids, offs, rows, feature_class=c, **kw))
        _distinct_merges(a)
    same_store(g, r)


@pytest.mark.parametrize("metric", ["euclidean", "cosine"])
def test_thousands_of_queries_on_a_handful_of_tracks(eng, metric):
    """4,000 queries of one or two rows on 6 tracks; many queries repeat the same rows, so their groups tie exactly
    and the lower query index must win."""
    rng = np.random.default_rng(9)
    g, r = store_pair(metric, voting="best_fit", max_observations=2, feature_dim=32, topn=4)
    base = rng.standard_normal((6, 32)).astype(F32)
    ids = np.repeat(np.arange(1, 7, dtype=np.uint64), 2)
    rows = base[ids - 1] + 0.2 * rng.standard_normal((12, 32)).astype(F32)
    g.add(ids, rows)
    r.add(ids, rows)
    pool = base[rng.integers(0, 6, 40)] + 0.3 * rng.standard_normal((40, 32)).astype(F32)
    n = 4000
    cnt = rng.integers(1, 3, n)
    offs = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int32)
    q = pool[rng.integers(0, 40, int(offs[-1]))]
    qid = np.arange(10_000, 10_000 + n, dtype=np.uint64)
    a = g.associate(qid, offs, q)
    same_results(a, r.associate(qid, offs, q))
    assert 0 < a["merged"].sum() <= 6
    _distinct_merges(a)
    ws = a["weights"][:, 0][a["counts"] > 0]
    assert len(np.unique(ws)) < len(ws)   # exact ties took part
    same_store(g, r)
    s = g.search(qid[:3000], offs[:3001], q[: offs[3000]])
    same_results(s, r.search(qid[:3000], offs[:3001], q[: offs[3000]]))
    same_results(g.search_owned(g.ids()[:5]), r.search_owned(r.ids()[:5]))


def test_switching_the_rule_between_calls(eng):
    """One store switches rules between calls, the oracle with it; a TopN call after switching back leaves it byte for
    byte as an untouched TopN twin that made the same calls under TopN."""
    w = World(77, 24, "f32", None, "newest")
    g, r = store_pair(voting="best_fit", **OPTS["euclidean"])
    twin = gpu_store(**OPTS["euclidean"])
    w.fill([g, r, twin], 1, 40, 0)
    rules = ["best_fit", "topn", "best_fit", "best_fit", "topn"]
    for k, rule in enumerate(rules):
        g.set_voting(rule)
        r.set_voting(rule)
        ids, offs, rows, _ = w.queries(1000 + 100 * k, 50, 0)
        if rule == "best_fit":
            same_results(g.search(ids, offs, rows), r.search(ids, offs, rows))
            same_results(g.search_owned(g.ids()[:9]), r.search_owned(r.ids()[:9]))
            continue   # searches change nothing, so the twin stays in step
        a = g.associate(ids, offs, rows)
        same_results(a, r.associate(ids, offs, rows))
        same_results(a, twin.associate(ids, offs, rows))
        assert np.array_equal(g.save(), twin.save())
    g.set_voting("best_fit")
    r.set_voting("best_fit")
    ids, offs, rows, _ = w.queries(9000, 50, 0)
    same_results(g.associate(ids, offs, rows), r.associate(ids, offs, rows))
    same_store(g, r)
    from similari_b200._lib import lib

    before = g.voting()
    assert lib().sb200_fstore_set_voting(g._h, 2) == -1 and g.voting() == before
    with pytest.raises(ValueError):
        g.set_voting("sort")


@pytest.mark.parametrize("metric,storage", [("euclidean", "f32"), ("cosine", "f16")])
def test_associate_wasted_equals_the_host_composition(eng, metric, storage):
    import test_gpu_wasted_store as tws

    dim, hist = 64, 10
    ta = tws._tracker(eng, 3, hist, dim)
    sa, sb = (tws._store(eng, dim, metric, storage, 3, voting="best_fit") for _ in range(2))
    tws._prefill([sa, sb], dim, 50, 3)
    d = tws.Driver(3, 40, dim, 0x5EEDBE57, "f32")
    merged = 0
    for fr in range(24):
        d.frame([ta])
        if fr % 4 == 3:
            a = tws._collect(eng, ta, None, sa, sb, tws.HIST[hist])
            _distinct_merges(a)
            merged += int(a["merged"].sum())
    assert merged > 0
