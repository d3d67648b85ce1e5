"""GPU checks of the feature store's storage type (sb200_fstore_set_storage_type, FeatureStore(storage=...)).  Every
comparison is for equality, weights as f64 bits:
- fed a column of its own type, an f16 / bf16 store returns what an f32 store fed the same column returns, through every
  call (add, search, associate, search_owned, merge_owned, fetch, fetch(remove)), host and device columns alike;
- fed any other column, it holds the rows rounded once (fstore_oracle.round_rows), searches like an f32 store that holds
  the rounded rows and is queried with the unrounded ones, and associates like that search followed by add(round(rows));
- its blob carries storage_type and a feat section of half the size, and continues exactly after a load."""
import numpy as np
import pytest

import fstore_oracle as fo
from fstore_checks import METRICS, bits, gpu_store, refused_blob, same_results, store_options

pytestmark = pytest.mark.gpu

CODES = {"f32": 0, "f16": 1, "bf16": 2}


def _store(metric, dim, K, column="f32", storage="f32", **kw):
    """A store of the storage type whose host calls send columns of type `column`."""
    s = gpu_store(metric, storage, max_observations=K, feature_dim=dim, **kw)
    s.set_feature_type(column)
    assert s.storage_type() == storage
    return s


def _pool(n, dim, t, seed, edges=True):
    """(rows as sent under column type `t`, their exact f32 widening).  With `edges` some rows carry +-0, subnormals of
    the column's type, the largest finite value and, for f32, values that round to the binary16 edges."""
    rng = np.random.default_rng(seed)
    f = rng.standard_normal((n, dim)).astype(np.float32)
    if t == "f32":
        if edges:
            vals = np.float32([0.0, -0.0, 65504.0, 65519.99, 65520.0, -65520.0, 2.0 ** -24, 2.0 ** -25, 3 * 2.0 ** -25,
                               2.0 ** -26, np.finfo(np.float32).max, np.finfo(np.float32).smallest_subnormal,
                               1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -11, 1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8])
            for i in range(min(n, 8)):
                f[i, ::3] = np.resize(np.roll(vals, i), f[i, ::3].shape)
        return f, f.copy()
    if t == "f16":
        h = f.astype(np.float16)
        if edges:
            u = h.view(np.uint16)
            for i, v in enumerate([0x0000, 0x8000, 0x0001, 0x83FF, 0x7BFF, 0xFBFF, 0x0400]):
                u[i, ::2] = v
        return h, h.astype(np.float32)
    bits = (f.view(np.uint32) >> 16).astype(np.uint16)
    if edges:
        for i, v in enumerate([0x0000, 0x8000, 0x0001, 0x807F, 0x7F7F, 0x3380, 0x477F, 0x4780]):
            bits[i, ::2] = v
    return bits, (bits.astype(np.uint32) << 16).view(np.float32)


def _flat(out):
    if isinstance(out, dict):
        return [out[k] for k in sorted(out)]
    return list(out)


def _state(s):
    return [s.ids()] + _flat(s.fetch(s.ids()))


# ------------------------------------------------------------------------------------------------ own-type feed
def _script(K, n_pool):
    """A fixed call sequence: (op, ids, offsets, pool rows) or (op, args).  Rings wrap, the capacity grows several
    times, owned merges run as chains and stars, with and without removal."""
    nxt = [0]

    def take(n):
        idx = (np.arange(n) + nxt[0]) % n_pool
        nxt[0] += n
        return idx

    def queries(first_id, n):
        lens = [1 + (i * 2) % (K + 2) for i in range(n)]   # fewer than, exactly and more than K rows
        return np.arange(first_id, first_id + n, dtype=np.uint64), np.cumsum([0] + lens).astype(np.int32), take(sum(lens))

    rng = np.random.default_rng(K)
    u64 = lambda *v: np.array(v, np.uint64)  # noqa: E731
    ids = lambda n, rnd: np.concatenate([np.arange(1, n + 1), rng.integers(1, n + 1, rnd)]).astype(np.uint64)  # noqa
    steps = [("add", ids(4, 5), None, take(9)),                                   # small first capacity
             ("add", ids(12, 18), None, take(30)),                                # grow, wrap
             ("search",) + queries(100, 6),
             ("associate",) + queries(200, 7),
             ("owned", 0, u64(1, 2, 3, 777)),
             ("owned", 1, None),                                                  # every stored track
             ("merge", u64(1, 3, 2), u64(2, 1, 3), False),                        # chain 1 <- 2, 3 <- 1, 2 <- 3
             ("merge", u64(4, 4, 4), u64(5, 6, 7), True),                         # star with removal
             ("fetch",),
             ("remove", u64(3, 999, 7, 202)),
             ("add", ids(40, 20), None, take(60)),                                # new tracks: grows again
             ("associate",) + queries(300, 9),
             ("owned", 1, None),
             ("owned", 0, u64(300, 301, 8, 9)),
             ("merge", u64(10, 12, 12, 20), u64(11, 10, 13, 14), True),           # chain with removal
             ("search",) + queries(400, 4),
             ("fetch",)]
    return steps


def _run(store, steps, rows, device=None):
    """Runs the script; with `device` the add / search / associate columns are torch CUDA tensors of the same bits."""
    outs = []
    for st in steps:
        op = st[0]
        if op == "fetch":
            outs += _state(store)
        elif op == "remove":
            outs += _flat(store.fetch(st[1], remove=True)) + [store.ids()]
        elif op == "owned":
            ids = store.ids() if st[2] is None else st[2]
            outs += _flat(store.search_owned(ids, each=bool(st[1])))
        elif op == "merge":
            store.merge_owned(st[1], st[2], remove=st[3])
            outs += [store.ids()]
        else:
            _, ids, offs, idx = st
            col = rows[idx]
            if device is None:
                if op == "add":
                    store.add(ids, col)
                else:
                    outs += _flat(getattr(store, op)(ids, offs, col))
            else:
                import torch

                t = torch.from_numpy(np.ascontiguousarray(col).view(np.int16) if col.dtype == np.uint16 else
                                     np.ascontiguousarray(col)).cuda()
                if col.dtype == np.uint16:
                    t = t.view(torch.bfloat16)
                torch.cuda.synchronize()
                if op == "add":
                    store.add_device(ids, t.data_ptr())
                else:
                    outs += _flat(getattr(store, op + "_device")(ids, offs, t.data_ptr()))
    outs.append(np.array([store.size()]))
    return outs


@pytest.mark.parametrize("storage", ["f16", "bf16"])
@pytest.mark.parametrize("metric", ["euclidean", "cosine"])
@pytest.mark.parametrize("K", [1, 3, 8])
@pytest.mark.parametrize("dim", [8, 100, 512])
def test_own_type_feed_equals_an_f32_store(storage, metric, K, dim):
    steps = _script(K, 96)
    raw, wide = _pool(96, dim, storage, seed=dim * 10 + K)
    want = _run(_store(metric, dim, K, storage, "f32"), steps, raw)
    same_results(_run(_store(metric, dim, K, storage, storage), steps, raw), want)
    same_results(_run(_store(metric, dim, K, storage, storage), steps, raw, device=True), want)
    if K == 3 and dim != 512:   # the f32 store itself against the oracle, on the widened rows
        oracle = fo.FeatureStore(metric=METRICS[metric], **store_options(max_observations=K, feature_dim=dim))
        same_results(_run(oracle, steps, wide), want)


# ------------------------------------------------------------------------------------------------ rounding feed
def _fetched_equal_model(store, ids, want):
    counts, feats = store.fetch(ids)
    for i, c in enumerate(counts):
        got, exp = feats[i, :c], want[i][:c]
        nan = np.isnan(exp)
        assert np.array_equal(np.isnan(got), nan)
        assert np.array_equal(bits(got[~nan]), bits(exp[~nan]))


@pytest.mark.parametrize("storage,column", [("f16", "f32"), ("f16", "bf16"), ("bf16", "f32"), ("bf16", "f16")])
@pytest.mark.parametrize("metric", ["euclidean", "cosine"])
def test_rounding_feed(storage, column, metric):
    dim, K, n = 40, 3, 72
    raw, wide = _pool(n, dim, column, seed=CODES[storage] * 7 + CODES[column])
    if column == "f32":   # NaN and +-inf inside ordinary rows as well
        raw[9, 5], raw[10, 0], raw[11, dim - 1] = np.nan, np.inf, -np.inf
        wide = raw.copy()
    rounded = fo.round_rows(wide, storage)
    ids = np.repeat(np.arange(1, 13, dtype=np.uint64), 4)   # 12 tracks, rings wrap
    half = _store(metric, dim, K, column, storage)
    ref = _store(metric, dim, K, "f32", "f32")   # an f32 store holding the rounded rows
    half.add(ids, raw[:48])
    ref.add(ids, rounded[:48])
    per_track = [rounded[:48][ids == t][-K:] for t in range(1, 13)]
    _fetched_equal_model(half, np.arange(1, 13, dtype=np.uint64), per_track)
    # search: queries are never rounded
    qids = np.arange(100, 106, dtype=np.uint64)
    offs = np.array([0, 1, 3, 6, 10, 14, 16], np.int32)
    same_results(_flat(half.search(qids, offs, raw[48:64])), _flat(ref.search(qids, offs, wide[48:64])))
    # associate = search with the unrounded rows, then add(dest, round(rows)) query by query (the newest K rows)
    aids = np.arange(200, 206, dtype=np.uint64)
    aoffs = np.array([0, 2, 3, 7, 9, 12, 16], np.int32)
    a_raw, a_wide = raw[56:72], wide[56:72]
    got = half.associate(aids, aoffs, a_raw)
    s = ref.search(aids, aoffs, a_wide)
    for q in range(len(aids)):
        dest = s["winners"][q, 0] if s["counts"][q] > 0 else aids[q]
        lo = max(aoffs[q], aoffs[q + 1] - K)
        ref.add(np.full(aoffs[q + 1] - lo, dest, np.uint64), fo.round_rows(a_wide[lo:aoffs[q + 1]], storage))
    want = dict(s, merged=(s["counts"] > 0).astype(np.uint8),
                track_ids=np.where(s["counts"] > 0, s["winners"][:, 0], aids).astype(np.uint64))
    same_results(_flat(got), _flat(want))
    assert np.array_equal(half.ids(), ref.ids())
    rc, rf = ref.fetch(ref.ids())
    _fetched_equal_model(half, ref.ids(), [rf[i] for i in range(len(rc))])
    # owned calls compare widened stored rows
    same_results(_flat(half.search_owned(half.ids(), each=True)), _flat(ref.search_owned(ref.ids(), each=True)))


# ------------------------------------------------------------------------------------------------ blob
def _header(blob):
    from similari_b200 import _lib

    return _lib.FstoreBlobHeader.from_buffer_copy(blob[:128].tobytes())


def _worn(storage, column, metric="euclidean", dim=40, K=3):
    raw, _ = _pool(96, dim, column, seed=5)
    s = _store(metric, dim, K, column, storage)
    steps = [st for st in _script(K, 96) if st[0] not in ("search", "fetch")]
    _run(s, steps, raw)
    s.add(np.array([7777], np.uint64), raw[[40]])   # one track that has not filled its ring
    counts, _ = s.fetch(s.ids())
    assert counts.min() < K == counts.max() and s.size() > 4
    return s, raw


@pytest.mark.parametrize("storage", ["f16", "bf16"])
@pytest.mark.parametrize("metric", ["euclidean", "cosine"])
def test_blob_of_a_half_store(storage, metric):
    import torch

    import similari_b200.engine as eng

    dim, K = 40, 3
    s, raw = _worn(storage, storage, metric, dim, K)
    f, _ = _worn("f32", storage, metric, dim, K)   # the same calls on an f32 store
    blob, fblob = s.save(), f.save()
    h, fh = _header(blob), _header(fblob)
    assert (h.storage_type, fh.storage_type, h.live) == (CODES[storage], 0, fh.live)
    assert h.sec_bytes[3] * 2 == fh.sec_bytes[3] == h.live * K * h.d8 * 4
    feat = blob[h.sec_off[3]: h.sec_off[3] + h.sec_bytes[3]].view(np.uint16)
    if storage == "f16":
        wide = feat.view(np.float16).astype(np.float32)
    else:
        wide = (feat.astype(np.uint32) << 16).view(np.float32)
    assert np.array_equal(wide.view(np.uint32), fblob[fh.sec_off[3]: fh.sec_off[3] + fh.sec_bytes[3]].view(np.uint32))
    n = s.save_device(0, 0)
    assert n == len(blob) < len(fblob)
    dblob = torch.zeros(n, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    assert s.save_device(dblob.data_ptr(), n) == n
    assert np.array_equal(dblob.cpu().numpy(), blob)
    copies = [eng.FeatureStore.load(blob), eng.FeatureStore.load(dblob.data_ptr(), n)]
    for c in copies:
        assert c.storage_type() == storage and c.feature_type() == storage
        same_results(_state(c), _state(s))
        assert np.array_equal(c.save(), blob)
    steps = _script(K, 96)
    for st in steps:   # fresh ids: the script's query ids must not be stored yet
        if st[0] in ("search", "associate"):
            st[1][:] += 5000
    want = _run(s, steps, raw)
    for c in copies:
        same_results(_run(c, steps, raw), want)


def test_blob_storage_type_is_checked():
    from similari_b200 import _lib

    s, _ = _worn("f16", "f16")
    f, _ = _worn("f32", "f16")
    for blob in (s.save(), f.save()):
        b = blob.copy()
        _lib.FstoreBlobHeader.from_buffer(b).storage_type = 7
        refused_blob(b, "storage_type")
        b = blob.copy()
        _lib.FstoreBlobHeader.from_buffer(b).storage_type = -1
        refused_blob(b, "storage_type")
    b = f.save().copy()
    _lib.FstoreBlobHeader.from_buffer(b).storage_type = 1   # an f32 blob relabelled: its feat section is twice too big
    refused_blob(b, "feat holds")
    b = s.save().copy()
    _lib.FstoreBlobHeader.from_buffer(b).storage_type = 0
    refused_blob(b, "feat holds")


def test_empty_half_store_blob():
    import similari_b200.engine as eng

    s = _store("cosine", 100, 5, "f32", "bf16", topn=7)
    blob = s.save()
    h = _header(blob)
    assert (len(blob), h.storage_type, h.sec_bytes[3]) == (256, 2, 0)
    c = eng.FeatureStore.load(blob)
    assert (c.size(), c.storage_type(), c.feature_type()) == (0, "bf16", "f32")


# ------------------------------------------------------------------------------------------------ setter
def test_setter_refusals_and_reuse_after_removal():
    from similari_b200 import _lib

    dim, K = 24, 3
    raw, wide = _pool(400, dim, "f16", seed=9, edges=False)
    L = _lib.lib()
    s = _store("euclidean", dim, K, "f16", "f16")
    assert L.sb200_fstore_set_storage_type(s._h, 3) == -1 and "storage type" in L.sb200_last_error().decode()
    assert L.sb200_fstore_set_storage_type(s._h, -1) == -1
    assert s.storage_type() == "f16"
    ids = np.repeat(np.arange(1, 51, dtype=np.uint64), 2)
    s.add(ids, raw[:100])
    before, blob = _state(s), s.save()
    for t in (0, 1, 2, 7):
        assert L.sb200_fstore_set_storage_type(s._h, t) == -1
        assert ("holds tracks" if t != 7 else "unknown") in L.sb200_last_error().decode()
    assert s.storage_type() == "f16"
    same_results(_state(s), before)
    assert np.array_equal(s.save(), blob)
    # emptied by fetch(remove): allowed again, also to a wider type than the columns were allocated for
    s.fetch(s.ids(), remove=True)
    assert s.size() == 0
    for t in ("f32", "bf16", "f32"):
        assert L.sb200_fstore_set_storage_type(s._h, CODES[t]) == 0 and s.storage_type() == t
    fresh = _store("euclidean", dim, K, "f16", "f32")
    ids = np.repeat(np.arange(1, 151, dtype=np.uint64), 2)
    for x in (s, fresh):
        x.add(ids[:100], raw[100:200])
        x.add(ids[100:], raw[200:400])   # grows past the old columns
    same_results(_state(s), _state(fresh))
    assert np.array_equal(s.save(), fresh.save())


# ------------------------------------------------------------------------------------------------ gallery size
def test_gallery_search_is_identical_at_100k_tracks():
    import similari_b200.engine as eng

    tracks, K, dim, Q = 100_000, 3, 512, 256
    rng = np.random.default_rng(12)
    stores = {t: eng.FeatureStore(metric="euclidean", distance_filter=1e30, max_observations=K, feature_dim=dim, topn=5,
                                  max_distance=1e30, min_votes=1, storage=t) for t in ("f32", "f16")}
    chunk = 20_000
    for b in range(0, tracks, chunk):
        ids = np.repeat(np.arange(b + 1, b + 1 + chunk, dtype=np.uint64), K)
        rows = rng.standard_normal((chunk * K, dim)).astype(np.float16)
        for s in stores.values():
            s.add(ids, rows)
    q = rng.standard_normal((Q, dim)).astype(np.float16)
    qid = np.arange(10**9, 10**9 + Q, dtype=np.uint64)
    offs = np.arange(Q + 1, dtype=np.int32)
    a, b = (_flat(s.search(qid, offs, q)) for s in stores.values())
    same_results(a, b)
    assert a[0].min() == 5
