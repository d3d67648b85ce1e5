"""GPU checks of the feature store's I/O surface: FP16 / BF16 feature columns, device-resident columns ordered against the
caller's stream, and the store blob (sb200_fstore_set_feature_type, _add_device / _search_device / _associate_device,
_save / _load).  Widening a 2-byte element is exact, so every comparison is for equality: a typed or device-fed store
against an f32 store fed the widened rows, a loaded store against the one that was saved."""
import ctypes as C

import numpy as np
import pytest

import fstore_oracle as fo
from fstore_checks import METRICS, gpu_store, refused_blob, same_results, store_options

pytestmark = pytest.mark.gpu

TORCH_TYPES = {"f32": "float32", "f16": "float16", "bf16": "bfloat16"}


def _store(metric, dim, K, t="f32", **kw):
    """A store whose host calls send columns of type t."""
    s = gpu_store(metric, max_observations=K, feature_dim=dim, **kw)
    s.set_feature_type(t)
    return s


def _pool(n, dim, t, seed):
    """(rows as sent under type `t`, their exact f32 widening); the first rows hold +-0, subnormals, +-Inf, NaN with
    payloads and the largest finite value in every lane, the rest are random."""
    rng = np.random.default_rng(seed)
    f = rng.standard_normal((n, dim)).astype(np.float32)
    if t == "f32":
        u = f.view(np.uint32)
        for i, v in enumerate([0x00000000, 0x80000000, 0x00000001, 0x807FFFFF, 0x7F800000, 0xFF800000, 0x7FC00001]):
            u[i] = v
        return f, f.copy()
    if t == "f16":
        h = f.astype(np.float16)
        u = h.view(np.uint16)
        for i, v in enumerate([0x0000, 0x8000, 0x0001, 0x83FF, 0x7C00, 0xFC00, 0x7E01, 0xFE55, 0x7BFF]):
            u[i] = v
        u[9][::2] = 0x0001   # subnormals mixed into an ordinary row
        return h, h.astype(np.float32)
    bits = (f.view(np.uint32) >> 16).astype(np.uint16)
    for i, v in enumerate([0x0000, 0x8000, 0x0001, 0x807F, 0x7F80, 0xFF80, 0x7FC1, 0xFFE5, 0x7F7F]):
        bits[i] = v
    bits[9][::2] = 0x0001
    return bits, (bits.astype(np.uint32) << 16).view(np.float32)


def _script(dim, K, n_pool, seed):
    """One fixed sequence of calls as (op, ids, offsets or None, row indices into the pool)."""
    rng = np.random.default_rng(seed)
    nxt = [0]

    def take(n):
        idx = (np.arange(n) + nxt[0]) % n_pool
        nxt[0] += n
        return idx

    def queries(first_id, n):
        lens = [1 + (i * 2) % (K + 2) for i in range(n)]   # fewer than, exactly and more than K rows
        return np.arange(first_id, first_id + n, dtype=np.uint64), np.cumsum([0] + lens).astype(np.int32), take(sum(lens))

    steps = [("add", rng.integers(1, 13, 30).astype(np.uint64), None, take(30))]
    steps.append(("search",) + queries(100, 6))
    steps.append(("associate",) + queries(200, 7))
    steps.append(("fetch", None, None, None))
    steps.append(("remove", np.array([3, 999, 5, 201], np.uint64), None, None))
    steps.append(("add", rng.integers(1, 16, 11).astype(np.uint64), None, take(11)))
    steps.append(("associate",) + queries(300, 5))
    steps.append(("search",) + queries(400, 3))
    steps.append(("fetch", None, None, None))
    return steps


def _flat(out):
    if isinstance(out, dict):
        return [out[k] for k in sorted(out)]
    return list(out)


def _run(store, steps, rows, feed=None):
    """Runs the script; `feed(op, ids, offs, rows)` replaces the host-pointer call when given.  Returns every output."""
    outs = []
    for op, ids, offs, idx in steps:
        if op == "fetch":
            outs += [store.ids()] + _flat(store.fetch(store.ids()))
        elif op == "remove":
            outs += _flat(store.fetch(ids, remove=True)) + [store.ids()]
        elif feed is not None:
            outs += _flat(feed(op, ids, offs, rows[idx]) or {})
        elif op == "add":
            store.add(ids, rows[idx])
        else:
            outs += _flat(getattr(store, op)(ids, offs, rows[idx]))
    outs.append(np.array([store.size()]))
    return outs


# ------------------------------------------------------------------------------------------------ element types
@pytest.mark.parametrize("metric", ["euclidean", "cosine"])
@pytest.mark.parametrize("dim", [8, 100, 256, 513])
@pytest.mark.parametrize("K", [1, 3])
def test_typed_columns_equal_the_widened_request(metric, dim, K):
    steps = _script(dim, K, 64, seed=dim + K)
    for t in ("f16", "bf16"):
        raw, wide = _pool(64, dim, t, seed=7 * dim + K)
        typed, plain = _store(metric, dim, K, t), _store(metric, dim, K)
        oracle = fo.FeatureStore(metric=METRICS[metric], **store_options(max_observations=K, feature_dim=dim))
        want = _run(plain, steps, wide)
        same_results(_run(typed, steps, raw), want)
        same_results(_run(oracle, steps, wide), want)
        assert typed.feature_type() == t and plain.feature_type() == "f32"


def test_float16_arrays_are_sent_as_they_are():
    """Without a declared type a float16 array goes up as 2-byte rows; a later float32 array switches back."""
    raw, wide = _pool(40, 24, "f16", seed=1)
    a, b = _store("euclidean", 24, 3), _store("euclidean", 24, 3)
    ids = np.arange(1, 21, dtype=np.uint64)
    a.add(ids, raw[:20])
    assert a.feature_type() == "f16"
    a.add(ids, wide[20:])
    assert a.feature_type() == "f32"
    b.add(ids, wide[:20])
    b.add(ids, wide[20:])
    same_results(_flat(a.fetch(ids)), _flat(b.fetch(ids)))
    with pytest.raises(ValueError):
        _store("euclidean", 24, 3, "bf16").add(ids, wide[:20])   # a declared 2-byte type takes 2-byte elements only


# ------------------------------------------------------------------------------------------------ device columns
def _device_feed(store, t, dim, shift):
    """Feeds each call from a torch CUDA tensor that a side stream is still writing when the call is made.  The column
    starts `shift` elements into its allocation."""
    import torch

    side = torch.cuda.Stream()
    dt = getattr(torch, TORCH_TYPES[t])
    ballast = torch.ones((4096, 4096), device="cuda")
    keep = []

    def feed(op, ids, offs, rows):
        n = rows.shape[0]
        host = torch.from_numpy(rows.view(np.int16) if t == "bf16" else rows).contiguous().pin_memory()
        if t == "bf16":
            host = host.view(torch.bfloat16)
        buf = torch.zeros(shift + n * dim, dtype=dt, device="cuda")
        col = buf[shift:].view(n, dim)
        torch.cuda.current_stream().synchronize()   # the zeros are in place; only the side stream writes from here
        with torch.cuda.stream(side):
            for _ in range(2):   # work in front of the copy, so the call is made while the column is still unwritten
                ballast @ ballast
            col.copy_(host, non_blocking=True)
        keep.append((host, buf))
        assert col.data_ptr() == buf.data_ptr() + shift * buf.element_size()
        if op == "add":
            return store.add_device(ids, col.data_ptr(), side.cuda_stream)
        return getattr(store, op + "_device")(ids, offs, col.data_ptr(), side.cuda_stream)

    return feed


@pytest.mark.parametrize("metric", ["euclidean", "cosine"])
@pytest.mark.parametrize("t", ["f32", "f16", "bf16"])
@pytest.mark.parametrize("dim,shift", [(256, 0), (256, 3), (513, 513), (100, 0)])
def test_device_columns_equal_the_host_request(metric, t, dim, shift):
    """(256, 3) and (513, one row) put the column's base off 16 bytes: the scalar loads of fs_stage_kernel."""
    K = 3
    steps = _script(dim, K, 64, seed=dim)
    raw, wide = _pool(64, dim, t, seed=dim + shift)
    dev, host, plain = _store(metric, dim, K, t), _store(metric, dim, K, t), _store(metric, dim, K)
    want = _run(plain, steps, wide)
    same_results(_run(host, steps, raw), want)
    same_results(_run(dev, steps, raw, feed=_device_feed(dev, t, dim, shift)), want)


def test_device_calls_on_the_default_stream_and_empty_store():
    import torch

    dim, K = 64, 2
    raw, wide = _pool(32, dim, "f16", seed=5)
    dev, plain = _store("euclidean", dim, K, "f16"), _store("euclidean", dim, K)
    col = torch.from_numpy(raw).cuda()   # written on the legacy default stream, which stream == 0 names
    ids = np.arange(50, 58, dtype=np.uint64)
    offs = np.arange(0, 9, dtype=np.int32) * 4
    same_results(_flat(dev.associate_device(ids, offs, col.data_ptr())), _flat(plain.associate(ids, offs, wide)))
    same_results(_flat(dev.search_device(ids + 100, offs, col.data_ptr())), _flat(plain.search(ids + 100, offs, wide)))
    same_results([dev.ids()] + _flat(dev.fetch(dev.ids())), [plain.ids()] + _flat(plain.fetch(plain.ids())))


def test_a_host_pointer_is_not_a_device_column():
    from similari_b200._lib import Sb200Error, pinned_empty

    dim = 16
    raw, _ = _pool(24, dim, "f32", seed=2)
    s = _store("euclidean", dim, 3)
    s.add(np.arange(1, 13, dtype=np.uint64), raw[:12])
    before = [s.ids()] + _flat(s.fetch(s.ids()))
    pinned = pinned_empty((12, dim), np.float32)
    pinned[:] = raw[12:]
    ids = np.arange(100, 104, dtype=np.uint64)
    offs = np.arange(0, 5, dtype=np.int32) * 3
    for host in (np.ascontiguousarray(raw[12:]), pinned):
        for call in (lambda p: s.add_device(ids, p), lambda p: s.search_device(ids, offs, p),
                     lambda p: s.associate_device(ids, offs, p)):
            with pytest.raises(Sb200Error, match="-1.*d_features"):
                call(host.ctypes.data)
            same_results([s.ids()] + _flat(s.fetch(s.ids())), before)


# ------------------------------------------------------------------------------------------------ the store blob
def _worn_store(metric="euclidean", dim=40, K=3, t="f32"):
    """A store after adds, merges that wrapped the rings, and removals."""
    raw, _ = _pool(64, dim, t, seed=3)
    s = _store(metric, dim, K, t)
    for op, ids, offs, idx in _script(dim, K, 64, seed=11):
        if op == "add":
            s.add(ids, raw[idx])
        elif op == "associate":
            s.associate(ids, offs, raw[idx])
        elif op == "remove":
            s.fetch(ids, remove=True)
    s.add(np.array([7777], np.uint64), raw[[40]])   # one track that has not filled its ring
    counts, _ = s.fetch(s.ids())
    assert counts.min() < K == counts.max() and s.size() > 4
    return s, raw


@pytest.mark.parametrize("metric", ["euclidean", "cosine"])
@pytest.mark.parametrize("t", ["f32", "bf16"])
def test_save_load_continues_exactly(metric, t):
    import torch

    import similari_b200.engine as eng

    dim, K = 40, 3
    s, raw = _worn_store(metric, dim, K, t)
    blob = s.save()
    assert np.array_equal(blob, s.save())
    n = s.save_device(0, 0)
    assert n == len(blob)
    dblob = torch.full((n + 32,), 0xAB, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    assert s.save_device(dblob.data_ptr() + 16, n) == n   # 16-byte aligned: written in place
    assert np.array_equal(dblob[16:16 + n].cpu().numpy(), blob)
    assert bool((dblob[:16] == 0xAB).all()) and bool((dblob[16 + n:] == 0xAB).all())
    copies = [eng.FeatureStore.load(blob), eng.FeatureStore.load(dblob.data_ptr() + 16, n),
              eng.FeatureStore.load(blob.tobytes())]
    state = [s.ids()] + _flat(s.fetch(s.ids()))
    for c in copies:
        assert (c.K, c.D, c.topn, c.feature_type()) == (K, dim, 4, t)
        same_results([c.ids()] + _flat(c.fetch(c.ids())), state)
        assert np.array_equal(c.save(), blob)
    steps = _script(dim, K, 64, seed=23)
    for st in steps:   # fresh ids: the script's query ids must not be stored yet
        if st[0] in ("search", "associate"):
            st[1][:] += 5000
    want = _run(s, steps, raw)
    for c in copies:
        same_results(_run(c, steps, raw), want)


def test_equal_states_give_equal_blobs():
    """Two call histories that end in the same tracks, order and ring state, with different leftovers in the ring slots
    that hold no observation."""
    dim, K = 24, 3
    raw, _ = _pool(32, dim, "f32", seed=4)
    one = np.array([1], np.uint64)
    a = _store("euclidean", dim, K)
    a.add(np.array([1, 1, 1, 1, 2], np.uint64), raw[[20, 21, 22, 23, 24]])   # track 1 wraps: holds 21, 22, 23
    b = _store("euclidean", dim, K)
    b.associate(one, np.array([0, 1], np.int32), raw[[30]])                   # a new track through associate
    b.add(np.array([1, 1, 7, 7, 7, 1], np.uint64), raw[[21, 22, 25, 26, 27, 23]])
    b.fetch(np.array([7], np.uint64), remove=True)                            # compaction into fresh columns
    b.add(np.array([2], np.uint64), raw[[24]])
    same_results([a.ids()] + _flat(a.fetch(a.ids())), [b.ids()] + _flat(b.fetch(b.ids())))
    blob = a.save()
    assert np.array_equal(blob, b.save())
    # the unfilled slots of track 2 are zeros in the blob
    from similari_b200 import _lib

    h = _lib.FstoreBlobHeader.from_buffer_copy(blob[:128].tobytes())
    d8 = h.d8
    feat = blob[h.sec_off[3]: h.sec_off[3] + h.sec_bytes[3]].view(np.float32).reshape(2, K, d8)
    assert not feat[1, 1:].any() and feat[1, 0].any()


def test_empty_store_round_trips():
    import similari_b200.engine as eng

    s = _store("cosine", 100, 5, "f16", topn=7)
    blob = s.save()
    assert len(blob) == 256
    c = eng.FeatureStore.load(blob)
    assert (c.size(), len(c.ids()), c.K, c.D, c.topn, c.feature_type()) == (0, 0, 5, 100, 7, "f16")
    assert np.array_equal(c.save(), blob)
    raw, _ = _pool(16, 100, "f16", seed=6)
    ids = np.arange(1, 9, dtype=np.uint64)
    for x in (s, c):
        x.add(ids, raw[:8])
    same_results(_flat(c.fetch(ids)), _flat(s.fetch(ids)))


def test_damaged_blobs_are_refused():
    import similari_b200.engine as eng
    from similari_b200 import _lib

    K = 3
    s, _ = _worn_store(K=K)
    blob = s.save()
    hdr = _lib.FstoreBlobHeader.from_buffer_copy(blob[:128].tobytes())
    live = hdr.live

    def damaged(edit):
        b = blob.copy()
        edit(b, _lib.FstoreBlobHeader.from_buffer(b))   # the header aliases the copy
        return b

    def column(b, sec, dtype):
        return b[hdr.sec_off[sec]: hdr.sec_off[sec] + hdr.sec_bytes[sec]].view(dtype)

    refused_blob(blob[:-1], "truncated")
    refused_blob(blob[:100], "truncated")
    refused_blob(damaged(lambda b, h: setattr(h, "version", 2)), "version")
    refused_blob(damaged(lambda b, h: setattr(h, "magic", 0x42534253)), "magic")
    refused_blob(damaged(lambda b, h: column(b, 1, np.int32).__setitem__(live // 2, 0)), "cnt")
    refused_blob(damaged(lambda b, h: column(b, 1, np.int32).__setitem__(0, K + 1)), "cnt")
    refused_blob(damaged(lambda b, h: column(b, 2, np.int32).__setitem__(live - 1, K)), "start")
    refused_blob(damaged(lambda b, h: column(b, 2, np.int32).__setitem__(0, -1)), "start")
    refused_blob(damaged(lambda b, h: column(b, 0, np.uint64).__setitem__(1, column(b, 0, np.uint64)[0])), "twice")
    refused_blob(damaged(lambda b, h: h.sec_off.__setitem__(1, h.sec_off[1] + 8)), "cnt is not 256-byte aligned")
    refused_blob(damaged(lambda b, h: h.sec_off.__setitem__(2, h.sec_off[1])), "start lies outside")
    refused_blob(damaged(lambda b, h: h.sec_bytes.__setitem__(3, h.sec_bytes[3] - 4)), "feat holds")
    refused_blob(damaged(lambda b, h: setattr(h, "max_observations", 65)), "max_observations")
    refused_blob(damaged(lambda b, h: setattr(h, "topn", 0)), "topn")
    refused_blob(damaged(lambda b, h: setattr(h, "feature_dim", 8193)), "feature_dim")
    refused_blob(damaged(lambda b, h: setattr(h, "metric", 2)), "metric")
    refused_blob(damaged(lambda b, h: setattr(h, "d8", h.d8 + 8)), "d8")
    refused_blob(damaged(lambda b, h: setattr(h, "feature_type", 3)), "feature_type")
    # a tracker blob is not a store blob, and the other way round
    tracker = eng.Tracker(_lib.default_options())
    refused_blob(tracker.save(), "magic")
    with pytest.raises(_lib.Sb200Error, match="-1"):
        eng.Tracker.load(blob)
    # the undamaged blob still loads, and the store that wrote it is as it was
    assert np.array_equal(eng.FeatureStore.load(blob).save(), blob)
    assert np.array_equal(s.save(), blob)


def test_save_into_a_short_buffer_writes_nothing():
    from similari_b200 import _lib

    s, _ = _worn_store()
    L = _lib.lib()
    n = C.c_uint64(0)
    assert L.sb200_fstore_save(s._h, None, 0, C.byref(n)) == 0
    total = n.value
    buf = np.full(total, 0xAB, np.uint8)
    n = C.c_uint64(0)
    assert L.sb200_fstore_save(s._h, _lib.ptr(buf), total - 1, C.byref(n)) == -3
    assert n.value == total and (buf == 0xAB).all()
    assert str(total) in L.sb200_last_error().decode()
    assert L.sb200_fstore_save(s._h, _lib.ptr(buf), total, C.byref(n)) == 0 and n.value == total
    assert np.array_equal(buf, s.save())
