"""GPU checks of the feature store's gate (track attributes): search / associate through host and device columns, the
owned calls and the attribute columns bit for bit against the CPU oracle, every refusal leaving the store's blob as it
was, and the version-2 blob: round trip, byte-equal twins, load refusals; an ungated store's blob stays version 1."""
import ctypes as C
import zlib

import numpy as np
import pytest

import fstore_oracle as fo
from fstore_checks import gpu_store, refused_blob, same_results, same_store, store_pair

pytestmark = pytest.mark.gpu


def _windows(rng, n, span=400, length=40, sources=2):
    t0 = rng.integers(0, span, n).astype(np.int64)
    return dict(sources=rng.integers(1, sources + 1, n).astype(np.uint64), t_start=t0,
                t_end=t0 + rng.integers(0, length, n).astype(np.int64))


def _feats(rng, n, dim, storage):
    """Rows the storage type holds exactly, so that a merged query row is stored unchanged by both stores."""
    return fo.round_rows(rng.standard_normal((n, dim)).astype(np.float32), storage)


def _fill(stores, rng, n_tracks, dim, storage, K):
    lens = 1 + (np.arange(n_tracks) * 7 + 3) % (2 * K + 1)
    ids = np.repeat(np.arange(1, n_tracks + 1, dtype=np.uint64), lens)
    rng.shuffle(ids)
    f = _feats(rng, len(ids), dim, storage)
    w = _windows(rng, n_tracks)
    at = {k: v[ids.astype(np.int64) - 1] for k, v in w.items()}   # one source per id; windows hull per track
    at["t_start"] = at["t_start"] - rng.integers(0, 5, len(ids))
    for part in np.array_split(np.arange(len(ids)), 3):
        for s in stores:
            s.add(ids[part], f[part], **{k: v[part] for k, v in at.items()})


def _queries(rng, Q, dim, storage, first_id):
    lens = 1 + rng.integers(0, 4, Q)
    offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    return np.arange(first_id, first_id + Q, dtype=np.uint64), offs, _feats(rng, int(offs[-1]), dim, storage)


def _device(x):
    import torch

    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


@pytest.mark.parametrize("storage", ["f32", "f16", "bf16"])
@pytest.mark.parametrize("metric", ["euclidean", "cosine"])
@pytest.mark.parametrize("gate", ["same_source", "any_source"])
def test_search_and_associate_match_the_oracle(storage, metric, gate):
    import torch

    rng = np.random.default_rng(zlib.crc32(f"{storage} {metric} {gate}".encode()))
    dim, K = 24, 3
    g, o = store_pair(metric, storage, gate, max_observations=K, feature_dim=dim, topn=4, min_votes=1)
    _fill((g, o), rng, 60, dim, storage, K)
    refused = 0   # queries whose first winner the gate refused in associate
    for it in range(4):
        ids, offs, f = _queries(rng, 40, dim, storage, 1000 + 100 * it)
        at = _windows(rng, len(ids))
        on_device = it % 2 == 1
        if on_device:
            d = _device(f)
            rg = g.search_device(ids, offs, d.data_ptr(), **at)
            torch.cuda.synchronize()
        else:
            rg = g.search(ids, offs, f, **at)
        same_results(rg, o.search(ids, offs, f, **at), "search")
        if on_device:
            rg = g.associate_device(ids, offs, d.data_ptr(), **at)
        else:
            rg = g.associate(ids, offs, f, **at)
        ro = o.associate(ids, offs, f, **at)
        same_results(rg, ro, "associate")
        refused += int(((ro["counts"] > 0) & (ro["merged"] == 0)).sum())
        same_store(g, o)
    assert refused > 0
    # the device column path of add
    ids = np.array([1, 2, 5000], np.uint64)
    src, t0, t1 = o.attributes(ids)
    at = dict(sources=np.where(src == 0, 9, src), t_start=np.minimum(t1, 10_000), t_end=np.minimum(t1, 10_000) + 3)
    f = _feats(rng, 3, dim, storage)
    g.add_device(ids, _device(f).data_ptr(), **at)
    torch.cuda.synchronize()
    o.add(ids, f, **at)
    same_store(g, o)


@pytest.mark.parametrize("metric", ["euclidean", "cosine"])
def test_gallery_scale(metric):
    """20,000 tracks x K = 3 x 512-d with random windows: a search and an associate of 64 queries."""
    rng = np.random.default_rng(11)
    dim, K, n = 512, 3, 20_000
    g, o = store_pair(metric, gate="same_source", max_observations=K, feature_dim=dim, topn=5, min_votes=1)
    ids = np.repeat(np.arange(1, n + 1, dtype=np.uint64), K)
    f = rng.standard_normal((len(ids), dim)).astype(np.float32)
    w = _windows(rng, n, span=100_000, length=2_000, sources=4)
    at = {k: np.repeat(v, K) for k, v in w.items()}
    for s in (g, o):
        s.add(ids, f, **at)
    q, offs, qf = _queries(rng, 64, dim, "f32", 10 ** 6)
    qa = _windows(rng, 64, span=100_000, length=2_000, sources=4)
    same_results(g.search(q, offs, qf, **qa), o.search(q, offs, qf, **qa), "search")
    same_results(g.associate(q, offs, qf, **qa), o.associate(q, offs, qf, **qa), "associate")
    sel = np.concatenate([o.ids()[:100], o.ids()[-64:]])
    same_results(g.attributes(sel), o.attributes(sel))


@pytest.mark.parametrize("metric", ["euclidean", "cosine"])
@pytest.mark.parametrize("gate", ["same_source", "any_source"])
def test_owned_calls_match_the_oracle(metric, gate):
    rng = np.random.default_rng(5)
    dim, K = 16, 3
    g, o = store_pair(metric, gate=gate, max_observations=K, feature_dim=dim, topn=5)
    _fill((g, o), rng, 50, dim, "f32", K)
    ids = o.ids()
    q = np.concatenate([ids[rng.permutation(len(ids))[:12]], [777777]]).astype(np.uint64)
    for each in (False, True):
        same_results(g.search_owned(q, each=each), o.search_owned(q, each=each), f"owned each={each}")
    same_results(g.search_owned(ids, each=True), o.search_owned(ids, each=True), "owned whole store")
    # merge_owned: random pairs, applied when the oracle accepts them, refused by both when it does not
    accepted = refused = 0
    for _ in range(30):
        d, s = (int(x) for x in rng.choice(o.ids(), 2, replace=False))
        remove = bool(rng.integers(0, 2))
        try:
            o.merge_owned([d], [s], remove=remove)
            ok = True
        except ValueError:
            ok = False
        if ok:
            g.merge_owned([d], [s], remove=remove)
            accepted += 1
        else:
            blob = g.save()
            with pytest.raises(Exception):
                g.merge_owned([d], [s], remove=remove)
            assert np.array_equal(g.save(), blob)
            refused += 1
        same_store(g, o)
    assert accepted and refused


def test_fetch_attr_after_merges_and_removals():
    g, o = store_pair(gate="same_source", max_observations=2, feature_dim=8, topn=5)
    rng = np.random.default_rng(2)
    f = rng.standard_normal((6, 8)).astype(np.float32)
    at = dict(sources=np.array([1, 1, 1, 2, 1, 1], np.uint64), t_start=np.array([0, 10, 20, 0, 40, 50], np.int64),
              t_end=np.array([5, 15, 25, 100, 45, 55], np.int64))
    ids = np.arange(1, 7, dtype=np.uint64)
    for s in (g, o):
        s.add(ids, f, **at)
        s.merge_owned([1, 1], [2, 3], remove=True)
        s.fetch([5], remove=True)
    same_store(g, o)
    src, t0, t1 = g.attributes([1, 2, 3, 4, 5, 6])
    assert src.tolist() == [1, 0, 0, 2, 0, 1]
    assert t0.tolist() == [0, 0, 0, 0, 0, 50] and t1.tolist() == [25, 0, 0, 100, 0, 55]
    assert g.ids().tolist() == [1, 4, 6]


def _rc(L, fn, *args):
    return fn(*args), L.sb200_last_error().decode()


def test_refusals_leave_the_store_unchanged():
    import similari_b200.engine as eng
    from similari_b200 import _lib

    L = _lib.lib()
    p = _lib.ptr
    g = gpu_store(gate="same_source", max_observations=2, feature_dim=8, topn=5)
    f = np.ones((3, 8), np.float32)
    g.add([1, 2, 3], f, sources=[1, 1, 2], t_start=[0, 10, 0], t_end=[5, 15, 5])
    blob = g.save()
    ids = np.array([9], np.uint64)
    offs = np.array([0, 1], np.int32)
    cnt, win, w = np.zeros(1, np.int32), np.zeros((1, 5), np.uint64), np.zeros((1, 5), np.float64)
    tid, mg = np.zeros(1, np.uint64), np.zeros(1, np.uint8)
    src, t0, t1 = np.array([1], np.uint64), np.array([3], np.int64), np.array([2], np.int64)
    bad = _lib.FstoreAttrs(src.ctypes.data, t0.ctypes.data, t1.ctypes.data)
    checks = [
        (L.sb200_fstore_add, (g._h, 1, p(ids), p(f)), "_attr"),
        (L.sb200_fstore_search, (g._h, 1, p(ids), p(offs), p(f), p(cnt), p(win), p(w)), "_attr"),
        (L.sb200_fstore_associate, (g._h, 1, p(ids), p(offs), p(f), p(cnt), p(win), p(w), p(tid), p(mg)), "_attr"),
        (L.sb200_fstore_add_attr, (g._h, 1, p(ids), C.byref(bad), p(f), None, None), "t_start"),
        (L.sb200_fstore_search_attr, (g._h, 1, p(ids), p(offs), C.byref(bad), p(f), None, p(cnt), p(win), p(w), None),
         "t_start"),
        (L.sb200_fstore_associate_attr, (g._h, 1, p(ids), p(offs), C.byref(bad), p(f), None, p(cnt), p(win), p(w),
                                         p(tid), p(mg), None), "t_start"),
        (L.sb200_fstore_set_gate, (g._h, 2), "holds tracks"),
        (L.sb200_fstore_set_gate, (g._h, 3), "unknown gate"),
    ]
    d = _device(f)
    checks += [
        (L.sb200_fstore_add_device, (g._h, 1, p(ids), C.c_void_p(d.data_ptr()), None), "_attr"),
        (L.sb200_fstore_search_device, (g._h, 1, p(ids), p(offs), C.c_void_p(d.data_ptr()), p(cnt), p(win), p(w), None),
         "_attr"),
        (L.sb200_fstore_associate_device, (g._h, 1, p(ids), p(offs), C.c_void_p(d.data_ptr()), p(cnt), p(win), p(w),
                                           p(tid), p(mg), None), "_attr"),
    ]
    for fn, args, word in checks:
        rc, msg = _rc(L, fn, *args)
        assert rc == -1 and word in msg, (fn.__name__, rc, msg)
        assert np.array_equal(g.save(), blob), fn.__name__
    good = dict(sources=[3], t_start=[0], t_end=[1])
    with pytest.raises(_lib.Sb200Error):
        g.add([1], f[:1], sources=[2], t_start=[50], t_end=[60])   # another source than track 1's
    assert "source" in L.sb200_last_error().decode()
    with pytest.raises(_lib.Sb200Error):
        g.merge_owned([1], [3])   # different sources under same_source
    with pytest.raises(_lib.Sb200Error):
        g.associate_wasted(eng.Tracker(_lib.default_options()), cap=1)
    assert "window" in L.sb200_last_error().decode()
    assert np.array_equal(g.save(), blob)
    # the _attr calls on an ungated store
    u = gpu_store(feature_dim=8, topn=5)
    t0g, t1g = np.array([0], np.int64), np.array([1], np.int64)
    a = _lib.FstoreAttrs(src.ctypes.data, t0g.ctypes.data, t1g.ctypes.data)
    rc, msg = _rc(L, L.sb200_fstore_add_attr, u._h, 1, p(ids), C.byref(a), p(f), None, None)
    assert rc == -1 and "gate" in msg
    rc, msg = _rc(L, L.sb200_fstore_fetch_attr, u._h, 1, p(ids), p(src), p(t0), p(t1))
    assert rc == -1 and "gate" in msg
    with pytest.raises(ValueError):
        u.add([1], f[:1], **good)
    assert u.size() == 0


def test_gated_blob_round_trips_and_twins_are_byte_equal():
    import similari_b200.engine as eng
    from similari_b200 import _lib

    rng = np.random.default_rng(8)
    for storage in ("f32", "bf16"):
        g1, o = store_pair(storage=storage, gate="any_source", max_observations=3, feature_dim=20, topn=5)
        g2 = gpu_store(storage=storage, gate="any_source", max_observations=3, feature_dim=20, topn=5)
        _fill((g1, g2, o), rng, 30, 20, storage, 3)
        for src in range(2, 30):   # the first track whose window track 1 can absorb
            try:
                o.merge_owned([1], [src], remove=True)
            except ValueError:
                continue
            for x in (g1, g2):
                x.merge_owned([1], [src], remove=True)
            break
        assert g1.size() == o.size() == 29
        b1, b2 = g1.save(), g2.save()
        assert np.array_equal(b1, b2)
        h = _lib.FstoreBlobHeaderV2.from_buffer_copy(b1[:C.sizeof(_lib.FstoreBlobHeaderV2)].tobytes())
        assert (h.version, h.gate, h.live) == (2, 2, g1.size())
        assert [h.sec_bytes[i] for i in (4, 5, 6)] == [8 * h.live] * 3
        c = eng.FeatureStore.load(b1)
        assert c.gate == "any_source"
        assert np.array_equal(c.save(), b1)
        same_store(c, o)
        q, offs, qf = _queries(rng, 10, 20, storage, 5000)
        at = _windows(rng, 10)
        same_results(c.associate(q, offs, qf, **at), o.associate(q, offs, qf, **at))
        same_store(c, o)


def test_an_ungated_store_still_writes_version_1():
    import similari_b200.engine as eng
    from similari_b200 import _lib

    s = gpu_store(feature_dim=8, topn=5)
    s.add([1, 2], np.ones((2, 8), np.float32))
    b = s.save()
    h = _lib.FstoreBlobHeader.from_buffer_copy(b[:128].tobytes())
    assert (h.version, h.live) == (1, 2)
    assert h.sec_off[0] == 256 and h.total_bytes == len(b)
    c = eng.FeatureStore.load(b)
    assert c.gate is None and np.array_equal(c.save(), b)


def test_damaged_version_2_blobs_are_refused():
    import similari_b200.engine as eng
    from similari_b200 import _lib

    g = gpu_store(gate="same_source", feature_dim=8, topn=5)
    g.add([1, 2, 3], np.ones((3, 8), np.float32), sources=[1, 1, 1], t_start=[0, 10, 20], t_end=[5, 15, 25])
    blob = g.save()
    hdr = _lib.FstoreBlobHeaderV2.from_buffer_copy(blob[:C.sizeof(_lib.FstoreBlobHeaderV2)].tobytes())

    def damaged(edit):
        b = blob.copy()
        edit(b, _lib.FstoreBlobHeaderV2.from_buffer(b))
        return b

    def column(b, sec):
        return b[hdr.sec_off[sec]: hdr.sec_off[sec] + hdr.sec_bytes[sec]].view(np.int64)

    refused_blob(damaged(lambda b, h: setattr(h, "gate", 0)), "gate")
    refused_blob(damaged(lambda b, h: setattr(h, "gate", 3)), "gate")
    refused_blob(damaged(lambda b, h: column(b, 5).__setitem__(1, 16)), "t_start > t_end")
    refused_blob(damaged(lambda b, h: column(b, 6).__setitem__(2, -1)), "t_start > t_end")
    refused_blob(damaged(lambda b, h: h.sec_bytes.__setitem__(6, h.sec_bytes[6] - 8)), "t_end holds")
    refused_blob(damaged(lambda b, h: h.sec_off.__setitem__(4, h.sec_off[4] + 8)), "source is not 256-byte aligned")
    refused_blob(blob[:150], "truncated")
    assert np.array_equal(eng.FeatureStore.load(blob).save(), blob)
