"""GPU check of the feature store's columns through growth, compaction and a gate switch on an emptied store that keeps
its capacity (where set_gate allocates the attribute columns at the capacity): after every step the store matches the CPU
oracle bit for bit, and the final blob equals a fresh twin's and loads into a store that continues like the original."""
import zlib

import numpy as np
import pytest

import fstore_oracle as fo
from fstore_checks import gpu_store, same_results, same_store, store_options, store_pair

pytestmark = pytest.mark.gpu

K, DIM = 3, 20   # d8 = 24: every stored row has a zero tail
OPTS = dict(max_observations=K, feature_dim=DIM, topn=3)
NEXT_TYPE = {"f32": "f16", "f16": "bf16", "bf16": "f32"}


def _rows(rng, track_ids, storage, gated):
    """An add of 1..2K rows for each of `track_ids`, shuffled, with one source per id when the store is gated."""
    ids = np.repeat(np.asarray(track_ids, np.uint64), 1 + rng.integers(0, 2 * K, len(track_ids)))
    rng.shuffle(ids)
    f = fo.round_rows(rng.standard_normal((len(ids), DIM)).astype(np.float32), storage)
    if not gated:
        return ids, f, {}
    t0 = rng.integers(0, 1000, len(ids)).astype(np.int64)
    return ids, f, dict(sources=(1 + ids % 3).astype(np.uint64), t_start=t0, t_end=t0 + rng.integers(0, 50, len(ids)))


def _add(stores, call):
    ids, f, at = call
    for s in stores:
        s.add(ids, f, **at)


@pytest.mark.parametrize("start_gated", [False, True])
@pytest.mark.parametrize("storage", ["f32", "f16", "bf16"])
def test_columns_survive_growth_compaction_and_a_gate_switch(storage, start_gated):
    import similari_b200.engine as eng
    from similari_b200._lib import check

    rng = np.random.default_rng(zlib.crc32(f"columns {storage} {start_gated}".encode()))
    gate = "same_source" if start_gated else None
    g, o = store_pair(storage=storage, gate=gate, **OPTS)
    # growth: eight adds of ten new tracks each (and rows for tracks already stored), through several reserves
    for step in range(8):
        new = np.arange(10 * step + 1, 10 * step + 11, dtype=np.uint64)
        old = rng.choice(np.arange(1, 10 * step + 1, dtype=np.uint64), min(5, 10 * step), replace=False)
        _add((g, o), _rows(rng, np.concatenate([new, old]), storage, start_gated))
        same_store(g, o)
    # compaction: a scattered third of the tracks leaves, then the store grows again
    gone = o.ids()[rng.permutation(o.size())[: o.size() // 3]]
    same_results(g.fetch(gone, remove=True), o.fetch(gone, remove=True))
    same_store(g, o)
    for step in range(8, 12):
        _add((g, o), _rows(rng, np.arange(10 * step + 1, 10 * step + 11, dtype=np.uint64), storage, start_gated))
        same_store(g, o)
    most = o.size()
    # emptied, the store keeps its capacity; the gate and the storage type change there
    same_results(g.fetch(o.ids(), remove=True), o.fetch(o.ids(), remove=True))
    assert g.size() == 0
    gate = None if start_gated else "same_source"
    storage = NEXT_TYPE[storage]
    check(g._L.sb200_fstore_set_gate(g._h, eng.GATES[gate]))
    check(g._L.sb200_fstore_set_storage_type(g._h, eng.FEATURE_TYPES[storage]))
    g.gate = gate
    assert g.storage_type() == storage
    o = fo.FeatureStore(gate=gate, **store_options(**OPTS))
    same_store(g, o)
    # refill past the old capacity (below 1.5x the most tracks ever stored)
    twin = gpu_store(storage=storage, gate=gate, **OPTS)
    first = 1000
    while o.size() < 2 * most:
        call = _rows(rng, np.arange(first, first + 25, dtype=np.uint64), storage, gate is not None)
        _add((g, o, twin), call)
        same_store(g, o)
        first += 25
    blob = g.save()
    assert np.array_equal(blob, twin.save())
    loaded = eng.FeatureStore.load(blob)
    assert loaded.storage_type() == storage and loaded.gate == gate
    # the loaded store continues like the original: an associate, a removal and an add, then equal blobs
    ids = np.arange(5000, 5012, dtype=np.uint64)
    offs = np.arange(0, 2 * len(ids) + 1, 2, dtype=np.int32)
    f = fo.round_rows(rng.standard_normal((int(offs[-1]), DIM)).astype(np.float32), storage)
    at = {}
    if gate is not None:
        t0 = rng.integers(2000, 3000, len(ids)).astype(np.int64)
        at = dict(sources=(1 + ids % 3).astype(np.uint64), t_start=t0, t_end=t0 + 5)
    same_results(g.associate(ids, offs, f, **at), loaded.associate(ids, offs, f, **at))
    gone = g.ids()[::4]
    for s in (g, loaded):
        s.fetch(gone, remove=True)
    call = _rows(rng, np.arange(6000, 6030, dtype=np.uint64), storage, gate is not None)
    _add((g, loaded), call)
    assert np.array_equal(g.save(), loaded.save())
