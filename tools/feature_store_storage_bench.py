"""Feature track store with 2-byte stored rows: one JSON line per measurement.

  python tools/feature_store_storage_bench.py [--rounds N] [--tracks N]

Three stores hold the same gallery (100,000 tracks x K = 3 x 512-d, euclidean): an f32 store and an f16 store fed an
FP16 column, and a bf16 store fed a BF16 column.
1. `search` of 1,024 single-observation queries (FP16 column for the f32 and f16 stores, BF16 for the bf16 store), the
   stores alternated over rounds in one process: distance-stage device time (sb200_fstore_last_stage_ms) and host call
   time, median of each round's calls; the line reports the median and range of the rounds.  Before anything is timed
   the f16 store's outputs are compared with the f32 store's for equality (own-type feed: they must be identical), and
   the bf16 store's with an f32 store fed the same BF16 column.
2. Device bytes of the stored rows (`feat`) and blob bytes of each store.
3. `save` / `load` of each store to a device blob and to a pageable host blob: host wall clock (the calls return when
   the copy is complete).
Seeded.  The card's name and power limit are read in the same run; without a CUDA device the script fails.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = [x.strip() for x in out.split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def emit(d):
    print(json.dumps(d), flush=True)


def stats(v):
    return {"median": float(np.median(v)), "min": float(min(v)), "max": float(max(v))}


def bf16_bits(x):
    """Round-to-nearest-even bfloat16 bits of f32 values (finite inputs)."""
    u = x.astype(np.float32).view(np.uint32).astype(np.uint64)
    return ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)


def build_stores(tracks, K, dim, seed=0):
    """{name: (store, query column type)}; the same random rows go into every store, as FP16 or BF16."""
    import similari_b200.engine as eng

    def make(storage, column):
        st = eng.FeatureStore(metric="euclidean", distance_filter=1e30, max_observations=K, feature_dim=dim, topn=5,
                              max_distance=1e30, min_votes=1, storage=storage)
        st.set_feature_type(column)
        return st

    stores = {"f32": (make("f32", "f16"), "f16"), "f16": (make("f16", "f16"), "f16"),
              "bf16": (make("bf16", "bf16"), "bf16"), "f32_bf16_fed": (make("f32", "bf16"), "bf16")}
    rng = np.random.default_rng(seed)
    chunk = 20_000
    for b in range(0, tracks, chunk):
        n = min(chunk, tracks - b)
        ids = np.repeat(np.arange(b + 1, b + 1 + n, dtype=np.uint64), K)
        rows = rng.standard_normal((n * K, dim)).astype(np.float32)
        cols = {"f16": rows.astype(np.float16), "bf16": bf16_bits(rows)}
        for st, t in stores.values():
            st.add(ids, cols[t])
    return stores


def same(a, b):
    for k in a:
        x, y = a[k], b[k]
        if x.dtype == np.float64:
            x, y = x.view(np.uint64), y.view(np.uint64)
        if not np.array_equal(x, y):
            return False
    return True


def search_bench(stores, queries, dim, rounds, calls, info):
    rng = np.random.default_rng(1)
    q = rng.standard_normal((queries, dim)).astype(np.float32)
    cols = {"f16": q.astype(np.float16), "bf16": bf16_bits(q)}
    qid = np.arange(10**9, 10**9 + queries, dtype=np.uint64)
    offs = np.arange(queries + 1, dtype=np.int32)
    res = {name: st.search(qid, offs, cols[t]) for name, (st, t) in stores.items()}   # also the warm-up
    if not same(res["f16"], res["f32"]):
        raise SystemExit("the f16 store's search differs from the f32 store's")
    if not same(res["bf16"], res["f32_bf16_fed"]):
        raise SystemExit("the bf16 store's search differs from the f32 store fed the same BF16 column")
    timed = ["f32", "f16", "bf16"]
    dist = {n: [] for n in timed}
    call = {n: [] for n in timed}
    for _ in range(rounds):
        for name in timed:
            st, t = stores[name]
            d, w = [], []
            for _ in range(calls):
                t0 = time.perf_counter()
                st.search(qid, offs, cols[t])
                w.append((time.perf_counter() - t0) * 1e3)
                d.append(float(st.last_stage_ms()[0]))
            dist[name].append(float(np.median(d)))
            call[name].append(float(np.median(w)))
    st = stores["f32"][0]
    emit({"bench": "storage_search", "queries": queries, "tracks": st.size(), "K": st.K, "dim": dim, "rounds": rounds,
          "calls_per_round": calls, "outputs_identical": True, **info,
          "distance_stage_ms": {n: stats(v) for n, v in dist.items()},
          "ms_per_call": {n: stats(v) for n, v in call.items()}})


def sizes(stores, info):
    out = {}
    for name in ("f32", "f16", "bf16"):
        st = stores[name][0]
        d8 = (st.D + 7) // 8 * 8
        out[name] = {"feat_bytes_live": st.size() * st.K * d8 * (4 if name == "f32" else 2),
                     "blob_bytes": int(st.save_device(0, 0))}
    emit({"bench": "storage_bytes", "tracks": stores["f32"][0].size(), **info, "bytes": out})


def blob_times(stores, reps, info):
    import torch

    import similari_b200.engine as eng

    out = {}
    for name in ("f32", "f16", "bf16"):
        st = stores[name][0]
        n = st.save_device(0, 0)
        dblob = torch.empty(n, dtype=torch.uint8, device="cuda")
        hblob = np.empty(n, np.uint8)
        hblob[:] = 0   # touch the pages: the first save is not charged with page faults
        torch.cuda.synchronize()
        res = {"save_device": [], "load_device": [], "save_host_pageable": [], "load_host_pageable": []}
        for _ in range(reps + 1):   # the first repetition warms up
            t0 = time.perf_counter()
            st.save_device(dblob.data_ptr(), n)
            t1 = time.perf_counter()
            c = eng.FeatureStore.load(dblob.data_ptr(), n)
            t2 = time.perf_counter()
            c.close()
            t3 = time.perf_counter()
            if st._L.sb200_fstore_save(st._h, hblob.ctypes.data, n, C.byref(C.c_uint64(0))) != 0:
                raise SystemExit("save to the host blob failed")
            t4 = time.perf_counter()
            c = eng.FeatureStore.load(hblob)
            t5 = time.perf_counter()
            c.close()
            for k, v in zip(res, (t1 - t0, t2 - t1, t4 - t3, t5 - t4)):
                res[k].append(v * 1e3)
        if not np.array_equal(dblob.cpu().numpy(), hblob):
            raise SystemExit(f"{name}: the device blob and the host blob differ")
        out[name] = {"blob_bytes": int(n), **{k: stats(v[1:]) for k, v in res.items()}}
        del dblob
    emit({"bench": "storage_blob_wall", "tracks": stores["f32"][0].size(), "reps": reps, **info, "ms": out})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--tracks", type=int, default=100_000)
    a = ap.parse_args()
    from similari_b200._lib import lib

    if lib().sb200_device_count() <= 0:
        raise SystemExit("feature_store_storage_bench needs a CUDA device")
    info = card()
    stores = build_stores(a.tracks, 3, 512)
    search_bench(stores, 1024, 512, a.rounds, a.calls, info)
    sizes(stores, info)
    blob_times(stores, 3, info)


if __name__ == "__main__":
    main()
