"""Feature track store with a gate (track attributes): what the gate costs.  One JSON line per measurement.

  python tools/feature_store_gate_bench.py [--rounds N] [--tracks N] [--iters N]

1. Gallery search: two stores hold the same gallery (100,000 tracks x K = 3 x 512-d, euclidean), one ungated and one
   gated (same_source; every track in one source, windows in [0, 10^5)).  `search` of 1,024 single-observation queries
   whose windows lie after every track's, so no pair is gated out; the stores alternate over rounds in one process:
   distance-stage device time (sb200_fstore_last_stage_ms) and host call time, median of each round's calls; the line
   reports the median and range of the rounds.
2. Feature-tracker loop: 500 objects, each iteration one drifting observation per object associated with the store
   (benches/feature_tracker.rs), with point windows [i, i] at iteration i, which never conflict.  An ungated and a gated
   store run the same iterations alternately; host time per iteration, median and range over the rounds' medians.
Before anything is timed, each gated store's outputs are compared with the ungated store's for equality (windows that
never conflict must not change a result).  Seeded.  The card's name and power limit are read in the same run; without
a CUDA device the script fails.
"""
from __future__ import annotations

import argparse
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


def same(a, b, what):
    for k in b:
        if not np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8)):
            raise AssertionError(f"{what}: the gated store's {k} differs from the ungated store's")


def gallery(tracks, K, dim, rounds, calls=5, Q=1024, seed=0):
    import similari_b200.engine as eng

    kw = dict(metric="euclidean", distance_filter=1e30, max_observations=K, feature_dim=dim, topn=5, max_distance=1e30,
              min_votes=1)
    stores = {"ungated": eng.FeatureStore(**kw), "gated": eng.FeatureStore(gate="same_source", **kw)}
    rng = np.random.default_rng(seed)
    chunk = 20_000
    for b in range(0, tracks, chunk):
        n = min(chunk, tracks - b)
        ids = np.repeat(np.arange(b + 1, b + 1 + n, dtype=np.uint64), K)
        rows = rng.standard_normal((n * K, dim)).astype(np.float32)
        t0 = np.repeat(rng.integers(0, 100_000, n), K).astype(np.int64)
        stores["ungated"].add(ids, rows)
        stores["gated"].add(ids, rows, sources=np.ones(n * K, np.uint64), t_start=t0, t_end=t0 + 10)
    qids = np.arange(10**7, 10**7 + Q, dtype=np.uint64)
    offs = np.arange(Q + 1, dtype=np.int32)
    qf = rng.standard_normal((Q, dim)).astype(np.float32)
    at = dict(sources=np.ones(Q, np.uint64), t_start=np.full(Q, 200_000, np.int64), t_end=np.full(Q, 200_000, np.int64))
    args = {"ungated": {}, "gated": at}
    same(stores["gated"].search(qids, offs, qf, **at), stores["ungated"].search(qids, offs, qf), "gallery search")
    dist = {k: [] for k in stores}
    call = {k: [] for k in stores}
    for r in range(rounds):
        for name in (("ungated", "gated") if r % 2 == 0 else ("gated", "ungated")):
            s = stores[name]
            d, c = [], []
            for _ in range(calls):
                t = time.perf_counter()
                s.search(qids, offs, qf, **args[name])
                c.append((time.perf_counter() - t) * 1e3)
                d.append(float(s.last_stage_ms()[0]))
            dist[name].append(float(np.median(d)))
            call[name].append(float(np.median(c)))
    for name in stores:
        emit({"what": "gallery_search", "store": name, "tracks": tracks, "K": K, "dim": dim, "queries": Q,
              "rounds": rounds, "dist_ms": stats(dist[name]), "call_ms": stats(call[name]), **CARD})


def tracker_loop(objects, iters, rounds, dim=128, K=3, seed=1):
    import similari_b200.engine as eng

    kw = dict(metric="euclidean", distance_filter=1e30, max_observations=K, feature_dim=dim, topn=1, max_distance=1e30,
              min_votes=1)
    rng = np.random.default_rng(seed)
    base = rng.standard_normal((objects, dim)).astype(np.float32)
    offs = np.arange(objects + 1, dtype=np.int32)
    src = np.ones(objects, np.uint64)

    def run(gated, timed):
        s = eng.FeatureStore(gate="same_source" if gated else None, **kw)
        r = np.random.default_rng(seed + 1)
        outs, ms = [], []
        for i in range(iters):
            f = base + 0.05 * r.standard_normal(base.shape).astype(np.float32)
            ids = np.arange(1 + i * objects, 1 + (i + 1) * objects, dtype=np.uint64)
            at = dict(sources=src, t_start=np.full(objects, i, np.int64), t_end=np.full(objects, i, np.int64))
            t = time.perf_counter()
            o = s.associate(ids, offs, f, **(at if gated else {}))
            ms.append((time.perf_counter() - t) * 1e3)
            if not timed:
                outs.append(o)
        return outs, ms

    for a, b in zip(run(True, False)[0], run(False, False)[0]):
        same(a, b, "tracker loop")
    per = {"ungated": [], "gated": []}
    for r in range(rounds):
        for name in (("ungated", "gated") if r % 2 == 0 else ("gated", "ungated")):
            per[name].append(float(np.median(run(name == "gated", True)[1])))
    for name in per:
        emit({"what": "tracker_associate_loop", "store": name, "objects": objects, "iters": iters, "dim": dim, "K": K,
              "rounds": rounds, "iter_ms": stats(per[name]), **CARD})


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--tracks", type=int, default=100_000)
    ap.add_argument("--iters", type=int, default=50)
    a = ap.parse_args()
    CARD = card()
    gallery(a.tracks, 3, 512, a.rounds)
    tracker_loop(500, a.iters, a.rounds)
