"""Feature track store with quality retention: what keeping the best observations costs.  One JSON line per measurement.

  python tools/feature_store_quality_bench.py [--rounds N] [--tracks N] [--iters N]

0. Before anything is timed, a small quality store (f16 rows, gated and ungated) runs a seeded mix of add / associate /
   merge_owned calls beside the CPU oracle (fstore_oracle), and its outputs, rows, qualities and histories must be
   identical.
1. Gallery search: two stores hold the same gallery (100,000 tracks x 12 rows x 512-d, euclidean, f32 rows), one newest
   and one quality store (initial_capacity 12, so every track holds its 12 rows too).  `search` of 512 single-observation
   queries per call (1,024 per measurement pair would exceed the 2^30-pair bound of one call at K = 12); the stores
   alternate over rounds in one process: distance-stage device time (sb200_fstore_last_stage_ms) and host call time,
   median of each round's calls; the line reports the median and range of the rounds.
2. Feature-tracker loop: 500 objects, each iteration one drifting observation per object associated with the store
   (benches/feature_tracker.rs, K = 12), the quality store with a random quality per observation (defaults 4 / 1.5).  A
   newest and a quality store run the same iterations alternately; host time per iteration and the apply-stage device
   time, median and range over the rounds' medians.
Seeded.  The card's name and power limit are read in the same run; without a CUDA device the script fails.
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


def equal(a, b, what):
    if not np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8)):
        raise AssertionError(f"{what} differs from the oracle")


def check_against_oracle(seed=5):
    import fstore_oracle as fo
    import similari_b200.engine as eng

    rng = np.random.default_rng(seed)
    dim = 64
    for gate in (None, "any_source"):
        kw = dict(distance_filter=1e9, max_observations=12, feature_dim=dim, topn=3, max_distance=1e9, min_votes=1,
                  retention="quality", gate=gate)
        g, o = eng.FeatureStore(storage="f16", **kw), fo.FeatureStore(threads=8, **kw)
        next_id = 1
        for it in range(30):
            Q = 40
            lens = 1 + rng.integers(0, 9, Q)
            offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
            f = fo.round_rows(rng.standard_normal((int(offs[-1]), dim)).astype(np.float32), "f16")
            q = rng.integers(0, 5, int(offs[-1])).astype(np.float32)
            ids = np.arange(next_id, next_id + Q, dtype=np.uint64)
            next_id += Q
            t0 = np.full(Q, it, np.int64)
            at = {} if gate is None else dict(sources=np.ones(Q, np.uint64), t_start=t0, t_end=t0)
            rg, ro = g.associate(ids, offs, f, quality=q, **at), o.associate(ids, offs, f, quality=q, **at)
            for k in ro:
                equal(rg[k], ro[k], f"associate {k}")
            if it % 10 == 9:
                live = o.ids()
                pick = live[rng.choice(len(live), 6, replace=False)]
                g.merge_owned(pick[1:], pick[:-1])
                o.merge_owned(pick[1:], pick[:-1])
        live = o.ids()
        equal(g.ids(), live, "ids")
        for x, y in zip(g.fetch_quality(live), o.fetch_quality(live)):
            equal(x, y, "fetch_quality")
        for x, y in zip(g.merge_history(live), o.merge_history(live)):
            equal(x, y, "merge_history")
    emit({"what": "oracle_check", "ok": True, **CARD})


def gallery(tracks, K, dim, rounds, calls=5, Q=512, seed=0):
    import similari_b200.engine as eng

    kw = dict(metric="euclidean", distance_filter=1e30, max_observations=K, feature_dim=dim, topn=5, max_distance=1e30,
              min_votes=1)
    stores = {"newest": eng.FeatureStore(**kw),
              "quality": eng.FeatureStore(retention="quality", initial_capacity=K, merge_extension=1.0, **kw)}
    rng = np.random.default_rng(seed)
    chunk = 10_000
    for b in range(0, tracks, chunk):
        n = min(chunk, tracks - b)
        ids = np.repeat(np.arange(b + 1, b + 1 + n, dtype=np.uint64), K)
        rows = rng.standard_normal((n * K, dim)).astype(np.float32)
        stores["newest"].add(ids, rows)
        stores["quality"].add(ids, rows, quality=np.zeros(n * K, np.float32))   # equal qualities: insertion order
    qids = np.arange(10**7, 10**7 + Q, dtype=np.uint64)
    offs = np.arange(Q + 1, dtype=np.int32)
    qf = rng.standard_normal((Q, dim)).astype(np.float32)
    qq = np.zeros(Q, np.float32)
    args = {"newest": {}, "quality": {"quality": qq}}
    a, b = stores["quality"].search(qids, offs, qf, quality=qq), stores["newest"].search(qids, offs, qf)
    for k in b:   # the same rows in the same order: the same results
        equal(a[k], b[k], f"gallery search {k} (quality store against newest store)")
    dist = {k: [] for k in stores}
    call = {k: [] for k in stores}
    for r in range(rounds):
        for name in (("newest", "quality") if r % 2 == 0 else ("quality", "newest")):
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


def tracker_loop(objects, iters, rounds, dim=128, K=12, seed=1):
    import similari_b200.engine as eng

    kw = dict(metric="euclidean", distance_filter=1e30, max_observations=K, feature_dim=dim, topn=1, max_distance=1e30,
              min_votes=1)
    rng = np.random.default_rng(seed)
    base = rng.standard_normal((objects, dim)).astype(np.float32)
    offs = np.arange(objects + 1, dtype=np.int32)

    def run(quality):
        s = eng.FeatureStore(retention="quality" if quality else "newest", **kw)
        r = np.random.default_rng(seed + 1)
        ms, apply_ms = [], []
        for i in range(iters):
            f = base + 0.05 * r.standard_normal(base.shape).astype(np.float32)
            q = r.random(objects).astype(np.float32)
            ids = np.arange(1 + i * objects, 1 + (i + 1) * objects, dtype=np.uint64)
            t = time.perf_counter()
            s.associate(ids, offs, f, **({"quality": q} if quality else {}))
            ms.append((time.perf_counter() - t) * 1e3)
            apply_ms.append(float(s.last_stage_ms()[2]))
        return float(np.median(ms)), float(np.median(apply_ms))

    per = {"newest": [], "quality": []}
    app = {"newest": [], "quality": []}
    for r in range(rounds):
        for name in (("newest", "quality") if r % 2 == 0 else ("quality", "newest")):
            m, a = run(name == "quality")
            per[name].append(m)
            app[name].append(a)
    for name in per:
        emit({"what": "tracker_associate_loop", "store": name, "objects": objects, "iters": iters, "dim": dim, "K": K,
              "rounds": rounds, "iter_ms": stats(per[name]), "apply_ms": stats(app[name]), **CARD})


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--tracks", type=int, default=100_000)
    ap.add_argument("--iters", type=int, default=50)
    a = ap.parse_args()
    CARD = card()
    check_against_oracle()
    gallery(a.tracks, 12, 512, a.rounds)
    tracker_loop(500, a.iters, a.rounds)
