"""Feature track store: TopN voting against BestFit voting (sb200_fstore_set_voting), the two arms alternated in one
process.  One JSON line per result.

  python tools/feature_store_bestfit_bench.py [--rounds 6] [--tracks 100000] [--iters 50] [--scenes 64]

First both rules are checked against the CPU oracle at a small size (associate and search on a contended store).  Then:
- gallery search: 512 single-row queries x 100,000 tracks x K = 12 x 512-d, euclidean, f32 rows (DESIGN 3d.6).  One
  store; the rule is switched before each call.  Per arm the distance and voting stages (sb200_fstore_last_stage_ms:
  BestFit's voting stage holds TopN and the two claim passes) and the host call time.  Results checked equal in counts
  and weights, which the rule does not change.
- feature-tracker associate loop: 500 objects, 128-d, K = 12, topn 1, a fresh store per arm and round, iterated --iters
  times; per iteration host time.
- wasted tracks into a store (tools/wasted_store_bench.py's shape: a BatchVisualSort tracker of --scenes scenes x 512
  objects x 512-d, kept history 10, a 2,000-track gallery, one collection per frame): a TopN store and a BestFit store
  start from the same gallery; each round the tracker is cloned and each arm collects from one of the two.  Per arm the
  wall time of the call, and the number of stored tracks the call merged more than one query into (TopN's fused
  identities; BestFit's must be 0).
Each cell is the median (min - max) of the rounds' medians.  Times are host clocks around calls that return after their
device work.  Seeded.  The card's name, power limit and clock are read in the same run; without a device the script
fails.
"""
from __future__ import annotations

import argparse
import dataclasses
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

RULES = ("topn", "best_fit")


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
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype == np.float64:
        a, b = a.view(np.uint64), b.view(np.uint64)
    if not np.array_equal(a, b):
        raise SystemExit(f"{what} differs")


def fused(out):
    """Stored tracks that more than one query of the call was merged into."""
    t = out["track_ids"][out["merged"].astype(bool)]
    _, n = np.unique(t, return_counts=True)
    return int((n > 1).sum())


def check_against_oracle():
    import fstore_oracle as fo
    import similari_b200.engine as eng

    rng = np.random.default_rng(3)
    kw = dict(distance_filter=1e9, max_observations=4, feature_dim=64, topn=3, max_distance=1e9, min_votes=1)
    for rule in RULES:
        g, o = eng.FeatureStore(voting=rule, **kw), fo.FeatureStore(voting=rule, **kw)
        base = rng.standard_normal((20, 64)).astype(np.float32)
        ids = np.repeat(np.arange(1, 21, dtype=np.uint64), 3)
        rows = base[ids - 1] + 0.2 * rng.standard_normal((60, 64)).astype(np.float32)
        g.add(ids, rows)
        o.add(ids, rows)
        for it in range(5):
            Q = 200
            offs = np.arange(Q + 1, dtype=np.int32) * 2
            f = base[rng.integers(0, 6, 2 * Q)] + 0.3 * rng.standard_normal((2 * Q, 64)).astype(np.float32)
            qid = np.arange(1000 + it * Q, 1000 + (it + 1) * Q, dtype=np.uint64)
            for k, v in g.search(qid, offs, f).items():
                equal(v, o.search(qid, offs, f)[k], f"{rule} search {k}")
            rg, ro = g.associate(qid, offs, f), o.associate(qid, offs, f)
            for k in ro:
                equal(rg[k], ro[k], f"{rule} associate {k}")
        equal(g.ids(), o.ids(), f"{rule} ids")
        live = o.ids()
        for x, y in zip(g.fetch(live), o.fetch(live)):
            equal(x, y, f"{rule} fetch")
    emit({"what": "oracle_check", "ok": True, **CARD})


def gallery(tracks, rounds, K=12, dim=512, Q=512, calls=5):
    import similari_b200.engine as eng

    s = eng.FeatureStore(metric="euclidean", distance_filter=1e30, max_observations=K, feature_dim=dim, topn=5,
                         max_distance=1e30, min_votes=1)
    rng = np.random.default_rng(0)
    for b in range(0, tracks, 10_000):
        n = min(10_000, tracks - b)
        s.add(np.repeat(np.arange(b + 1, b + 1 + n, dtype=np.uint64), K), rng.standard_normal((n * K, dim)).astype(np.float32))
    qids = np.arange(10**7, 10**7 + Q, dtype=np.uint64)
    offs = np.arange(Q + 1, dtype=np.int32)
    qf = rng.standard_normal((Q, dim)).astype(np.float32)
    res = {}
    for rule in RULES:
        s.set_voting(rule)
        res[rule] = s.search(qids, offs, qf)
    for k in ("counts", "weights"):
        equal(res["topn"][k], res["best_fit"][k], f"gallery search {k}")
    dist, vote, call = ({r: [] for r in RULES} for _ in range(3))
    for r in range(rounds):
        for rule in (RULES if r % 2 == 0 else RULES[::-1]):
            s.set_voting(rule)
            d, v, c = [], [], []
            for _ in range(calls):
                t = time.perf_counter()
                s.search(qids, offs, qf)
                c.append((time.perf_counter() - t) * 1e3)
                st = s.last_stage_ms()
                d.append(float(st[0]))
                v.append(float(st[1]))
            dist[rule].append(float(np.median(d)))
            vote[rule].append(float(np.median(v)))
            call[rule].append(float(np.median(c)))
    pairs = Q * tracks * K
    for rule in RULES:
        emit({"what": "gallery_search", "voting": rule, "tracks": tracks, "K": K, "dim": dim, "queries": Q,
              "rounds": rounds, "dist_ms": stats(dist[rule]), "voting_ms": stats(vote[rule]),
              "call_ms": stats(call[rule]), "distance_matrix_bytes": pairs * 4, **CARD})


def tracker_loop(objects, iters, rounds, dim=128, K=12, seed=1):
    import similari_b200.engine as eng

    kw = dict(metric="euclidean", distance_filter=1e30, max_observations=K, feature_dim=dim, topn=1, max_distance=1e30,
              min_votes=1)
    base = np.random.default_rng(seed).standard_normal((objects, dim)).astype(np.float32)
    offs = np.arange(objects + 1, dtype=np.int32)

    def run(rule):
        s = eng.FeatureStore(voting=rule, **kw)
        r = np.random.default_rng(seed + 1)
        ms = []
        for i in range(iters):
            f = base + 0.05 * r.standard_normal(base.shape).astype(np.float32)
            ids = np.arange(1 + i * objects, 1 + (i + 1) * objects, dtype=np.uint64)
            t = time.perf_counter()
            s.associate(ids, offs, f)
            ms.append((time.perf_counter() - t) * 1e3)
        return float(np.median(ms))

    per = {r: [] for r in RULES}
    for r in range(rounds):
        for rule in (RULES if r % 2 == 0 else RULES[::-1]):
            per[rule].append(run(rule))
    for rule in RULES:
        emit({"what": "tracker_associate_loop", "voting": rule, "objects": objects, "iters": iters, "dim": dim, "K": K,
              "rounds": rounds, "iter_ms": stats(per[rule]), **CARD})


def wasted(scenes, rounds, objects=512, dim=512, hist=10, gallery_n=2000, warmup=2):
    import similari_b200.engine as eng
    from similari_b200._lib import default_options
    from similari_b200.workload import CONFIGS, Workload

    cfg = dataclasses.replace(CONFIGS["cfg5"], n_scenes=scenes, n_objects=objects, feature_dim=dim, drop_frac=0.1,
                              seed=0x5EED5700)
    opts = dict(kind=3, positional_kind=0, iou_threshold=0.3, max_idle_epochs=1, history_length=hist, visual_kind=0,
                visual_threshold=0.7, feature_dim=dim, visual_max_observations=3, visual_min_votes=1,
                visual_minimal_track_length=1, min_confidence=0.1)
    tracker = eng.Tracker(default_options(**opts))
    tracker.set_feature_history(True)
    stores = {rule: eng.FeatureStore(metric="euclidean", distance_filter=1.0, max_observations=3, feature_dim=dim,
                                     topn=1, max_distance=1.0, min_votes=1, voting=rule) for rule in RULES}
    g = np.random.default_rng(7).standard_normal((gallery_n, dim)).astype(np.float32)
    g /= np.linalg.norm(g, axis=1, keepdims=True)
    for s in stores.values():
        s.add(np.arange(1 << 40, (1 << 40) + gallery_n, dtype=np.uint64), g)
    wl = Workload(cfg)
    ms, fuse, merged = ({r: [] for r in RULES} for _ in range(3))
    for rnd in range(warmup + rounds):
        f = wl.next_frame()
        tracker.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=f["features"])
        trackers = {"topn": tracker, "best_fit": eng.Tracker.load(tracker.save())}
        for rule in (RULES if rnd % 2 == 0 else RULES[::-1]):
            trackers[rule].sync()
            t0 = time.perf_counter()
            r = stores[rule].associate_wasted(trackers[rule], history_cap=hist)
            if rnd >= warmup:
                ms[rule].append((time.perf_counter() - t0) * 1e3)
                fuse[rule].append(fused(r))
                merged[rule].append(int(r["merged"].sum()))
    if sum(fuse["best_fit"]):
        raise SystemExit("BestFit merged two queries of one call into one track")
    for rule in RULES:
        emit({"what": "wasted_to_store", "voting": rule, "scenes": scenes, "objects": objects, "dim": dim,
              "kept_history_length": hist, "gallery": gallery_n, "rounds": rounds, "ms_per_collection": stats(ms[rule]),
              "merged_per_collection": stats(merged[rule]), "tracks_fused_per_collection": stats(fuse[rule]),
              "tracks_fused_total": int(sum(fuse[rule])), "store_size_after": stores[rule].size(), **CARD})


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--tracks", type=int, default=100_000)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--scenes", type=int, default=64)
    a = ap.parse_args()
    from similari_b200._lib import lib

    if lib().sb200_device_count() <= 0:
        raise SystemExit("needs a CUDA device")
    CARD = card()
    check_against_oracle()
    gallery(a.tracks, a.rounds)
    tracker_loop(500, a.iters, a.rounds)
    wasted(a.scenes, a.rounds)
