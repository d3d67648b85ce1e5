"""Feature track store timings (sb200_fstore_*): prints one JSON line per measurement.

  python tools/feature_store_bench.py [--iters N] [--warmup W] [--skip-gallery]

1. The feature-tracker loop of the reference's benches/feature_tracker.rs (10 / 100 / 500 objects, 256-d, K = 3,
   TopN(1, 100.0, 1), d < 100.0): milliseconds per associate call on the GPU (host wall clock; the call returns after
   its results are on the host) and per iteration of the CPU oracle on all host cores.  The reference's own published
   figures (assets/benchmarks/benchmarks.md:76-86, a laptop CPU) are quoted beside them as the reference's numbers.
2. A gallery-scale search: 1024 single-observation queries against 100,000 tracks x K = 3 x 512-d (euclidean): per-stage
   device times, observation pairs per second and the distance kernel's FP32 operation rate.  The operation count is
   3 non-fused FP32 operations per pair and feature (sub, mul, add); the yardstick is the H100 SXM data sheet's 67
   TFLOP/s FP32 halved (it counts an FMA as two operations), i.e. 33.5 T non-fused operations per second at 700 W.
The card's name and power limit are read in the same run.
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

REFERENCE_NS = {10: 101_465, 100: 4_020_673, 500: 61_716_729}   # benchmarks.md:76-86, ns per iteration


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = [x.strip() for x in out.split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def emit(d):
    print(json.dumps(d), flush=True)


def feature_tracker(objects, iters, warmup, info):
    import fstore_oracle as fo
    import similari_b200.engine as eng
    from similari_b200.workload import FeatGen

    opts = dict(distance_filter=100.0, max_observations=3, feature_dim=256, topn=1, max_distance=100.0, min_votes=1)
    res = {}
    for impl in ("gpu", "oracle"):
        st = eng.FeatureStore(metric="euclidean", **opts) if impl == "gpu" else \
            fo.FeatureStore(metric=fo.EUCLIDEAN, threads=os.cpu_count() or 1, **opts)
        gens = [FeatGen(1000.0 * i, 256, 0.1, seed=1000 + i) for i in range(objects)]
        offs = np.arange(objects + 1, dtype=np.int32)
        nid, times = 1, []
        for it in range(warmup + iters):
            ids = np.arange(nid, nid + objects, dtype=np.uint64)
            nid += objects
            feats = np.stack([g.next() for g in gens])
            t0 = time.perf_counter()
            st.associate(ids, offs, feats)
            if it >= warmup:
                times.append((time.perf_counter() - t0) * 1e3)
        res[impl] = times
        if impl == "gpu":
            res["stage_ms"] = [float(x) for x in st.last_stage_ms()]
            res["size"] = st.size()
    emit({"bench": "feature_tracker", "objects": objects, "dim": 256, "K": 3, "iters": iters, **info,
          "gpu_ms_per_iter_median": float(np.median(res["gpu"])), "gpu_ms_per_iter_min": float(np.min(res["gpu"])),
          "gpu_last_stage_ms": res["stage_ms"], "store_size": res["size"],
          "oracle_ms_per_iter_median": float(np.median(res["oracle"])), "oracle_threads": os.cpu_count(),
          "reference_published_ms_per_iter": REFERENCE_NS[objects] / 1e6,
          "reference_published_on": "the reference's own laptop-CPU figure; not measured here"})


def gallery(iters, info, tracks=100_000, K=3, dim=512, queries=1024):
    import similari_b200.engine as eng

    rng = np.random.default_rng(0)
    st = eng.FeatureStore(metric="euclidean", distance_filter=1e30, max_observations=K, feature_dim=dim, topn=5,
                          max_distance=1e30, min_votes=1)
    chunk = 20_000
    for b in range(0, tracks, chunk):
        n = min(chunk, tracks - b)
        ids = np.repeat(np.arange(b + 1, b + 1 + n, dtype=np.uint64), K)
        st.add(ids, rng.standard_normal((n * K, dim)).astype(np.float32))
    qid = np.arange(10**9, 10**9 + queries, dtype=np.uint64)
    offs = np.arange(queries + 1, dtype=np.int32)
    q = rng.standard_normal((queries, dim)).astype(np.float32)
    st.search(qid, offs, q)   # warm-up (allocations, module load)
    stages, walls = [], []
    for _ in range(iters):
        t0 = time.perf_counter()
        st.search(qid, offs, q)
        walls.append((time.perf_counter() - t0) * 1e3)
        stages.append(st.last_stage_ms().astype(float))
    stages = np.array(stages)
    dist_ms = float(np.median(stages[:, 0]))
    pairs = queries * tracks * K
    ops = 3.0 * pairs * dim
    emit({"bench": "gallery_search", "queries": queries, "tracks": tracks, "K": K, "dim": dim, "iters": iters, **info,
          "stage_ms_median": {"distance": dist_ms, "topn": float(np.median(stages[:, 1]))},
          "call_ms_median": float(np.median(walls)), "pairs": pairs, "pairs_per_s": pairs / (dist_ms * 1e-3),
          "fp32_ops_per_s": ops / (dist_ms * 1e-3),
          "fraction_of_33.5T_nonfused": ops / (dist_ms * 1e-3) / 33.5e12})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--skip-gallery", action="store_true")
    a = ap.parse_args()
    from similari_b200._lib import lib

    if lib().sb200_device_count() <= 0:
        raise SystemExit("feature_store_bench needs a CUDA device")
    info = card()
    for objects in (10, 100, 500):
        feature_tracker(objects, a.iters, a.warmup, info)
    if not a.skip_gallery:
        gallery(max(5, a.iters // 4), info)


if __name__ == "__main__":
    main()
