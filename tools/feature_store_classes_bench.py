"""Feature track store with two feature classes against two single-class stores holding the same rows.  One JSON line
per measurement.

  python tools/feature_store_classes_bench.py [--gallery N] [--rounds N] [--reps N]

A gallery of --gallery tracks (default 100,000), each holding K = 3 rows of a 128-d class and of a 512-d class (f32), is
built once in a two-class store (classes={0: 128, 1: 512}) and once in two single-class stores (128-d and 512-d).  Then:
- search: 64 queries of 3 rows against each class, the class search of the two-class store and the search of the
  single-class store of that dim alternated in one process, outputs checked equal before the timings count;
- merge_owned: 256 pairs of stored tracks merged (remove=True) in the two-class store, against the same pairs merged in
  both single-class stores;
- associate_store: 256 tracks of a two-class collecting store taken into the gallery (remove=True), against the same
  tracks of two single-class collecting stores taken into the single-class galleries.
Times are host clocks around calls that end in a device synchronise; per arm the median and range over the rounds'
medians of --reps calls.  Seeded.  The card's name and power limit are read in the same run; without a CUDA device the
script fails.
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

K = 3
CLASSES = {0: 128, 1: 512}


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = [x.strip() for x in out.split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def emit(d):
    print(json.dumps(d), flush=True)


def store(classes=None, dim=128):
    import similari_b200.engine as eng

    return eng.FeatureStore(metric="euclidean", distance_filter=1e9, max_observations=K, feature_dim=dim, topn=5,
                            max_distance=1e9, min_votes=1, classes=classes)


def fill(multi, singles, ids, rng):
    rows = np.repeat(ids, K)
    for c, d in CLASSES.items():
        f = rng.standard_normal((len(rows), d)).astype(np.float32)
        multi.add(rows, f, feature_class=c)
        singles[c].add(rows, f)


def same(a, b):
    for k in a:
        x, y = a[k], b[k]
        if x.dtype == np.float64:
            x, y = x.view(np.uint64), y.view(np.uint64)
        if not np.array_equal(x, y):
            raise SystemExit(f"outputs differ in {k}")


def timed(fn):
    t = time.perf_counter()
    fn()
    return (time.perf_counter() - t) * 1e3


def summary(name, rounds, **kw):
    med = [float(np.median(r)) for r in rounds]
    emit({"measure": name, "median_ms": float(np.median(med)), "min_ms": min(med), "max_ms": max(med), **kw, **card()})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gallery", type=int, default=100_000)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    from similari_b200._lib import lib

    if lib().sb200_device_count() <= 0:
        raise SystemExit("needs a CUDA device")
    rng = np.random.default_rng(0)
    multi = store(CLASSES)
    singles = {c: store(dim=d) for c, d in CLASSES.items()}
    fill(multi, singles, np.arange(1, a.gallery + 1, dtype=np.uint64), rng)

    # search per class
    for c, d in CLASSES.items():
        q = rng.standard_normal((64 * K, d)).astype(np.float32)
        qid, off = np.arange(10**9, 10**9 + 64, dtype=np.uint64), np.arange(0, 64 * K + 1, K, dtype=np.int32)
        same(multi.search(qid, off, q, feature_class=c), singles[c].search(qid, off, q))
        rm, rs = [], []
        for r in range(a.rounds):
            tm, ts = [], []
            for i in range(a.reps):
                arms = [(tm, lambda: multi.search(qid, off, q, feature_class=c)), (ts, lambda: singles[c].search(qid, off, q))]
                for out, fn in arms[:: 1 if i % 2 == 0 else -1]:
                    out.append(timed(fn))
            rm.append(tm)
            rs.append(ts)
        summary("search", rm, store="two_classes", feature_class=c, dim=d, gallery=a.gallery, queries=64)
        summary("search", rs, store="single_class", dim=d, gallery=a.gallery, queries=64)

    # merge_owned: fresh pairs every call, in both arms
    nxt = a.gallery
    rm, rs = [], []
    for r in range(a.rounds):
        tm, ts = [], []
        for i in range(a.reps):
            pairs = np.arange(nxt - 511, nxt + 1, dtype=np.uint64)
            nxt -= 512
            dst, src = pairs[0::2], pairs[1::2]
            arms = [(tm, lambda: multi.merge_owned(dst, src)),
                    (ts, lambda: [singles[c].merge_owned(dst, src) for c in CLASSES])]
            for out, fn in arms[:: 1 if i % 2 == 0 else -1]:
                out.append(timed(fn))
        rm.append(tm)
        rs.append(ts)
    for c in CLASSES:
        ids = multi.ids()[:1000]
        cm, fm = multi.fetch(ids, feature_class=c)
        cs, fs = singles[c].fetch(ids)
        if not (np.array_equal(cm, cs) and np.array_equal(fm, fs)):
            raise SystemExit("merge_owned results differ")
    summary("merge_owned", rm, store="two_classes", pairs=256, gallery=a.gallery)
    summary("merge_owned", rs, store="two_single_class_stores", pairs=256, gallery=a.gallery)

    # associate_store: 256 collected tracks of both classes into the gallery
    rm, rs = [], []
    base = 2 * 10**9
    for r in range(a.rounds):
        tm, ts = [], []
        for i in range(a.reps):
            cm_, cs_ = store(CLASSES), {c: store(dim=d) for c, d in CLASSES.items()}
            ids = np.arange(base, base + 256, dtype=np.uint64)
            base += 256
            fill(cm_, cs_, ids, rng)
            res = {}
            arms = [(tm, lambda: res.__setitem__("m", multi.associate_store(cm_, ids, feature_class=0))),
                    (ts, lambda: res.__setitem__("s", [singles[c].associate_store(cs_[c], ids) for c in CLASSES]))]
            for out, fn in arms[:: 1 if i % 2 == 0 else -1]:
                out.append(timed(fn))
            same(res["m"], res["s"][0])
        rm.append(tm)
        rs.append(ts)
    summary("associate_store", rm, store="two_classes", tracks=256, gallery=a.gallery,
            note="one search on class 0, then both classes applied")
    summary("associate_store", rs, store="two_single_class_stores", tracks=256, gallery=a.gallery,
            note="a search and apply in each store")


if __name__ == "__main__":
    main()
