"""Feature track store owned-call timings (sb200_fstore_search_owned / _merge_owned): one JSON line per measurement.

  python tools/feature_store_owned_bench.py [--tracks N] [--rounds R] [--subset Q] [--pairs P]

a. An each-mode self-join of a gallery (N tracks x K = 3 x 512-d, euclidean; default 20,000): search_owned(all ids,
   each=True), ms per call and observation pairs per second (query rows x stored rows, the distance matrix it computes).
b. The host path that gives the same results, on Q queries (default 200): fetch the query's rows, then one search per
   query, against search_owned(those ids, each=True).  The two arms are alternated within each round.
c. merge_owned of P pairs (default 10,000) that include chains and stars, without removal, and of P / 10 pairs with
   removal, against the host emulation (fetch src, add its rows to dest, fetch src with remove).  Each arm starts from
   the same store, reloaded from a device blob, and the arms alternate.
Every arm's outputs (results, or the whole store blob) are compared for equality before anything is timed.  Seeded.  The
card's name and power limit are read in the same run; without a CUDA device the script fails.
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


def build_store(tracks, K, dim, seed=0):
    import similari_b200.engine as eng

    rng = np.random.default_rng(seed)
    st = eng.FeatureStore(metric="euclidean", distance_filter=1e30, max_observations=K, feature_dim=dim, topn=5,
                          max_distance=1e30, min_votes=1)
    chunk = 20_000
    for b in range(0, tracks, chunk):
        n = min(chunk, tracks - b)
        ids = np.repeat(np.arange(b + 1, b + 1 + n, dtype=np.uint64), K)
        st.add(ids, rng.standard_normal((n * K, dim)).astype(np.float32))
    return st


def timed(fn):
    t0 = time.perf_counter()
    r = fn()
    return r, time.perf_counter() - t0


def same(a, b):
    return all(np.array_equal(np.asarray(a[k]).view(np.uint8), np.asarray(b[k]).view(np.uint8)) for k in a)


def host_search(st, ids):
    """fetch + one search per query: the rows cross PCIe twice."""
    out = {"counts": [], "winners": [], "weights": []}
    cnt, f = st.fetch(ids)
    for i, q in enumerate(ids):
        r = st.search(np.array([q], np.uint64), np.array([0, cnt[i]], np.int32), f[i, :cnt[i]])
        for k in out:
            out[k].append(r[k])
    return {k: np.concatenate(v) for k, v in out.items()}


def pairs(rng, ids, n, remove):
    """n pairs: a third chains (the previous destination becomes the source), a third are stars into a few hubs."""
    ids = np.asarray(ids)
    hubs = [int(x) for x in ids[:8]]
    dest, src, gone = [], [], set()
    while len(dest) < n:
        k = rng.integers(3)
        if k == 0 and dest:
            c, d = dest[-1], int(ids[rng.integers(len(ids))])
        elif k == 1:
            d, c = hubs[rng.integers(len(hubs))], int(ids[rng.integers(len(ids))])
        else:
            d, c = int(ids[rng.integers(len(ids))]), int(ids[rng.integers(len(ids))])
        if d == c or d in gone or c in gone:
            continue
        dest.append(d)
        src.append(c)
        if remove:
            gone.add(c)
    return dest, src


def emulate(st, dest, src, remove):
    for d, c in zip(dest, src):
        cnt, f = st.fetch([c])
        st.add(np.full(cnt[0], d, np.uint64), f[0, :cnt[0]])
        if remove:
            st.fetch([c], remove=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tracks", type=int, default=20_000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--subset", type=int, default=200)
    ap.add_argument("--pairs", type=int, default=10_000)
    a = ap.parse_args()

    import torch
    import similari_b200.engine as eng

    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    info = card()
    K, D = 3, 512
    st = build_store(a.tracks, K, D)
    ids = st.ids()
    rows = K * len(ids)   # every track holds K observations
    pair_count = rows * len(ids) * K

    # a. the each-mode self-join
    whole = st.search_owned(ids, each=True)   # warm-up, and the reference for b
    times = []
    for _ in range(a.rounds):
        r, t = timed(lambda: st.search_owned(ids, each=True))
        assert same(r, whole)
        times.append(t)
    emit(dict(info, measure="search_owned_each_self_join", tracks=len(ids), K=K, dim=D, pairs=pair_count,
              ms=[round(t * 1e3, 2) for t in times], pairs_per_s=round(pair_count / float(np.median(times)), -7),
              stage_ms=[round(float(x), 2) for x in st.last_stage_ms()]))

    # b. the host path on a subset, alternated with the owned call on the same subset
    rng = np.random.default_rng(3)
    sub = ids[rng.choice(len(ids), a.subset, replace=False)]
    pos = {int(x): i for i, x in enumerate(ids)}
    want = {k: v[[pos[int(x)] for x in sub]] for k, v in whole.items()}
    dev, host = st.search_owned(sub, each=True), host_search(st, sub)
    assert same(dev, want) and same(host, want), "the two paths differ"
    td, th = [], []
    for _ in range(a.rounds):
        td.append(timed(lambda: st.search_owned(sub, each=True))[1])
        th.append(timed(lambda: host_search(st, sub))[1])
    emit(dict(info, measure="owned_search_subset", tracks=len(ids), queries=len(sub), equal=True,
              device_ms_per_query=[round(t * 1e3 / len(sub), 3) for t in td],
              host_ms_per_query=[round(t * 1e3 / len(sub), 3) for t in th]))

    # c. merge_owned against the host emulation, from the same reloaded store
    nbytes = st.save_device(0, 0)
    blob = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    st.save_device(blob.data_ptr(), nbytes)
    for remove, n in ((False, a.pairs), (True, max(1, a.pairs // 10))):
        dest, src = pairs(np.random.default_rng(7 + remove), ids, n, remove)
        g = eng.FeatureStore.load(blob.data_ptr(), nbytes)
        g.merge_owned(dest, src, remove=remove)
        e = eng.FeatureStore.load(blob.data_ptr(), nbytes)
        emulate(e, dest, src, remove)
        assert bytes(g.save()) == bytes(e.save()), "merge_owned differs from the emulation"
        del g, e
        tm, te = [], []
        for _ in range(a.rounds):
            g = eng.FeatureStore.load(blob.data_ptr(), nbytes)
            tm.append(timed(lambda: g.merge_owned(dest, src, remove=remove))[1])
            apply_ms = float(g.last_stage_ms()[2])
            del g
            e = eng.FeatureStore.load(blob.data_ptr(), nbytes)
            te.append(timed(lambda: emulate(e, dest, src, remove))[1])
            del e
        emit(dict(info, measure="merge_owned", tracks=len(ids), pairs=n, remove=remove, blob_equal=True,
                  device_ms=[round(t * 1e3, 2) for t in tm], device_move_kernels_ms=round(apply_ms, 3),
                  host_emulation_ms=[round(t * 1e3, 1) for t in te]))


if __name__ == "__main__":
    main()
