"""Feature track store I/O timings (typed and device-resident feature columns, the store blob): one JSON line per
measurement.

  python tools/feature_store_io_bench.py [--rounds N] [--profile]

1. `search` per call with the same query values sent three ways -- f32 host, f16 host, f16 device-resident -- alternated
   in one process over several rounds (median of each round's calls; the line reports the median and range of the rounds).
   Two sizes: the gallery of DESIGN 3d (1024 single-observation queries against 100,000 tracks x K = 3 x 512-d) and the
   500-object feature-tracker loop (500 queries against 500 tracks x K = 3 x 256-d).  The three results are compared for
   equality before anything is timed.
2. `save` / `load` of the gallery to a device blob and to a pageable host blob: host wall clock (the calls return when
   the copy is complete).
3. With --profile (a run of its own: tracing slows the host): device time of the blob's copy kernel (xfer_copy_kernel)
   under torch.profiler during one save and one load to a device blob, against the HBM bound of the rows it moves
   (bytes read + bytes written over the H100 SXM data sheet's 3.35 TB/s, a 700 W figure).
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

HBM_BYTES_PER_S = 3.35e12


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


def search_paths(st, queries, dim, rounds, calls, info, label):
    import torch

    rng = np.random.default_rng(1)
    q16 = rng.standard_normal((queries, dim)).astype(np.float16)
    q32 = q16.astype(np.float32)
    dq = torch.from_numpy(q16).cuda()
    torch.cuda.synchronize()
    qid = np.arange(10**9, 10**9 + queries, dtype=np.uint64)
    offs = np.arange(queries + 1, dtype=np.int32)

    def f32_host():
        return st.search(qid, offs, q32)

    def f16_host():
        return st.search(qid, offs, q16)

    def f16_device():
        st.set_feature_type("f16")
        r = st.search_device(qid, offs, dq.data_ptr())
        st.set_feature_type("f32")
        return r

    paths = {"f32_host": f32_host, "f16_host": f16_host, "f16_device": f16_device}
    ref = f32_host()
    for name, fn in paths.items():   # warm-up of every path, and the three must agree exactly
        r = fn()
        for k in ref:
            if not np.array_equal(r[k].view(np.uint64) if r[k].dtype == np.float64 else r[k],
                                  ref[k].view(np.uint64) if ref[k].dtype == np.float64 else ref[k]):
                raise SystemExit(f"{label}: {name} differs from f32_host in {k}")
    per_round = {name: [] for name in paths}
    for _ in range(rounds):
        for name, fn in paths.items():
            ts = []
            for _ in range(calls):
                t0 = time.perf_counter()
                fn()
                ts.append((time.perf_counter() - t0) * 1e3)
            per_round[name].append(float(np.median(ts)))
    emit({"bench": "search_paths", "size": label, "queries": queries, "tracks": st.size(), "K": st.K, "dim": dim,
          "rounds": rounds, "calls_per_round": calls, **info,
          "ms_per_call": {name: {"median": float(np.median(v)), "min": min(v), "max": max(v)}
                          for name, v in per_round.items()},
          "request_bytes": {"f32_host": queries * dim * 4, "f16_host": queries * dim * 2, "f16_device": 0}})


def blob_times(st, reps, info):
    import torch

    import similari_b200.engine as eng

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
        if st._L.sb200_fstore_save(st._h, hblob.ctypes.data, n, C.byref(C.c_uint64(0))) != 0:   # into the array that exists
            raise SystemExit("save to the host blob failed")
        t4 = time.perf_counter()
        c = eng.FeatureStore.load(hblob)
        t5 = time.perf_counter()
        c.close()
        for k, v in zip(res, (t1 - t0, t2 - t1, t4 - t3, t5 - t4)):
            res[k].append(v * 1e3)
    if not np.array_equal(dblob.cpu().numpy(), hblob):
        raise SystemExit("the device blob and the host blob differ")
    rows = st.size() * st.K * ((st.D + 7) // 8 * 8) * 4
    emit({"bench": "blob_wall", "tracks": st.size(), "K": st.K, "dim": st.D, "blob_bytes": n, "row_bytes": rows,
          "reps": reps, **info,
          "ms": {k: {"median": float(np.median(v[1:])), "min": min(v[1:]), "max": max(v[1:])} for k, v in res.items()}})


def blob_profile(st, info):
    import torch
    from torch.profiler import ProfilerActivity, profile

    import similari_b200.engine as eng

    n = st.save_device(0, 0)
    dblob = torch.empty(n, dtype=torch.uint8, device="cuda")
    st.save_device(dblob.data_ptr(), n)   # warm-up
    eng.FeatureStore.load(dblob.data_ptr(), n).close()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        st.save_device(dblob.data_ptr(), n)
        c = eng.FeatureStore.load(dblob.data_ptr(), n)
        torch.cuda.synchronize()
    c.close()
    kernels = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and "kernel" in e.name:
            name = next((k for k in ("xfer_copy_kernel", "fs_blob_scrub_kernel", "fs_class_check_kernel") if k in e.name),
                        e.name)
            kernels.setdefault(name, []).append(e.device_time if hasattr(e, "device_time") else e.cuda_time)
    copy_us = [v for k, v in kernels.items() if "xfer_copy_kernel" in k]
    if not copy_us or len(copy_us[0]) != 2:
        raise SystemExit(f"expected two launches of xfer_copy_kernel in the trace, found {kernels}")
    moved = sum(st.size() * w for w in (8, 4, 4, st.K * ((st.D + 7) // 8 * 8) * 4))
    bound_us = 2 * moved / HBM_BYTES_PER_S * 1e6
    emit({"bench": "blob_copy_kernel", "tracks": st.size(), "K": st.K, "dim": st.D, "bytes_read_plus_written": 2 * moved,
          **info, "xfer_copy_kernel_us": {"save": copy_us[0][0], "load": copy_us[0][1]},
          "hbm_bound_us_at_3.35TB/s": bound_us,
          "fraction_of_hbm_bound": {"save": bound_us / copy_us[0][0], "load": bound_us / copy_us[0][1]},
          "other_kernels_us": {k: v for k, v in kernels.items() if "xfer_copy_kernel" not in k}})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--profile", action="store_true", help="only the copy kernel's time under torch.profiler")
    ap.add_argument("--tracks", type=int, default=100_000)
    a = ap.parse_args()
    from similari_b200._lib import lib

    if lib().sb200_device_count() <= 0:
        raise SystemExit("feature_store_io_bench needs a CUDA device")
    info = card()
    gallery = build_store(a.tracks, 3, 512)
    if a.profile:
        blob_profile(gallery, info)
        return
    search_paths(gallery, 1024, 512, a.rounds, 3, info, "gallery")
    loop = build_store(500, 3, 256, seed=2)
    search_paths(loop, 500, 256, a.rounds, 200, info, "tracker_loop_500")
    loop.close()
    blob_times(gallery, 3, info)


if __name__ == "__main__":
    main()
