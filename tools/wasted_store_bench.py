"""Wasted tracks into a feature track store: the device call against the host composition, one JSON line per result.

  python tools/wasted_store_bench.py [--scenes 64] [--objects 512] [--dim 512] [--rounds 8] [--gallery 2000]

A BatchVisualSort tracker (kept_history_length 10, max_idle_epochs 1, 10% of the detections dropped per frame so
tracks expire) is fed seeded frames, and two twin euclidean stores (K = 3, topn 1) start from the same gallery.  Each
round (one collection per frame keeps each call within the 2^30-pair bound of one distance matrix) feeds `--frames` frames, clones the tracker (sb200_tracker_load of its blob, untimed: a multi-scene frame appends
its scenes' wasted records in the order their blocks finish, so a second tracker fed the same frames may hold them in
another order) and collects every wasted record once per arm, the original in one and the clone in the other:
  device: FeatureStore.associate_wasted (sb200_fstore_associate_wasted), the history rows never leave the device;
  host:   Tracker.wasted_visual, the present rows of each record gathered in numpy, one FeatureStore.associate.
The arms alternate which goes first.  Each round's outputs (records, counts, winners, f64 weights, track ids, merged)
are compared for equality before its times count, and the store blobs after the last round.  Times are host wall clock
around each arm's calls, which return after their device work is complete.  The PCIe bytes are those the host path
moves, counted from shapes: the history rows and present bytes down (H x d8 x 4 + H per record), the request rows up
(d8 x 4 per kept row).  The card's name, power limit and clock are read in the same run; without a device the script
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


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = [x.strip() for x in out.split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def emit(d):
    print(json.dumps(d), flush=True)


def stats(v):
    return {"median": float(np.median(v)), "min": float(min(v)), "max": float(max(v))}


def host_arm(t, s, H):
    """wasted_visual + one associate of the present rows; returns the per-record outputs and the PCIe bytes."""
    w = t.wasted_visual(history_cap=H)
    n, D = len(w["ids"]), s.D
    rows, offs, qi = [], [0], []
    for i in range(n):
        p = w["feature_present"][i]
        if p.any():
            rows.append(w["features"][i][p][:, :D])
            offs.append(offs[-1] + int(p.sum()))
            qi.append(i)
    out = {"ids": w["ids"], "counts": np.zeros(n, np.int32), "winners": np.zeros((n, s.topn), np.uint64),
           "weights": np.zeros((n, s.topn), np.float64), "track_ids": np.zeros(n, np.uint64),
           "merged": np.zeros(n, np.uint8)}
    kept = 0
    if qi:
        r = s.associate(w["ids"][qi], offs, np.concatenate(rows))
        for k in ("counts", "winners", "weights", "track_ids", "merged"):
            out[k][qi] = r[k]
        kept = int(np.minimum(np.diff(offs), s.K).sum())
    d8 = (D + 7) // 8 * 8
    return out, {"d2h": n * H * (d8 * 4 + 1), "h2d": kept * d8 * 4, "records": n, "queried": len(qi)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", type=int, default=64)
    ap.add_argument("--objects", type=int, default=512)
    ap.add_argument("--dim", type=int, default=512)
    ap.add_argument("--hist", type=int, default=10)
    ap.add_argument("--frames", type=int, default=1)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=8)
    ap.add_argument("--gallery", type=int, default=2000)
    a = ap.parse_args()

    import similari_b200.engine as eng
    from similari_b200._lib import default_options, lib
    from similari_b200.workload import CONFIGS, Workload

    if lib().sb200_device_count() <= 0:
        raise SystemExit("wasted_store_bench needs a CUDA device")
    emit({"card": card()})
    cfg = dataclasses.replace(CONFIGS["cfg5"], n_scenes=a.scenes, n_objects=a.objects, feature_dim=a.dim,
                              drop_frac=0.1, seed=0x5EED5700)
    opts = dict(kind=3, positional_kind=0, iou_threshold=0.3, max_idle_epochs=1, history_length=a.hist, visual_kind=0,
                visual_threshold=0.7, feature_dim=a.dim, visual_max_observations=3, visual_min_votes=1,
                visual_minimal_track_length=1, min_confidence=0.1)
    tracker = eng.Tracker(default_options(**opts))
    tracker.set_feature_history(True)
    stores = [eng.FeatureStore(metric="euclidean", distance_filter=1.0, max_observations=3, feature_dim=a.dim, topn=1,
                               max_distance=1.0, min_votes=1) for _ in range(2)]
    rng = np.random.default_rng(7)
    g = rng.standard_normal((a.gallery, a.dim)).astype(np.float32)
    g /= np.linalg.norm(g, axis=1, keepdims=True)
    for s in stores:
        s.add(np.arange(1 << 40, (1 << 40) + a.gallery, dtype=np.uint64), g)
    wl = Workload(cfg)
    ms = {"device": [], "host": []}
    io = []
    for rnd in range(a.warmup + a.rounds):
        for _ in range(a.frames):
            f = wl.next_frame()
            tracker.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=f["features"])
        trackers = [tracker, eng.Tracker.load(tracker.save())]
        res = {}
        for arm in (("device", "host") if rnd % 2 == 0 else ("host", "device")):
            t, s = trackers[arm == "host"], stores[arm == "host"]
            t.sync()
            t0 = time.perf_counter()
            if arm == "device":
                r = s.associate_wasted(t, history_cap=a.hist)
            else:
                r, b = host_arm(t, s, a.hist)
            res[arm] = (time.perf_counter() - t0) * 1e3, r
        for k in ("ids", "counts", "winners", "track_ids", "merged"):
            if not np.array_equal(res["device"][1][k], res["host"][1][k]):
                raise SystemExit(f"round {rnd}: {k} differs between the arms")
        if not np.array_equal(res["device"][1]["weights"].view(np.uint64), res["host"][1]["weights"].view(np.uint64)):
            raise SystemExit(f"round {rnd}: weights differ between the arms")
        if rnd >= a.warmup:
            ms["device"].append(res["device"][0])
            ms["host"].append(res["host"][0])
            io.append(b)
    if not np.array_equal(stores[0].save(), stores[1].save()):
        raise SystemExit("the store blobs differ between the arms")
    rec = [x["records"] for x in io]
    emit({"config": {"scenes": a.scenes, "objects": a.objects, "dim": a.dim, "kept_history_length": a.hist,
                     "frames_per_collection": a.frames, "gallery": a.gallery, "rounds": a.rounds},
          "records_per_collection": stats(rec), "queried_per_collection": stats([x["queried"] for x in io]),
          "store_size_after": stores[0].size(), "outputs_equal": True})
    emit({"arm": "device", "ms_per_collection": stats(ms["device"])})
    emit({"arm": "host", "ms_per_collection": stats(ms["host"]),
          "pcie_mb_per_collection": {"d2h": stats([x["d2h"] / 1e6 for x in io]),
                                     "h2d": stats([x["h2d"] / 1e6 for x in io])}})


if __name__ == "__main__":
    main()
