"""Live tracks searched in a feature track store: the device call against the host composition, one JSON line per result.

  python tools/feature_store_live_bench.py [--scenes 64] [--objects 512] [--dim 512] [--rounds 8] [--gallery 100000]

A BatchVisualSort tracker (visual_max_observations 5, max_idle_epochs 2) is fed seeded frames, and one euclidean store
(K = 3, topn 1) holds a gallery of `--gallery` tracks with three rows each.  Each round feeds one frame and queries the
tracks that frame created (the re-identification lookup of new tracks; at most 2^30 / (3 x gallery) of them, the
pair bound of one call), once per arm:
  device: FeatureStore.search_tracks (sb200_fstore_search_tracks), the rows never leave the device;
  host:   Tracker.scene_observations of every scene of the frame, the present rows gathered in numpy, one
          FeatureStore.search.
The arms alternate which goes first.  Each round's outputs (counts, winners, f64 weights) are compared for equality
before its times count.  Times are host wall clock around each arm, which returns after its device work is complete.
The PCIe bytes are counted from shapes: the host arm reads whole scenes back (per live track 8 + 4 bytes, and per
observation slot 1 + 4 + 4 x dim bytes) and uploads its request rows (d8 x 4 per kept row); the device arm moves 24
bytes up and 8 down per pair, 4 up per query and request row, and 4 down per row on a quality store (not this one).
The card's name, power limit and clock are read in the same run; without a device the script fails.
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


def host_arm(t, s, scenes, sc, ti):
    """scene_observations of the scenes, the present rows of the pairs, one search; outputs and PCIe bytes."""
    obs = {sid: t.scene_observations(sid) for sid in scenes}
    n, K = len(ti), s.K
    rows, offs, qi = [], [0], []
    where = {(sid, int(i)): j for sid, ob in obs.items() for j, i in enumerate(ob["ids"])}
    for i, (sid, tid) in enumerate(zip(sc, ti)):
        j = where.get((int(sid), int(tid)))
        if j is None:
            continue
        ob = obs[int(sid)]
        p = ob["has_feat"][j, : ob["n_obs"][j]].astype(bool)
        if p.any():
            rows.append(ob["feats"][j, : ob["n_obs"][j]][p])
            offs.append(offs[-1] + int(p.sum()))
            qi.append(i)
    out = {"counts": np.zeros(n, np.int32), "winners": np.zeros((n, s.topn), np.uint64),
           "weights": np.zeros((n, s.topn), np.float64)}
    kept = 0
    if qi:
        r = s.search(ti[qi], offs, np.concatenate(rows))
        for k in out:
            out[k][qi] = r[k]
        kept = int(np.minimum(np.diff(offs), K).sum())
    live = sum(len(ob["ids"]) for ob in obs.values())
    Kt, D = next(iter(obs.values()))["has_feat"].shape[1], s.D
    d8 = (D + 7) // 8 * 8
    return out, {"d2h": live * (12 + Kt * (5 + 4 * D)), "h2d": kept * d8 * 4, "pairs": n, "queried": len(qi),
                 "rows": kept}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", type=int, default=64)
    ap.add_argument("--objects", type=int, default=512)
    ap.add_argument("--dim", type=int, default=512)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=8)
    ap.add_argument("--gallery", type=int, default=100000)
    a = ap.parse_args()

    import similari_b200.engine as eng
    from similari_b200._lib import default_options, lib
    from similari_b200.workload import CONFIGS, Workload

    if lib().sb200_device_count() <= 0:
        raise SystemExit("feature_store_live_bench needs a CUDA device")
    emit({"card": card()})
    cfg = dataclasses.replace(CONFIGS["cfg5"], n_scenes=a.scenes, n_objects=a.objects, feature_dim=a.dim,
                              drop_frac=0.1, seed=0x5EED5800)
    opts = dict(kind=3, positional_kind=0, iou_threshold=0.3, max_idle_epochs=2, visual_kind=0, visual_threshold=0.7,
                feature_dim=a.dim, visual_max_observations=5, visual_min_votes=1, visual_minimal_track_length=1,
                min_confidence=0.1)
    t = eng.Tracker(default_options(**opts))
    s = eng.FeatureStore(metric="euclidean", distance_filter=1.0, max_observations=3, feature_dim=a.dim, topn=1,
                         max_distance=1.0, min_votes=1)
    rng = np.random.default_rng(7)
    ids = np.arange(1 << 40, (1 << 40) + a.gallery, dtype=np.uint64)
    for _ in range(3):
        g = rng.standard_normal((a.gallery, a.dim)).astype(np.float32)
        g /= np.linalg.norm(g, axis=1, keepdims=True)
        s.add(ids, g)
    wl = Workload(cfg)
    ms = {"device": [], "host": []}
    io, stage = [], []
    known = set()
    bound = (1 << 30) // (a.gallery * 3)   # a new track holds one row: pairs = rows x gallery x K within 2^30
    for rnd in range(-1, a.warmup + a.rounds):
        f = wl.next_frame()
        r = t.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=f["features"])
        det_sc = np.repeat(f["scene_ids"], np.diff(f["det_offsets"])).astype(np.uint64)
        new = [(int(sc), int(i)) for sc, i in zip(det_sc, r["ids"]) if (int(sc), int(i)) not in known][:bound]
        known |= {(int(sc), int(i)) for sc, i in zip(det_sc, r["ids"])}
        if rnd < 0:   # the first frame creates every track
            continue
        sc = np.array([p[0] for p in new], np.uint64)
        ti = np.array([p[1] for p in new], np.uint64)
        scenes = sorted(set(map(int, sc)))
        res = {}
        for arm in (("device", "host") if rnd % 2 == 0 else ("host", "device")):
            t.sync()
            t0 = time.perf_counter()
            if arm == "device":
                out = s.search_tracks(t, sc, ti)
            else:
                out, b = host_arm(t, s, scenes, sc, ti)
            res[arm] = (time.perf_counter() - t0) * 1e3, out
            if arm == "device":
                st = s.last_stage_ms()
        for k in ("counts", "winners"):
            if not np.array_equal(res["device"][1][k], res["host"][1][k]):
                raise SystemExit(f"round {rnd}: {k} differs between the arms")
        if not np.array_equal(res["device"][1]["weights"].view(np.uint64), res["host"][1]["weights"].view(np.uint64)):
            raise SystemExit(f"round {rnd}: weights differ between the arms")
        if rnd >= a.warmup:
            ms["device"].append(res["device"][0])
            ms["host"].append(res["host"][0])
            io.append(b)
            stage.append(st)
    pairs = [x["pairs"] for x in io]
    emit({"config": {"scenes": a.scenes, "objects": a.objects, "dim": a.dim, "tracker_K": 5, "store_K": 3,
                     "gallery": a.gallery, "rounds": a.rounds},
          "pairs_per_call": stats(pairs), "rows_per_call": stats([x["rows"] for x in io]), "outputs_equal": True})
    emit({"ms_per_call": {k: stats(v) for k, v in ms.items()},
          "device_stage_ms": {"distance": stats([x[0] for x in stage]), "vote": stats([x[1] for x in stage])},
          "pcie_bytes_per_call": {
              "host": stats([x["d2h"] + x["h2d"] for x in io]),
              "device": stats([24 * x["pairs"] + 8 * x["pairs"] + 4 * (x["queried"] + 1) + 4 * x["queried"]
                               + 4 * x["rows"] for x in io])}})


if __name__ == "__main__":
    main()
