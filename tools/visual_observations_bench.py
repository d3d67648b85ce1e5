"""How the visual frame scales with the observations kept per track (visual_max_observations = K).

cfg5's shape (BatchVisualSort, 256 scenes x 512 objects, D = 512) under the options of the reference's
python/visual_sort/batch_visual_sort.py example (Euclidean(0.7), Mahalanobis positional metric, minimal track length 7,
minimal area 5, quality gates 0.45 / 0.5, 5 votes, 15 idle epochs), for K in {3, 5, 8, 16, 25, 32} on the three visual
paths: e4m3 screen (SB200_VIS_KERNEL=tc8), BF16 screen (tc16) and the dense path (a threshold that cuts nothing,
f32::MAX, as --visual-threshold max does in bench.py).  Each (K, path) arm is a fresh tracker fed the same seeded,
device-resident frames through predict_batch_device; the first `warmup` frames fill the observation lists and are not
timed.  Reported per arm: ms / frame (CUDA events, median and minimum), the median of last_stage_ms() per stage, the
live tracks at the end, and the feature-arena bytes of one track block (f32, BF16 and e4m3 rows, norms, scales, and the
three per-observation columns).  The card's name, power limit and maximum SM clock are read in the same run.

    python tools/visual_observations_bench.py [steps] [warmup] [K,K,...]
"""
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PATHS = {"e4m3": ("tc8", None), "bf16": ("tc16", None), "dense": (None, 3.402823466e38)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def arena_bytes_per_track(K, d8):
    fp8_pitch = (d8 + 15) // 16 * 16
    return K * (4 * d8 + 2 * d8 + (fp8_pitch if d8 <= 512 else 0) + 4 + 4) + K * (1 + 1 + 4)


def main():
    import torch

    import similari_b200.engine as eng
    from similari_b200._lib import KIND_BATCH_VISUAL_SORT, POS_MAHA, VIS_EUCLIDEAN, Sb200Error, default_options, lib
    from similari_b200.workload import CONFIGS, Workload

    if lib().sb200_device_count() <= 0:
        raise SystemExit("visual_observations_bench needs a CUDA device")
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    warmup = int(sys.argv[2]) if len(sys.argv) > 2 else 24
    ks = [int(k) for k in sys.argv[3].split(",")] if len(sys.argv) > 3 else [3, 5, 8, 16, 25, 32]
    cfg = CONFIGS["cfg5"]
    wl = Workload(cfg)
    frames = []
    for _ in range(steps + warmup):
        f = wl.next_frame()
        frames.append((f, torch.from_numpy(f["boxes"]).cuda(), torch.from_numpy(f["features"]).cuda()))
    d8 = (cfg.feature_dim + 7) // 8 * 8
    example = dict(kind=KIND_BATCH_VISUAL_SORT, feature_dim=cfg.feature_dim, max_idle_epochs=15, history_length=25,
                   visual_kind=VIS_EUCLIDEAN, visual_threshold=0.7, positional_kind=POS_MAHA,
                   visual_minimal_track_length=7, visual_minimal_area=5.0, visual_minimal_quality_use=0.45,
                   visual_minimal_quality_collect=0.5, visual_min_votes=5, max_scenes_hint=cfg.n_scenes,
                   max_dets_per_scene_hint=cfg.n_objects)
    stream = torch.cuda.current_stream()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ids = torch.zeros(cfg.n_scenes * cfg.n_objects, dtype=torch.int64, device="cuda")
    res = {"card": card(), "shape": [cfg.n_scenes, cfg.n_objects, cfg.n_objects, cfg.feature_dim], "steps": steps,
           "warmup": warmup, "arms": []}
    for K in ks:
        for path, (env, thr) in PATHS.items():
            if env:
                os.environ["SB200_VIS_KERNEL"] = env
            else:
                os.environ.pop("SB200_VIS_KERNEL", None)
            kw = dict(example, visual_max_observations=K)
            if thr is not None:
                kw["visual_threshold"] = thr
            t = eng.Tracker(default_options(**kw))
            t.set_stream(stream.cuda_stream)
            ms, stages = [], []
            try:
                for i, (f, db, dfe) in enumerate(frames):
                    ev0.record(stream)
                    t.predict_batch_device(f["scene_ids"], f["det_offsets"], db.data_ptr(), dfe.data_ptr(),
                                           d_ids=ids.data_ptr())
                    ev1.record(stream)
                    t.sync()
                    ev1.synchronize()
                    if i >= warmup:
                        ms.append(ev0.elapsed_time(ev1))
                        stages.append(t.last_stage_ms())
            except Sb200Error as e:   # e.g. the store outgrowing device memory: this arm is not measured
                res["arms"].append({"K": K, "path": path, "not_measured": str(e)})
                print(json.dumps(res["arms"][-1]), flush=True)
                del t
                continue
            wc = t.work_counters()
            res["arms"].append({
                "K": K, "path": path, "ms_per_frame_median": float(np.median(ms)), "ms_per_frame_min": float(np.min(ms)),
                "stage_ms_median": {k: float(np.median([s[k] for s in stages])) for k in stages[0]},
                "live_tracks": t.active_tracks(), "arena_bytes_per_track": arena_bytes_per_track(K, d8),
                "tc_frames": wc["tc_frames"], "dense_fallback_scenes": wc["dense_fallback_scenes"]})
            print(json.dumps(res["arms"][-1]), flush=True)
            del t
    os.environ.pop("SB200_VIS_KERNEL", None)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
