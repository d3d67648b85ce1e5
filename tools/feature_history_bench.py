"""Cost of the feature history on the cfg5 workload (BatchVisualSort, 256 scenes x 512 objects, D = 512).

Four arms in one process, alternated frame by frame so that clock and thermal drift hit them alike: feature history off
and on at history_length H = 1, and off and on at H = 10.  The off and on arms of one H differ only in the feature history
(the box history is the same), so their difference is its cost.  Each arm is a tracker fed the same device-resident frames
through predict_batch_device; every `collect` frames (outside the timed region) each arm collects its wasted tracks, as a
caller following the reference's advice does.  Reported per arm: ms/step from CUDA events, kernel launches per step; for
the on arms the pool's allocated bytes, the bytes of the blocks in use, and the extra algorithmic HBM traffic per step
(M * d8 * 4 bytes of history rows plus M present bytes, M = detections).  Then the time of one wasted_visual()
collection of 10^4 records.

    python tools/feature_history_bench.py [steps] [warmup] [collect]
"""
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    import torch

    import similari_b200.engine as eng
    from similari_b200._lib import default_options
    from similari_b200.workload import CONFIGS, Workload, tracker_options_for

    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    warmup = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    collect = int(sys.argv[3]) if len(sys.argv) > 3 else 5
    cfg = CONFIGS["cfg5"]
    wl = Workload(cfg)
    frames = []
    for _ in range(steps + warmup):
        f = wl.next_frame()
        frames.append((f, torch.from_numpy(f["boxes"]).cuda(), torch.from_numpy(f["features"]).cuda()))
    hint = dict(max_scenes_hint=cfg.n_scenes, max_tracks_per_scene_hint=2 * cfg.n_objects,
                max_dets_per_scene_hint=cfg.n_objects)
    arms = {}
    for H in (1, 10):
        for on in (False, True):
            t = eng.Tracker(tracker_options_for("cfg5", default_options, history_length=H, **hint))
            if on:
                t.set_feature_history(True)
            arms[f"H={H} {'on' if on else 'off'}"] = {"t": t, "ms": [], "launches": [], "H": H, "on": on}
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ids = torch.zeros(cfg.n_scenes * cfg.n_objects, dtype=torch.int64, device="cuda")
    stream = torch.cuda.current_stream()
    for name, a in arms.items():
        a["t"].set_stream(stream.cuda_stream)
    for i, (f, db, dfe) in enumerate(frames):
        for name, a in arms.items():
            t = a["t"]
            l0 = eng.launch_count()
            ev0.record(stream)
            t.predict_batch_device(f["scene_ids"], f["det_offsets"], db.data_ptr(), dfe.data_ptr(), d_ids=ids.data_ptr())
            ev1.record(stream)
            t.sync()
            ev1.synchronize()
            if i >= warmup:
                a["ms"].append(ev0.elapsed_time(ev1))
                a["launches"].append(eng.launch_count() - l0)
        if (i + 1) % collect == 0:
            for a in arms.values():
                if a["on"]:
                    a["t"].wasted_visual()   # drains every record
                else:
                    while len(a["t"].wasted_history()["ids"]):
                        pass
    M = float(np.mean([int(f["det_offsets"][-1]) for f, _, _ in frames]))
    d8 = (cfg.feature_dim + 7) // 8 * 8
    res = {"card": card(), "steps": steps, "warmup": warmup, "arms": {}}
    for name, a in arms.items():
        r = {"ms_per_step_median": float(np.median(a["ms"])), "ms_per_step_min": float(np.min(a["ms"])),
             "launches_per_step": sorted(set(a["launches"]))}
        r["live_tracks"] = a["t"].active_tracks()
        if a["on"]:
            pool = a["t"].feature_history_pool()
            r["pool_blocks"] = pool
            r["pool_bytes"] = pool["capacity"] * a["H"] * (4 * d8 + 1)
            r["pool_bytes_in_use"] = (pool["handed_out"] - pool["free"]) * a["H"] * (4 * d8 + 1)
            r["extra_hbm_bytes_per_step"] = M * (d8 * 4 + 1)
        res["arms"][name] = r
    # one collection of 10^4 records: the H = 10 arm's tracks expire (skip_epochs), then wasted_visual() drains them
    t = arms["H=10 on"]["t"]
    t.wasted_visual()   # empty the bin first
    per_scene = -(-10000 // cfg.n_objects)
    for s in range(per_scene):
        t.skip_epochs(10, int(f["scene_ids"][s]))
    t.sync()
    t0 = time.perf_counter()
    w = t.wasted_visual()
    res["collect_records"] = int(len(w["ids"]))
    res["collect_ms"] = (time.perf_counter() - t0) * 1e3
    print(json.dumps(res))


if __name__ == "__main__":
    main()
