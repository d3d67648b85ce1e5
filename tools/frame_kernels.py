#!/usr/bin/env python
"""Per-kernel device time of steady-state frames of a BASELINE config, from torch.profiler (CUPTI kernel records):
    python tools/frame_kernels.py cfg5 [--warm 9] [--frames 5] [--visual-threshold max] [--csv out.csv]
Inputs are resident in HBM, as in bench.py's device-timed arm.  After the warm-up, the given number of frames run
under the profiler, each followed by a synchronise; the table lists, per kernel name, the launches and the device
time per frame (mean over the profiled frames), the sum of kernel time, and the wall time per frame with the
profiler on (tracing slows the host: take end-to-end times from bench.py)."""
import argparse
import os
import re
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def short(name: str) -> str:
    """A kernel's name without its argument list; template arguments stay (they tell the element types apart)."""
    depth, out = 0, []
    for ch in name:
        if ch == "(" and depth == 0:
            break
        if ch == "<":
            depth += 1
        elif ch == ">":
            depth -= 1
        out.append(ch)
    s = "".join(out).replace("void ", "").replace("sb::", "")
    return re.sub(r"\s+", " ", s).strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("config", nargs="?", default="cfg5")
    ap.add_argument("--warm", type=int, default=9)
    ap.add_argument("--frames", type=int, default=5)
    ap.add_argument("--visual-threshold", default=None)
    ap.add_argument("--csv", default=None)
    a = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    import similari_b200.engine as eng
    from similari_b200._lib import default_options
    from similari_b200.workload import CONFIGS, Workload, tracker_options_for

    over = {}
    if a.visual_threshold is not None:
        over["visual_threshold"] = 3.402823466e38 if a.visual_threshold == "max" else float(a.visual_threshold)
    cfg = CONFIGS[a.config]
    dev = torch.device("cuda", 0)
    t = eng.Tracker(tracker_options_for(a.config, default_options, max_scenes_hint=cfg.n_scenes,
                                        max_tracks_per_scene_hint=4 * cfg.n_objects, max_dets_per_scene_hint=cfg.n_objects, **over))
    t.set_stream(torch.cuda.current_stream().cuda_stream)
    wl = Workload(cfg)
    d_ids = torch.zeros(cfg.n_scenes * cfg.n_objects, dtype=torch.int64, device=dev)
    frames = []
    for _ in range(a.warm + a.frames):   # inputs of every frame resident before the first one runs
        f = wl.next_frame()
        db = torch.from_numpy(np.ascontiguousarray(f["boxes"])).to(dev)
        df = torch.from_numpy(f["features"]).to(dev) if f["features"] is not None else None
        frames.append((f, db, df))
    torch.cuda.synchronize()

    def run(fr):
        f, db, df = fr
        t.predict_batch_device(f["scene_ids"], f["det_offsets"], db.data_ptr(), df.data_ptr() if df is not None else 0,
                               d_ids=d_ids.data_ptr())
        t.sync()

    for fr in frames[:a.warm]:
        run(fr)
    l0 = eng.launch_count()
    wall = []
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for fr in frames[a.warm:]:
            w0 = time.perf_counter()
            run(fr)
            wall.append(time.perf_counter() - w0)
    launches = (eng.launch_count() - l0) / a.frames

    rows = {}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        r = rows.setdefault(short(e.name), [0, 0.0])
        r[0] += 1
        r[1] += e.time_range.elapsed_us()
    items = sorted(rows.items(), key=lambda kv: -kv[1][1])
    tot = sum(v[1] for _, v in items) / a.frames
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:   # the table is still useful without the card's settings
        pl = f"unavailable ({ex})"
    wc = t.work_counters()
    print(f"{a.config} {'visual_threshold=' + a.visual_threshold if a.visual_threshold else ''} on {name} "
          f"(power limit, max SM clock: {pl}); {a.frames} frames after {a.warm}; launches per frame (sb200): {launches:.2f}; "
          f"tc_frames {wc['tc_frames']} of {wc['frames']}")
    print(f"| kernel | launches/frame | us/frame |\n|---|---|---|")
    for n, (c, us) in items:
        print(f"| `{n}` | {c / a.frames:.2f} | {us / a.frames:.1f} |")
    print(f"| sum of kernel time | | {tot:.1f} |")
    print(f"wall time per frame, profiler on: {1e3 * np.mean(wall):.3f} ms (min {1e3 * np.min(wall):.3f})")
    if a.csv:
        os.makedirs(os.path.dirname(os.path.abspath(a.csv)), exist_ok=True)
        with open(a.csv, "w") as fo:
            fo.write("kernel,launches_per_frame,us_per_frame\n")
            for n, (c, us) in items:
                fo.write(f"\"{n}\",{c / a.frames:.3f},{us / a.frames:.2f}\n")


if __name__ == "__main__":
    main()
