"""The visual screen on e4m3 and on BF16 operands, side by side on one workload (default cfg5).

Two trackers fed the same device-resident frames, alternated frame by frame so that clock and thermal drift hit them
alike: one with SB200_VIS_KERNEL=tc8 (e4m3 screen), one with tc16 (BF16 screen).  Reported per arm: ms/step from CUDA
events, the screen and refine kernel times (the library's counters), survivors per frame and how many of them the exact
test cut (sb200_screen_counters), and the screen's share of the dense tensor peak of its operand type: 2 * M * rows * D
FLOP per frame over the kernel time, against the H100 SXM data sheet's 1979 TFLOP/s (FP8) and 989 TFLOP/s (BF16),
figures for a 700 W card.  The card's name, power limit and clocks are read in the same run.

    python tools/screen_fp8_bench.py [config] [steps] [warmup]
"""
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PEAK = {"tc8": 1979.0, "tc16": 989.0}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    import torch

    import similari_b200.engine as eng
    from similari_b200._lib import default_options
    from similari_b200.workload import CONFIGS, Workload, tracker_options_for

    name = sys.argv[1] if len(sys.argv) > 1 else "cfg5"
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 20
    warmup = int(sys.argv[3]) if len(sys.argv) > 3 else 5
    cfg = CONFIGS[name]
    wl = Workload(cfg)
    frames = []
    for _ in range(steps + warmup):
        f = wl.next_frame()
        frames.append((f, torch.from_numpy(f["boxes"]).cuda(), torch.from_numpy(f["features"]).cuda()))
    hint = dict(max_scenes_hint=cfg.n_scenes, max_tracks_per_scene_hint=4 * cfg.n_objects,
                max_dets_per_scene_hint=cfg.n_objects)
    arms = {m: {"t": eng.Tracker(tracker_options_for(name, default_options, **hint)), "ms": []} for m in ("tc8", "tc16")}
    stream = torch.cuda.current_stream()
    ids = torch.zeros(cfg.n_scenes * cfg.n_objects, dtype=torch.int64, device="cuda")
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for a in arms.values():
        a["t"].set_stream(stream.cuda_stream)
    for i, (f, db, dfe) in enumerate(frames):
        if i == warmup:
            for a in arms.values():
                a["w0"], a["s0"] = a["t"].work_counters(), a["t"].screen_counters()
        for mode, a in arms.items():
            os.environ["SB200_VIS_KERNEL"] = mode
            ev0.record(stream)
            a["t"].predict_batch_device(f["scene_ids"], f["det_offsets"], db.data_ptr(), dfe.data_ptr(), d_ids=ids.data_ptr())
            ev1.record(stream)
            a["t"].sync()
            ev1.synchronize()
            if i >= warmup:
                a["ms"].append(ev0.elapsed_time(ev1))
    out = {"config": name, "card": card(), "steps": steps, "arms": {}}
    D = cfg.feature_dim
    for mode, a in arms.items():
        w1, s1 = a["t"].work_counters(), a["t"].screen_counters()
        w0, s0 = a["w0"], a["s0"]
        tcf = max(1, w1["tc_frames"] - w0["tc_frames"])
        screen_ms = (w1["vis_screen_ms"] - w0["vis_screen_ms"]) / tcf
        dots = (w1["visual_dot_products"] - w0["visual_dot_products"]) / steps
        tflops = 2.0 * dots * D / (screen_ms * 1e-3) / 1e12 if screen_ms > 0 else None
        frames_s = (s1["fp8_frames"] - s0["fp8_frames"]) + (s1["bf16_frames"] - s0["bf16_frames"])
        out["arms"][mode] = {
            "ms_per_step": float(np.median(a["ms"])), "ms_spread": [float(np.min(a["ms"])), float(np.max(a["ms"]))],
            "vis_screen_ms": screen_ms, "vis_refine_ms": (w1["vis_refine_ms"] - w0["vis_refine_ms"]) / tcf,
            "survivors_per_frame": (s1["survivors"] - s0["survivors"]) / max(1, frames_s),
            "cut_per_frame": (s1["cut"] - s0["cut"]) / max(1, frames_s),
            "screen_tflops": tflops, "peak_tflops_datasheet": PEAK[mode],
            "screen_frac_of_peak": tflops / PEAK[mode] if tflops else None,
        }
        a["t"].close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
