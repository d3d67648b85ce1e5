"""FP16 / BF16 feature columns against f32 on the cfg5 workload (BatchVisualSort, 256 scenes x 512 objects, D = 512).

Two paths, each with the features as f32, f16 (numpy astype) and bf16 (torch), the three types alternated round by round
in one process so that clock and thermal drift hit them alike:
  host   : pinned host columns, sb200_prefetch_inputs of frame i + 1 + sb200_predict_batch_async of frame i (bench.py's
           end-to-end loop); the features cross PCIe at their own element size.
  device : the columns already in HBM, one sb200_predict_batch_device per step, stream-ordered.
Reported per path and type: ms/step (CUDA events around the timed steps, then a device synchronise) as the mean over the
rounds with its min / max.  A separate run under torch.profiler gives the per-call device times of cand_norm_kernel and
feat_store_kernel, the two kernels that read whole feature rows.  Before timing, every f16 / bf16 tracker is checked frame
by frame against an f32 tracker fed the widened copy of its own features (ids, epochs, lengths, voting types, both boxes).

    python tools/feature_type_bench.py [steps] [warmup] [rounds]
"""
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

TYPES = ("f32", "f16", "bf16")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    import torch

    import similari_b200.engine as eng
    from similari_b200._lib import default_options, pinned_empty
    from similari_b200.workload import CONFIGS, Workload, tracker_options_for

    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    warmup = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    rounds = int(sys.argv[3]) if len(sys.argv) > 3 else 3
    if torch.cuda.device_count() == 0:
        raise SystemExit("feature_type_bench needs a CUDA device")
    cfg = CONFIGS["cfg5"]
    wl = Workload(cfg)
    n = warmup + steps + 1   # the host loop prefetches one frame ahead
    frames = [wl.next_frame() for _ in range(n)]
    D = cfg.feature_dim

    # the three columns of every frame: as sent (host pinned, device) and the exact f32 widening of the sent values
    col = {t: [] for t in TYPES}
    for f in frames:
        x = f["features"]
        tb = torch.from_numpy(x).to(torch.bfloat16)
        col["f32"].append((x, x))
        h = x.astype(np.float16)
        col["f16"].append((h, h.astype(np.float32)))
        col["bf16"].append((tb.view(torch.int16).numpy().view(np.uint16).copy(), tb.float().numpy()))
    host = {t: [] for t in TYPES}
    dev = {t: [] for t in TYPES}
    for t in TYPES:
        for f, (a, _) in zip(frames, col[t]):
            b = pinned_empty(f["boxes"].shape, np.float32)
            b[...] = f["boxes"]
            p = pinned_empty(a.shape, a.dtype)
            p[...] = a
            host[t].append((b, p))
            dev[t].append((torch.from_numpy(f["boxes"]).cuda(), torch.from_numpy(a.view(np.int16) if a.dtype != np.float32
                                                                                   else a).cuda()))
    dboxes = [d[0] for d in dev["f32"]]
    max_total = cfg.n_scenes * cfg.n_objects
    stream = torch.cuda.current_stream()

    def new_tracker():
        t = eng.Tracker(tracker_options_for("cfg5", default_options, max_scenes_hint=cfg.n_scenes,
                                            max_tracks_per_scene_hint=4 * cfg.n_objects,
                                            max_dets_per_scene_hint=cfg.n_objects))
        t.set_stream(stream.cuda_stream)
        return t

    # ---- outputs: each narrow type against f32 fed its widened copy, at the timed size, every frame
    cols = ("ids", "epochs", "lengths", "voting_types", "predicted", "observed")
    checked = 0
    for t in ("f16", "bf16"):
        a, b = new_tracker(), new_tracker()
        for i, f in enumerate(frames):
            ra = a.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=col[t][i][0], feature_type=t)
            rb = b.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=col[t][i][1])
            for k in cols:
                assert ra[k].tobytes() == rb[k].tobytes(), f"{t}: frame {i}: {k} differs from the widened f32 run"
            checked += len(f["boxes"])
        a.close()
        b.close()

    # ---- timing
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    res = {p: {t: [] for t in TYPES} for p in ("host", "device")}
    ring = [{"ids": pinned_empty((max_total,), np.uint64), "lengths": pinned_empty((max_total,), np.uint32),
             "predicted": pinned_empty((max_total, 6), np.float32)} for _ in range(5)]

    def run_host(t):
        tr = new_tracker()
        ft = None if t == "f32" else t
        tr.prefetch_inputs(host[t][0][0], features=host[t][0][1], feature_type=ft)
        for i in range(warmup + steps):
            f = frames[i]
            if i == warmup:
                tr.sync()
                torch.cuda.synchronize()
                ev0.record()
            out = {k: v[: len(f["boxes"])] for k, v in ring[i % 5].items()}
            tr.prefetch_inputs(host[t][i + 1][0], features=host[t][i + 1][1], feature_type=ft)
            tr.predict_batch(f["scene_ids"], f["det_offsets"], host[t][i][0], features=host[t][i][1], out=out, wait=False,
                             feature_type=ft)
        tr.sync()
        torch.cuda.synchronize()
        ev1.record()
        ev1.synchronize()
        tr.close()
        return ev0.elapsed_time(ev1) / steps

    def run_device(t, n_steps=steps, n_warm=warmup):
        tr = new_tracker()
        tr.set_stream(stream.cuda_stream, join_per_call=False)
        ids = torch.zeros(max_total, dtype=torch.int64, device="cuda")
        for i in range(n_warm + n_steps):
            f = frames[i]
            if i == n_warm:
                tr.sync()
                torch.cuda.synchronize()
                ev0.record()
            tr.predict_batch_device(f["scene_ids"], f["det_offsets"], dboxes[i].data_ptr(), dev[t][i][1].data_ptr(),
                                    d_ids=ids.data_ptr(), feature_type=t)
        tr.stream_join(stream.cuda_stream)
        ev1.record()
        ev1.synchronize()
        tr.sync()
        tr.close()
        return ev0.elapsed_time(ev1) / n_steps

    for r in range(rounds):
        order = TYPES if r % 2 == 0 else TYPES[::-1]
        for t in order:
            res["host"][t].append(run_host(t))
        for t in order:
            res["device"][t].append(run_device(t))

    # ---- kernel times under the profiler (a run of its own)
    from torch.profiler import ProfilerActivity, profile

    kern = {}
    for t in TYPES:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            run_device(t, n_steps=4, n_warm=0)
        for e in prof.key_averages():
            for k in ("cand_norm_kernel", "feat_store_kernel"):
                if k in e.key:
                    d = kern.setdefault(t, {}).setdefault(k, [0.0, 0])
                    d[0] += e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
                    d[1] += e.count
    kernels_us = {t: {k: round(v[0] / max(1, v[1]), 1) for k, v in d.items()} for t, d in kern.items()}

    stat = lambda v: {"mean": round(float(np.mean(v)), 4), "min": round(float(np.min(v)), 4),  # noqa: E731
                      "max": round(float(np.max(v)), 4)}
    total = int(np.mean([len(f["boxes"]) for f in frames]))
    out = {"card": card(), "config": "cfg5 BatchVisualSort 256 scenes x 512 objects, D = 512", "steps": steps,
           "warmup": warmup, "rounds": rounds, "checked_detections": checked,
           "feature_mb_per_frame": {t: round(total * D * (4 if t == "f32" else 2) / 1e6, 1) for t in TYPES},
           "ms_per_step": {p: {t: stat(v) for t, v in d.items()} for p, d in res.items()},
           "kernel_us_per_call": kernels_us}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
