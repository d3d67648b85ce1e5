#!/usr/bin/env python
"""Times the point Kalman filter, the box filter's distance and the intersection-area matrix on the GPU.

Workloads: Vec2DKalmanFilter predict + update on 2^20 points; Universal2DBoxKalmanFilter distance on 2^20 (state, box)
pairs; intersection_areas of 4096 x 4096 oriented boxes (1920 x 1080 scene, heights 40-160 px).  Each is timed as the
host call (wall clock, median of `reps`; inputs and outputs are host arrays, so the PCIe copies and the per-call
allocations are inside) and as kernel time (torch.profiler with CUDA activities over `reps` host calls after a warm-up;
the device time of the named kernel divided by the number of calls).  For each kernel it prints the FLOPs and bytes the
shapes imply and the bound (HBM or FP64) that the data sheet rates would put on it; the intersection FLOPs are counted
by replaying the clip on a sample of pairs.  One per-object call, Universal2DBoxKalmanFilter.predict on one state, is
timed as well.  Needs a GPU; prints one JSON object.

usage: geom_kalman_bench.py [reps]"""
import json
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, __file__.rsplit("/tools/", 1)[0])
import similari_b200.api as api  # noqa: E402
import similari_b200.engine as eng  # noqa: E402

HBM_BPS = 3.35e12     # H100 SXM data sheet, HBM3
FP64_FLOPS = 34e12    # H100 SXM data sheet, FP64 (non-tensor)
FP32_FLOPS = 67e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def host_ms(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return 1e3 * float(np.median(ts)), 1e3 * float(min(ts))


def kernel_ms(fn, reps, names):
    """Mean device time per call of the kernels whose names contain one of `names` (torch.profiler, CUDA activity)."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    tot = {n: 0.0 for n in names}
    cnt = {n: 0 for n in names}
    for e in prof.events():
        for n in names:
            if n in e.name and e.device_type.name == "CUDA":
                tot[n] += e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
                cnt[n] += 1
    return {n: (tot[n] / 1e3 / reps if cnt[n] else None) for n in names}, cnt


def bound(flops, nbytes, peak_flops, label):
    t_mem, t_alu = nbytes / HBM_BPS, flops / peak_flops
    return {"flops": flops, "bytes": nbytes, "min_us_hbm": 1e6 * t_mem, f"min_us_{label}": 1e6 * t_alu,
            "bound": "HBM" if t_mem >= t_alu else label.upper()}


def clip_flops(s, c):
    """FP64 operations of one clip_poly pass sequence + shoelace on vertex arrays s, c ([4][2]), as sb_math.cuh runs it:
    2 per clip edge, 5 per inside test, 22 per intersection (one division counted as one), 6 per shoelace term + 2."""
    poly = [tuple(p) for p in s]
    f = 0
    for i in range(4):
        c1, c2 = c[i - 1], c[i]
        ex, ey = c2[0] - c1[0], c2[1] - c1[1]
        f += 2
        if not poly:
            continue
        inside = [ex * (q[1] - c1[1]) - ey * (q[0] - c1[0]) <= 0.0 for q in poly]
        f += 5 * (len(poly) + 1)
        out = []
        for j, q in enumerate(poly):
            p, p_in, q_in = poly[j - 1], inside[j - 1], inside[j]
            if q_in != p_in:
                f += 22
                dcx, dcy = p[0] - q[0], p[1] - q[1]
                dpx, dpy = c1[0] - c2[0], c1[1] - c2[1]
                n1, n2 = p[0] * q[1] - p[1] * q[0], c1[0] * c2[1] - c1[1] * c2[0]
                n3 = 1.0 / (dcx * dpy - dcy * dpx)
                out.append(((n1 * dpx - n2 * dcx) * n3, (n1 * dpy - n2 * dcy) * n3))
            if q_in:
                out.append(q)
        poly = out
    if len(poly) >= 3:
        f += 6 * len(poly) + 2
    return f


def main():
    import torch

    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    res = {"card": card(), "torch_device": torch.cuda.get_device_name(0)}
    r = np.random.default_rng(0x6E0)

    # -------- Vec2DKalmanFilter predict + update, 2^20 points
    n = 1 << 20
    pts = np.stack([r.uniform(0, 1920, n), r.uniform(0, 1080, n)], 1).astype(np.float32)
    f = api.Vec2DKalmanFilter()
    st = f.initiate(pts)
    pts_list = pts  # the API takes any (x, y) sequence; a [n][2] array avoids building 2^20 tuples

    def vec_step():
        return f.update(f.predict(st), pts_list)

    h = host_ms(vec_step, reps)
    k, _ = kernel_ms(vec_step, reps, ["point_kalman_kernel"])
    kp = k["point_kalman_kernel"]
    res["vec2d_predict_update"] = {
        "n": n, "host_ms_median": h[0], "host_ms_min": h[1],
        "kernel_ms_predict_plus_update": kp,
        **bound(n * (18 + 38), n * (96 + 104), FP32_FLOPS, "fp32")}
    if kp:
        res["vec2d_predict_update"]["achieved_hbm_TBps"] = n * 200 / (kp * 1e-3) / 1e12

    # -------- box filter distance, 2^20 pairs
    boxes = np.stack([r.uniform(0, 1920, n), r.uniform(0, 1080, n), np.full(n, np.nan), r.uniform(0.3, 0.8, n),
                      r.uniform(40, 160, n), np.ones(n)], 1).astype(np.float32)
    states = eng.kalman_predict(eng.kalman_initiate(boxes))
    z = boxes.copy()
    z[:, :2] += r.normal(0, 3, (n, 2)).astype(np.float32)
    h = host_ms(lambda: eng.kalman_distance(states, z), reps)
    k, _ = kernel_ms(lambda: eng.kalman_distance(states, z), reps, ["kalman_distance_kernel"])
    kd = k["kalman_distance_kernel"]
    res["box_distance"] = {"n": n, "host_ms_median": h[0], "host_ms_min": h[1], "kernel_ms": kd,
                           **bound(n * 44, n * (120 + 24 + 4), FP32_FLOPS, "fp32")}
    if kd:
        res["box_distance"]["achieved_hbm_TBps"] = n * 148 / (kd * 1e-3) / 1e12

    # -------- intersection areas, 4096 x 4096
    m = 4096
    a = np.stack([r.uniform(0, 1920, m), r.uniform(0, 1080, m), r.uniform(-1.5, 1.5, m), r.uniform(0.3, 0.8, m),
                  r.uniform(40, 160, m), np.ones(m)], 1).astype(np.float32)
    b = a[r.permutation(m)].copy()
    ireps = max(3, reps // 4)
    h = host_ms(lambda: eng.intersection_areas(a, b), ireps)
    subj = [api.Universal2DBox(*row[:5]) for row in a]
    clip = [api.Universal2DBox(*row[:5]) for row in b]
    h_api = host_ms(lambda: api.intersection_areas(subj, clip), ireps)
    k, _ = kernel_ms(lambda: eng.intersection_areas(a, b), ireps, ["intersection_areas_kernel", "box_vertices_kernel"])
    ki = k["intersection_areas_kernel"]
    va, vb = eng.box_vertices(a), eng.box_vertices(b)
    sample = r.integers(0, m, (4000, 2))
    per_pair = float(np.mean([clip_flops(va[i], vb[j]) for i, j in sample]))
    flops = per_pair * m * m
    res["intersection_areas"] = {
        "m": m, "n": m, "host_ms_median": h[0], "host_ms_min": h[1], "api_host_ms_median": h_api[0],
        "kernel_ms": ki, "box_vertices_kernel_ms": k["box_vertices_kernel"],
        "fp64_ops_per_pair_sampled": per_pair, **bound(flops, 2 * m * 64 + m * m * 8, FP64_FLOPS, "fp64")}
    if ki:
        res["intersection_areas"]["achieved_fp64_TFLOPs"] = flops / (ki * 1e-3) / 1e12
        res["intersection_areas"]["achieved_hbm_TBps"] = (2 * m * 64 + m * m * 8) / (ki * 1e-3) / 1e12

    # -------- one per-object call of the reference-shaped API
    bf = api.Universal2DBoxKalmanFilter()
    s1 = bf.initiate(api.Universal2DBox.ltwh(10.0, 20.0, 5.0, 10.0))
    h = host_ms(lambda: bf.predict(s1), 200)
    res["per_object_predict"] = {"host_ms_median": h[0], "host_ms_min": h[1]}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
