#!/usr/bin/env python
"""Times sb200_nms on the cfg5 NMS workload of SURVEY.md section 8d: 10 000 oriented boxes = 2 000 clusters x 5
near-duplicates (jitter 3 px / 0.03 rad) on 3840x2160, scores U(0,1), nms_threshold 0.8.  Host-pointer call
(H2D + kernels + D2H inside), best and median of `reps` runs; optional oracle check on a sub-sample.

--batch: the same suppression over a frame of 256 scenes (cameras), each 100 clusters x 5 near-duplicates on 3840x2160
with its own seed, timed three ways: (a) one sb200_nms_batch call (host pointers, wall clock), (b) sb200_nms_batch_device
on inputs resident in HBM (CUDA events over repeated calls on one stream, after warm-up), (c) the same scenes through 256
sb200_nms calls.  --check compares every scene of (a) and (b) with oracle.nms.

usage: nms_bench.py [reps] [--check] [--batch]"""
import json
import sys
import time

import numpy as np

sys.path.insert(0, __file__.rsplit("/tools/", 1)[0])
from similari_b200.engine import nms_batch, nms_batch_device, nms_indices  # noqa: E402


def make_boxes(n_clusters=2000, dup=5, seed=0x5EED00A5):
    r = np.random.default_rng(seed)
    xc = r.uniform(0, 3840, n_clusters)
    yc = r.uniform(0, 2160, n_clusters)
    ang = r.uniform(-np.pi / 2, np.pi / 2, n_clusters)
    asp = r.uniform(0.3, 0.8, n_clusters)
    h = r.uniform(40, 160, n_clusters)
    b = np.empty((n_clusters, dup, 6), np.float32)
    b[..., 0] = xc[:, None] + r.normal(0, 3, (n_clusters, dup))
    b[..., 1] = yc[:, None] + r.normal(0, 3, (n_clusters, dup))
    b[..., 2] = ang[:, None] + r.normal(0, 0.03, (n_clusters, dup))
    b[..., 3] = asp[:, None]
    b[..., 4] = h[:, None]
    b[..., 5] = 1.0
    b = b.reshape(-1, 6)
    s = r.uniform(0, 1, len(b)).astype(np.float32)
    p = r.permutation(len(b))
    return np.ascontiguousarray(b[p]), s[p]


def batch_scenes(n_scenes=256, n_clusters=100, dup=5, seed=0x5EED00A5):
    parts = [make_boxes(n_clusters, dup, seed + 1 + s) for s in range(n_scenes)]
    offsets = np.arange(n_scenes + 1, dtype=np.int32) * (n_clusters * dup)
    return np.concatenate([b for b, _ in parts]), np.concatenate([s for _, s in parts]), offsets


def _stats(ts):
    return 1e3 * min(ts), 1e3 * float(np.median(ts))


def main_batch(reps, check):
    import torch

    boxes, scores, offsets = batch_scenes()
    n_sets, total = len(offsets) - 1, len(boxes)
    out = {"workload": "NMS oriented, 256 scenes x 500 boxes (100 clusters x 5), thr 0.8", "n_scenes": n_sets,
           "boxes_per_scene": int(offsets[1]), "gpu": torch.cuda.get_device_name(0)}

    # (a) one host-pointer call for the whole frame
    nms_batch(boxes, scores, offsets, 0.8)
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        keep_a = nms_batch(boxes, scores, offsets, 0.8)
        ts.append(time.perf_counter() - t0)
    out["a_batch_host_ms_best"], out["a_batch_host_ms_median"] = _stats(ts)
    out["kept"] = int(sum(len(k) for k in keep_a))

    # (b) device pointers, inputs resident, one stream; CUDA events around `calls` back-to-back calls
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        d_boxes, d_scores = torch.from_numpy(boxes).cuda(), torch.from_numpy(scores).cuda()
        d_idx = torch.empty(total, dtype=torch.int32, device="cuda")
        d_cnt = torch.empty(n_sets, dtype=torch.int32, device="cuda")
    args = (offsets, d_boxes.data_ptr(), d_scores.data_ptr(), 0.8, None, d_idx.data_ptr(), d_cnt.data_ptr())
    for _ in range(5):
        nms_batch_device(*args, stream=st.cuda_stream)
    st.synchronize()
    calls, per_call = 50, []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        for _ in range(calls):
            nms_batch_device(*args, stream=st.cuda_stream)
        e1.record(st)
        e1.synchronize()
        per_call.append(e0.elapsed_time(e1) / calls / 1e3)
    out["b_batch_device_ms_best"], out["b_batch_device_ms_median"] = _stats(per_call)
    idx, cnt = d_idx.cpu().numpy(), d_cnt.cpu().numpy()
    keep_b = [idx[offsets[s]:offsets[s] + cnt[s]] for s in range(n_sets)]

    # (c) one sb200_nms call per scene
    scenes = [(boxes[offsets[s]:offsets[s + 1]], scores[offsets[s]:offsets[s + 1]]) for s in range(n_sets)]
    nms_indices(*scenes[0], 0.8)
    ts = []
    for _ in range(max(1, reps // 2)):
        t0 = time.perf_counter()
        keep_c = [nms_indices(b, s, 0.8) for b, s in scenes]
        ts.append(time.perf_counter() - t0)
    out["c_loop_of_single_calls_ms_best"], out["c_loop_of_single_calls_ms_median"] = _stats(ts)
    out["speedup_a_vs_c"] = out["c_loop_of_single_calls_ms_median"] / out["a_batch_host_ms_median"]
    out["speedup_b_vs_c"] = out["c_loop_of_single_calls_ms_median"] / out["b_batch_device_ms_median"]
    out["a_b_c_identical"] = all(np.array_equal(a, b) and np.array_equal(a, c) for a, b, c in zip(keep_a, keep_b, keep_c))
    if check:
        import oracle

        out["identical_to_oracle"] = all(
            np.array_equal(oracle.nms(b, s, 0.8), a) and np.array_equal(a, kb)
            for (b, s), a, kb in zip(scenes, keep_a, keep_b))
    print(json.dumps(out))


def main():
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    reps = int(args[0]) if args else 10
    if "--batch" in sys.argv:
        return main_batch(reps, "--check" in sys.argv)
    boxes, scores = make_boxes()
    nms_indices(boxes, scores, 0.8)   # warm-up (context, allocations)
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        keep = nms_indices(boxes, scores, 0.8)
        ts.append(time.perf_counter() - t0)
    out = {"workload": "NMS oriented 10k boxes (2000 clusters x 5), thr 0.8", "n": len(boxes), "kept": int(len(keep)),
           "ms_best": 1e3 * min(ts), "ms_median": 1e3 * float(np.median(ts)),
           "pair_tests_upper": len(boxes) * (len(boxes) - 1) // 2}
    if "--check" in sys.argv:
        import oracle

        t0 = time.perf_counter()
        ref = oracle.nms(boxes, scores, 0.8)
        out["oracle_ms"] = 1e3 * (time.perf_counter() - t0)
        out["identical_to_oracle"] = bool(np.array_equal(ref, keep))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
