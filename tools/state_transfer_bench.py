"""State blob throughput at cfg5 steady state (256 scenes x 512 objects, D = 512, BatchVisualSort).

Reports the bytes each direction must move, computed from the shapes (live tracks and arena blocks times the row widths
of the store's columns), next to the blob size the library reports (which adds only the header and section alignment),
then times
  - sb200_tracker_save / _load with a device blob and with a host blob (pinned staging, PCIe),
  - sb200_scenes_export / _import of 32 scenes (device blob),
by wall clock around the (synchronous) calls and by the device time of the pack / unpack kernels (torch.profiler).
The kernels are compared with the HBM bound (read + write of the blob at the 3.35 TB/s of the H100 SXM data sheet) and the
host blob with PCIe.  Prints one JSON line; the card name and its power limit are part of it.

    python tools/state_transfer_bench.py [--frames 6] [--reps 3]
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

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_BPS = 3.35e12
PCIE_BPS = 64e9   # PCIe 5.0 x16, one direction, data sheet


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:
        return None


def state_bytes(o, live, blocks, n_scenes):
    """Bytes of the tracker's state a save moves, from the shapes alone: per live track every store column, per arena
    block its f32 and BF16 feature rows, norms and owner, per free block a free-list entry, per scene a table row.  (The
    wasted buffer is drained before the measurement; the feature history is off at cfg5.)"""
    K, d8 = int(o.visual_max_observations), (int(o.feature_dim) + 7) // 8 * 8
    H = 64 if o.history_length <= 0 else min(int(o.history_length), 64)
    track = 8 + 4 + 4 + 8 + 1 + 24 + 24 + 4 + 128   # id, epoch, length, custom id, voting type, boxes, radius, Kalman row
    track += 64 if o.positional_kind == 1 else 0     # IoU: vertex cache
    track += 2 * 24 * H if H > 1 else 0              # box-history rings
    track += K + K + 4 * K + 1 + 1 + 4               # observation permutation / present / quality, counts, arena block
    block = 4 * K * d8 + 2 * K * d8 + 4 * K + 4      # f32 rows, BF16 rows, norms, owner
    return live * track + blocks * block + (blocks - live) * 4 + n_scenes * 24


def save_into(g, host):
    """sb200_tracker_save into an existing host array (no allocation inside the timed call)."""
    from similari_b200._lib import check

    n = C.c_size_t(0)
    check(g._L.sb200_tracker_save(g._h, host.ctypes.data_as(C.c_void_p), host.nbytes, C.byref(n)))


def kernel_ms(fn, name_part="xfer_"):
    """Wall ms of fn() and the summed device ms of the kernels whose name contains name_part."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        t0 = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        wall = (time.perf_counter() - t0) * 1e3
    dev = sum(e.device_time_total for e in prof.key_averages() if name_part in e.key) / 1e3
    return r, wall, dev


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=6)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import torch

    import similari_b200.engine as eng
    from similari_b200._lib import default_options
    from similari_b200.workload import CONFIGS, Workload, tracker_options_for

    wl = Workload(CONFIGS["cfg5"])
    g = eng.Tracker(tracker_options_for("cfg5", default_options))
    for _ in range(args.frames):
        f = wl.next_frame()
        g.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=f["features"])
    g.wasted()   # a collection point: the blob then holds the live state alone
    live, blocks = g.scene_live_counts(np.arange(256, dtype=np.uint64))
    sb = state_bytes(g.opts, int(live.sum()), int(blocks.sum()), 256)
    n = g.save_device(0, 0)
    assert 0 <= n - sb <= 64 * 1024, (n, sb)   # header and section alignment only
    dev = torch.empty(n, dtype=torch.uint8, device="cuda")
    host = np.empty(n, np.uint8)
    res = {"card": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(), "frames": args.frames,
           "live_tracks": int(live.sum()), "arena_blocks": int(blocks.sum()), "blob_bytes": int(n),
           "bytes_each_direction": int(sb), "format_overhead_bytes": int(n - sb)}
    rows = {k: [] for k in ("save_dev", "load_dev", "save_host", "load_host", "export32", "import32")}
    for _ in range(args.reps):
        _, w, d = kernel_ms(lambda: g.save_device(dev.data_ptr(), n))
        rows["save_dev"].append((w, d))
        h, w, d = kernel_ms(lambda: eng.Tracker.load(dev.data_ptr(), n))
        rows["load_dev"].append((w, d))
        h.close()
        del h
        _, w, d = kernel_ms(lambda: save_into(g, host))
        rows["save_host"].append((w, d))
        h, w, d = kernel_ms(lambda: eng.Tracker.load(host))
        rows["load_host"].append((w, d))
        h.close()
        del h
        scenes = np.arange(32, dtype=np.uint64)
        ne = g.export_scenes(scenes, d_ptr=0)
        eb = torch.empty(ne, dtype=torch.uint8, device="cuda")
        _, w, d = kernel_ms(lambda: g.export_scenes(scenes, remove=True, d_ptr=eb.data_ptr(), cap=ne))
        rows["export32"].append((w, d))
        _, w, d = kernel_ms(lambda: g.import_scenes(eb.data_ptr(), ne))
        rows["import32"].append((w, d))
        res["export32_bytes"] = int(ne)
    for k, v in rows.items():
        w = min(x[0] for x in v)
        d = min(x[1] for x in v)
        nb = res["export32_bytes"] if k.endswith("32") else sb
        res[k] = {"wall_ms": round(w, 3), "kernel_ms": round(d, 3),
                  "kernel_fraction_of_hbm_bound": round((2 * nb / HBM_BPS * 1e3) / d, 3) if d > 0 else None}
        if k.endswith("_host"):
            res[k]["wall_fraction_of_pcie"] = round((nb / PCIE_BPS * 1e3) / w, 3)
    res["hbm_bound_ms"] = round(2 * sb / HBM_BPS * 1e3, 3)
    res["pcie_bound_ms"] = round(sb / PCIE_BPS * 1e3, 3)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
