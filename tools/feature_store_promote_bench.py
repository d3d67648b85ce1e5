"""Feature track store, store to store: the main loop of the reference's examples/track_merging.rs at a user's scale.
One JSON line per measurement.

  python tools/feature_store_promote_bench.py [--rounds N] [--frames N] [--gallery N]

Every frame, 16 cameras x 32 objects add one observation each (D = 512, K = 12) to a gated collecting store; each object
is a tracklet of about 30 frames (20..40) of one of 400 people.  Then the baked tracklets (now > t_end + 3) move into a
gated gallery preloaded with `--gallery` tracks (default 100,000, 3 rows each, windows long before the run):
- device arm: find_baked + associate_store(remove=True), the rows never leaving the device;
- host arm: the same loop without them: attributes(ids()) of the whole collecting store, the bake rule in Python,
  attributes + fetch(remove=True) of the baked ids, and associate of the fetched rows;
- quality arm: the device arm on quality stores (defaults 4 / 1.5), with a random quality per observation.
The device and host arms are twin pipelines fed the same observations, alternated every frame (which one runs first
alternates too); their outputs are checked equal every frame before the timings count.  A run warms up for 40 frames
(the first tracklets bake after about 30), then each round times --frames frames.  Per frame: host time of the promote
step (a host clock around calls that end in a device synchronise), median and range over the rounds' medians; and the
bytes each arm moves over PCIe, computed from the shapes the calls stage and read back (not measured).
Seeded.  The card's name and power limit are read in the same run; without a CUDA device the script fails.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CAMS, OBJS, DIM, K, PERIOD, PEOPLE = 16, 32, 512, 12, 3, 400


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = [x.strip() for x in out.split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def emit(d):
    print(json.dumps(d), flush=True)


def stats(v):
    return {"median": float(np.median(v)), "min": float(min(v)), "max": float(max(v))}


def store(retention="newest"):
    import similari_b200.engine as eng

    return eng.FeatureStore(distance_filter=1e9, max_observations=K, feature_dim=DIM, topn=1, max_distance=14.0,
                            min_votes=3, gate="same_source", retention=retention)


def gallery_blob(n, rng, retention):
    g = store(retention)
    for a in range(0, n, 10000):
        m = min(10000, n - a)
        ids = np.repeat(np.arange(10**9 + a, 10**9 + a + m, dtype=np.uint64), 3)
        rows = rng.standard_normal((3 * m, DIM), np.float32)
        t = np.repeat(-(10**7) + np.arange(a, a + m, dtype=np.int64) * 10, 3)
        kw = dict(quality=np.ones(3 * m, np.float32)) if retention == "quality" else {}
        g.add(ids, rows, sources=ids % CAMS + 1, t_start=t, t_end=t + 5, **kw)
    return g.save()


def promote_device(col, gal, frame):
    baked = col.find_baked(frame, PERIOD)
    return gal.associate_store(col, baked, remove=True), baked, None


def promote_host(col, gal, frame):
    live = col.ids()
    _, _, t1 = col.attributes(live)
    baked = live[[frame > int(e) + PERIOD for e in t1]] if len(live) else live
    s, t0, t1 = col.attributes(baked)
    counts, feats = col.fetch(baked, remove=True)
    offs = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    rows = np.concatenate([feats[i, :counts[i]] for i in range(len(baked))]) if len(baked) else feats.reshape(0, DIM)
    return gal.associate(baked, offs, rows, sources=s, t_start=t0, t_end=t1), baked, int(offs[-1])


def pcie_bytes(live, nb, rows, topn=1):
    """Bytes over PCIe of one promote step (both directions), from the shapes each call stages and reads back.  d8 =
    DIM here.  Common to both arms: the associate request tables (ids, offsets, row -> query, dest, max_dist) and its
    results (weights, counts, positions, the destinations read back on a gated store)."""
    tables = nb * 8 + (nb + 1) * 4 + rows * 4 + nb * 4 + 4
    results = nb * topn * 8 + nb * 4 + nb * topn * 4 + nb * 4
    device = 4 + 4 * nb + 4 * nb + 8 * nb + tables + results   # find_baked count and positions; ring peek of src
    host = (24 * live + 4 * live                               # attributes(ids()) of the collecting store
            + 24 * nb + 4 * nb                                  # attributes(baked)
            + nb * K * DIM * 4 + 4 * nb + 4 * nb                # fetch: K rows per id back, counts, positions
            + rows * DIM * 4 + 24 * nb + tables + results)      # associate: the rows and triples go back down
    return device, host


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--frames", type=int, default=20)
    ap.add_argument("--gallery", type=int, default=100000)
    ap.add_argument("--seed", type=int, default=3)
    a = ap.parse_args()
    import similari_b200.engine as eng

    emit({"what": "card", **card()})
    rng = np.random.default_rng(a.seed)
    people = rng.standard_normal((PEOPLE, DIM)).astype(np.float32)
    blob_n, blob_q = gallery_blob(a.gallery, rng, "newest"), gallery_blob(a.gallery, rng, "quality")
    arms = {"device": (store(), eng.FeatureStore.load(blob_n), promote_device),
            "host": (store(), eng.FeatureStore.load(blob_n), promote_host),
            "quality": (store("quality"), eng.FeatureStore.load(blob_q), promote_device)}
    del blob_n, blob_q
    slots, next_id = [], 1   # per object: [tracklet id, person, camera, last frame]
    for c in range(CAMS):
        for _ in range(OBJS):
            slots.append([next_id, int(rng.integers(0, PEOPLE)), c + 1, int(rng.integers(0, 40))])
            next_id += 1
    times = {k: [] for k in arms}
    sizes = []
    warm = 40
    for frame in range(warm + a.rounds * a.frames):
        for s in slots:
            if s[3] < frame:
                s[:] = [next_id, int(rng.integers(0, PEOPLE)), s[2], frame + int(rng.integers(20, 41))]
                next_id += 1
        ids = np.array([s[0] for s in slots], np.uint64)
        rows = people[[s[1] for s in slots]] + 0.2 * rng.standard_normal((len(slots), DIM), np.float32)
        attrs = dict(sources=[s[2] for s in slots], t_start=[frame] * len(slots), t_end=[frame] * len(slots))
        qual = rng.integers(0, 5, len(slots)).astype(np.float32)
        for k, (col, _, _) in arms.items():
            col.add(ids, rows, **attrs, **(dict(quality=qual) if k == "quality" else {}))
        order = ["device", "host"] if frame % 2 == 0 else ["host", "device"]
        out = {}
        for k in order + ["quality"]:
            col, gal, fn = arms[k]
            live = col.size()
            t = time.perf_counter()
            r, baked, nrows = fn(col, gal, frame)
            dt = time.perf_counter() - t
            out[k] = (r, baked, live, nrows)
            if frame >= warm:
                times[k].append(dt * 1e3)
        (rd, bd, live, _), (rh, bh, _, nrows) = out["device"], out["host"]
        if not np.array_equal(bd, bh) or any(not np.array_equal(rd[x], rh[x]) for x in rd):
            raise AssertionError(f"frame {frame}: the device and host arms differ")
        if frame >= warm:
            sizes.append((len(bd), nrows, *pcie_bytes(live, len(bd), nrows)))
    per_round = lambda v: [float(np.median(v[i * a.frames:(i + 1) * a.frames])) for i in range(a.rounds)]
    common = {"rounds": a.rounds, "frames_per_round": a.frames, "gallery_tracks_at_start": a.gallery,
              "objects_per_frame": CAMS * OBJS, "dim": DIM, "K": K}
    for k in arms:
        emit({"what": f"promote_step_ms_{k}", "per_frame": stats(per_round(times[k])), **common})
    sz = np.array(sizes, np.float64)
    emit({"what": "promoted_per_frame", "tracks": stats(per_round(sz[:, 0])), "rows": stats(per_round(sz[:, 1])),
          **common})
    for i, k in ((2, "device"), (3, "host")):
        emit({"what": f"pcie_bytes_per_frame_{k}", "bytes": stats(per_round(sz[:, i])), "source": "computed from shapes",
              **common})


if __name__ == "__main__":
    main()
