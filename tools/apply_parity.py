#!/usr/bin/env python
"""Runs the same seeded frames on two builds of the package and checks that they leave identical trackers and outputs:
    python tools/apply_parity.py dump --root TREE --out DIR [--frames 20]
    python tools/apply_parity.py compare DIR_A DIR_B
`dump` imports similari_b200 from TREE (a checkout with its library built), runs cfg5, cfg3 (one scene), cfg4 (positional
only) and a VisualSort tracker with 25 observations per track, box history and feature history on, for --frames frames
each, and writes every frame's SortTrack columns, the wasted records, and the SHA-256 of each tracker's state blob
(Tracker.save()) after the last frame.  It then runs TREE/bench.py --dump-outputs into DIR/bench.  `compare` checks the
two directories file by file, byte for byte, and exits non-zero on any difference.  Needs a GPU."""
import argparse
import dataclasses
import hashlib
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

COLUMNS = ("ids", "epochs", "lengths", "voting_types", "predicted", "observed")


def cases(Workload, CONFIGS, tracker_options_for, default_options, KIND_VISUAL_SORT):
    """(name, options, workload, extra per-frame columns) of every tracker the dump runs."""
    out = []
    for name in ("cfg5", "cfg3", "cfg4"):
        cfg = CONFIGS[name]
        hints = dict(max_scenes_hint=cfg.n_scenes, max_tracks_per_scene_hint=4 * cfg.n_objects,
                     max_dets_per_scene_hint=cfg.n_objects)
        out.append((name, tracker_options_for(name, default_options, **hints), Workload(cfg), False))
    # K above kMaxObs (the warp-per-row observation lists), box history rings and the feature history pool.  One scene:
    # history blocks return to the pool in the order the records are collected, and that order is only fixed within a scene
    cfg = dataclasses.replace(CONFIGS["cfg3"], n_objects=512, feature_dim=128, seed=0x5EEDA125)
    opts = tracker_options_for("cfg3", default_options, kind=KIND_VISUAL_SORT, feature_dim=128,
                               visual_max_observations=25, history_length=6, max_idle_epochs=3)
    out.append(("visual_k25_history", opts, Workload(cfg), True))
    return out


def dump(root, out_dir, frames, bench_steps, bench_warmup):
    sys.path.insert(0, os.path.abspath(root))
    import similari_b200.engine as eng
    from similari_b200._lib import KIND_VISUAL_SORT, default_options
    from similari_b200.workload import CONFIGS, Workload, tracker_options_for

    os.makedirs(out_dir, exist_ok=True)
    summary = {}
    for name, opts, wl, varied in cases(Workload, CONFIGS, tracker_options_for, default_options, KIND_VISUAL_SORT):
        t = eng.Tracker(opts)
        if varied:
            t.set_feature_history(True)
        rng = np.random.default_rng(0x5EEDA000)
        cols = {k: [] for k in COLUMNS}
        for _ in range(frames):
            f = wl.next_frame()
            n = len(f["boxes"])
            extra = {}
            if varied:   # qualities with ties and observations without a feature: the observation lists reorder and drop
                extra = dict(quality=rng.choice(np.array([0.3, 0.5, 0.8, 0.8, 1.0], np.float32), n),
                             has_feature=(rng.random(n) >= 0.1).astype(np.uint8))
            r = t.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=f["features"], **extra)
            for k in COLUMNS:
                cols[k].append(np.asarray(r[k]))
        for k in COLUMNS:
            np.save(os.path.join(out_dir, f"{name}_{k}.npy"), np.concatenate(cols[k]))
        # The sweep appends the records of a frame's scenes to the wasted buffer in the order its CTAs finish (DESIGN §3b):
        # collect them before the blob is taken, and compare them sorted by (scene, id)
        rec = {}
        while True:
            w = t.wasted()
            if len(w["ids"]) == 0:
                break
            for k, v in w.items():
                rec.setdefault(k, []).append(v)
        rec = {k: np.concatenate(v) for k, v in rec.items()}
        if rec:
            order = np.lexsort((rec["ids"], rec["scene_ids"]))
            for k, v in rec.items():
                np.save(os.path.join(out_dir, f"{name}_wasted_{k}.npy"), v[order])
        blob = np.asarray(t.save()).tobytes()
        summary[name] = {"blob_bytes": len(blob), "blob_sha256": hashlib.sha256(blob).hexdigest()}
        t.close()
        print(name, summary[name], flush=True)
    with open(os.path.join(out_dir, "blobs.json"), "w") as fo:
        json.dump(summary, fo, indent=1, sort_keys=True)
    with tempfile.TemporaryDirectory() as tmp:   # bench.py writes nothing into the tree it runs from
        cmd = [sys.executable, os.path.join(os.path.abspath(root), "bench.py"), "--gpus", "1", "--steps", str(bench_steps),
               "--warmup", str(bench_warmup), "--dump-outputs", os.path.join(os.path.abspath(out_dir), "bench")]
        subprocess.run(cmd, check=True, cwd=tmp, stdout=subprocess.DEVNULL)


def compare(a, b):
    names = sorted(set(os.listdir(a)) | set(os.listdir(os.path.join(b))))
    files = []
    for n in names:
        if n == "bench":
            files += [os.path.join("bench", m) for m in sorted(set(os.listdir(os.path.join(a, n))) |
                                                                   set(os.listdir(os.path.join(b, n))))]
        else:
            files.append(n)
    bad = 0
    for n in files:
        pa, pb = os.path.join(a, n), os.path.join(b, n)
        if not (os.path.exists(pa) and os.path.exists(pb)):
            print(f"{n}: only in {'the first' if os.path.exists(pa) else 'the second'} directory")
            bad += 1
            continue
        with open(pa, "rb") as fa, open(pb, "rb") as fb:
            same = fa.read() == fb.read()
        print(f"{n}: {'identical' if same else 'DIFFERS'}")
        bad += 0 if same else 1
    print(f"{len(files) - bad} of {len(files)} files identical")
    return 1 if bad else 0


def main():
    ap = argparse.ArgumentParser()
    sub = ap.add_subparsers(dest="cmd", required=True)
    d = sub.add_parser("dump")
    d.add_argument("--root", required=True)
    d.add_argument("--out", required=True)
    d.add_argument("--frames", type=int, default=20)
    d.add_argument("--bench-steps", type=int, default=4)
    d.add_argument("--bench-warmup", type=int, default=2)
    c = sub.add_parser("compare")
    c.add_argument("a")
    c.add_argument("b")
    a = ap.parse_args()
    if a.cmd == "dump":
        dump(a.root, a.out, a.frames, a.bench_steps, a.bench_warmup)
        return 0
    return compare(a.a, a.b)


if __name__ == "__main__":
    sys.exit(main())
