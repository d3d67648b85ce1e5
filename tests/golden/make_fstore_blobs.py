"""Writes tests/golden/fstore_blobs.npz: one feature track store blob per blob shape the store writes (versions 1 to 4),
each from a seeded script of store calls, with the state of the store that wrote it.
tests/test_gpu_feature_store_blob_versions.py loads every blob with the current build, checks the state and that save()
gives the same bytes back, and runs each script again on a fresh store.  The fixture was written by the build before
save and load shared one section plan, so the test pins what an older build's blobs hold.

    python tests/golden/make_fstore_blobs.py [--tree DIR] [--out FILE]

--tree: the source tree whose similari_b200 package (built in place) writes the blobs; default this one.  Needs a GPU."""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np


def _rows(rng, n, dim):
    return rng.standard_normal((n, dim)).astype(np.float32)


def _windows(rng, n, base):
    t0 = base + 100 * np.arange(n, dtype=np.int64)
    return dict(sources=rng.integers(1, 3, n).astype(np.uint64), t_start=t0, t_end=t0 + 40)


def v1_f32_partial(eng, rng):
    """version 1, f32: one track wraps its ring, the others hold fewer than K rows; associate, then fetch(remove)"""
    s = eng.FeatureStore(feature_dim=20, max_observations=4, topn=2, max_distance=1e6, distance_filter=1e6)
    s.add(np.array([1, 1, 1, 1, 1, 1, 2, 3, 3, 4], np.uint64), _rows(rng, 10, 20))
    s.associate(np.array([7, 8], np.uint64), np.array([0, 2, 3], np.int32), _rows(rng, 3, 20))
    s.fetch(np.array([4], np.uint64), remove=True)
    s.add(np.array([5], np.uint64), _rows(rng, 1, 20))
    return s


def v1_bf16(eng, rng):
    """version 1, bf16 rows"""
    s = eng.FeatureStore(metric="cosine", feature_dim=12, max_observations=3, storage="bf16", distance_filter=2.0,
                         max_distance=2.0)
    s.add(np.repeat(np.arange(1, 6, dtype=np.uint64), 2), _rows(rng, 10, 12))
    s.associate(np.array([9], np.uint64), np.array([0, 2], np.int32), _rows(rng, 2, 12))
    s.fetch(np.array([2], np.uint64), remove=True)
    return s


def empty_f16(eng, rng):
    """version 1 of an empty f16 store"""
    return eng.FeatureStore(metric="cosine", feature_dim=100, max_observations=5, storage="f16", topn=7)


def _gated(eng, rng, gate):
    s = eng.FeatureStore(feature_dim=16, max_observations=3, gate=gate, max_distance=1e6, distance_filter=1e6)
    ids = np.repeat(np.arange(1, 7, dtype=np.uint64), 2)
    t0 = ids.astype(np.int64) * 10
    s.add(ids, _rows(rng, 12, 16), sources=(ids % 2 + 1).astype(np.uint64), t_start=t0, t_end=t0 + 5)
    s.associate(np.array([11, 12, 13], np.uint64), np.array([0, 1, 3, 4], np.int32), _rows(rng, 4, 16),
                **_windows(rng, 3, 1000))
    s.fetch(np.array([3], np.uint64), remove=True)
    return s


def v2_same_source(eng, rng):
    """version 2, gate same_source"""
    return _gated(eng, rng, "same_source")


def v2_any_source(eng, rng):
    """version 2, gate any_source"""
    return _gated(eng, rng, "any_source")


def _quality(eng, rng, gate, storage):
    s = eng.FeatureStore(feature_dim=20, max_observations=4, gate=gate, storage=storage, retention="quality",
                         max_distance=1e6, distance_filter=1e6)
    ids = np.repeat(np.arange(1, 9, dtype=np.uint64), 3)
    t0 = ids.astype(np.int64) * 10
    at = {} if gate is None else dict(sources=np.ones(len(ids), np.uint64), t_start=t0, t_end=t0 + 5)
    s.add(ids, _rows(rng, len(ids), 20), quality=rng.random(len(ids)).astype(np.float32), **at)
    s.merge_owned([1, 1, 4], [2, 3, 5], remove=True)
    qa = {} if gate is None else _windows(rng, 2, 1000)
    s.associate(np.array([21, 22], np.uint64), np.array([0, 2, 3], np.int32), _rows(rng, 3, 20),
                quality=rng.random(3).astype(np.float32), **qa)
    s.fetch(np.array([6], np.uint64), remove=True)
    return s


def v3_ungated(eng, rng):
    """version 3, quality retention, ungated f32"""
    return _quality(eng, rng, None, "f32")


def v3_gated_f16(eng, rng):
    """version 3, quality retention, gate any_source, f16 rows"""
    return _quality(eng, rng, "any_source", "f16")


def v4_three_classes(eng, rng):
    """version 4: three classes of different dims, newest"""
    dims = {0: 8, 3: 16, 9: 5}
    s = eng.FeatureStore(feature_dim=8, max_observations=3, classes=dims, max_distance=1e6, distance_filter=1e6)
    s.add(np.array([1, 1, 2, 3, 3, 3, 3], np.uint64), _rows(rng, 7, 8))
    s.add(np.array([2, 4, 4], np.uint64), _rows(rng, 3, 16), feature_class=3)
    s.add(np.array([1, 5], np.uint64), _rows(rng, 2, 5), feature_class=9)
    s.associate(np.array([6], np.uint64), np.array([0, 2], np.int32), _rows(rng, 2, 16), feature_class=3)
    s.merge_owned([1], [5], remove=True)
    s.fetch(np.array([2], np.uint64), remove=True)
    return s


def v4_gated_quality(eng, rng):
    """version 4: two classes, gate same_source, quality retention"""
    s = eng.FeatureStore(feature_dim=8, max_observations=4, classes={0: 8, 2: 12}, gate="same_source",
                         retention="quality", max_distance=1e6, distance_filter=1e6)
    ids = np.array([1, 1, 2, 3, 3], np.uint64)
    t0 = ids.astype(np.int64) * 10
    s.add(ids, _rows(rng, 5, 8), quality=rng.random(5).astype(np.float32), sources=np.ones(5, np.uint64), t_start=t0,
          t_end=t0 + 5)
    ids = np.array([2, 4, 4], np.uint64)
    t0 = ids.astype(np.int64) * 10
    s.add(ids, _rows(rng, 3, 12), quality=rng.random(3).astype(np.float32), sources=np.ones(3, np.uint64), t_start=t0,
          t_end=t0 + 5, feature_class=2)
    s.merge_owned([1], [2], remove=True)
    s.fetch(np.array([4], np.uint64), remove=True)
    return s


def v4_one_class(eng, rng):
    """version 4: the single class 5"""
    s = eng.FeatureStore(feature_dim=12, max_observations=3, classes={5: 12}, max_distance=1e6, distance_filter=1e6)
    s.add(np.array([1, 1, 2, 3, 3, 3, 3], np.uint64), _rows(rng, 7, 12), feature_class=5)
    s.associate(np.array([4], np.uint64), np.array([0, 1], np.int32), _rows(rng, 1, 12), feature_class=5)
    return s


SCRIPTS = [v1_f32_partial, v1_bf16, empty_f16, v2_same_source, v2_any_source, v3_ungated, v3_gated_f16,
           v4_three_classes, v4_gated_quality, v4_one_class]


def run(eng, script):
    """the store of `script`, from its own seed"""
    return script(eng, np.random.default_rng(SCRIPTS.index(script) + 1))


def state(s):
    """what a store of the fixture is checked against: ids, per class the fetched counts and rows (and qualities), the
    class counts, and the attributes and merge histories where the store has them"""
    ids = s.ids()
    out = {"ids": ids, "class_counts": s.class_counts(ids)}
    quality = s.retention()[0] == "quality"
    for c in s.classes():
        if quality:
            out[f"c{c}_counts"], out[f"c{c}_rows"], out[f"c{c}_qual"] = s.fetch_quality(ids, feature_class=c)
        else:
            out[f"c{c}_counts"], out[f"c{c}_rows"] = s.fetch(ids, feature_class=c)
    if s.gate is not None:
        out["src"], out["t_start"], out["t_end"] = s.attributes(ids)
    if quality:
        h = s.merge_history(ids)
        out["hist_len"] = np.array([len(x) for x in h], np.int32)
        out["hist"] = np.concatenate(h) if h else np.zeros(0, np.uint64)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tree", default=os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
    ap.add_argument("--out", default=os.path.join(os.path.dirname(os.path.abspath(__file__)), "fstore_blobs.npz"))
    a = ap.parse_args()
    sys.path.insert(0, os.path.abspath(a.tree))
    import similari_b200.engine as eng

    arrays = {}
    for script in SCRIPTS:
        s = run(eng, script)
        arrays[f"{script.__name__}/blob"] = s.save()
        for k, v in state(s).items():
            arrays[f"{script.__name__}/{k}"] = v
        s.close()
    np.savez_compressed(a.out, **arrays)
    print(a.out, sum(v.nbytes for v in arrays.values()), "bytes before compression")


if __name__ == "__main__":
    main()
