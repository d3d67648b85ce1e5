"""Checks shared by the feature-store tests: bit-exact comparison of call results and of whole stores, a GPU store and
its CPU-oracle twin (fstore_oracle) built from one set of options, and the refusal of a damaged store blob.

Results and stores are compared bit for bit: floats through unsigned views of their size, so NaN payloads and the sign
of zero count, and arrays must agree in dtype and shape as well."""
import ctypes as C
import os

import numpy as np

import fstore_oracle as fo

METRICS = {"euclidean": fo.EUCLIDEAN, "cosine": fo.COSINE}
THREADS = max(1, min(16, os.cpu_count() or 1))
DEFAULTS = dict(distance_filter=1e9, max_observations=3, feature_dim=16, topn=4, max_distance=1e9, min_votes=1)


def bits(a):
    """A floating-point array as the unsigned integers of its element size; any other array as it is."""
    a = np.ascontiguousarray(a)
    return a.view(f"u{a.dtype.itemsize}") if a.dtype.kind == "f" else a


def same_results(a, b, what=""):
    """a and b are the same results: dicts with the same keys, or lists / tuples of the same length, down to arrays of
    equal dtype, shape and bits."""
    if isinstance(b, dict):
        assert isinstance(a, dict) and a.keys() == b.keys(), (what, list(a), list(b))
        for k in b:
            same_results(a[k], b[k], (what, k))
    elif isinstance(b, (list, tuple)):
        assert isinstance(a, (list, tuple)) and len(a) == len(b), (what, len(a), len(b))
        for i, (x, y) in enumerate(zip(a, b)):
            same_results(x, y, (what, i))
    else:
        assert a.dtype == b.dtype and a.shape == b.shape, (what, a.dtype, b.dtype, a.shape, b.shape)
        assert np.array_equal(bits(a), bits(b)), (what, a, b)


def _rules(s):
    """The rules that decide what a store holds.  The capacity parameters count on a quality store alone: a newest
    store ignores them (the library reports its defaults, the oracle the values it was given)."""
    rule, init, ext = s.retention()
    return ((rule, init, np.float32(ext)) if rule == "quality" else (rule,)), s.gate, s.classes()


def same_store(g, o):
    """g and o hold the same tracks under the same rules: ids and size; each class's rows; on a quality store the rows'
    qualities and the merge histories; on a gated store the attributes; with several classes the rows per class.  The
    per-track reads also ask for an id neither store holds."""
    assert _rules(g) == _rules(o), (_rules(g), _rules(o))
    stored = o.ids()
    same_results(g.ids(), stored, "ids")
    assert g.size() == o.size() == len(stored)
    ids = np.concatenate([stored, np.setdiff1d(np.array([12345], np.uint64), stored)])
    quality = o.retention()[0] == "quality"
    for c in o.classes():
        same_results(g.fetch(ids, feature_class=c), o.fetch(ids, feature_class=c), ("fetch", c))
        if quality:
            same_results(g.fetch_quality(ids, feature_class=c), o.fetch_quality(ids, feature_class=c),
                         ("fetch_quality", c))
    if quality:
        same_results(g.merge_history(ids), o.merge_history(ids), "merge_history")
    if o.gate is not None:
        same_results(g.attributes(ids), o.attributes(ids), "attributes")
    if len(o.classes()) > 1:
        same_results(g.class_counts(ids), o.class_counts(ids), "class_counts")


def store_options(**over):
    """The options of a test store: DEFAULTS with `over` on top."""
    return dict(DEFAULTS, **over)


def gpu_store(metric="euclidean", storage="f32", **over):
    """An engine.FeatureStore of store_options(**over)."""
    import similari_b200.engine as eng

    return eng.FeatureStore(metric=metric, storage=storage, **store_options(**over))


def store_pair(metric="euclidean", storage="f32", gate=None, retention="newest", voting="topn", classes=None, **over):
    """A GPU store and its fstore_oracle twin, built from the same options (the oracle keeps f32 rows whatever the
    storage type)."""
    o = store_options(gate=gate, retention=retention, voting=voting, classes=classes, **over)
    return gpu_store(metric, storage, **o), fo.FeatureStore(metric=METRICS[metric], threads=THREADS, **o)


def refused_blob(blob, field):
    """sb200_fstore_load refuses the damaged `blob` with SB200_ERR_INVALID, hands back no handle, and names `field`."""
    from similari_b200 import _lib

    L = _lib.lib()
    h = C.c_void_p()
    blob = np.ascontiguousarray(blob)
    assert L.sb200_fstore_load(_lib.ptr(blob), len(blob), 0, C.byref(h)) == -1
    assert h.value is None
    assert field in L.sb200_last_error().decode(), L.sb200_last_error()
