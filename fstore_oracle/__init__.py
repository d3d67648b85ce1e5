"""CPU oracle of the feature track store -- TEST INFRASTRUCTURE ONLY.

ctypes binding of ``fstore_oracle/libfstore_oracle.so`` (built from ``feature_store.cpp`` by ``build()``), which calls
the distance code of ``oracle/liboracle.so``.  It restates the reference's TrackStore for feature-only tracks and
TopNVoting::winners, and defines the orders the reference leaves to its shards and HashMaps (see feature_store.cpp).
Only ``tests/``, ``__graft_entry__`` and the store benchmarks under ``tools/`` import it; ``similari_b200`` never does.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

import oracle

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "feature_store.cpp")
_LIB_PATH = os.path.join(_HERE, "libfstore_oracle.so")
_ORACLE_DIR = os.path.dirname(os.path.abspath(oracle.__file__))

EUCLIDEAN, COSINE = 0, 1
# track attribute rules (feature_store.cpp): None = no attributes
GATES = {None: 0, "same_source": 1, "any_source": 2}
# retention rules (feature_store.cpp): the newest K, or the best by quality with a capacity growing with the merges
RETENTIONS = {"newest": 0, "quality": 1}
# voting rules (feature_store.cpp): TopNVoting or BestFitVoting
VOTINGS = {"topn": 0, "best_fit": 1}


def build(force: bool = False) -> str:
    """Compile libfstore_oracle.so if missing or stale (g++ only; -ffp-contract=off as for liboracle.so)."""
    base = oracle.build()
    deps = [_SRC, os.path.join(_ORACLE_DIR, "similari_oracle.h"), base]
    if force or not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < max(os.path.getmtime(d) for d in deps):
        subprocess.check_call([
            "g++", "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-Wextra", "-pthread",
            "-shared", "-o", _LIB_PATH, _SRC, "-L" + _ORACLE_DIR, "-l:liboracle.so", "-Wl,-rpath,$ORIGIN/../oracle"])
    return _LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB_PATH)
        vp, i32, i64, f32 = C.c_void_p, C.c_int32, C.c_int64, C.c_float
        sig = {
            "ofs_create": (vp, [i32, f32, i32, i32, i32, f32, i32]),
            "ofs_destroy": (None, [vp]),
            "ofs_add": (C.c_int, [vp, i32, vp, vp]),
            "ofs_search": (C.c_int, [vp, i32, vp, vp, vp, vp, vp, vp, i32]),
            "ofs_associate": (C.c_int, [vp, i32, vp, vp, vp, vp, vp, vp, vp, vp, i32]),
            "ofs_fetch": (i64, [vp, i32, vp, i32, vp, vp]),
            "ofs_size": (i64, [vp]),
            "ofs_ids": (i64, [vp, i64, vp]),
            "ofs_topn_voting": (C.c_int, [f32, i32, i32, i32, vp, vp, vp, vp, vp, vp]),
            "ofs_search_owned": (C.c_int, [vp, i32, vp, i32, vp, vp, vp, i32]),
            "ofs_merge_owned": (C.c_int, [vp, i32, vp, vp, i32]),
            "ofs_set_gate": (C.c_int, [vp, i32]),
            "ofs_add_attr": (C.c_int, [vp, i32, vp, vp, vp, vp, vp]),
            "ofs_search_attr": (C.c_int, [vp, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, i32]),
            "ofs_associate_attr": (C.c_int, [vp, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, i32]),
            "ofs_fetch_attr": (i64, [vp, i32, vp, vp, vp, vp]),
            "ofs_set_retention": (C.c_int, [vp, i32, i32, f32]),
            "ofs_add_quality": (C.c_int, [vp, i32, vp, vp, vp, vp, vp, vp]),
            "ofs_search_quality": (C.c_int, [vp, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, i32]),
            "ofs_associate_quality": (C.c_int, [vp, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, i32]),
            "ofs_fetch_quality": (i64, [vp, i32, vp, i32, vp, vp, vp]),
            "ofs_merge_history": (i64, [vp, i32, vp, vp, i64, vp]),
            "ofs_find_baked": (i64, [vp, i64, i64, i64, vp]),
            "ofs_associate_store": (C.c_int, [vp, vp, i32, vp, i32, vp, vp, vp, vp, vp, i32]),
            "ofs_set_classes": (C.c_int, [vp, i32, vp, vp]),
            "ofs_use_class": (C.c_int, [vp, C.c_uint64]),
            "ofs_class_counts": (i64, [vp, i32, vp, vp]),
            "ofs_set_voting": (C.c_int, [vp, i32]),
            "ofs_bestfit_voting": (C.c_int, [f32, i32, i32, i32, vp, vp, vp, vp, vp, vp]),
        }
        for name, (res, args) in sig.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def round_rows(x, storage):
    """What a store of storage type `storage` ("f32", "f16", "bf16") holds for the f32 values `x`, widened back to f32:
    each value rounded once to the type, to nearest with ties to even, overflow to +-inf, subnormals kept; NaN stays NaN
    (its payload is not modelled).  Written from the formats' definitions, without numpy's or torch's casts, so that the
    tests can check it against both."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    if storage == "f32":
        return x.copy()
    nan = np.isnan(x)
    if storage == "bf16":
        u = x.view(np.uint32).astype(np.uint64)
        r = ((u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000).astype(np.uint32).view(np.float32)
        return np.where(nan, np.float32(np.nan), r)
    if storage != "f16":
        raise ValueError(f"unknown storage type {storage!r}")
    with np.errstate(invalid="ignore", over="ignore"):
        a = np.abs(x.astype(np.float64))   # exact
        _, ex = np.frexp(np.where(np.isfinite(a) & (a > 0), a, 1.0))   # a = m * 2^ex, m in [0.5, 1)
        ulp = np.ldexp(1.0, np.maximum(ex - 1, -14) - 10)              # binary16: 11 significant bits, emin = -14
        r = np.rint(a / ulp) * ulp                                     # a / ulp is exact; rint ties to even
        r = np.where(np.isinf(a) | (r > 65504.0), np.inf, r)
        return np.where(nan, np.float32(np.nan), np.copysign(r, x).astype(np.float32))


def topn_voting(topn, max_distance, min_votes, ents):
    """TopNVoting::winners.  ents: list of (from, to, distance or None).  Returns {query: [(winner, weight), ...]}."""
    return _voting(lib().ofs_topn_voting, topn, max_distance, min_votes, ents)


def bestfit_voting(topn, max_distance, min_votes, ents):
    """BestFitVoting::winners on TopN's groups: every element claims its track in the order weight descending, then
    the group's first appearance; a loser's winner is its own query.  Each query's list is cut at topn after the claims.
    ents and the result as for topn_voting."""
    return _voting(lib().ofs_bestfit_voting, topn, max_distance, min_votes, ents)


def _voting(fn, topn, max_distance, min_votes, ents):
    fr = np.array([e[0] for e in ents], dtype=np.uint64)
    to = np.array([e[1] for e in ents], dtype=np.uint64)
    fe = np.array([np.nan if e[2] is None else e[2] for e in ents], dtype=np.float32)
    cap = max(1, len(ents))
    q, w, wt = np.zeros(cap, np.uint64), np.zeros(cap, np.uint64), np.zeros(cap, np.float64)
    n = fn(max_distance, min_votes, topn, len(ents), _p(fr), _p(to), _p(fe), _p(q), _p(w), _p(wt))
    res = {}
    for i in range(n):
        res.setdefault(int(q[i]), []).append((int(w[i]), float(wt[i])))
    return res


class FeatureStore:
    """The oracle's feature track store; same calls and results as similari_b200.engine.FeatureStore."""

    def __init__(self, metric=EUCLIDEAN, distance_filter=100.0, max_observations=3, feature_dim=256, topn=1,
                 max_distance=100.0, min_votes=1, threads=1, gate=None, retention="newest", initial_capacity=4,
                 merge_extension=1.5, classes=None, voting="topn"):
        self._L = lib()
        self.K, self.D, self.topn, self.threads = int(max_observations), int(feature_dim), int(topn), int(threads)
        self._h = self._L.ofs_create(metric, distance_filter, self.K, self.D, self.topn, max_distance, min_votes)
        if not self._h:
            raise ValueError("invalid feature store options")
        if gate not in GATES:
            raise ValueError(f"gate must be one of {list(GATES)}")
        self.gate = gate
        if self._L.ofs_set_gate(self._h, GATES[gate]):
            raise ValueError("invalid gate")
        if retention not in RETENTIONS:
            raise ValueError(f"retention must be one of {list(RETENTIONS)}")
        if self._L.ofs_set_retention(self._h, RETENTIONS[retention], int(initial_capacity), float(merge_extension)):
            raise ValueError("invalid retention parameters")
        self._retention = (retention, int(initial_capacity), float(merge_extension))
        self._classes = {0: self.D} if classes is None else {int(k): int(v) for k, v in dict(classes).items()}
        cid = np.array(list(self._classes), np.uint64)
        dims = np.array(list(self._classes.values()), np.int32)
        if self._L.ofs_set_classes(self._h, len(cid), _p(cid), _p(dims)):
            raise ValueError("invalid classes")
        self._use(None)
        self.set_voting(voting)

    def set_voting(self, voting):
        """"topn" or "best_fit": how every later search / associate / search_owned / associate_store votes."""
        if voting not in VOTINGS or self._L.ofs_set_voting(self._h, VOTINGS[voting]):
            raise ValueError(f"voting must be one of {list(VOTINGS)}")
        self._voting = voting

    def voting(self):
        return self._voting

    def _use(self, feature_class):
        """Selects the class of the next call (None: the first declared one)."""
        c = next(iter(self._classes)) if feature_class is None else int(feature_class)
        if c not in self._classes or self._L.ofs_use_class(self._h, c):
            raise ValueError(f"feature_class {c} is not declared")
        self.D = self._classes[c]

    def classes(self):
        return dict(self._classes)

    def class_counts(self, ids):
        """counts[n][len(classes())]: each track's rows per class, declared order (0 where not stored)."""
        ids = np.ascontiguousarray(ids, dtype=np.uint64)
        out = np.zeros((len(ids), len(self._classes)), np.int32)
        self._L.ofs_class_counts(self._h, len(ids), _p(ids), _p(out))
        return out

    def retention(self):
        """(rule, initial_capacity, merge_extension)."""
        return self._retention

    def _quality(self, n, quality):
        """The quality column of a call: required on a quality store, refused on a newest one."""
        if self._retention[0] == "newest":
            if quality is not None:
                raise ValueError("quality= needs a quality store")
            return None
        if quality is None:
            raise ValueError("a quality store needs quality=")
        q = np.ascontiguousarray(quality, dtype=np.float32)
        if q.shape != (n,):
            raise ValueError("quality needs one value per row")
        return q

    def _attrs(self, n, sources, t_start, t_end):
        """The three attribute columns of a call: required on a gated store, refused on an ungated one."""
        given = [a is not None for a in (sources, t_start, t_end)]
        if self.gate is None:
            if any(given):
                raise ValueError("sources / t_start / t_end need a gated store")
            return None
        if not all(given):
            raise ValueError("a gated store needs sources, t_start and t_end")
        a = (np.ascontiguousarray(sources, dtype=np.uint64), np.ascontiguousarray(t_start, dtype=np.int64),
             np.ascontiguousarray(t_end, dtype=np.int64))
        if any(len(x) != n for x in a):
            raise ValueError("sources / t_start / t_end need one entry per row")
        return a

    def __del__(self):
        if getattr(self, "_h", None):
            self._L.ofs_destroy(self._h)
            self._h = None

    def add(self, ids, features, sources=None, t_start=None, t_end=None, quality=None, feature_class=None):
        self._use(feature_class)
        ids = np.ascontiguousarray(ids, dtype=np.uint64)
        f = np.ascontiguousarray(features, dtype=np.float32).reshape(len(ids), self.D)
        a = self._attrs(len(ids), sources, t_start, t_end)
        q = self._quality(len(ids), quality)
        if q is not None:
            if self._L.ofs_add_quality(self._h, len(ids), _p(ids), _p(q), *(map(_p, a) if a else (None,) * 3), _p(f)):
                raise ValueError("invalid add request")
        elif a is None:
            self._L.ofs_add(self._h, len(ids), _p(ids), _p(f))
        elif self._L.ofs_add_attr(self._h, len(ids), _p(ids), *map(_p, a), _p(f)):
            raise ValueError("invalid add request")

    def _queries(self, ids, offsets, features):
        ids = np.ascontiguousarray(ids, dtype=np.uint64)
        offs = np.ascontiguousarray(offsets, dtype=np.int32)
        f = np.ascontiguousarray(features, dtype=np.float32).reshape(-1, self.D)
        q = len(ids)
        out = {"counts": np.zeros(q, np.int32), "winners": np.zeros((q, self.topn), np.uint64),
               "weights": np.zeros((q, self.topn), np.float64)}
        return ids, offs, f, out

    def search(self, ids, offsets, features, sources=None, t_start=None, t_end=None, quality=None, feature_class=None):
        self._use(feature_class)
        ids, offs, f, out = self._queries(ids, offsets, features)
        a = self._attrs(len(ids), sources, t_start, t_end)
        q = self._quality(len(f), quality)
        if q is not None:
            rc = self._L.ofs_search_quality(self._h, len(ids), _p(ids), _p(offs), _p(q),
                                            *(map(_p, a) if a else (None,) * 3), _p(f), _p(out["counts"]),
                                            _p(out["winners"]), _p(out["weights"]), self.threads)
        elif a is None:
            rc = self._L.ofs_search(self._h, len(ids), _p(ids), _p(offs), _p(f), _p(out["counts"]),
                                    _p(out["winners"]), _p(out["weights"]), self.threads)
        else:
            rc = self._L.ofs_search_attr(self._h, len(ids), _p(ids), _p(offs), *map(_p, a), _p(f), _p(out["counts"]),
                                         _p(out["winners"]), _p(out["weights"]), self.threads)
        if rc:
            raise ValueError("invalid search request")
        return out

    def associate(self, ids, offsets, features, sources=None, t_start=None, t_end=None, quality=None, feature_class=None):
        self._use(feature_class)
        ids, offs, f, out = self._queries(ids, offsets, features)
        a = self._attrs(len(ids), sources, t_start, t_end)
        q = self._quality(len(f), quality)
        out["track_ids"] = np.zeros(len(ids), np.uint64)
        out["merged"] = np.zeros(len(ids), np.uint8)
        res = [_p(out[k]) for k in ("counts", "winners", "weights", "track_ids", "merged")]
        if q is not None:
            rc = self._L.ofs_associate_quality(self._h, len(ids), _p(ids), _p(offs), _p(q),
                                               *(map(_p, a) if a else (None,) * 3), _p(f), *res, self.threads)
        elif a is None:
            rc = self._L.ofs_associate(self._h, len(ids), _p(ids), _p(offs), _p(f), *res, self.threads)
        else:
            rc = self._L.ofs_associate_attr(self._h, len(ids), _p(ids), _p(offs), *map(_p, a), _p(f), *res,
                                            self.threads)
        if rc:
            raise ValueError("invalid associate request")
        return out

    def search_owned(self, ids, each=False, feature_class=None):
        """owned_track_distances + TopNVoting::winners for stored tracks; each=True: once per id."""
        self._use(feature_class)
        ids = np.ascontiguousarray(ids, dtype=np.uint64)
        q = len(ids)
        out = {"counts": np.zeros(q, np.int32), "winners": np.zeros((q, self.topn), np.uint64),
               "weights": np.zeros((q, self.topn), np.float64)}
        rc = self._L.ofs_search_owned(self._h, q, _p(ids), int(bool(each)), _p(out["counts"]), _p(out["winners"]),
                                      _p(out["weights"]), self.threads)
        if rc:
            raise ValueError("invalid owned search request")
        return out

    def merge_owned(self, dest_ids, src_ids, remove=True):
        """merge_owned for each pair (dest_ids[i], src_ids[i]) in order."""
        d = np.ascontiguousarray(dest_ids, dtype=np.uint64)
        s = np.ascontiguousarray(src_ids, dtype=np.uint64)
        if len(d) != len(s):
            raise ValueError("dest_ids and src_ids must have the same length")
        if self._L.ofs_merge_owned(self._h, len(d), _p(d), _p(s), int(bool(remove))):
            raise ValueError("invalid merge request")

    def fetch(self, ids, remove=False, feature_class=None):
        self._use(feature_class)
        ids = np.ascontiguousarray(ids, dtype=np.uint64)
        counts = np.zeros(len(ids), np.int32)
        feats = np.zeros((len(ids), self.K, self.D), np.float32)
        self._L.ofs_fetch(self._h, len(ids), _p(ids), int(bool(remove)), _p(counts), _p(feats))
        return counts, feats

    def fetch_quality(self, ids, remove=False, feature_class=None):
        """(counts, features, qualities[n][K]) of a quality store, rows in the track's order (best first)."""
        self._use(feature_class)
        ids = np.ascontiguousarray(ids, dtype=np.uint64)
        counts = np.zeros(len(ids), np.int32)
        feats = np.zeros((len(ids), self.K, self.D), np.float32)
        qual = np.zeros((len(ids), self.K), np.float32)
        if self._L.ofs_fetch_quality(self._h, len(ids), _p(ids), int(bool(remove)), _p(counts), _p(feats), _p(qual)) < 0:
            raise ValueError("fetch_quality() needs a quality store")
        return counts, feats, qual

    def merge_history(self, ids):
        """The merge history of each of the tracks `ids` (an empty array where an id is not stored)."""
        ids = np.ascontiguousarray(ids, dtype=np.uint64)
        lens = np.zeros(len(ids), np.int32)
        total = self._L.ofs_merge_history(self._h, len(ids), _p(ids), _p(lens), 0, None)
        if total < 0:
            raise ValueError("merge_history() needs a quality store")
        out = np.zeros(max(1, total), np.uint64)
        self._L.ofs_merge_history(self._h, len(ids), _p(ids), _p(lens), total, _p(out))
        offs = np.concatenate([[0], np.cumsum(lens)])
        return [out[offs[i]: offs[i + 1]].copy() for i in range(len(ids))]

    def attributes(self, ids):
        """(sources, t_start, t_end) of the tracks `ids` (0 where an id is not stored) of a gated store."""
        ids = np.ascontiguousarray(ids, dtype=np.uint64)
        src, t0, t1 = np.zeros(len(ids), np.uint64), np.zeros(len(ids), np.int64), np.zeros(len(ids), np.int64)
        if self._L.ofs_fetch_attr(self._h, len(ids), _p(ids), _p(src), _p(t0), _p(t1)) < 0:
            raise ValueError("attributes() needs a gated store")
        return src, t0, t1

    def find_baked(self, now, baked_period=0):
        """The ids (store order) of the tracks of a gated store with now > t_end + baked_period, exactly."""
        n = self.size()
        out = np.zeros(max(1, n), np.uint64)
        total = self._L.ofs_find_baked(self._h, int(now), int(baked_period), n, _p(out))
        if total < 0:
            raise ValueError("find_baked() needs a gated store")
        return out[:total]

    def associate_store(self, src, ids, remove=True, feature_class=None):
        """fetch_tracks(ids) of the oracle store `src`, then one associate of this store with those tracks as its
        queries (each merged into its winner with its list and history, or added whole); remove=True takes them out of
        `src`.  Returns the associate dict."""
        self._use(feature_class)
        src._use(feature_class)
        ids = np.ascontiguousarray(ids, dtype=np.uint64)
        q = len(ids)
        out = {"counts": np.zeros(q, np.int32), "winners": np.zeros((q, self.topn), np.uint64),
               "weights": np.zeros((q, self.topn), np.float64), "track_ids": np.zeros(q, np.uint64),
               "merged": np.zeros(q, np.uint8)}
        if self._L.ofs_associate_store(self._h, src._h, q, _p(ids), int(bool(remove)),
                                       *(_p(v) for v in out.values()), self.threads):
            raise ValueError("invalid associate_store request")
        return out

    def size(self):
        return int(self._L.ofs_size(self._h))

    def ids(self):
        n = self.size()
        out = np.zeros(max(1, n), np.uint64)
        self._L.ofs_ids(self._h, n, _p(out))
        return out[:n]
