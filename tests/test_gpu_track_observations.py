"""The state the apply stage leaves in the device store, track by track, against the oracle: the Kalman mean and covariance
of all four tracker kinds, and for the visual trackers each track's kept observations (order, feature flag, quality, the
f32 arena row and its norm), the arena's block bookkeeping and the BF16 copy of every kept row.  The device state is read
from Tracker.save(), whose sections follow DESIGN §3b.

The workloads vary what the end-to-end tests keep fixed: qualities with ties and on the collect / use thresholds, missing
features, boxes on the area gate, and short idle limits, so that feature blocks are freed and reused every frame.  One
constructed case fills a block with NaN, inf and overflowing rows and hands it to a new track: the stale rows must not
reach the screen or the dense weight sums."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

F32MAX = float(np.finfo(np.float32).max)
MAX_SECTIONS = 48
MAHA, IOU = 0, 1
KST_FLOATS = 32   # Kalman state row of the store: 30 floats padded to 128 bytes


@pytest.fixture(scope="module")
def eng():
    import similari_b200.engine as e
    from similari_b200._lib import lib

    if lib().sb200_device_count() <= 0:
        pytest.fail("no CUDA device: the gpu-marked tests must run on an H100")
    return e


def both(eng, oracle, **kw):
    from similari_b200._lib import default_options

    return eng.Tracker(default_options(**kw)), oracle.Tracker(oracle.make_options(**kw))


def below(x):
    """The f32 value one ulp below x."""
    return np.nextafter(np.float32(x), np.float32(0))


# ------------------------------------------------------------------------------------------------ device state reader
def _blob_header():
    from similari_b200._lib import Options

    class BlobHeader(C.Structure):
        _fields_ = [("magic", C.c_uint32), ("version", C.c_uint32), ("type", C.c_uint32), ("n_sections", C.c_uint32),
                    ("total_bytes", C.c_uint64), ("opts", Options),
                    ("feature_history", C.c_int32), ("hist_len", C.c_int32), ("d8", C.c_int32), ("n_scenes", C.c_int32),
                    ("seen_features", C.c_int32), ("adapt_dense", C.c_int32), ("auto_waste_counter", C.c_int32),
                    ("auto_waste_periodicity", C.c_int32), ("scene_cap", C.c_int32), ("track_cap", C.c_int32),
                    ("pad0", C.c_int32), ("pad1", C.c_int32),
                    ("live_total", C.c_int64), ("blk_total", C.c_int64), ("free_total", C.c_int64),
                    ("wasted_count", C.c_int64), ("revealed", C.c_int64), ("hpool_top", C.c_int64),
                    ("hpool_free", C.c_int64), ("hpool_cap", C.c_int64), ("id_counter", C.c_uint64),
                    ("sec_off", C.c_uint64 * MAX_SECTIONS), ("sec_bytes", C.c_uint64 * MAX_SECTIONS)]

    return BlobHeader


class BlobScene(C.Structure):
    _fields_ = [("scene_id", C.c_uint64), ("epoch", C.c_uint32), ("n_tracks", C.c_int32), ("n_hidden", C.c_int32),
                ("arena_top", C.c_int32)]


def read_state(blob):
    """{scene_id: columns} of a tracker blob without box history or feature history.  Track columns hold the scene's
    live tracks in store order; feat / feat_bf16 / fnorm2 / blk_owner its arena blocks [0, arena_top); free its free
    list.  Sections are located through the header's table, in the order of DESIGN §3b."""
    H = _blob_header()
    h = H.from_buffer_copy(blob[: C.sizeof(H)].tobytes())
    assert (h.magic, h.version, h.type) == (0x42534253, 1, 1)
    assert h.hist_len == 1 and h.feature_history == 0, "the reader knows the layout without histories only"
    o = h.opts
    K, d8 = max(1, o.visual_max_observations), h.d8
    visual = o.kind >= 2
    # (name, type, elements per row; 0: one element, read as a vector)
    per_track = [("id", np.uint64, 0), ("epoch", np.uint32, 0), ("length", np.uint32, 0), ("custom", np.int64, 0),
                 ("vt", np.int8, 0), ("pred", np.float32, 6), ("obs", np.float32, 6), ("radius", np.float32, 0),
                 ("kst", np.float32, KST_FLOATS)]
    if o.positional_kind == IOU:
        per_track.append(("vert", np.float64, 8))
    per_block, per_free = [], []
    if visual:
        per_track += [("obs_phys", np.uint8, K), ("obs_hasf", np.uint8, K), ("obs_q", np.float32, K),
                      ("obs_n", np.uint8, 0), ("feat_cnt", np.uint8, 0), ("fblk", np.int32, 0)]
        per_block = [("feat", np.float32, K * d8), ("feat_bf16", np.uint16, K * d8), ("fnorm2", np.float32, K),
                     ("blk_owner", np.int32, 0)]
        per_free = [("free", np.int32, 0)]
    raw = np.ascontiguousarray(blob)
    table = (BlobScene * h.n_scenes).from_buffer_copy(raw[h.sec_off[0]: h.sec_off[0] + h.sec_bytes[0]].tobytes())
    counts = {"track": [s.n_tracks for s in table], "block": [s.arena_top for s in table],
              "free": [s.arena_top - s.n_tracks if visual else 0 for s in table]}
    cols, sec = {}, 1
    for unit, spec in (("track", per_track), ("block", per_block), ("free", per_free)):
        rows = sum(counts[unit])
        for name, dt, w in spec:
            n = rows * max(w, 1)
            assert h.sec_bytes[sec] == n * np.dtype(dt).itemsize, name
            a = np.frombuffer(raw, dtype=dt, count=n, offset=int(h.sec_off[sec]))
            cols[name] = (unit, a.reshape(rows, w) if w else a)
            sec += 1
    out = {}
    pre = {u: np.concatenate([[0], np.cumsum(c)]).astype(int) for u, c in counts.items()}
    for i, s in enumerate(table):
        sc = {"scene_epoch": s.epoch, "n_tracks": s.n_tracks, "arena_top": s.arena_top}
        for name, (unit, a) in cols.items():
            sc[name] = a[pre[unit][i]: pre[unit][i + 1]]
        if visual:
            sc["feat"] = sc["feat"].reshape(-1, K, d8)
            sc["feat_bf16"] = sc["feat_bf16"].reshape(-1, K, d8)
        out[int(s.scene_id)] = sc
    return out


# ------------------------------------------------------------------------------------------------ comparisons
def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def same_f32(a, b):
    """Bit-equal, or NaN on both sides (the payload of a NaN is not part of the result)."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return bool(np.all((bits(a) == bits(b)) | (np.isnan(a) & np.isnan(b))))


def bf16_rne(x):
    """uint16 bits of RNE(x) to BF16 for finite and infinite x; NaN lanes are flagged separately."""
    u = bits(x).astype(np.uint64)
    return ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16), np.isnan(x)


KALMAN_PAIRS = [(i, j) for i in range(5) for j in ((i, i), (i, i + 5), (i + 5, i), (i + 5, i + 5))]


def check_kalman(s30, s110, where):
    """The device's 30 floats against the oracle's mean[10] + P[10][10]: the mean and the four entries of every 2 x 2
    (position, velocity) block bit-equal, every other covariance entry exactly 0."""
    assert np.array_equal(bits(s30[:, :10]), bits(s110[:, :10])), where
    P = s110[:, 10:].reshape(-1, 10, 10)
    rest = np.ones((10, 10), bool)
    for c, (i, (r, q)) in enumerate(KALMAN_PAIRS):
        assert np.array_equal(bits(s30[:, 10 + c]), bits(P[:, r, q])), (where, r, q)
        rest[r, q] = False
    assert np.all(P[:, rest] == 0.0), where


def oracle_live(o, sid, max_idle):
    """Store positions of the oracle's tracks with epoch + max_idle >= the scene's epoch: the tracks the device still
    holds (it drops the others at the end of the frame in which they expire, the oracle at its next collection point)."""
    cur = o.current_epoch(sid)
    idle = o.idle_tracks(sid)
    ep = {int(i): int(e) for i, e in zip(idle["ids"], idle["epochs"])}
    ids = o.scene_tracks(sid)["ids"]
    return [j for j, i in enumerate(ids) if ep.get(int(i), cur) + max_idle >= cur]


def check_state(g, o, opts_kw, scene_ids, where):
    """Every check of the device store against the oracle, per scene, matched by track id.  Returns the blob state."""
    kind, max_idle = opts_kw["kind"], opts_kw["max_idle_epochs"]
    visual = kind >= 2
    st = read_state(g.save()) if visual else None
    for sid in map(int, scene_ids):
        dg, do = g.scene_tracks(sid), o.scene_tracks(sid)
        live = oracle_live(o, sid, max_idle)
        w = (where, sid)
        assert dg["ids"].tolist() == do["ids"][live].tolist(), w
        check_kalman(dg["states"], do["states"][live], w)
        if not visual:
            continue
        s = st[sid]
        assert s["id"].tolist() == dg["ids"].tolist() and s["scene_epoch"] == o.current_epoch(sid), w
        assert np.array_equal(s["kst"][:, :30], dg["states"]), w
        ob = o.scene_observations(sid)
        n_obs, hasf, q, feats, norm2 = (ob[k][live] for k in ("n_obs", "has_feat", "quality", "feats", "norm2"))
        assert s["obs_n"].tolist() == n_obs.tolist(), w
        assert s["feat_cnt"].tolist() == do["feat_counts"][live].tolist(), w
        # arena: owned blocks and the free list partition [0, arena_top); every owner is its track
        top, fblk, owner, free = s["arena_top"], s["fblk"], s["blk_owner"], s["free"]
        assert sorted(fblk.tolist() + free.tolist()) == list(range(top)), w
        assert np.array_equal(owner[fblk], np.arange(len(fblk))), w
        assert np.all(owner[free] == -1), w
        for t in range(len(fblk)):
            on = int(n_obs[t])
            assert np.array_equal(s["obs_hasf"][t, :on], hasf[t, :on]), (w, t)
            assert np.array_equal(bits(s["obs_q"][t, :on]), bits(q[t, :on])), (w, t)
            kept = [k for k in range(on) if hasf[t, k]]
            phys = s["obs_phys"][t, kept].astype(int)
            assert len(set(phys.tolist())) == len(kept), (w, t)
            assert int(s["feat_cnt"][t]) == len(kept), (w, t)
            for k, p in zip(kept, phys):
                row = s["feat"][fblk[t], p]
                assert same_f32(row, feats[t, k]), (w, t, k)
                assert same_f32(s["fnorm2"][fblk[t], p], norm2[t, k]), (w, t, k)
                want, nan = bf16_rne(row)
                got = s["feat_bf16"][fblk[t], p]
                assert np.array_equal(got[~nan], want[~nan]), (w, t, k)
                assert np.all((got[nan] & 0x7F80) == 0x7F80) and np.all(got[nan] & 0x7F), (w, t, k)
    return st


def check_outputs(rg, ro, where):
    for key in ("ids", "epochs", "lengths", "voting_types"):
        assert np.array_equal(np.asarray(rg[key]).astype(np.uint64), ro[key].astype(np.uint64)), (where, key)


# ------------------------------------------------------------------------------------------------ workloads
class ObservationWorkload:
    """Workload frames with the inputs that steer the observation lists: qualities from a small set (ties are the rule)
    that holds the collect and use thresholds and the f32 values one ulp below them, about a fifth of the detections
    without a feature, and about a sixth of the objects sized onto the area gate (h * h * aspect == min_area), which the
    size jitter moves them across."""

    Q_COLLECT, Q_USE, MIN_AREA = 0.5, 0.8, 3000.0

    def __init__(self, n_scenes, n_objects, d, seed):
        from similari_b200.workload import CONFIGS, Workload

        cfg = dataclasses.replace(CONFIGS["cfg5"], name="observations", n_scenes=n_scenes, n_objects=n_objects,
                                  oriented=False, feature_dim=d, canvas=(1500.0, 1000.0), drop_frac=0.2,
                                  fresh_frac=0.12, seed=seed)
        self.wl = Workload(cfg)
        self.rng = np.random.default_rng(seed ^ 0x0B5E)
        gate = self.rng.random(self.wl.h.shape) < 0.17
        self.wl.h[gate] = np.sqrt(np.float32(self.MIN_AREA) / self.wl.a[gate]).astype(np.float32)
        self.qset = np.array([0.3, 0.5, 0.5, 0.8, 0.8, 1.0, 1.0, below(self.Q_COLLECT), below(self.Q_USE)], np.float32)

    def next_frame(self):
        f = self.wl.next_frame()
        n = len(f["boxes"])
        f["quality"] = self.rng.choice(self.qset, n).astype(np.float32)
        f["has_feature"] = (self.rng.random(n) >= 0.2).astype(np.uint8)
        return f

    @classmethod
    def options(cls, kind, K, d, vis, path, max_idle, min_track_length):
        dense = path.startswith("dense")
        thr = (F32MAX if vis == 0 else -1.0) if dense else (0.7 if vis == 0 else 0.2)   # dense: a threshold that cuts nothing
        return dict(kind=kind, positional_kind=IOU, iou_threshold=0.3, max_idle_epochs=max_idle, visual_kind=vis,
                    visual_threshold=thr, feature_dim=d, visual_max_observations=K, visual_min_votes=min(2, K),
                    visual_minimal_track_length=min_track_length, min_confidence=0.1,
                    visual_minimal_area=cls.MIN_AREA, visual_minimal_quality_use=cls.Q_USE,
                    visual_minimal_quality_collect=cls.Q_COLLECT)


def predict_both(g, o, f, **kw):
    args = (f["scene_ids"], f["det_offsets"], f["boxes"])
    fk = dict(features=f.get("features"), has_feature=f.get("has_feature"), quality=f.get("quality"))
    return g.predict_batch(*args, **fk, **kw), o.predict_batch(*args, **fk)


def set_path(monkeypatch, path):
    monkeypatch.setenv("SB200_VIS_KERNEL", "dense" if path.startswith("dense") else path)
    if path == "dense-generic":
        monkeypatch.setenv("SB200_DENSE_GENERIC", "1")


KS = [1, 2, 3, 5, 7, 8]
D_OF_K = {1: 60, 2: 32, 3: 64, 5: 128, 7: 60, 8: 64}
PATHS = ["simt", "tc16", "tc8", "dense"]
CASES = [(K, kind, path) for K in KS for kind in (2, 3) for path in PATHS + (["dense-generic"] if K <= 5 else [])]
FRAMES = 18


def _case(K, kind, path):
    d = D_OF_K[K]
    vis = (K + kind) % 2
    opts = ObservationWorkload.options(kind, K, d, vis, path, max_idle=1 + (K + kind) % 2,
                                       min_track_length=2 if K >= 5 else 1)
    wl = ObservationWorkload(1 if kind == 2 else 3, 140 if kind == 2 else 70, d, 0x5EED7000 + 97 * K + 13 * kind)
    return opts, wl


@pytest.mark.parametrize("K,kind,path", CASES, ids=[f"K{c[0]}-k{c[1]}-{c[2]}" for c in CASES])
def test_track_state_matches_oracle(eng, oracle, K, kind, path, monkeypatch):
    """Frame after frame: the SortTrack columns, and the whole device store of every scene (Kalman states, observation
    lists, arena rows, norms, BF16 copies, block bookkeeping) against the oracle."""
    set_path(monkeypatch, path)
    opts, wl = _case(K, kind, path)
    g, o = both(eng, oracle, **opts)
    for fr in range(FRAMES):
        f = wl.next_frame()
        rg, ro = predict_both(g, o, f)
        check_outputs(rg, ro, fr)
        check_state(g, o, opts, f["scene_ids"], fr)
    wc, sc = g.work_counters(), g.screen_counters()
    if path != "simt":   # the forced path ran
        assert wc["tc_frames"] >= FRAMES - 2, wc
    if path == "tc8":
        assert sc["fp8_frames"] >= FRAMES - 2, sc
    if path == "tc16":
        assert sc["bf16_frames"] >= FRAMES - 2, sc


def test_frames_in_flight_leave_the_oracle_state(eng, oracle, monkeypatch):
    """Frames enqueued back to back without waiting (four in flight at most): after sync() every frame's columns and the
    final store are the frame-by-frame oracle's."""
    from similari_b200._lib import pinned_empty

    set_path(monkeypatch, "tc8")
    opts, wl = _case(3, 3, "tc8")
    g, o = both(eng, oracle, **opts)
    frames = [wl.next_frame() for _ in range(14)]
    ref, outs = [], []
    for f in frames:
        total = len(f["boxes"])
        out = {"ids": pinned_empty((total,), np.uint64), "epochs": pinned_empty((total,), np.uint32),
               "lengths": pinned_empty((total,), np.uint32), "voting_types": pinned_empty((total,), np.uint8)}
        rg, ro = predict_both(g, o, f, out=out, wait=False)
        outs.append(rg)
        ref.append(ro)
    g.sync()
    for fr, (rg, ro) in enumerate(zip(outs, ref)):
        check_outputs(rg, ro, fr)
    check_state(g, o, opts, frames[-1]["scene_ids"], "final")


# ------------------------------------------------------------------------------------------------ Kalman across scales
class ScaleSweep:
    """Objects with heights from 1e-3 to 1e4 on one row, each spaced from the next by more than both their sizes, moving
    by a few percent of their own size per frame (so IoU and Mahalanobis matching work at every scale); a tenth of the
    detections are missed each frame.  Oriented boxes carry an angle, axis-aligned ones none (NaN: 0 in the state)."""

    def __init__(self, n_scenes, n, oriented, d, seed):
        r = self.rng = np.random.default_rng(seed)
        self.h = np.tile(np.logspace(-3, 4, n), (n_scenes, 1))
        self.a = r.uniform(0.3, 0.8, (n_scenes, n))
        gap = 1.5 * (self.h[:, :-1] + self.h[:, 1:])
        self.x = np.concatenate([np.zeros((n_scenes, 1)), np.cumsum(gap, axis=1)], axis=1)
        self.y = 0.5 * self.h
        self.ang = r.uniform(-1.0, 1.0, (n_scenes, n)) if oriented else None
        self.conf = r.uniform(0.3, 1.0, (n_scenes, n))
        self.cent = r.standard_normal((n_scenes, n, d)) if d else None
        self.d, self.fr = d, 0

    def next_frame(self):
        r, S, n = self.rng, *self.h.shape
        if self.fr:
            self.x += r.normal(0, 0.03, (S, n)) * self.h
            self.y += r.normal(0, 0.03, (S, n)) * self.h
            self.h *= r.uniform(0.98, 1.02, (S, n))
            if self.ang is not None:
                self.ang += r.normal(0, 0.02, (S, n))
        self.fr += 1
        boxes, feats, offs = [], [], [0]
        for s in range(S):
            idx = np.flatnonzero(r.random(n) >= 0.1)
            r.shuffle(idx)
            b = np.stack([self.x[s, idx], self.y[s, idx], self.ang[s, idx] if self.ang is not None else np.full(len(idx), np.nan),
                          self.a[s, idx], self.h[s, idx], self.conf[s, idx]], axis=1)
            boxes.append(b.astype(np.float32))
            if self.d:
                feats.append((self.cent[s, idx] + 0.02 * r.standard_normal((len(idx), self.d))).astype(np.float32))
            offs.append(offs[-1] + len(idx))
        return {"scene_ids": np.arange(S, dtype=np.uint64), "det_offsets": np.asarray(offs, np.int32),
                "boxes": np.concatenate(boxes), "features": np.concatenate(feats) if self.d else None}


@pytest.mark.parametrize("kind", [0, 1, 2, 3])
@pytest.mark.parametrize("pos", [MAHA, IOU])
@pytest.mark.parametrize("oriented", [False, True])
def test_kalman_state_across_scales_matches_oracle(eng, oracle, kind, pos, oriented):
    d = 32 if kind >= 2 else 0
    opts = dict(kind=kind, positional_kind=pos, iou_threshold=0.3, max_idle_epochs=2)
    if kind >= 2:
        opts.update(visual_kind=0, visual_threshold=0.7, feature_dim=d, visual_max_observations=3, visual_min_votes=2,
                    visual_minimal_track_length=1)
    g, o = both(eng, oracle, **opts)
    wl = ScaleSweep(1 if kind in (0, 2) else 3, 40, oriented, d, 0x5CA1E + 8 * kind + 2 * pos + oriented)
    merged = 0
    for fr in range(12):
        f = wl.next_frame()
        rg, ro = predict_both(g, o, f)
        check_outputs(rg, ro, fr)
        check_state(g, o, opts, f["scene_ids"], fr)
        merged += int(np.sum(ro["lengths"] > 1))
    assert merged > 200   # the update path ran at every scale, not only initiate


# ------------------------------------------------------------------------------------------------ poisoned reused blocks
POISON_K, POISON_D = 3, 64


def _poison_rows(rng):
    nan_row = rng.standard_normal(POISON_D).astype(np.float32)
    nan_row[3] = np.nan
    inf_row = rng.standard_normal(POISON_D).astype(np.float32)
    inf_row[5] = np.inf
    huge_row = np.full(POISON_D, 1.3e18, np.float32)   # |x|^2 ~ 1.1e38 > FLT_MAX / 4, finite
    return [nan_row, inf_row, huge_row]


# Euclidean dense is left out: under the f32::MAX threshold the overflowing row, stored in a live track, lies ~1e19 from
# every candidate, and BestFit's weights (max_dist - d, track/voting/best.rs) then tie for every pair of the scene.
POISON_CASES = [("dense", 1), ("tc8", 0), ("tc8", 1), ("tc16", 0), ("tc16", 1)]


@pytest.mark.parametrize("path,vis", POISON_CASES, ids=[f"{p}-{'cos' if v else 'euclid'}" for p, v in POISON_CASES])
def test_reused_block_with_poisoned_rows(eng, oracle, path, vis, monkeypatch):
    """Track P collects a NaN, an inf and an overflowing feature, one per physical slot of its block, then expires; the
    next new track Q takes the block (checked in the blob: same block, the three rows still there) and keeps at most
    one feature of its own there for several frames.  While P lives, the oracle decides whatever the fallback rules do;
    once its block belongs to Q, the dense path takes no scene back to the exact kernels, and tc8 screens every frame on
    e4m3 operands."""
    set_path(monkeypatch, path)
    rng = np.random.default_rng(0xBAD0 + vis)
    K, d, n = POISON_K, POISON_D, 40
    opts = dict(kind=2, positional_kind=IOU, iou_threshold=0.3, max_idle_epochs=1, visual_kind=vis,
                visual_threshold=(F32MAX if vis == 0 else -1.0) if path == "dense" else (0.7 if vis == 0 else 0.2),
                feature_dim=d, visual_max_observations=K, visual_min_votes=2, visual_minimal_track_length=1,
                min_confidence=0.1, visual_minimal_quality_use=0.9, visual_minimal_quality_collect=0.5)
    g, o = both(eng, oracle, **opts)
    grid = [(60.0 + 150.0 * (i % 8), 60.0 + 150.0 * (i // 8)) for i in range(n + 2)]
    cent = rng.standard_normal((n + 2, d)).astype(np.float32)
    cent /= np.linalg.norm(cent, axis=1, keepdims=True)
    poison = _poison_rows(rng)
    P, Q = n, n + 1
    # frame -> the extra detection: (object, feature or None, quality)
    # P's and Q's features are stored (quality >= collect) but never query (quality < use): both merge by position alone
    script = {0: (P, poison[0], 0.6), 1: (P, poison[1], 0.6), 2: (P, poison[2], 0.6), 5: (Q, None, 0.6),
              6: (Q, "own", 0.6), 7: (Q, None, 0.6), 8: (Q, "own", 0.4), 9: (Q, "own", 0.6), 10: (Q, "own", 0.6),
              11: (Q, "own", 0.6)}
    p_id = q_id = p_blk = None
    q_written = set()   # physical slots of the block that Q has stored a feature in
    fb_after_p = fp8_after_p = None
    for fr in range(12):
        objs = list(range(n)) + ([script[fr][0]] if fr in script else [])
        boxes = np.array([oracle.box(*grid[i], None, 0.5, 60.0, 0.9) for i in objs], np.float32)
        feats = cent[objs] + np.float32(0.02) * rng.standard_normal((len(objs), d)).astype(np.float32)
        hasf = np.ones(len(objs), np.uint8)
        qual = np.ones(len(objs), np.float32)
        if fr in script:
            _, feat, q = script[fr]
            qual[-1] = q
            if feat is None:
                hasf[-1] = 0
            elif isinstance(feat, np.ndarray):
                feats[-1] = feat
        f = {"scene_ids": np.zeros(1, np.uint64), "det_offsets": np.array([0, len(objs)], np.int32), "boxes": boxes,
             "features": feats, "has_feature": hasf, "quality": qual}
        rg, ro = predict_both(g, o, f)
        check_outputs(rg, ro, fr)
        st = check_state(g, o, opts, [0], fr)[0]
        ids = st["id"].tolist()
        if fr == 0:
            p_id = int(ro["ids"][-1])
        if fr == 2:   # P's three slots hold the three poisoned rows
            t = ids.index(p_id)
            p_blk = int(st["fblk"][t])
            assert int(st["obs_n"][t]) == K and int(st["feat_cnt"][t]) == K
            assert sorted(st["obs_phys"][t].tolist()) == list(range(K))
            for p, row in enumerate(poison):
                assert same_f32(st["feat"][p_blk, p], row), p
        if fr == 4:   # P expired at the end of this frame: its block is on the free list
            assert p_id not in ids and p_blk in st["free"].tolist()
            fb_after_p = g.work_counters()["dense_fallback_scenes"]
            fp8_after_p = g.screen_counters()["fp8_frames"]
        if fr == 5:
            q_id = int(ro["ids"][-1])
            assert q_id != p_id and int(ro["lengths"][-1]) == 1
        if fr >= 5:   # Q owns P's block; the slots Q has not written still hold P's rows
            t = ids.index(q_id)
            assert int(st["fblk"][t]) == p_blk, fr
            q_written |= {int(st["obs_phys"][t, k]) for k in range(int(st["obs_n"][t])) if st["obs_hasf"][t, k]}
            stale = [p for p in range(K) if p not in q_written]
            if fr <= 8:   # no feature at 5, one at 6, none stored at 7 (missing) and 8 (below the collect threshold)
                assert len(stale) == (K if fr == 5 else K - 1), (fr, q_written)
            for p in stale:
                assert same_f32(st["feat"][p_blk, p], poison[p]), (fr, p)
    assert p_blk is not None and q_id is not None
    if path == "dense":
        assert g.work_counters()["dense_fallback_scenes"] == fb_after_p
    if path == "tc8":
        assert g.screen_counters()["fp8_frames"] - fp8_after_p == 7
