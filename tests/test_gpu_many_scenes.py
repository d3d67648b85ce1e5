"""The batch trackers along the scene axis, frame by frame against the CPU oracle: requests past the one-CTA frame
tables (1,024 scenes: the carried prefix sums of frame_setup_kernel; 512: apply_rank_kernel's new-track prefix), past
the 65,535 blocks a grid's y (or z) dimension holds (the per-scene cost, metadata and own-area launches stride over the
scenes), with scenes joining, leaving and reordering between frames, and across a save / load.

Each frame's ids, epochs, lengths and voting types must be the oracle's, its predicted and observed boxes bit-equal
(NaN normalised), and active_tracks() the same; at the end wasted() and the scene_tracks() of scenes on both sides of
every boundary (first, last, 511 / 512, 1023 / 1024, 65,534 / 65,535).  The frames are ragged: about one scene in ten
is empty (more where a case's device memory would grow past the budget), as many hold one detection, most 2 to 6, and
a few chosen scenes hundreds.

Device memory: every case stays under MEM_BUDGET, measured as the drop in free device memory; the peak is printed.
At 70,001 scenes one visual tracker takes about 3.1 GiB (H100 80 GB): its store keeps at least 64 track rows per scene."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

F32 = np.float32
MEM_BUDGET = 4 << 30
BOUNDARY = (0, 511, 512, 1023, 1024, 65534, 65535)


@pytest.fixture(scope="module")
def eng():
    import similari_b200.engine as e
    from similari_b200._lib import lib

    if lib().sb200_device_count() <= 0:
        pytest.fail("no CUDA device: the gpu-marked tests must run on an H100")
    return e


def _threads():
    try:
        return max(4, min(24, len(os.sched_getaffinity(0))))
    except Exception:
        return 8


class DeviceMemory:
    """Device memory in use since construction (free memory before, less the least seen after each frame)."""

    def __init__(self):
        import torch

        torch.cuda.mem_get_info()   # the context exists before the first reading
        self._info = torch.cuda.mem_get_info
        self.free0 = self._info()[0]
        self.peak = 0

    def sample(self):
        self.peak = max(self.peak, self.free0 - self._info()[0])

    def check(self, what):
        self.sample()
        print(f"{what}: peak device memory {self.peak / 2**30:.2f} GiB")
        assert self.peak < MEM_BUDGET, (what, self.peak)


class Ragged:
    """Seeded ragged multi-scene frames, vectorised over every object of every scene.

    Scene s holds m[s] objects: 0 for a fraction `empty` of the scenes, 1 for about 10 %, else 2..max_m; `big` {scene: m}
    overrides chosen scenes.  A scene's canvas grows with its crowd (400 x 300 up to four objects), so small scenes
    overlap a lot.  Each frame moves every object, replaces `fresh` of them by new identities and drops `drop` of them
    (none in the first frame); frame(order) sends the scenes `order` (indices into scene_ids) in that order, each
    scene's detections shuffled."""

    def __init__(self, n_scenes, seed, dim=0, oriented=False, max_m=6, big=None, scene_ids=None, drop=0.1, fresh=0.05,
                 empty=0.1):
        r = self.rng = np.random.default_rng(seed)
        u = r.random(n_scenes)
        m = np.where(u < empty, 0, np.where(u < empty + 0.1, 1, r.integers(2, max_m + 1, n_scenes)))
        for s, k in (big or {}).items():
            m[s] = k
        self.m = m
        self.n_scenes, self.dim, self.oriented, self.drop, self.fresh = n_scenes, dim, oriented, drop, fresh
        self.scene_ids = (np.arange(n_scenes, dtype=np.uint64) if scene_ids is None
                          else np.ascontiguousarray(scene_ids, dtype=np.uint64))
        self.of = np.repeat(np.arange(n_scenes), m)
        self.scale = np.sqrt(np.maximum(m, 4) / 4.0)[self.of].astype(F32)
        n = len(self.of)
        self.xc, self.yc, self.h, self.a, self.ang, self.conf = (np.zeros(n, F32) for _ in range(6))
        self.cent = np.zeros((n, dim), F32)
        self._fresh(np.arange(n))
        self.frame_no = 0

    @staticmethod
    def _unit(v):
        return (v / np.linalg.norm(v, axis=-1, keepdims=True)).astype(F32)

    def _fresh(self, idx):
        r, k = self.rng, len(idx)
        if k == 0:
            return
        self.xc[idx] = r.uniform(0, 400, k) * self.scale[idx]
        self.yc[idx] = r.uniform(0, 300, k) * self.scale[idx]
        self.h[idx] = r.uniform(40, 160, k)
        self.a[idx] = r.uniform(0.3, 0.8, k)
        self.ang[idx] = r.uniform(-np.pi / 2, np.pi / 2, k)
        self.conf[idx] = r.uniform(0.3, 1.0, k)
        if self.dim:
            self.cent[idx] = self._unit(r.standard_normal((k, self.dim), dtype=F32))

    def frame(self, order=None):
        r, n = self.rng, len(self.of)
        order = np.arange(self.n_scenes) if order is None else np.asarray(order)
        if self.frame_no > 0:
            self.xc += r.normal(0, 2.0, n).astype(F32)
            self.yc += r.normal(0, 2.0, n).astype(F32)
            self.h *= r.uniform(0.98, 1.02, n).astype(F32)
            self.a *= r.uniform(0.98, 1.02, n).astype(F32)
            if self.oriented:
                self.ang += r.normal(0, 0.02, n).astype(F32)
            self._fresh(np.flatnonzero(r.random(n) < self.fresh))
        keep = r.random(n) >= (self.drop if self.frame_no > 0 else 0.0)
        self.frame_no += 1
        rank = np.full(self.n_scenes, -1, np.int64)
        rank[order] = np.arange(len(order))
        rk = rank[self.of]
        sel = np.flatnonzero(keep & (rk >= 0))
        sel = sel[np.lexsort((r.random(len(sel)), rk[sel]))]
        counts = np.bincount(rk[sel], minlength=len(order))
        offs = np.zeros(len(order) + 1, np.int32)
        offs[1:] = np.cumsum(counts)
        boxes = np.stack([self.xc[sel], self.yc[sel], self.ang[sel] if self.oriented else np.full(len(sel), np.nan, F32),
                          self.a[sel], self.h[sel], self.conf[sel]], axis=1).astype(F32)
        feats = None
        if self.dim:
            feats = self._unit(self.cent[sel] + 0.02 * r.standard_normal((len(sel), self.dim), dtype=F32))
        return {"scene_ids": self.scene_ids[order], "det_offsets": offs, "boxes": boxes, "features": feats}


def _nan0(a):
    return np.nan_to_num(a, nan=-7.0)


def _same_frame(rg, ro, ctx):
    for key in ("ids", "epochs", "lengths", "voting_types"):
        bad = int((rg[key] != ro[key]).sum())
        assert bad == 0, (ctx, key, bad)
    for key in ("predicted", "observed"):
        assert np.array_equal(_nan0(rg[key]), _nan0(ro[key])), (ctx, key)


def _same_records(wg, wo, ctx):
    ig, io = np.argsort(wg["ids"], kind="stable"), np.argsort(wo["ids"], kind="stable")
    assert len(ig) == len(io), (ctx, len(ig), len(io))
    for key in ("ids", "scene_ids", "epochs", "lengths"):
        assert np.array_equal(wg[key][ig], wo[key][io]), (ctx, key)
    for key in ("predicted", "observed"):
        assert np.array_equal(_nan0(wg[key][ig]), _nan0(wo[key][io])), (ctx, key)


def _same_scene(g, o, sid, ctx):
    """The device store drops a track at the end of the frame in which it expires, the oracle at its next collection:
    the device holds the oracle's tracks with epoch + max_idle_epochs >= the scene's epoch, in the same order."""
    sid = int(sid)
    sg, so = g.scene_tracks(sid), o.scene_tracks(sid)
    cur, max_idle = o.current_epoch(sid), int(o.opts.max_idle_epochs)
    idle = o.idle_tracks(sid)
    ep = dict(zip(idle["ids"].tolist(), idle["epochs"].tolist()))
    live = [j for j, i in enumerate(so["ids"].tolist()) if ep.get(i, cur) + max_idle >= cur]
    assert g.current_epoch(sid) == cur, (ctx, sid)
    assert sg["ids"].tolist() == so["ids"][live].tolist(), (ctx, sid)
    assert np.array_equal(_nan0(sg["boxes"]), _nan0(so["boxes"][live])), (ctx, sid)
    assert np.array_equal(sg["feat_counts"], so["feat_counts"][live]), (ctx, sid)


def _sample(scene_ids):
    n = len(scene_ids)
    return [scene_ids[i] for i in sorted({i for i in BOUNDARY if i < n} | {n - 1})]


def _pair(eng, oracle, **kw):
    from similari_b200._lib import default_options

    return eng.Tracker(default_options(**kw)), oracle.Tracker(oracle.make_options(**kw), threads=_threads())


def _finish(g, o, sample, ctx, wasted_cap=1 << 20):
    """skip_epochs on the sampled scenes (each call sweeps every slot), then wasted() and the sampled scene stores."""
    for sid in sample:
        _same_scene(g, o, sid, ctx)
    for sid in sample:
        g.skip_epochs(2, int(sid))
        o.skip_epochs(2, int(sid))
    assert g.active_tracks() == o.active_tracks(), ctx
    wg, wo = g.wasted(wasted_cap), o.wasted(wasted_cap)
    _same_records(wg, wo, ctx)
    for sid in sample:
        _same_scene(g, o, sid, ctx)
    return len(wo["ids"])


def _run(g, o, wl, frames, ctx, mem=None, orders=None):
    for fr in range(frames):
        f = wl.frame(None if orders is None else orders[fr])
        rg = g.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=f["features"])
        ro = o.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=f["features"])
        _same_frame(rg, ro, (ctx, fr))
        assert g.active_tracks() == o.active_tracks(), (ctx, fr)
        if mem is not None:
            mem.sample()
    return f


BATCH_SORT_IOU = dict(kind=1, positional_kind=1, iou_threshold=0.3, max_idle_epochs=1)
BATCH_SORT_MAHA = dict(kind=1, positional_kind=0, max_idle_epochs=1)


def _visual(vis_kind=0, dim=32, k=3, **over):
    kw = dict(kind=3, positional_kind=1, iou_threshold=0.3, max_idle_epochs=1, visual_kind=vis_kind,
              visual_threshold=0.7 if vis_kind == 0 else 0.3, feature_dim=dim, visual_max_observations=k,
              visual_min_votes=1, visual_minimal_track_length=1, min_confidence=0.1)
    kw.update(over)
    return kw


KINDS = {
    "batch_sort_iou": (BATCH_SORT_IOU, False, 0),
    "batch_sort_maha_oriented": (BATCH_SORT_MAHA, True, 0),
    "batch_visual_euclidean": (_visual(0, dim=8), False, 8),
    "batch_visual_cosine": (_visual(1, dim=8), False, 8),
}


@pytest.mark.parametrize("kind", list(KINDS))
@pytest.mark.parametrize("n_scenes", [1023, 1024, 1025, 2049, 4097])
def test_past_the_one_cta_frame_tables(eng, oracle, kind, n_scenes):
    """Past 1,024 scenes the frame tables' prefix sums carry from chunk to chunk.  With 2,049 scenes, four scenes of
    513 to 600 detections at 511, 512, 1023 and 1024 also cross the 512-row chunk of the new-track prefix and the
    512-thread strides of the voting kernels.  The store has one row capacity for every scene, which those scenes
    raise for all 2,049 of them: the visual kinds keep 8-wide features to stay within MEM_BUDGET."""
    opts, oriented, dim = KINDS[kind]
    big = {511: 513, 512: 600, 1023: 577, 1024: 530} if n_scenes == 2049 else None
    mem = DeviceMemory()
    g, o = _pair(eng, oracle, **opts)
    wl = Ragged(n_scenes, 0x5CE0000 + n_scenes, dim=dim, oriented=oriented, big=big)
    _run(g, o, wl, 5, (kind, n_scenes), mem)
    assert _finish(g, o, _sample(wl.scene_ids), (kind, n_scenes)) > 0
    mem.check(f"{kind} x {n_scenes} scenes")
    g.close()


@pytest.mark.parametrize("path", ["simt", "tc", "dense", "own_area"])
def test_visual_paths_past_1024_scenes(eng, oracle, path, monkeypatch):
    """Each visual cost path over 2,049 scenes: the exact SIMT kernels, the tensor-core screen (its tile list carried
    across frame_setup_kernel's chunks) with the exact refinement, and the dense tensor-core weight sums with a
    threshold that cuts nothing; and the own-area gate, whose shares come from the scene's boxes on the device."""
    over = {}
    if path == "dense":
        over = dict(visual_kind=1, visual_threshold=-1.0)
    elif path == "own_area":
        over = dict(visual_minimal_own_area_percentage_use=0.6, visual_minimal_own_area_percentage_collect=0.8)
    monkeypatch.setenv("SB200_VIS_KERNEL", "tc" if path == "own_area" else path)
    mem = DeviceMemory()
    g, o = _pair(eng, oracle, **_visual(**over))
    wl = Ragged(2049, 0x5CE1000, dim=32)
    _run(g, o, wl, 5, path, mem)
    wc = g.work_counters()
    if path in ("tc", "own_area", "dense"):
        assert wc["tc_frames"] >= 4, wc
    if path == "dense":   # a scene the dense bounds cannot take falls back alone (to the exact kernels)
        assert wc["dense_fallback_scenes"] < 0.02 * 2049 * 5, wc
    assert _finish(g, o, _sample(wl.scene_ids), path) > 0
    mem.check(f"visual path {path} x 2049 scenes")
    g.close()


def _pad(rows, d8):
    out = np.zeros((len(rows), d8), F32)
    out[:, : rows.shape[1]] = rows
    return out


def _history_run(eng, oracle, n_scenes, frames, hist, dim, seed, big=None, empty=0.1):
    mem = DeviceMemory()
    g, o = _pair(eng, oracle, **_visual(dim=dim, k=2, history_length=hist))
    g.set_feature_history(True)
    wl = Ragged(n_scenes, seed, dim=dim, big=big, empty=empty)
    d8 = (dim + 7) // 8 * 8
    seen = {}
    apply_ms = []
    for fr in range(frames):
        f = wl.frame()
        rg = g.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=f["features"])
        apply_ms.append(g.last_stage_ms()["apply"])
        ro = o.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=f["features"])
        _same_frame(rg, ro, ("history", n_scenes, fr))
        assert g.active_tracks() == o.active_tracks()
        rows = _pad(f["features"], d8)
        for i, tid in enumerate(rg["ids"].tolist()):
            seen.setdefault(tid, []).append(rows[i])
        mem.sample()
    sample = _sample(wl.scene_ids)
    for sid in sample:
        _same_scene(g, o, sid, "history")
        g.skip_epochs(2, int(sid))
        o.skip_epochs(2, int(sid))
    w, wo = g.wasted_visual(), o.wasted(1 << 20)
    _same_records(w, wo, "history")
    for i, tid in enumerate(w["ids"].tolist()):
        exp = seen[tid][-hist:]
        assert int(w["lengths"][i]) == len(seen[tid])
        assert bool(w["feature_present"][i].all()) and len(w["features"][i]) == len(exp), tid
        assert np.array_equal(np.asarray(exp).view(np.uint32), w["features"][i].view(np.uint32)), tid
    mem.check(f"feature history x {n_scenes} scenes")
    print(f"feature history x {n_scenes} scenes: apply stage ms per frame", [round(x, 3) for x in apply_ms])
    g.close()
    return len(w["ids"])


def test_feature_history_past_1024_scenes(eng, oracle):
    """The feature-history pool blocks of new tracks come from the new-track prefix over the earlier scenes
    (apply_rank_kernel, 512 scenes at a time); the wasted records carry each observation's input row."""
    assert _history_run(eng, oracle, 2049, 5, 3, 8, 0x5CE2000, big={511: 520, 512: 513, 1100: 600}) > 1000


def test_feature_history_past_the_grid_limit(eng, oracle):
    """The same at 65,536 scenes, where each CTA of apply_rank_kernel sums the new tracks of every earlier scene."""
    assert _history_run(eng, oracle, 65536, 3, 2, 8, 0x5CE2100, empty=0.8) > 2000


GRID_CASES = {
    "batch_sort_iou": (BATCH_SORT_IOU, None),
    "visual_simt": (_visual(dim=8, k=2), "simt"),
    "visual_tc": (_visual(dim=8, k=2), "tc"),
    # the dense path gives every scene with tracks whole 128-detection tiles of weight sums: 9 scenes in 10 are empty here
    "visual_dense": (_visual(1, dim=8, k=2, visual_threshold=-1.0), "dense"),
    "visual_own_area": (_visual(dim=8, k=2, visual_minimal_own_area_percentage_use=0.6,
                                visual_minimal_own_area_percentage_collect=0.8), None),
}


@pytest.mark.parametrize("case", list(GRID_CASES))
@pytest.mark.parametrize("n_scenes", [65536, 70001])
def test_past_the_grid_limit(eng, oracle, case, n_scenes, monkeypatch):
    """More scenes than a grid's y dimension holds (65,535): 0 to 3 detections per scene, D = 8, K = 2."""
    opts, vk = GRID_CASES[case]
    if vk is not None:
        monkeypatch.setenv("SB200_VIS_KERNEL", vk)
    mem = DeviceMemory()
    g, o = _pair(eng, oracle, **opts)
    wl = Ragged(n_scenes, 0x5CE3000 + n_scenes, dim=opts.get("feature_dim", 0) if opts["kind"] == 3 else 0, max_m=3,
                empty=0.9 if vk == "dense" else 0.1)
    _run(g, o, wl, 3, (case, n_scenes), mem)
    print(f"{case} x {n_scenes} scenes: stage ms of the last frame", g.last_stage_ms())
    if vk in ("tc", "dense"):
        assert g.work_counters()["tc_frames"] >= 2
    assert _finish(g, o, _sample(wl.scene_ids), (case, n_scenes)) > 0
    mem.check(f"{case} x {n_scenes} scenes")
    g.close()


def test_scene_churn_past_the_grid_limit(eng, oracle):
    """Scene ids near 2^64 - 1; each frame sends another subset in another order (the request's scene table is
    rebuilt), and new scenes join mid-run: the store, sized for the first frame's 34,000 scenes, grows to 68,000 slots
    keeping the live rows, and requests of up to 67,000 scenes follow.  Most scenes are empty: the growth holds the old
    and the new store at once."""
    n_univ = 67000
    ids = np.uint64(0xFFFFFFFFFFFFFFFF) - np.arange(n_univ, dtype=np.uint64) * np.uint64(7)
    wl = Ragged(n_univ, 0x5CE4000, dim=8, max_m=3, scene_ids=ids, empty=0.7)
    r = np.random.default_rng(0x5CE4001)
    first, seen = np.arange(34000), np.arange(54000)
    orders = [first,
              r.permutation(np.concatenate([r.permutation(first)[:30000], np.arange(34000, 54000)])),
              r.permutation(np.concatenate([r.permutation(seen)[:47000], np.arange(54000, n_univ)])),
              r.permutation(n_univ),
              r.permutation(n_univ)[:66000]]
    mem = DeviceMemory()
    g, o = _pair(eng, oracle, **_visual(dim=8, k=2))
    _run(g, o, wl, len(orders), "churn", mem, orders=orders)
    sample = [ids[i] for i in sorted({0, 511, 512, 1023, 1024, 33999, 34000, 53999, 54000, 65534, 65535, n_univ - 1})]
    assert _finish(g, o, sample, "churn") > 0
    mem.check("scene churn")
    g.close()


def test_save_and_load_past_the_grid_limit(eng, oracle):
    """A 70,001-scene BatchVisualSort tracker saved after two frames; the original runs two more frames, then (one
    tracker at a time on the device) a tracker loaded from the blob runs the same two: identical results, the
    oracle's."""
    mem = DeviceMemory()
    g, o = _pair(eng, oracle, **_visual(dim=8, k=2))
    wl = Ragged(70001, 0x5CE5000, dim=8, max_m=3)
    _run(g, o, wl, 2, "before save", mem)
    blob = g.save()
    frames, outs = [wl.frame() for _ in range(2)], []
    for fr, f in enumerate(frames):
        args = (f["scene_ids"], f["det_offsets"], f["boxes"])
        outs.append(g.predict_batch(*args, features=f["features"]))
        ro = o.predict_batch(*args, features=f["features"])
        _same_frame(outs[-1], ro, ("original", fr))
        assert g.active_tracks() == o.active_tracks()
        mem.sample()
    sample = _sample(wl.scene_ids)
    for sid in sample:
        _same_scene(g, o, sid, "original")
    n_live, wg = g.active_tracks(), g.wasted(1 << 20)
    _same_records(wg, o.wasted(1 << 20), "original")
    stores = [g.scene_tracks(int(sid)) for sid in sample]
    g.close()
    g2 = eng.Tracker.load(blob)
    for fr, f in enumerate(frames):
        r2 = g2.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=f["features"])
        for key in r2:
            assert np.array_equal(outs[fr][key].view(np.uint8), r2[key].view(np.uint8)), ("loaded", fr, key)
        mem.sample()
    assert g2.active_tracks() == n_live
    for sid, st in zip(sample, stores):
        s2 = g2.scene_tracks(int(sid))
        for key in st:
            assert np.array_equal(st[key].view(np.uint8), s2[key].view(np.uint8)), ("loaded", sid, key)
    _same_records(g2.wasted(1 << 20), wg, "loaded")
    mem.check("save / load x 70001 scenes")
    g2.close()
