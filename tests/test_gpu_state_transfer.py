"""State blob: save / load of whole trackers and export / import of scenes (sb200_tracker_save / _load,
sb200_scenes_export / _import).

A loaded tracker is an exact continuation: fed the same requests as the original it returns the same results, bit for
bit, and answers every query the same way.  A moved scene continues as it would have in place (the sharding parity of
SURVEY 8e): epochs, lengths, voting types and boxes bit-identical, the ids of the tracks that existed at export
unchanged, new tracks the same partition of the detections.  Every comparison is exact (byte views)."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

MAHA, IOU = 0, 1


@pytest.fixture(scope="module")
def eng():
    import similari_b200.engine as e
    from similari_b200._lib import lib

    if lib().sb200_device_count() <= 0:
        pytest.fail("no CUDA device: the gpu-marked tests must run on an H100")
    return e


def _cfg(n_scenes, n_objects, dim, oriented, seed, scene_base=0):
    from similari_b200.workload import CONFIGS, Workload

    cfg = dataclasses.replace(CONFIGS["cfg5"], n_scenes=n_scenes, n_objects=n_objects, feature_dim=dim, oriented=oriented,
                              canvas=(900.0, 600.0), drop_frac=0.25, fresh_frac=0.15, feat_noise=0.05, seed=seed)
    return Workload(cfg, scene_base=scene_base)


def _opts(kind, pos, hist, dim, K, constraints=None, **over):
    from similari_b200._lib import default_options

    kw = dict(kind=kind, positional_kind=pos, iou_threshold=0.2, max_idle_epochs=2, history_length=hist,
              constraints=constraints)
    if kind >= 2:
        kw.update(visual_kind=0, visual_threshold=0.7, feature_dim=dim, visual_max_observations=K, visual_min_votes=1,
                  visual_minimal_track_length=1)
    kw.update(over)
    return default_options(**kw)


def _bytes(a):
    return np.ascontiguousarray(a).tobytes()


def _same(a, b, what=""):
    if isinstance(a, dict):
        assert a.keys() == b.keys(), what
        for k in a:
            _same(a[k], b[k], f"{what}.{k}")
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), what
        for i, (x, y) in enumerate(zip(a, b)):
            _same(x, y, f"{what}[{i}]")
    elif isinstance(a, np.ndarray):
        assert a.shape == b.shape and a.dtype == b.dtype and _bytes(a) == _bytes(b), what
    else:
        assert a == b, what


def _collect(g, fh):
    """wasted records grouped by scene (stable: each scene's records keep their order).  The end-of-frame sweep runs a CTA
    per scene and each appends its expired tracks where a counter places them, so the interleaving of the scenes of one
    frame is not fixed -- not even between two trackers created alike -- while the order within a scene is."""
    w = g.wasted_visual() if fh else g.wasted_history()
    order = np.argsort(w["scene_ids"], kind="stable")
    return {k: (v[order] if isinstance(v, np.ndarray) else [v[i] for i in order]) for k, v in w.items()}


def _queries(g, scenes, fh):
    q = {"epochs": [g.current_epoch(int(s)) for s in scenes], "counts": g.scene_track_counts(scenes),
         "live": g.scene_live_counts(scenes), "idle": [g.idle_tracks(int(s)) for s in scenes],
         "active": g.active_tracks()}
    if fh:
        q["pool"] = g.feature_history_pool()
    return q


def _predict(g, f):
    return g.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=f["features"])


# kind, positional metric, oriented, history_length, feature history, D, K, constraints
CASES = [
    (0, IOU, False, 1, False, 0, 1, None),
    (1, MAHA, True, 5, False, 0, 1, None),
    (1, IOU, False, 100, False, 0, 1, [(1, 3.0), (3, 6.0)]),
    (2, IOU, False, 5, True, 30, 1, None),
    (2, MAHA, True, 100, True, 512, 3, None),
    (3, IOU, True, 1, False, 512, 5, None),
    (3, MAHA, False, 100, True, 512, 3, None),
    (3, IOU, False, 5, True, 30, 5, [(2, 4.0)]),
]


def _case_id(c):
    return f"k{c[0]}-{'iou' if c[1] else 'maha'}{'-or' if c[2] else ''}-h{c[3]}-{'fh' if c[4] else 'nofh'}-D{c[5]}-K{c[6]}" + \
        ("-st" if c[7] else "")


def _make(eng, case):
    kind, pos, oriented, hist, fh, dim, K, cons = case
    g = eng.Tracker(_opts(kind, pos, hist, dim, K, cons))
    if fh:
        g.set_feature_history(True)
    g.set_auto_waste(7)
    wl = _cfg(3 if kind in (1, 3) else 1, 40, dim, oriented, seed=0x5EED7000 + 97 * kind + hist + dim)
    return g, wl


def _save_load(eng, g, where):
    """(blob bytes as a host array, loaded tracker)."""
    if where == "device":
        import torch

        n = g.save_device(0, 0)
        buf = torch.empty(n, dtype=torch.uint8, device="cuda")
        assert g.save_device(buf.data_ptr(), n) == n
        torch.cuda.synchronize()
        h = eng.Tracker.load(buf.data_ptr(), n)
        return buf.cpu().numpy(), h
    blob = g.save()
    return blob, eng.Tracker.load(blob)


def _continue(g, h, frames, fh, scenes):
    for i, f in enumerate(frames):
        _same(_predict(g, f), _predict(h, f), f"frame {i}")
        if i % 3 == 2:
            _same(_collect(g, fh), _collect(h, fh), f"wasted at frame {i}")
        if i % 4 == 1:
            _same(_queries(g, scenes, fh), _queries(h, scenes, fh), f"queries at frame {i}")
    _same(_collect(g, fh), _collect(h, fh), "final wasted")
    _same(_queries(g, scenes, fh), _queries(h, scenes, fh), "final queries")


@pytest.mark.parametrize("variant", ["host", "device", "async", "device_io"])
@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_save_load_is_an_exact_continuation(eng, case, variant):
    from similari_b200._lib import pinned_empty

    fh = case[4]
    g, wl = _make(eng, case)
    frames = [wl.next_frame() for _ in range(32)]
    scenes = frames[0]["scene_ids"]
    for f in frames[:10]:
        _predict(g, f)
    pending = []
    if variant == "async":   # two frames still in flight when the save is called
        for f in frames[10:12]:
            n = int(f["det_offsets"][-1])
            out = {"ids": pinned_empty(n, np.uint64), "epochs": pinned_empty(n, np.uint32),
                   "lengths": pinned_empty(n, np.uint32), "voting_types": pinned_empty(n, np.uint8),
                   "predicted": pinned_empty((n, 6), np.float32), "observed": pinned_empty((n, 6), np.float32)}
            g.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=f["features"], out=out, wait=False)
            pending.append(out)
    elif variant == "device_io":   # device-resident frames on a caller stream the tracker does not join
        import torch

        s = torch.cuda.Stream()
        g.set_stream(s.cuda_stream, join_per_call=False)
        with torch.cuda.stream(s):
            for f in frames[10:12]:
                n = int(f["det_offsets"][-1])
                db = torch.from_numpy(f["boxes"]).cuda()
                df = torch.from_numpy(f["features"]).cuda() if f["features"] is not None else None
                ids = torch.zeros(n, dtype=torch.int64, device="cuda")
                g.predict_batch_device(f["scene_ids"], f["det_offsets"], db.data_ptr(),
                                       df.data_ptr() if df is not None else 0, d_ids=ids.data_ptr())
                pending.append((db, df, ids))
    else:
        for f in frames[10:12]:
            _predict(g, f)
    blob, h = _save_load(eng, g, "device" if variant == "device" else "host")
    if variant == "async":
        assert all(len(o["ids"]) == 0 or o["epochs"].max() > 0 for o in pending)
    # save -> load -> save is the same blob
    assert _bytes(h.save()) == _bytes(blob)
    _continue(g, h, frames[12:], fh, scenes)


@pytest.mark.parametrize("case", [CASES[1], CASES[4], CASES[6]], ids=_case_id)
def test_save_of_a_fresh_tracker(eng, case):
    fh = case[4]
    g, wl = _make(eng, case)
    blob, h = _save_load(eng, g, "host")
    frames = [wl.next_frame() for _ in range(12)]
    _continue(g, h, frames, fh, frames[0]["scene_ids"])


def test_loaded_tracker_keeps_matching_the_oracle(eng, oracle):
    from similari_b200._lib import default_options
    from similari_b200.workload import tracker_options_for

    wl = _cfg(6, 60, 64, True, seed=0x5EED7A11)
    over = dict(feature_dim=64, visual_threshold=0.7)
    g = eng.Tracker(tracker_options_for("cfg5", default_options, **over))
    o = oracle.Tracker(tracker_options_for("cfg5", oracle.make_options, **over))
    for fr in range(16):
        f = wl.next_frame()
        if fr == 8:
            g = eng.Tracker.load(g.save())
        rg = _predict(g, f)
        ro = o.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=f["features"])
        for key in ("ids", "epochs", "lengths", "voting_types"):
            assert np.array_equal(rg[key], ro[key]), (fr, key)


# ------------------------------------------------------------------------------------------------------ migration
def _split(f, keep):
    """The request of frame f restricted to the scenes in `keep` (in frame order)."""
    sc, offs = f["scene_ids"], f["det_offsets"]
    rows, new_offs, new_sc = [], [0], []
    for i, s in enumerate(sc):
        if int(s) in keep:
            rows.append(np.arange(offs[i], offs[i + 1]))
            new_offs.append(new_offs[-1] + offs[i + 1] - offs[i])
            new_sc.append(s)
    idx = np.concatenate(rows) if rows else np.zeros(0, np.int64)
    return {"scene_ids": np.asarray(new_sc, np.uint64), "det_offsets": np.asarray(new_offs, np.int32),
            "boxes": f["boxes"][idx], "features": None if f["features"] is None else f["features"][idx]}, idx


def _merge(a, b):
    return {"scene_ids": np.concatenate([a["scene_ids"], b["scene_ids"]]),
            "det_offsets": np.concatenate([a["det_offsets"], a["det_offsets"][-1] + b["det_offsets"][1:]]).astype(np.int32),
            "boxes": np.concatenate([a["boxes"], b["boxes"]]),
            "features": None if a["features"] is None else np.concatenate([a["features"], b["features"]])}


class Partition:
    """Same partition of detections into tracks: a bijection between the reference's ids and the moved tracker's,
    identity on the ids that existed at export."""

    def __init__(self, first_new):
        self.first_new, self.fwd, self.back = first_new, {}, {}

    def check(self, ref_ids, got_ids):
        for r, g in zip(map(int, ref_ids), map(int, got_ids)):
            if r < self.first_new:
                assert r == g
            assert self.fwd.setdefault(r, g) == g and self.back.setdefault(g, r) == r


def _check_scene_parity(rr, rt, part):
    for key in ("epochs", "lengths", "voting_types", "predicted", "observed"):
        assert _bytes(rr[key]) == _bytes(rt[key]), key
    part.check(rr["ids"], rt["ids"])


def _tracker(eng, kind, dim, fh):
    t = eng.Tracker(_opts(kind, IOU, 5, dim, 3))
    if fh:
        t.set_feature_history(True)
    return t


def _first_rows(r, n):
    return {k: v[:n] for k, v in r.items()}


@pytest.mark.parametrize("holding", [False, True], ids=["fresh", "holding"])
@pytest.mark.parametrize("kind", [1, 3])
def test_migration_keeps_per_scene_parity(eng, kind, holding):
    dim, fh = (64, True) if kind == 3 else (0, False)
    wl = _cfg(8, 50, dim, False, seed=0x5EED7B00 + kind)
    frames = [wl.next_frame() for _ in range(20)]
    R, T1, T2 = (_tracker(eng, kind, dim, fh) for _ in range(3))
    other = _cfg(2, 30, dim, False, seed=0x5EED7C00, scene_base=8) if holding else None
    first_new = 0   # every id below it belongs to a track that existed at export
    for f in frames[:10]:
        first_new = max(first_new, int(_predict(R, f)["ids"].max()) + 1)
        _predict(T1, f)
        if holding:
            _predict(T2, other.next_frame())
    moved, rest = {2, 5, 6}, {0, 1, 3, 4, 7}
    blob = T1.export_scenes(sorted(moved), remove=True)
    # export -> import -> export is the same blob
    T3 = _tracker(eng, kind, dim, fh)
    T3.import_scenes(blob)
    assert _bytes(T3.export_scenes(sorted(moved))) == _bytes(blob)
    T2.import_scenes(blob)
    live, _ = T2.scene_live_counts(sorted(moved))
    assert list(T2.scene_track_counts(sorted(moved))) == list(live) and live.sum() > 0
    # the source reports the moved scenes' hidden records at its next collection, then counts nothing for them
    wr, w1 = R.wasted_history(), T1.wasted_history()
    for s in moved:
        a, b = wr["scene_ids"] == s, w1["scene_ids"] == s
        for key in ("ids", "epochs", "lengths", "predicted", "observed"):
            assert _bytes(wr[key][a]) == _bytes(w1[key][b]), (s, key)
    assert list(T1.scene_track_counts(sorted(moved))) == [0, 0, 0]
    p1, p2, owner = Partition(first_new), Partition(first_new), {}
    for f in frames[10:]:
        rr = _predict(R, f)
        f1, idx1 = _split(f, rest)
        f2, idx2 = _split(f, moved)
        r1 = _predict(T1, f1)
        n2 = int(f2["det_offsets"][-1])
        r2 = _first_rows(_predict(T2, _merge(f2, other.next_frame()) if holding else f2), n2)
        _check_scene_parity({k: v[idx1] for k, v in rr.items()}, r1, p1)
        _check_scene_parity({k: v[idx2] for k, v in rr.items()}, r2, p2)
        # among the moved scenes no id repeats: imported ids came from one counter, and every id T2 draws after the
        # import lies above it.  (T2's own scenes 8-9 hold ids of T2's own counter: those may equal imported ids of other
        # scenes -- ids are unique per scene -- so they are left out here.)
        for i, s in enumerate(f2["scene_ids"]):
            for tid in r2["ids"][f2["det_offsets"][i]: f2["det_offsets"][i + 1]]:
                assert owner.setdefault(int(tid), int(s)) == int(s), "an id repeats across the moved scenes"
    # re-adding a moved scene to the source starts it as a new scene
    assert T1.current_epoch(2) == 0
    f1, _ = _split(wl.next_frame(), {2})
    assert set(_predict(T1, f1)["epochs"].tolist()) == {1}


@pytest.mark.parametrize("kind", [1, 3])
def test_export_without_remove_changes_nothing(eng, kind):
    dim, fh = (64, True) if kind == 3 else (0, False)
    wl = _cfg(4, 40, dim, False, seed=0x5EED7D00 + kind)
    R, T = _tracker(eng, kind, dim, fh), _tracker(eng, kind, dim, fh)
    for fr in range(16):
        f = wl.next_frame()
        if fr == 8:
            T.export_scenes([1, 3])
        _same(_predict(R, f), _predict(T, f), f"frame {fr}")
    _same(_collect(R, fh), _collect(T, fh))


# ------------------------------------------------------------------------------------------------------ rejections
def _mutations():
    """(field, new value) of every option that an import compares."""
    return [("kind", 1), ("positional_kind", MAHA), ("iou_threshold", 0.25), ("min_confidence", 0.07),
            ("max_idle_epochs", 3), ("history_length", 6), ("kalman_position_weight", 0.06),
            ("kalman_velocity_weight", 0.007), ("constraints", [(1, 2.0)]), ("visual_kind", 1),
            ("visual_threshold", 0.6), ("feature_dim", 32), ("visual_max_observations", 4), ("visual_min_votes", 2),
            ("visual_minimal_track_length", 2), ("visual_minimal_area", 1.0), ("visual_minimal_quality_use", 0.1),
            ("visual_minimal_quality_collect", 0.1), ("visual_minimal_own_area_percentage_use", 0.1),
            ("visual_minimal_own_area_percentage_collect", 0.1)]


HDR_SEC_OFF = 24 + 160 + 12 * 4 + 8 * 8 + 8   # magic..total size, options, int32 fields, int64 fields, id counter


def test_rejections_change_nothing(eng):
    from similari_b200._lib import Sb200Error, lib

    dim = 64
    wl = _cfg(4, 40, dim, False, seed=0x5EED7E00)
    frames = [wl.next_frame() for _ in range(14)]
    src = _tracker(eng, 3, dim, True)
    T, twin = _tracker(eng, 3, dim, True), _tracker(eng, 3, dim, True)
    for f in frames[:6]:
        _predict(src, f)
        _predict(T, f)
        _predict(twin, f)
    blob = src.export_scenes([0, 1])
    tblob = src.save()

    def rejected(fn):
        with pytest.raises(Sb200Error):
            fn()

    def refused_without_side_effects(o, fh):
        """A destination with options `o` that holds scenes 50-51 refuses the blob, then runs like its twin."""
        d, dt = eng.Tracker(o), eng.Tracker(o)
        if fh:
            d.set_feature_history(True)
            dt.set_feature_history(True)
        own = _cfg(2, 20, max(int(o.feature_dim), 8) if o.kind >= 2 else 0, False, seed=0x5EED7E01, scene_base=50)
        fr = [own.next_frame() for _ in range(6)]
        for f in fr[:3]:
            _predict(d, f)
            _predict(dt, f)
        rejected(lambda: d.import_scenes(blob))
        assert d.scene_track_counts([0, 1]).sum() == 0
        for f in fr[3:]:
            _same(_predict(d, f), _predict(dt, f))
        _same(_collect(d, fh), _collect(dt, fh))

    # options of the destination differ in one field
    for field, val in _mutations():
        o = _opts(3, IOU, 5, dim, 3)
        if field == "constraints":
            o.n_constraints, o.constraint_epochs[0], o.constraint_max_dist[0] = 1, val[0][0], val[0][1]
        else:
            setattr(o, field, val)
        refused_without_side_effects(o, o.kind >= 2)
    # the feature-history flag differs
    refused_without_side_effects(_opts(3, IOU, 5, dim, 3), False)
    # a scene that already holds tracks here
    rejected(lambda: T.import_scenes(blob))
    # damaged blobs
    for off, val in ((0, 0x11), (4, 7)):
        b = blob.copy()
        b[off] ^= val
        rejected(lambda: T.import_scenes(b))
    rejected(lambda: T.import_scenes(blob[:-100]))
    b = blob.copy()
    b[HDR_SEC_OFF + 8: HDR_SEC_OFF + 16] = np.frombuffer(np.uint64(len(blob) + 4096).tobytes(), np.uint8)
    rejected(lambda: T.import_scenes(b))
    # the wrong blob type for the call, an unknown scene
    rejected(lambda: T.import_scenes(tblob))
    rejected(lambda: eng.Tracker.load(blob))
    rejected(lambda: T.export_scenes([0, 99]))
    # cap too small: *bytes is the size needed, nothing is written
    import torch

    need = T.export_scenes([0, 1], d_ptr=0)
    buf = torch.full((need,), 0xAB, dtype=torch.uint8, device="cuda")
    n = C.c_size_t(0)
    sc = np.array([0, 1], np.uint64)
    rc = lib().sb200_scenes_export(T._h, 2, sc.ctypes.data_as(C.c_void_p), 0, C.c_void_p(buf.data_ptr()), need - 1,
                                   C.byref(n))
    assert rc == -3 and n.value == need
    assert bool((buf == 0xAB).all())
    # ... and T still runs exactly like its twin
    for f in frames[6:]:
        _same(_predict(T, f), _predict(twin, f))
    _same(_collect(T, True), _collect(twin, True))


# ------------------------------------------------------------------------------------------------------ growth
def test_import_grows_the_store_the_scene_table_and_the_history_pool(eng):
    dim = 64
    wl = _cfg(6, 150, dim, False, seed=0x5EED7F00)
    frames = [wl.next_frame() for _ in range(10)]
    R, T1 = _tracker(eng, 3, dim, True), _tracker(eng, 3, dim, True)
    T2 = _tracker(eng, 3, dim, True)
    small = _cfg(1, 10, dim, False, seed=0x5EED7F01, scene_base=100)
    _predict(T2, small.next_frame())   # 4 scene slots, 64 rows per scene, a 256-block history pool
    pool0 = T2.feature_history_pool()["capacity"]
    first_new = 0
    for f in frames[:5]:
        first_new = max(first_new, int(_predict(R, f)["ids"].max()) + 1)
        _predict(T1, f)
    T2.import_scenes(T1.export_scenes(list(range(6)), remove=True))
    live, _ = T2.scene_live_counts(list(range(6)))
    assert live.max() > 64 and T2.feature_history_pool()["capacity"] > pool0
    part = Partition(first_new)
    for f in frames[5:]:
        _check_scene_parity(_predict(R, f), _predict(T2, f), part)


def test_cfg5_sized_save_load_round_trip(eng):
    import torch

    from similari_b200._lib import default_options
    from similari_b200.workload import CONFIGS, Workload, tracker_options_for

    wl = Workload(CONFIGS["cfg5"])
    g = eng.Tracker(tracker_options_for("cfg5", default_options))
    frames = [wl.next_frame() for _ in range(4)]
    for f in frames[:3]:
        _predict(g, f)
    n = g.save_device(0, 0)
    a = torch.empty(n, dtype=torch.uint8, device="cuda")
    assert g.save_device(a.data_ptr(), n) == n
    h = eng.Tracker.load(a.data_ptr(), n)
    b = torch.empty(n, dtype=torch.uint8, device="cuda")
    assert h.save_device(b.data_ptr(), n) == n
    torch.cuda.synchronize()
    assert torch.equal(a, b)
    del a, b
    _same(_predict(g, frames[3]), _predict(h, frames[3]))


def test_load_on_another_device(eng):
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU here: loading a device-0 blob on device 1 needs two")
    case = CASES[4]
    g, wl = _make(eng, case)
    frames = [wl.next_frame() for _ in range(16)]
    for f in frames[:8]:
        _predict(g, f)
    n = g.save_device(0, 0)
    buf = torch.empty(n, dtype=torch.uint8, device="cuda:0")
    g.save_device(buf.data_ptr(), n)
    torch.cuda.synchronize()
    h = eng.Tracker.load(buf.data_ptr(), n, device=1)
    _continue(g, h, frames[8:], True, frames[0]["scene_ids"])


def test_predict_launches_the_same_kernels_after_a_transfer(eng):
    dim = 64
    wl = _cfg(4, 40, dim, False, seed=0x5EED8000)
    T = _tracker(eng, 3, dim, True)
    for _ in range(4):
        _predict(T, wl.next_frame())

    def launches():
        f = wl.next_frame()
        c0 = eng.launch_count()
        _predict(T, f)
        return eng.launch_count() - c0

    before = launches()
    T.save()
    blob = T.export_scenes([0])
    d = _tracker(eng, 3, dim, True)
    d.import_scenes(blob)
    assert launches() == before


def test_unused_constraint_slots_do_not_count(eng):
    """Only the first n_constraints (epoch, distance) pairs are options: garbage in the unused slots is not a mismatch."""
    dim = 64
    wl = _cfg(2, 30, dim, False, seed=0x5EED8100)
    src = _tracker(eng, 3, dim, True)
    for _ in range(3):
        _predict(src, wl.next_frame())
    o = _opts(3, IOU, 5, dim, 3)
    for i in range(8):
        o.constraint_epochs[i], o.constraint_max_dist[i] = 1000 + i, float("nan")
    d = eng.Tracker(o)
    d.set_feature_history(True)
    d.import_scenes(src.export_scenes([0, 1]))
    assert list(d.scene_track_counts([0, 1])) == list(src.scene_track_counts([0, 1]))


def test_feature_history_cannot_be_switched_after_a_load_or_an_import(eng):
    from similari_b200._lib import Sb200Error

    dim = 64
    wl = _cfg(2, 30, dim, False, seed=0x5EED8200)
    for fh in (False, True):
        src = _tracker(eng, 3, dim, fh)
        for _ in range(4):
            _predict(src, wl.next_frame())
        loaded = eng.Tracker.load(src.save())
        with pytest.raises(Sb200Error):
            loaded.set_feature_history(not fh)
        d = _tracker(eng, 3, dim, fh)
        d.import_scenes(src.export_scenes([0]))
        with pytest.raises(Sb200Error):
            d.set_feature_history(not fh)
        # still usable, and the same as its source
        f = wl.next_frame()
        _same(_predict(src, f), _predict(loaded, f))


def test_device_blobs_are_ordered_after_the_caller_stream(eng):
    """save / export write, and import reads, a device blob in the order of the stream named with set_stream: work the
    caller queued on that stream before the call (here behind a long sleep) comes first, without a host synchronisation."""
    import torch

    dim = 64
    wl = _cfg(3, 40, dim, False, seed=0x5EED8300)
    frames = [wl.next_frame() for _ in range(10)]
    src, ref = _tracker(eng, 3, dim, True), _tracker(eng, 3, dim, True)
    for f in frames[:5]:
        _predict(src, f)
        _predict(ref, f)
    s = torch.cuda.Stream()
    # save: a fill the caller queued on its stream must land before the blob is written, not over it
    src.set_stream(s.cuda_stream)
    expect = src.save()
    n = len(expect)
    buf = torch.empty(n, dtype=torch.uint8, device="cuda")
    with torch.cuda.stream(s):
        torch.cuda._sleep(200_000_000)
        buf.fill_(0x5A)
        assert src.save_device(buf.data_ptr(), n) == n
    s.synchronize()
    assert _bytes(buf.cpu().numpy()) == _bytes(expect)
    # import: the blob arrives on the caller's stream (a receive) behind a long sleep; import is ordered after it
    blob = src.export_scenes([0, 1, 2], remove=True)
    host = torch.from_numpy(blob).pin_memory()
    dev = torch.empty(len(blob), dtype=torch.uint8, device="cuda")
    dst = _tracker(eng, 3, dim, True)
    dst.set_stream(s.cuda_stream)
    with torch.cuda.stream(s):
        torch.cuda._sleep(200_000_000)
        dev.copy_(host, non_blocking=True)
        dst.import_scenes(dev.data_ptr(), len(blob))
    for f in frames[5:]:
        _same(_predict(ref, f), _predict(dst, f))


def _api_obs(api, f, i0, i1):
    from similari_b200.api import Universal2DBox, VisualSortObservation

    out = []
    for i in range(i0, i1):
        b = f["boxes"][i]
        box = Universal2DBox.new_with_confidence(float(b[0]), float(b[1]), None if np.isnan(b[2]) else float(b[2]),
                                                 float(b[3]), float(b[4]), float(b[5]))
        out.append(VisualSortObservation(f["features"][i].tolist() if f["features"] is not None else None, 1.0, box, None))
    return out


def _api_step(api, t, f):
    """One frame through the api class; returns [(scene, [(id, epoch, length)])]."""
    from similari_b200.api import (BatchSort, BatchVisualSort, SortPredictionBatchRequest, Universal2DBox,
                                   VisualSort, VisualSortObservationSet, VisualSortPredictionBatchRequest)

    offs = f["det_offsets"]
    key = lambda tracks: [(int(x.id), int(x.epoch), int(x.length)) for x in tracks]   # noqa: E731
    if isinstance(t, (BatchVisualSort,)):
        req = VisualSortPredictionBatchRequest()
        for si, s in enumerate(f["scene_ids"]):
            for o in _api_obs(api, f, offs[si], offs[si + 1]):
                req.add(int(s), o)
        r = t.predict(req)
        return sorted((s, key(tr)) for s, tr in (r.get() for _ in range(r.batch_size())))
    if isinstance(t, VisualSort):
        os_ = VisualSortObservationSet()
        for o in _api_obs(api, f, offs[0], offs[1]):
            os_.add(o)
        return [(0, key(t.predict(os_)))]
    rows = [Universal2DBox.new_with_confidence(float(b[0]), float(b[1]), None, float(b[3]), float(b[4]), float(b[5]))
            for b in f["boxes"]]
    if isinstance(t, BatchSort):
        req = SortPredictionBatchRequest()
        for si, s in enumerate(f["scene_ids"]):
            for i in range(offs[si], offs[si + 1]):
                req.add(int(s), rows[i], None)
        r = t.predict(req)
        return sorted((s, key(tr)) for s, tr in (r.get() for _ in range(r.batch_size())))
    return [(0, key(t.predict([(b, None) for b in rows[offs[0]: offs[1]]])))]


@pytest.mark.parametrize("cls", ["Sort", "BatchSort", "VisualSort", "BatchVisualSort"])
def test_api_save_state_load_state_round_trip(eng, cls):
    import similari_b200.api as api

    visual = "Visual" in cls
    batch = cls.startswith("Batch")
    dim = 32 if visual else 0
    wl = _cfg(3 if batch else 1, 25, dim, False, seed=0x5EED8400 + len(cls))
    frames = [wl.next_frame() for _ in range(10)]

    def make():
        if not visual:
            return getattr(api, cls)(max_idle_epochs=2, method=api.PositionalMetricType.iou(0.2))
        o = api.VisualSortOptions()
        o.max_idle_epochs(2)
        o.visual_minimal_track_length(1)
        o.visual_metric(api.VisualSortMetricType.euclidean(0.7))
        return api.BatchVisualSort(1, 1, o) if batch else api.VisualSort(1, o)

    a = make()
    if visual:   # a tracker that has seen nothing saves an empty state, which loads as the same kind of tracker
        e = api.load_state(a.save_state())
        assert type(e) is type(a)
    for f in frames[:5]:
        _api_step(api, a, f)
    b = api.load_state(a.save_state())
    assert type(b) is type(a)
    for f in frames[5:]:
        assert _api_step(api, a, f) == _api_step(api, b, f)
    assert sorted((int(w.id), int(w.length)) for w in a.wasted()) == sorted((int(w.id), int(w.length)) for w in b.wasted())


@pytest.mark.parametrize("cls", ["BatchSort", "BatchVisualSort"])
def test_api_export_import_scenes(eng, cls):
    import similari_b200.api as api

    visual = cls == "BatchVisualSort"
    dim = 32 if visual else 0
    wl = _cfg(4, 25, dim, False, seed=0x5EED8500)
    frames = [wl.next_frame() for _ in range(10)]

    def make():
        if not visual:
            return api.BatchSort(max_idle_epochs=2, method=api.PositionalMetricType.iou(0.2))
        o = api.VisualSortOptions()
        o.max_idle_epochs(2)
        o.visual_minimal_track_length(1)
        o.visual_metric(api.VisualSortMetricType.euclidean(0.7))
        return api.BatchVisualSort(1, 1, o)

    R, A, B = make(), make(), make()   # B has never predicted: its engine tracker comes from the blob
    for f in frames[:5]:
        _api_step(api, R, f)
        _api_step(api, A, f)
    B.import_scenes(A.export_scenes([1, 3], remove=True))
    for f in frames[5:]:
        r = dict(_api_step(api, R, f))
        fb, _ = _split(f, {1, 3})
        got = dict(_api_step(api, B, fb))
        for s in (1, 3):
            assert [(e, l) for _, e, l in r[s]] == [(e, l) for _, e, l in got[s]]


def test_api_import_keeps_a_provisional_feature_dimension(eng):
    """A source that has seen no feature yet has a provisional dimension; so has a fresh importer."""
    import similari_b200.api as api

    o = api.VisualSortOptions()
    o.visual_minimal_track_length(1)
    A, B = api.BatchVisualSort(1, 1, o), api.BatchVisualSort(1, 1, o)
    wl = _cfg(1, 10, 0, False, seed=0x5EED8600)
    f = wl.next_frame()
    _api_step(api, A, f)   # boxes only
    B.import_scenes(A.export_scenes([0]))
    assert B._dim_provisional
    wf = _cfg(1, 10, 48, False, seed=0x5EED8601).next_frame()
    _api_step(api, B, wf)   # the first featured frame fixes the dimension, as it does for the source
    assert not B._dim_provisional
