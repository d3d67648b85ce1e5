"""End-to-end parity of the device-resident trackers (through sb200_predict_batch) against the CPU oracle:
identical ids / epochs / lengths / voting types frame after frame on seeded synthetic workloads, the reference's own
end-to-end sequences, lifecycle (skip_epochs / wasted / idle), and size-independent properties at BASELINE sizes."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


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


def run_frames(eng, oracle, wl_cfg, frames, opts_kw, exact_boxes=True, check_costs=True):
    import os

    from similari_b200.workload import Workload

    g, o = both(eng, oracle, **opts_kw)
    # Visual trackers evaluate the positional metric lazily (only for the pairs VisualVoting can still consult), so their
    # sb200_last_costs is partial by design.  A second tracker runs with SB200_FULL_COSTS=1 (every pair evaluated): its
    # matrix is compared with the oracle's, and both GPU trackers must produce the oracle's assignments.
    visual = opts_kw.get("kind", 0) in (2, 3)
    g_full = both(eng, oracle, **opts_kw)[0] if (check_costs and visual) else None
    wl = Workload(wl_cfg)
    for fr in range(frames):
        f = wl.next_frame()
        quality = None
        sid = int(f["scene_ids"][0])
        gc = g_full if g_full is not None else g     # the tracker whose cost matrix is checked
        if check_costs:   # columns of the cost matrices = the stores BEFORE the frame
            ids_g = [int(x) for x in gc.scene_tracks(sid)["ids"]]
            ids_o = [int(x) for x in o.scene_tracks(sid)["ids"]]
        rg = g.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=f["features"], quality=quality)
        ro = o.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=f["features"], quality=quality)
        results = [rg]
        if g_full is not None:
            os.environ["SB200_FULL_COSTS"] = "1"
            try:
                results.append(g_full.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=f["features"],
                                                    quality=quality))
            finally:
                del os.environ["SB200_FULL_COSTS"]
        for rr in results:
            for key in ("ids", "epochs", "lengths", "voting_types"):
                assert np.array_equal(rr[key], ro[key]), (fr, key)
            for key in ("predicted", "observed"):
                if exact_boxes:
                    assert np.array_equal(np.nan_to_num(rr[key], nan=-7.0), np.nan_to_num(ro[key], nan=-7.0)), (fr, key)
                else:
                    np.testing.assert_allclose(rr[key], ro[key], rtol=0, atol=1e-4, equal_nan=True)
        if check_costs:
            # The device store drops expired tracks at the end of the frame in which they expire (the reference keeps
            # them until its next collection point, where their column is all None): compare column by track id.
            cg, co = gc.last_costs(sid), o.last_costs(sid)
            assert (cg.size == 0 or cg.shape[1] == len(ids_g)) and (co.size == 0 or co.shape[1] == len(ids_o)), fr
            assert [i for i in ids_o if i in set(ids_g)] == ids_g, fr          # same store order
            if exact_boxes and co.size:
                col_of = {i: c for c, i in enumerate(ids_o)}
                live = [col_of[i] for i in ids_g]
                if cg.size:
                    assert np.array_equal(np.nan_to_num(cg, nan=-7.0), np.nan_to_num(co[:, live], nan=-7.0)), fr
                gone = np.setdiff1d(np.arange(len(ids_o)), live)
                assert np.all(np.isnan(co[:, gone])), fr                     # expired tracks never score
        assert g.active_tracks() == o.active_tracks()
    return g, o


def small(name, **over):
    import dataclasses

    from similari_b200.workload import CONFIGS

    return dataclasses.replace(CONFIGS[name], **over)


@pytest.mark.parametrize("kind_name,kind", [("sort", 0), ("batch_sort", 1)])
@pytest.mark.parametrize("pos", [0, 1])
@pytest.mark.parametrize("oriented", [False, True])
def test_sort_trackers_match_oracle(eng, oracle, kind_name, kind, pos, oriented):
    cfg = small("cfg2", n_scenes=1 if kind == 0 else 5, n_objects=60, oriented=oriented, canvas=(900.0, 600.0))
    # oriented IoU passes through device sin/cos: ids must still match, boxes are Kalman outputs (exact)
    run_frames(eng, oracle, cfg, 8, dict(kind=kind, positional_kind=pos, iou_threshold=0.3, max_idle_epochs=3),
               exact_boxes=True, check_costs=not (oriented and pos == 1))


@pytest.mark.parametrize("kind", [2, 3])
@pytest.mark.parametrize("pos", [0, 1])
@pytest.mark.parametrize("vis", [0, 1])
def test_visual_trackers_match_oracle(eng, oracle, kind, pos, vis):
    cfg = small("cfg5", n_scenes=1 if kind == 2 else 4, n_objects=40, oriented=False, canvas=(700.0, 500.0),
                feature_dim=64)
    run_frames(eng, oracle, cfg, 8,
               dict(kind=kind, positional_kind=pos, iou_threshold=0.3, max_idle_epochs=3, visual_kind=vis,
                    visual_threshold=0.7 if vis == 0 else 0.2, feature_dim=64, visual_max_observations=3,
                    visual_min_votes=2, visual_minimal_track_length=1, min_confidence=0.1))


@pytest.mark.parametrize("kind", [2, 3])
@pytest.mark.parametrize("vis", [0, 1])
def test_visual_trackers_tensor_core_path_match_oracle(eng, oracle, kind, vis, monkeypatch):
    """Same end-to-end comparison with the tensor-core visual-cost kernel forced on (the default for large frames)."""
    monkeypatch.setenv("SB200_VIS_KERNEL", "tc")
    cfg = small("cfg5", n_scenes=1 if kind == 2 else 3, n_objects=150, oriented=False, canvas=(1400.0, 900.0),
                feature_dim=128)
    run_frames(eng, oracle, cfg, 6,
               dict(kind=kind, positional_kind=1, iou_threshold=0.3, max_idle_epochs=3, visual_kind=vis,
                    visual_threshold=0.7 if vis == 0 else 0.2, feature_dim=128, visual_max_observations=3,
                    visual_min_votes=2, visual_minimal_track_length=1, min_confidence=0.1))


@pytest.mark.parametrize("mode", ["single", "multicast"])
@pytest.mark.parametrize("vis", [0, 1])
def test_screen_kernel_cta_organisations_match_oracle(eng, oracle, mode, vis, monkeypatch):
    """The two CTA organisations of the screen kernel (one CTA per tile; 2-CTA cluster with multicast B loads, the
    default) against the oracle; 300 candidates per scene exercise the ragged second candidate tile of a cluster
    (rows 256..299 valid, the rest masked) and D = 96 the zero-filled K tail."""
    monkeypatch.setenv("SB200_VIS_KERNEL", "tc")
    monkeypatch.setenv("SB200_SCREEN", mode)
    cfg = small("cfg5", n_scenes=3, n_objects=300, oriented=False, canvas=(2200.0, 1400.0), feature_dim=96)
    run_frames(eng, oracle, cfg, 5,
               dict(kind=3, positional_kind=1, iou_threshold=0.3, max_idle_epochs=3, visual_kind=vis,
                    visual_threshold=0.7 if vis == 0 else 0.2, feature_dim=96, visual_max_observations=3,
                    visual_min_votes=2, visual_minimal_track_length=1, min_confidence=0.1))


@pytest.mark.parametrize("kind,device_io", [(1, False), (3, False), (2, False), (0, False), (3, True), (1, True)])
def test_frames_in_flight_match_oracle(eng, oracle, kind, device_io):
    """Stream-ordered predict: frames are enqueued back to back (sb200_predict_batch_async / _device) without waiting for
    the device -- the per-frame tables (tracks per scene, offsets, tile list, id counter) are built by a kernel -- and the
    results, read after sb200_sync, are those of the frame-by-frame oracle.  Seven scenes, 11 frames: the ring of four
    frames in flight wraps, new tracks appear and expire while later frames are already queued."""
    import torch

    from similari_b200._lib import default_options, pinned_empty
    from similari_b200.workload import Workload

    visual = kind >= 2
    cfg = small("cfg5" if visual else "cfg2", n_scenes=7 if kind in (1, 3) else 1, n_objects=60, oriented=False,
                canvas=(800.0, 600.0), feature_dim=64 if visual else 0, drop_frac=0.15, fresh_frac=0.15)
    kw = dict(kind=kind, positional_kind=1, iou_threshold=0.3, max_idle_epochs=2)
    if visual:
        kw.update(visual_kind=0, visual_threshold=0.7, feature_dim=64, visual_max_observations=3, visual_min_votes=2,
                  visual_minimal_track_length=1, min_confidence=0.1)
    g, o = both(eng, oracle, **kw)
    wl = Workload(cfg)
    frames = [wl.next_frame() for _ in range(11)]
    ref = [o.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=f["features"]) for f in frames]
    outs = []
    keep = []
    for f in frames:
        total = len(f["boxes"])
        if device_io:
            dev = torch.device("cuda", 0)
            db = torch.from_numpy(np.ascontiguousarray(f["boxes"])).to(dev)
            df = torch.from_numpy(np.ascontiguousarray(f["features"])).to(dev) if visual else None
            d = {"ids": torch.zeros(total, dtype=torch.int64, device=dev), "epochs": torch.zeros(total, dtype=torch.int32, device=dev),
                 "lengths": torch.zeros(total, dtype=torch.int32, device=dev), "voting_types": torch.zeros(total, dtype=torch.uint8, device=dev)}
            keep.append((db, df))
            torch.cuda.synchronize()
            g.predict_batch_device(f["scene_ids"], f["det_offsets"], db.data_ptr(), df.data_ptr() if visual else 0,
                                   d_ids=d["ids"].data_ptr(), d_epochs=d["epochs"].data_ptr(),
                                   d_lengths=d["lengths"].data_ptr(), d_voting_types=d["voting_types"].data_ptr())
            outs.append(d)
        else:
            out = {"ids": pinned_empty((total,), np.uint64), "epochs": pinned_empty((total,), np.uint32),
                   "lengths": pinned_empty((total,), np.uint32), "voting_types": pinned_empty((total,), np.uint8)}
            g.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=f["features"], out=out, wait=False)
            outs.append(out)
    assert g.frames_in_flight() <= 4
    g.sync()
    assert g.frames_in_flight() == 0
    for fr, (r, ro) in enumerate(zip(outs, ref)):
        for key in ("ids", "epochs", "lengths", "voting_types"):
            got = r[key].cpu().numpy() if device_io else r[key]
            assert np.array_equal(got.astype(np.uint64), ro[key].astype(np.uint64)), (fr, key)
    assert g.active_tracks() == o.active_tracks()
    wc = g.work_counters()
    assert wc["frames"] == len(frames) and wc["pair_associations"] > 0


def test_ragged_batches_empty_and_single_detection_scenes(eng, oracle, monkeypatch):
    """A batch in which one scene is empty, one has a single detection and the others are full -- on the tensor-core path
    (the tile list skips the empty scene, the one-row scene is a 1 x N tile) and on the exact path."""
    from similari_b200.workload import Workload

    for vis_kernel in ("tc", "simt"):
        monkeypatch.setenv("SB200_VIS_KERNEL", vis_kernel)
        cfg = small("cfg5", n_scenes=5, n_objects=140, oriented=False, canvas=(1400.0, 900.0), feature_dim=128)
        kw = dict(kind=3, positional_kind=1, iou_threshold=0.3, max_idle_epochs=3, visual_kind=0, visual_threshold=0.7,
                  feature_dim=128, visual_max_observations=3, visual_min_votes=2, visual_minimal_track_length=1,
                  min_confidence=0.1)
        g, o = both(eng, oracle, **kw)
        wl = Workload(cfg)
        for fr in range(7):
            f = wl.next_frame()
            offs = f["det_offsets"].astype(np.int64)
            # scene (fr % 5) loses all its detections, scene ((fr + 2) % 5) keeps one
            keep = []
            for s in range(5):
                idx = np.arange(offs[s], offs[s + 1])
                if fr >= 2 and s == fr % 5:
                    idx = idx[:0]
                elif fr >= 2 and s == (fr + 2) % 5:
                    idx = idx[:1]
                keep.append(idx)
            new_offs = np.concatenate([[0], np.cumsum([len(k) for k in keep])]).astype(np.int32)
            sel = np.concatenate(keep)
            rg = g.predict_batch(f["scene_ids"], new_offs, f["boxes"][sel], features=f["features"][sel])
            ro = o.predict_batch(f["scene_ids"], new_offs, f["boxes"][sel], features=f["features"][sel])
            for key in ("ids", "epochs", "lengths", "voting_types"):
                assert np.array_equal(rg[key], ro[key]), (vis_kernel, fr, key)
        assert g.active_tracks() == o.active_tracks()


def test_expired_tracks_leave_the_device_store_but_not_the_api(eng, oracle):
    """Every detection is a fresh identity: the reference's store grows by ~400 expired tracks per frame until its
    next auto-waste tick.  The device store drops them at the end of the frame in which they expire (bounded scan
    width), while everything the API reports -- assignments, active_tracks, scene_track_counts, idle_tracks,
    wasted() -- is what the reference reports."""
    from similari_b200.workload import Workload

    cfg = small("cfg2", n_scenes=2, n_objects=400, oriented=False, canvas=(4000.0, 3000.0), drop_frac=0.0, fresh_frac=1.0)
    kw = dict(kind=1, positional_kind=1, iou_threshold=0.3, max_idle_epochs=1)
    g, o = both(eng, oracle, **kw)
    wl = Workload(cfg)
    for fr in range(22):
        f = wl.next_frame()
        rg = g.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"])
        ro = o.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"])
        for key in ("ids", "epochs", "lengths"):
            assert np.array_equal(rg[key], ro[key]), (fr, key)
        assert g.active_tracks() == o.active_tracks()
        live, _ = g.scene_live_counts(f["scene_ids"])
        assert live.max() <= 2 * 400                              # at most the last two frames' tracks can still match
        stored = g.scene_track_counts(f["scene_ids"])
        assert [int(x) for x in stored] == [len(o.scene_tracks(int(sid), cap=1 << 15)["ids"]) for sid in f["scene_ids"]]
    assert int(g.scene_track_counts(f["scene_ids"]).max()) > 4000    # the reference's store did grow
    for sid in f["scene_ids"]:
        ig, io = g.idle_tracks(int(sid), cap=1 << 15), o.idle_tracks(int(sid), cap=1 << 15)
        assert sorted(map(int, ig["ids"])) == sorted(map(int, io["ids"]))
    wg, wo = g.wasted(cap=1 << 17), o.wasted(cap=1 << 17)
    assert sorted(map(int, wg["ids"])) == sorted(map(int, wo["ids"])) and len(wg["ids"]) > 4000
    assert g.active_tracks() == o.active_tracks()


def test_visual_lifecycle_with_feature_arena_matches_oracle(eng, oracle, monkeypatch):
    """Visual tracker, short idle window, many frames: tracks expire every frame, their feature blocks are reused by new
    tracks, the small per-track arrays are compacted -- assignments, voting types, idle / wasted sets and the store order
    must stay those of the oracle.  Both visual kernels (tensor-core screen + refine, dense exact) are exercised."""
    from similari_b200.workload import Workload

    for vis_kernel in ("tc", "simt"):
        monkeypatch.setenv("SB200_VIS_KERNEL", vis_kernel)
        cfg = small("cfg5", n_scenes=3, n_objects=90, oriented=False, canvas=(1000.0, 700.0), feature_dim=64,
                    drop_frac=0.15, fresh_frac=0.15)
        kw = dict(kind=3, positional_kind=1, iou_threshold=0.3, max_idle_epochs=2, visual_kind=0, visual_threshold=0.7,
                  feature_dim=64, visual_max_observations=3, visual_min_votes=2, visual_minimal_track_length=1,
                  min_confidence=0.1)
        g, o = both(eng, oracle, **kw)
        wl = Workload(cfg)
        blocks_max = 0
        for fr in range(24):
            f = wl.next_frame()
            rg = g.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=f["features"])
            ro = o.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=f["features"])
            for key in ("ids", "epochs", "lengths", "voting_types"):
                assert np.array_equal(rg[key], ro[key]), (vis_kernel, fr, key)
            live, blocks = g.scene_live_counts(f["scene_ids"])
            blocks_max = max(blocks_max, int(blocks.max()))
            assert np.all(blocks >= live)
            if fr % 5 == 4:
                for sid in f["scene_ids"]:
                    ig, io = g.idle_tracks(int(sid)), o.idle_tracks(int(sid))
                    assert sorted(map(int, ig["ids"])) == sorted(map(int, io["ids"])), (vis_kernel, fr)
                wg, wo = g.wasted(), o.wasted()
                assert sorted(map(int, wg["ids"])) == sorted(map(int, wo["ids"])), (vis_kernel, fr)
                assert g.active_tracks() == o.active_tracks()
                for sid in f["scene_ids"]:
                    sg, so = g.scene_tracks(int(sid)), o.scene_tracks(int(sid))
                    assert list(map(int, sg["ids"])) == list(map(int, so["ids"]))
                    assert np.array_equal(sg["feat_counts"], so["feat_counts"])
        assert blocks_max < 2 * 90          # the arena recycles blocks: it never grows with the number of frames


def test_prefetched_inputs_give_identical_results(eng, oracle):
    """sb200_prefetch_inputs only moves the H2D copy earlier; results are those of the plain call."""
    from similari_b200.workload import Workload

    cfg = small("cfg5", n_scenes=3, n_objects=40, oriented=False, canvas=(700.0, 500.0), feature_dim=64)
    kw = dict(kind=3, positional_kind=1, iou_threshold=0.3, max_idle_epochs=3, visual_kind=0, visual_threshold=0.7,
              feature_dim=64, visual_max_observations=3, visual_min_votes=2, visual_minimal_track_length=1,
              min_confidence=0.1)
    g, o = both(eng, oracle, **kw)
    wl = Workload(cfg)
    frames = [wl.next_frame() for _ in range(6)]
    for f in frames:
        f["boxes"] = np.ascontiguousarray(f["boxes"], np.float32)
        f["features"] = np.ascontiguousarray(f["features"], np.float32)
    g.prefetch_inputs(frames[0]["boxes"], features=frames[0]["features"])
    for i, f in enumerate(frames):
        if i + 1 < len(frames) and i != 2:   # frame 3 is deliberately not prefetched
            g.prefetch_inputs(frames[i + 1]["boxes"], features=frames[i + 1]["features"])
        rg = g.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=f["features"])
        ro = o.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=f["features"])
        for key in ("ids", "epochs", "lengths", "voting_types"):
            assert np.array_equal(rg[key], ro[key]), (i, key)


def test_constraints_and_custom_ids(eng, oracle):
    from similari_b200.workload import Workload

    cfg = small("cfg1", n_objects=30)
    kw = dict(kind=0, positional_kind=1, iou_threshold=0.3, max_idle_epochs=1, constraints=[(1, 1.0)])
    g, o = both(eng, oracle, **kw)
    wl = Workload(cfg)
    for fr in range(5):
        f = wl.next_frame()
        cust = np.arange(len(f["boxes"]), dtype=np.int64) + 100 * fr
        rg = g.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], custom_ids=cust)
        ro = o.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], custom_ids=cust)
        for key in ("ids", "epochs", "lengths"):
            assert np.array_equal(rg[key], ro[key])


def test_reference_sort_sequence(eng):
    # src/trackers/sort/simple_api.rs:280-342 (sort) through the GPU tracker
    from similari_b200._lib import default_options
    import oracle as orc

    t = eng.Tracker(default_options(kind=0, positional_kind=1, iou_threshold=0.3, min_confidence=0.05, max_idle_epochs=2,
                                    history_length=10))
    assert t.current_epoch() == 0
    v = t.predict_batch([0], [0, 1], [orc.ltwh(0.0, 0.0, 10.0, 20.0)])
    assert len(t.wasted()["ids"]) == 0
    tid = int(v["ids"][0])
    assert v["lengths"][0] == 1 and v["epochs"][0] == 1 and t.current_epoch() == 1
    v = t.predict_batch([0], [0, 1], [orc.ltwh(0.1, 0.1, 10.1, 20.0)], custom_ids=[2])
    assert int(v["ids"][0]) == tid and v["lengths"][0] == 2 and v["epochs"][0] == 2
    v = t.predict_batch([0], [0, 1], [orc.ltwh(10.1, 10.1, 10.1, 20.0)], custom_ids=[3])
    assert int(v["ids"][0]) != tid and len(t.wasted()["ids"]) == 0 and t.current_epoch() == 3
    t.predict_batch([0], [0, 0], np.zeros((0, 6), np.float32))
    assert len(t.wasted()["ids"]) == 0 and t.current_epoch() == 4
    t.predict_batch([0], [0, 0], np.zeros((0, 6), np.float32))
    w = t.wasted()
    assert list(map(int, w["ids"])) == [tid] and t.current_epoch() == 5


def test_reference_visual_sort_sequence(eng):
    # src/trackers/visual_sort/simple_api.rs:328-666 (visual_sort) through the GPU tracker
    from similari_b200._lib import default_options
    import oracle as orc

    V, P = 0, 1
    t = eng.Tracker(default_options(kind=2, max_idle_epochs=3, history_length=3, visual_kind=0, visual_threshold=1.0,
                                    positional_kind=0, visual_minimal_track_length=2, visual_minimal_area=5.0,
                                    visual_minimal_quality_use=0.45, visual_minimal_quality_collect=0.7,
                                    visual_max_observations=3, visual_min_votes=2, feature_dim=2, min_confidence=0.1))

    def step(scene, feat, q, ltwh, custom):
        has = np.array([feat is not None], dtype=np.uint8)
        f = np.array([feat if feat is not None else [0.0, 0.0]], dtype=np.float32)
        r = t.predict_batch([scene], [0, 1], [orc.ltwh(*ltwh)], features=f, has_feature=has, quality=[q],
                            custom_ids=[custom])
        return int(r["ids"][0]), int(r["voting_types"][0]), int(r["epochs"][0]), int(r["lengths"][0])

    def feat_count(scene, tid):
        st = t.scene_tracks(scene)
        return int(st["feat_counts"][list(st["ids"]).index(tid)])

    first, vt, ep, ln = step(10, [1.0, 1.0], 0.9, (1.0, 1.0, 3.0, 5.0), 13)
    assert (vt, ep, ln) == (P, 1, 1) and feat_count(10, first) == 1
    other_scene, vt, ep, ln = step(1, [1.0, 1.0], 0.9, (1.0, 1.0, 3.0, 5.0), 133)
    assert (vt, ep, ln) == (P, 1, 1) and other_scene != first
    assert step(10, [0.95, 0.95], 0.93, (1.1, 1.1, 3.05, 5.01), 15) == (first, P, 2, 2) and feat_count(10, first) == 2
    assert step(10, None, 0.93, (1.11, 1.15, 3.15, 5.05), 25) == (first, P, 3, 3) and feat_count(10, first) == 2
    assert step(10, None, 0.93, (1.15, 1.25, 3.10, 5.05), 2) == (first, P, 4, 4) and feat_count(10, first) == 2
    assert step(10, [0.97, 0.97], 0.44, (1.15, 1.25, 3.10, 5.05), 2)[:2] == (first, P) and feat_count(10, first) == 2
    assert step(10, [0.97, 0.97], 0.6, (1.15, 1.25, 3.10, 5.05), 2)[:2] == (first, V) and feat_count(10, first) == 2
    assert step(10, [0.97, 0.97], 0.8, (1.15, 1.25, 3.10, 5.05), 2)[:2] == (first, V) and feat_count(10, first) == 3
    other, vt, ep, ln = step(10, [0.1, 0.1], 0.9, (10.0, 10.0, 3.0, 5.0), 33)
    assert (vt, ep, ln) == (P, 8, 1) and other != first and feat_count(10, other) == 1
    assert step(10, [0.12, 0.15], 0.88, (10.1, 10.1, 3.0, 5.0), 35) == (other, P, 9, 2) and feat_count(10, other) == 2
    assert step(10, [0.12, 0.14], 0.87, (10.1, 10.1, 3.0, 5.0), 31) == (other, V, 10, 3) and feat_count(10, other) == 3
    t.skip_epochs(5, scene_id=10)
    assert sorted(map(int, t.wasted()["ids"])) == sorted([first, other])


def test_lifecycle_waste_idle_matches_oracle(eng, oracle):
    from similari_b200.workload import Workload

    cfg = small("cfg2", n_scenes=3, n_objects=50, canvas=(800.0, 600.0), drop_frac=0.2, fresh_frac=0.2)
    kw = dict(kind=1, positional_kind=0, max_idle_epochs=1)
    g, o = both(eng, oracle, **kw)
    g.set_auto_waste(2)
    import ctypes as C

    o._L.orc_tracker_skip_epochs(o._h, 99, 0)  # no-op scene to mirror auto-waste cadence
    wl = Workload(cfg)
    for fr in range(9):
        f = wl.next_frame()
        rg = g.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"])
        ro = o.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"])
        assert np.array_equal(rg["ids"], ro["ids"]), fr
        if fr % 3 == 2:
            wg, wo = g.wasted(), o.wasted()
            assert sorted(map(int, wg["ids"])) == sorted(map(int, wo["ids"]))
            assert g.active_tracks() == o.active_tracks()
            for sid in f["scene_ids"]:
                ig, io = g.idle_tracks(int(sid)), o.idle_tracks(int(sid))
                assert sorted(map(int, ig["ids"])) == sorted(map(int, io["ids"]))
                sg, so = g.scene_tracks(int(sid)), o.scene_tracks(int(sid))
                assert list(map(int, sg["ids"])) == list(map(int, so["ids"]))  # store order preserved by compaction


def test_full_size_properties_cfg2(eng):
    """BASELINE cfg2 (64 scenes x 256 x 256, IoU): size-independent properties instead of an oracle run."""
    from similari_b200._lib import default_options
    from similari_b200.workload import CONFIGS, Workload, tracker_options_for

    t = eng.Tracker(tracker_options_for("cfg2", default_options))
    wl = Workload(CONFIGS["cfg2"])
    prev_ids = None
    for fr in range(5):
        f = wl.next_frame()
        r = t.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"])
        offs = f["det_offsets"]
        for s in range(len(f["scene_ids"])):
            ids = r["ids"][offs[s]:offs[s + 1]]
            assert len(np.unique(ids)) == len(ids)           # a track id is assigned at most once per scene & frame
        assert np.all(r["epochs"] == fr + 1)
        if prev_ids is not None:
            reused = np.isin(r["ids"], prev_ids).mean()
            assert reused > 0.8                               # most detections continue an existing track
            assert np.all(r["lengths"][~np.isin(r["ids"], prev_all)] == 1)
        prev_ids = r["ids"].copy()
        prev_all = r["ids"].copy() if fr == 0 else np.union1d(prev_all, r["ids"])


F32MAX = float(np.finfo(np.float32).max)


@pytest.mark.parametrize("kind", [2, 3])
@pytest.mark.parametrize("vis,thr", [(0, F32MAX), (1, -1.0), (0, 10.0)])
@pytest.mark.parametrize("kobs,min_votes", [(3, 2), (5, 1), (2, 2), (4, 3)])
def test_dense_tensor_core_path_matches_oracle(eng, oracle, kind, vis, thr, kobs, min_votes, monkeypatch):
    """Thresholds that cut nothing -- the reference's default Euclidean(f32::MAX), cosine(-1), the published bench's
    Euclidean(10.0) on unit vectors -- on the dense tensor-core path (kernels_feat_dense.cu): wgmma weight sums with error
    bounds, exact max_dist, selection of the groups that can be a BestFit row / column maximum, exact refinement, voting.
    Every id / voting type must be the oracle's.  K = 2..5 observations exercise column tiles of 256, 255, 256 and 255
    feature rows (tiles end at block boundaries), min_votes the block filter."""
    monkeypatch.setenv("SB200_VIS_KERNEL", "dense")
    cfg = small("cfg5", n_scenes=1 if kind == 2 else 3, n_objects=170, oriented=False, canvas=(1500.0, 1000.0),
                feature_dim=128, drop_frac=0.1, fresh_frac=0.1)
    g, o = run_frames(eng, oracle, cfg, 7,
                      dict(kind=kind, positional_kind=1, iou_threshold=0.3, max_idle_epochs=3, visual_kind=vis,
                           visual_threshold=thr, feature_dim=128, visual_max_observations=kobs,
                           visual_min_votes=min_votes, visual_minimal_track_length=1, min_confidence=0.1),
                      check_costs=False)
    wc = g.work_counters()
    assert wc["tc_frames"] >= 5 and wc["dense_fallback_scenes"] == 0    # the tensor-core path did the work, no scene fell back


def test_dense_path_preconditions_fall_back_per_scene(eng, oracle, monkeypatch):
    """The dense path forced onto a threshold that DOES cut (1.38 on unit vectors: about a third of the distances pass): the
    exact max_dist exceeds the threshold, the scene is flagged on the device and the exact SIMT kernels take it -- slow, but
    the assignments are still the oracle's."""
    monkeypatch.setenv("SB200_VIS_KERNEL", "dense")
    cfg = small("cfg5", n_scenes=2, n_objects=120, oriented=False, canvas=(1200.0, 800.0), feature_dim=64)
    g, o = run_frames(eng, oracle, cfg, 5,
                      dict(kind=3, positional_kind=1, iou_threshold=0.3, max_idle_epochs=3, visual_kind=0,
                           visual_threshold=1.38, feature_dim=64, visual_max_observations=3, visual_min_votes=2,
                           visual_minimal_track_length=1, min_confidence=0.1), check_costs=False)
    assert g.work_counters()["dense_fallback_scenes"] > 0


def test_threshold_that_cuts_nothing_switches_to_the_dense_path(eng, oracle):
    """Euclidean(10.0) on unit vectors looks selective to the host (finite threshold), so the first frames take the screen,
    whose survivor lists overflow in every scene (device-side exact fallback).  The tracker notices and moves to the dense
    tensor-core path: after the switch no scene falls back any more, and every frame matches the oracle."""
    from similari_b200._lib import default_options
    from similari_b200.workload import Workload

    cfg = small("cfg5", n_scenes=3, n_objects=420, oriented=False, canvas=(2600.0, 1600.0), feature_dim=256)
    kw = dict(kind=3, positional_kind=1, iou_threshold=0.3, max_idle_epochs=3, visual_kind=0, visual_threshold=10.0,
              feature_dim=256, visual_max_observations=3, visual_min_votes=2, visual_minimal_track_length=1,
              min_confidence=0.1)
    g, o = both(eng, oracle, **kw)
    wl = Workload(cfg)
    fallback = []
    for fr in range(9):
        f = wl.next_frame()
        rg = g.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=f["features"])
        ro = o.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=f["features"])
        for key in ("ids", "epochs", "lengths", "voting_types"):
            assert np.array_equal(rg[key], ro[key]), (fr, key)
        fallback.append(g.work_counters()["dense_fallback_scenes"])
    assert fallback[2] > 0                      # the screen's lists overflowed at first
    assert fallback[-1] == fallback[3]          # ... and nothing fell back once the dense path had taken over


@pytest.mark.parametrize("kind,hist", [(1, 4), (0, 7), (3, 3)])
def test_wasted_tracks_carry_their_box_history(eng, kind, hist):
    """WastedSortTrack.predicted_boxes / observed_boxes (src/trackers/sort.rs:316-341): the last `history_length` boxes of
    the track, oldest first, as SortAttributes::update_history keeps them (sort.rs:157-171).  The expected history of a
    track is rebuilt from the per-frame SortTrack records the tracker itself returned."""
    from similari_b200._lib import default_options
    from similari_b200.workload import Workload

    visual = kind >= 2
    cfg = small("cfg5" if visual else "cfg2", n_scenes=3 if kind in (1, 3) else 1, n_objects=50, oriented=True,
                canvas=(900.0, 600.0), feature_dim=32 if visual else 0, drop_frac=0.2, fresh_frac=0.15)
    kw = dict(kind=kind, positional_kind=0, max_idle_epochs=1, history_length=hist)
    if visual:
        kw.update(visual_kind=0, visual_threshold=0.7, feature_dim=32, visual_max_observations=3, visual_min_votes=1,
                  visual_minimal_track_length=1)
    g = eng.Tracker(default_options(**kw))
    wl = Workload(cfg)
    seen = {}
    n_checked = 0
    for fr in range(14):
        f = wl.next_frame()
        r = g.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=f["features"])
        for i, tid in enumerate(r["ids"]):
            seen.setdefault(int(tid), []).append((r["predicted"][i].copy(), r["observed"][i].copy()))
        if fr % 4 == 3:
            w = g.wasted_history()
            for i, tid in enumerate(w["ids"]):
                exp = seen[int(tid)][-hist:]
                assert int(w["lengths"][i]) == len(seen[int(tid)])
                gp, go = w["predicted_history"][i], w["observed_history"][i]
                assert len(gp) == len(exp) == len(go)
                for (ep, eo), p_, o_ in zip(exp, gp, go):
                    assert np.array_equal(np.nan_to_num(ep, nan=-7.0), np.nan_to_num(p_, nan=-7.0))
                    assert np.array_equal(np.nan_to_num(eo, nan=-7.0), np.nan_to_num(o_, nan=-7.0))
                assert np.array_equal(np.nan_to_num(w["predicted"][i], nan=-7.0), np.nan_to_num(gp[-1], nan=-7.0))
                n_checked += 1
    assert n_checked > 30


@pytest.mark.parametrize("kind", [1, 3])
def test_positional_list_overflow_takes_the_dense_voting_kernels(eng, oracle, kind, monkeypatch):
    """A crowd: 260 boxes on a 500 x 400 canvas, Mahalanobis metric -- nearly every (candidate, track) pair passes the 2R
    gate, ~60 k positional entries per scene against a list of 6 k.  That scene's entry list overflows, the device flags
    it, fills and rescans its dense matrix and the dense Kuhn-Munkres kernel solves it, while the sparse scene next to it
    stays on the lists.  Assignments must be the oracle's."""
    from similari_b200.workload import Workload

    visual = kind == 3
    if visual:
        monkeypatch.setenv("SB200_VIS_KERNEL", "tc")
    crowd = small("cfg5" if visual else "cfg2", n_scenes=1, n_objects=260, oriented=False, canvas=(500.0, 400.0),
                  feature_dim=64 if visual else 0, seed=11)
    sparse = small("cfg5" if visual else "cfg2", n_scenes=1, n_objects=120, oriented=False, canvas=(2500.0, 1800.0),
                   feature_dim=64 if visual else 0, seed=12)
    kw = dict(kind=kind, positional_kind=0, max_idle_epochs=3)
    if visual:
        kw.update(visual_kind=0, visual_threshold=0.7, feature_dim=64, visual_max_observations=3, visual_min_votes=2,
                  visual_minimal_track_length=1, min_confidence=0.1)
    g, o = both(eng, oracle, **kw)
    w1, w2 = Workload(crowd), Workload(sparse, scene_base=1)
    for fr in range(5):
        f1, f2 = w1.next_frame(), w2.next_frame()
        if visual and fr >= 1:     # half of the crowd's detections carry no feature: they go to the positional stage
            hasf = np.ones(len(f1["boxes"]) + len(f2["boxes"]), np.uint8)
            hasf[: len(f1["boxes"]) : 2] = 0
        else:
            hasf = None
        boxes = np.concatenate([f1["boxes"], f2["boxes"]])
        feats = np.concatenate([f1["features"], f2["features"]]) if visual else None
        offs = np.array([0, len(f1["boxes"]), len(boxes)], np.int32)
        rg = g.predict_batch([0, 1], offs, boxes, features=feats, has_feature=hasf)
        ro = o.predict_batch([0, 1], offs, boxes, features=feats, has_feature=hasf)
        for key in ("ids", "epochs", "lengths", "voting_types"):
            assert np.array_equal(rg[key], ro[key]), (fr, key, int((rg[key] != ro[key]).sum()))
    assert g.active_tracks() == o.active_tracks()


@pytest.mark.parametrize("join_per_call", [True, False])
def test_caller_stream_is_joined_by_events(eng, oracle, join_per_call):
    """sb200_tracker_set_stream: the tracker runs on its own streams and is ordered with the caller's by events.  Inputs are
    produced on the caller's stream right before each call (a device copy from a staging tensor into the buffer the call
    reads -- the call must wait for it), outputs are consumed on that stream right after it (a device copy out of a buffer
    the NEXT call overwrites): with join_per_call the stream waits for every frame by itself, without it
    sb200_stream_join makes it wait.  Either way the snapshots must be the oracle's, frame by frame."""
    import torch

    from similari_b200.workload import Workload

    cfg = small("cfg5", n_scenes=5, n_objects=50, oriented=False, canvas=(800.0, 600.0), feature_dim=64, drop_frac=0.1,
                fresh_frac=0.1)
    kw = dict(kind=3, positional_kind=1, iou_threshold=0.3, max_idle_epochs=2, visual_kind=0, visual_threshold=0.7,
              feature_dim=64, visual_max_observations=3, visual_min_votes=2, visual_minimal_track_length=1, min_confidence=0.1)
    g, o = both(eng, oracle, **kw)
    dev = torch.device("cuda", 0)
    side = torch.cuda.Stream(device=dev)
    g.set_stream(side.cuda_stream, join_per_call=join_per_call)
    wl = Workload(cfg)
    frames = [wl.next_frame() for _ in range(8)]
    ref = [o.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=f["features"]) for f in frames]
    cap = max(len(f["boxes"]) for f in frames)
    # staging tensors per frame (filled up front), ONE input buffer and ONE output buffer reused by every call
    st_b = [torch.from_numpy(np.ascontiguousarray(f["boxes"])).to(dev) for f in frames]
    st_f = [torch.from_numpy(np.ascontiguousarray(f["features"])).to(dev) for f in frames]
    in_b = torch.zeros(cap, 6, dtype=torch.float32, device=dev)
    in_f = torch.zeros(cap, 64, dtype=torch.float32, device=dev)
    d_ids = torch.zeros(cap, dtype=torch.int64, device=dev)
    snaps = []
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        for f, sb_, sf_ in zip(frames, st_b, st_f):
            n = len(f["boxes"])
            in_b[:n].copy_(sb_, non_blocking=True)      # on the caller's stream, right before the call
            in_f[:n].copy_(sf_, non_blocking=True)
            g.predict_batch_device(f["scene_ids"], f["det_offsets"], in_b.data_ptr(), in_f.data_ptr(), d_ids=d_ids.data_ptr())
            if not join_per_call:
                g.stream_join(side.cuda_stream)
            snaps.append(d_ids[:n].clone())             # on the caller's stream, right after the call
    side.synchronize()
    g.sync()
    for fr, (sn, ro) in enumerate(zip(snaps, ref)):
        assert np.array_equal(sn.cpu().numpy().astype(np.uint64), ro["ids"].astype(np.uint64)), fr
