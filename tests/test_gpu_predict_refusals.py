"""Refused predict requests change nothing.

Two trackers get the same frames; one of them also gets one malformed (or too large) request, through the C ABI because
the Python wrapper cannot pass most of these arguments.  The call must return its error code, and from then on the two
trackers must agree: epochs and track counts right after the refusal, every later frame's outputs and track counts,
and wasted() after the 100-call auto-waste tick.  A refused call that counted as a call would move the tick by one
frame: the tracks swept early are counted until the tick collects them, so the counts of that frame would differ.  Each
refusal also comes once with a frame in flight on both trackers (the solver bound then waits for it and checks again).

A prefetched input set whose columns the predict call has to grow is copied again, not read after the growth."""
import ctypes as C

import numpy as np
import pytest

from test_gpu_voting import smem_fits

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_CAPACITY = -1, -3
BIG_SCENE = 987654321   # the scene of the solver_capacity request: never created
REFUSE_AT, FRAMES = 4, 106   # the tick falls on the 101st call


@pytest.fixture(scope="module")
def eng():
    import similari_b200.engine as e
    from similari_b200._lib import lib

    if lib().sb200_device_count() <= 0:
        pytest.fail("no CUDA device: the gpu-marked tests must run on an H100")
    return e


def _solver_overflow_m():
    """The smallest scene of m detections (no stored tracks) that the on-chip assignment solver cannot hold (Sort: no
    visual list)."""
    m = 1
    while smem_fits(m, 0, viscap=0):
        m += 1
    return m


def _refusal(case, frame):
    """(n_scenes, scene_ids, det_offsets, boxes, expected status) of a refused request built around `frame`."""
    sids = np.ascontiguousarray(frame["scene_ids"][:2], dtype=np.uint64)
    offs = np.ascontiguousarray(frame["det_offsets"][:3], dtype=np.int32)
    boxes = np.ascontiguousarray(frame["boxes"][: int(offs[-1])], dtype=np.float32)
    if case == "negative_n_scenes":
        return -1, sids, offs, boxes, ERR_INVALID
    if case == "null_scene_ids":
        return 2, None, offs, boxes, ERR_INVALID
    if case == "null_det_offsets":
        return 2, sids, None, boxes, ERR_INVALID
    if case == "first_offset_not_zero":
        return 2, sids, offs + 1, boxes, ERR_INVALID
    if case == "decreasing_offsets":
        bad = offs.copy()
        bad[1] = bad[2] + 1
        return 2, sids, bad, boxes, ERR_INVALID
    if case == "null_boxes":
        return 2, sids, offs, None, ERR_INVALID
    if case == "scene_twice":
        return 2, np.array([sids[0], sids[0]], np.uint64), offs, boxes, ERR_INVALID
    if case == "solver_capacity":
        m = _solver_overflow_m()
        big = np.resize(np.asarray(frame["boxes"], np.float32).reshape(-1, 6), (m, 6))
        return 1, np.array([BIG_SCENE], np.uint64), np.array([0, m], np.int32), np.ascontiguousarray(big), ERR_CAPACITY
    raise AssertionError(case)


def _call_abi(t, n, sids, offs, boxes):
    from similari_b200._lib import PredictOut, lib, ptr

    total = max(len(boxes) if boxes is not None else 0, 1)
    ids = np.zeros(total, np.uint64)
    po = PredictOut(ptr(ids), None, None, None, None, None)
    return lib().sb200_predict_batch(t._h, n, ptr(sids), ptr(offs), ptr(boxes), None, None, None, None, None, C.byref(po))


@pytest.mark.parametrize("in_flight", [False, True])
@pytest.mark.parametrize("case", ["negative_n_scenes", "null_scene_ids", "null_det_offsets", "first_offset_not_zero",
                                  "decreasing_offsets", "null_boxes", "scene_twice", "solver_capacity"])
def test_refused_request_changes_nothing(eng, case, in_flight):
    import dataclasses

    from similari_b200._lib import default_options
    from similari_b200.workload import CONFIGS, Workload

    cfg = dataclasses.replace(CONFIGS["cfg2"], n_scenes=3, n_objects=24, fresh_frac=0.1)
    kw = dict(kind=1, positional_kind=1, iou_threshold=0.3, max_idle_epochs=1)
    ref, t = eng.Tracker(default_options(**kw)), eng.Tracker(default_options(**kw))
    wl = Workload(cfg)
    scene_ids = None
    for fr in range(FRAMES):
        f = wl.next_frame()
        scene_ids = f["scene_ids"]
        queued = fr == REFUSE_AT and in_flight
        ro = ref.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], wait=False) if queued else None
        rt = t.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], wait=False) if queued else None
        if fr == REFUSE_AT:
            n, sids, offs, boxes, want = _refusal(case, f)
            assert _call_abi(t, n, sids, offs, boxes) == want
            if queued:
                ref.sync()
                t.sync()
            for s in scene_ids:
                assert t.current_epoch(int(s)) == ref.current_epoch(int(s)), fr
            assert np.array_equal(t.scene_track_counts(scene_ids), ref.scene_track_counts(scene_ids))
            assert t.current_epoch(BIG_SCENE) == 0 and t.scene_track_counts([BIG_SCENE])[0] == 0
        if not queued:
            ro = ref.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"])
            rt = t.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"])
        for key in ro:
            assert np.array_equal(np.nan_to_num(rt[key], nan=-7.0), np.nan_to_num(ro[key], nan=-7.0)), (fr, key)
        assert np.array_equal(t.scene_track_counts(scene_ids), ref.scene_track_counts(scene_ids)), fr
    for s in scene_ids:
        assert t.current_epoch(int(s)) == ref.current_epoch(int(s))
    # the end-of-frame sweeps append the records in device order: compare them by id
    wo, wt = ref.wasted(), t.wasted()
    assert len(wo["ids"]) > 0
    so, st = np.argsort(wo["ids"], kind="stable"), np.argsort(wt["ids"], kind="stable")
    for key in wo:
        assert np.array_equal(np.nan_to_num(wt[key][st], nan=-7.0), np.nan_to_num(wo[key][so], nan=-7.0)), key


def test_prefetched_set_grown_by_predict_is_copied_again(eng):
    """The prefetch sizes its staging set without the scene count; a predict call with more scenes than the hint sizes
    the columns for more rows.  Boxes and features are already big enough from earlier frames, the quality column is
    not: predict grows it, which drops its contents, so it must copy the request again rather than use the set."""
    import dataclasses

    from similari_b200._lib import default_options
    from similari_b200.workload import CONFIGS, Workload

    cfg = dataclasses.replace(CONFIGS["cfg5"], n_scenes=4, n_objects=8, feature_dim=32, canvas=(1920.0, 1080.0))
    kw = dict(kind=3, positional_kind=1, iou_threshold=0.3, max_idle_epochs=5, visual_kind=0, visual_threshold=1.0,
              feature_dim=32, visual_max_observations=3, visual_min_votes=1, visual_minimal_track_length=1,
              visual_minimal_quality_use=0.5, visual_minimal_quality_collect=0.5, max_scenes_hint=1,
              max_dets_per_scene_hint=16)
    ref, t = eng.Tracker(default_options(**kw)), eng.Tracker(default_options(**kw))
    wl = Workload(cfg)
    for fr in range(8):
        f = wl.next_frame()
        boxes = np.ascontiguousarray(f["boxes"], np.float32).reshape(-1, 6)
        feats = np.ascontiguousarray(f["features"], np.float32)
        quality = np.full(len(boxes), 0.9, np.float32) if fr >= 2 else None
        if quality is not None:
            t.prefetch_inputs(boxes, features=feats, quality=quality)
        ro = ref.predict_batch(f["scene_ids"], f["det_offsets"], boxes, features=feats, quality=quality)
        rt = t.predict_batch(f["scene_ids"], f["det_offsets"], boxes, features=feats, quality=quality)
        for key in ro:
            assert np.array_equal(np.nan_to_num(rt[key], nan=-7.0), np.nan_to_num(ro[key], nan=-7.0)), (fr, key)
    assert t.active_tracks() == ref.active_tracks()
