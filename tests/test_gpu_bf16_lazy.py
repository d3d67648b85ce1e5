"""BF16 arena rows on the e4m3 screen.

Frames on the e4m3 screen do not write the BF16 copies of the stored feature rows; the tracker converts the rows they
skipped again before the first frame or blob that reads them.  A tracker that switches between the screens must hold,
return and save exactly what a tracker on the BF16 screen throughout holds: every predict column and the state blob
(which carries the BF16 rows) are compared byte for byte.  No track expires here: the scenes of a frame append their
expired tracks to the wasted buffer concurrently, in an order no two runs share, and that buffer is part of the blob."""
import dataclasses

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

COLS = ("ids", "epochs", "lengths", "voting_types", "predicted", "observed")


@pytest.fixture(scope="module")
def eng():
    import similari_b200.engine as e
    from similari_b200._lib import lib

    if lib().sb200_device_count() <= 0:
        pytest.fail("no CUDA device: the gpu-marked tests must run on an H100")
    return e


def _same(a, b, what=""):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape and a.dtype == b.dtype, what
    assert a.tobytes() == b.tobytes(), what


def _opts(metric, threshold, dim, **over):
    from similari_b200._lib import default_options

    kw = dict(kind=3, positional_kind=1, iou_threshold=0.3, max_idle_epochs=1000, visual_kind=metric,
              visual_threshold=threshold, feature_dim=dim, visual_max_observations=3, visual_min_votes=1,
              visual_minimal_track_length=1)
    kw.update(over)
    return default_options(**kw)


def _copy(opts):
    import ctypes as C

    o = type(opts)()
    C.memmove(C.byref(o), C.byref(opts), C.sizeof(opts))
    return o


def _frames(n_scenes, n_objects, dim, n_frames, seed, fresh=0.1):
    from similari_b200.workload import CONFIGS, Workload

    cfg = dataclasses.replace(CONFIGS["cfg5"], n_scenes=n_scenes, n_objects=n_objects, feature_dim=dim,
                              canvas=(900.0, 600.0), drop_frac=0.2, fresh_frac=fresh, seed=seed)
    wl = Workload(cfg)
    return [wl.next_frame() for _ in range(n_frames)]


def _column(feats, t):
    if t == "f32":
        return feats, None
    if t == "f16":
        return np.ascontiguousarray(feats.astype(np.float16)), t
    import torch

    tb = torch.from_numpy(np.ascontiguousarray(feats, dtype=np.float32)).to(torch.bfloat16)
    return tb.view(torch.int16).numpy().view(np.uint16).copy(), t


def _step(monkeypatch, trackers, f, t="f32"):
    """One frame on each (tracker, SB200_VIS_KERNEL) pair; the predict columns must agree."""
    feats, ft = _column(f["features"], t)
    res = []
    for tr, env in trackers:
        monkeypatch.setenv("SB200_VIS_KERNEL", env)
        res.append(tr.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=feats, feature_type=ft))
    for k in COLS:
        for r in res[1:]:
            _same(res[0][k], r[k], k)


@pytest.mark.parametrize("t", ["f32", "f16", "bf16"])
@pytest.mark.parametrize("metric", [0, 1], ids=["euclidean", "cosine"])
def test_e4m3_streak_then_bf16(eng, monkeypatch, metric, t):
    frames = _frames(4, 96, 512, 9, seed=0xB16 + metric)
    opts = _opts(metric, 0.7 if metric == 0 else 0.5, 512)
    a, b = eng.Tracker(opts), eng.Tracker(_copy(opts))
    for f in frames[:5]:
        _step(monkeypatch, [(a, "tc8"), (b, "tc16")], f, t)
    _same(a.save(), b.save(), "blob after the e4m3 streak")
    for f in frames[5:]:
        _step(monkeypatch, [(a, "tc16"), (b, "tc16")], f, t)
    _same(a.save(), b.save(), "blob after the switch")
    c = a.screen_counters()
    e8, e16 = c["fp8_frames"], c["bf16_frames"]
    assert e8 >= 4 and e16 == 4, (e8, e16)   # (the first frame has no tracks to screen)


def test_automatic_fallback(eng, monkeypatch):
    """Cosine at a threshold in the bulk of the distribution: the e4m3 screen keeps too many pairs, the tracker goes back
    to the BF16 screen after its first frame, and the BF16 rows that frame skipped are converted first."""
    frames = _frames(4, 128, 512, 6, seed=0xFA11)
    opts = _opts(1, 0.2, 512)
    a, b = eng.Tracker(opts), eng.Tracker(_copy(opts))
    for f in frames:
        _step(monkeypatch, [(a, "tc"), (b, "tc16")], f)
    c = a.screen_counters()
    e8, e16 = c["fp8_frames"], c["bf16_frames"]
    assert e8 >= 1 and e16 >= 1, (e8, e16)
    _same(a.save(), b.save(), "blob")


def test_dense_after_e4m3(eng, monkeypatch):
    frames = _frames(4, 96, 512, 7, seed=0xDE5E)
    opts = _opts(0, 0.7, 512)
    a, b = eng.Tracker(opts), eng.Tracker(_copy(opts))
    for f in frames[:4]:
        _step(monkeypatch, [(a, "tc8"), (b, "tc16")], f)
    for f in frames[4:]:
        _step(monkeypatch, [(a, "dense"), (b, "dense")], f)
    _same(a.save(), b.save(), "blob")


def test_export_import_after_e4m3(eng, monkeypatch):
    frames = _frames(4, 96, 256, 8, seed=0xE4)
    opts = _opts(0, 0.7, 256)
    a, b = eng.Tracker(opts), eng.Tracker(_copy(opts))
    for f in frames[:4]:
        _step(monkeypatch, [(a, "tc8"), (b, "tc16")], f)
    ids = [int(s) for s in frames[0]["scene_ids"][:2]]
    xa, xb = a.export_scenes(ids, remove=True), b.export_scenes(ids, remove=True)
    _same(xa, xb, "scene blob")
    a2, b2 = eng.Tracker(opts), eng.Tracker(_copy(opts))
    a2.import_scenes(xa)
    b2.import_scenes(xb)
    a.import_scenes(xa)
    b.import_scenes(xb)
    for f in frames[4:6]:
        _step(monkeypatch, [(a, "tc8"), (b, "tc16")], f)
        _step(monkeypatch, [(a2, "tc8"), (b2, "tc16")], f)
    # (whole-tracker blobs after an import are not compared: they differ between two runs of the same tracker)
    for f in frames[6:]:
        _step(monkeypatch, [(a, "tc16"), (b, "tc16")], f)
        _step(monkeypatch, [(a2, "tc16"), (b2, "tc16")], f)


def test_store_regrow_after_e4m3(eng, monkeypatch):
    """Frames of 40 detections per scene on e4m3, then frames of 300: the store grows (its row pitch changes) after rows
    were skipped."""
    small = _frames(4, 40, 512, 3, seed=0x6A0)
    big = _frames(4, 300, 512, 4, seed=0x6A1)
    opts = _opts(0, 0.7, 512)
    a, b = eng.Tracker(opts), eng.Tracker(_copy(opts))
    for f in small + big[:2]:
        _step(monkeypatch, [(a, "tc8"), (b, "tc16")], f)
    # (blobs after a regrow are not compared: they differ between two runs of the same tracker)
    for f in big[2:]:
        _step(monkeypatch, [(a, "tc16"), (b, "tc16")], f)


def test_streak_past_the_dirty_log(eng, monkeypatch):
    """More stored rows than the dirty-row log holds (2^18): every arena row is converted at the switch."""
    frames = _frames(6, 1024, 64, 70, seed=0x10C, fresh=0.0)
    opts = _opts(0, 0.7, 64)
    a, b = eng.Tracker(opts), eng.Tracker(_copy(opts))
    for f in frames[:66]:
        _step(monkeypatch, [(a, "tc8"), (b, "tc16")], f)
    assert sum(int(f["det_offsets"][-1]) for f in frames[:66]) > (1 << 18)
    for f in frames[66:]:
        _step(monkeypatch, [(a, "tc16"), (b, "tc16")], f)
    _same(a.save(), b.save(), "blob")
