"""FP16 and BF16 feature columns (sb200_set_feature_type).

Widening binary16 or bfloat16 to f32 is exact, so a tracker fed half-precision rows must return exactly what a tracker
with the same options returns when fed the widened f32 copy of the same rows: every predict column, the cost matrices,
the work counters (the same kernel path ran), the stored feature histories and the state blob.  Every comparison here
is on the raw bytes."""
import dataclasses

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

F32MAX = float(np.finfo(np.float32).max)
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


def _opts(kind, metric, threshold, dim, **over):
    from similari_b200._lib import default_options

    kw = dict(kind=kind, positional_kind=1, iou_threshold=0.3, max_idle_epochs=2, history_length=3, visual_kind=metric,
              visual_threshold=threshold, feature_dim=dim, visual_max_observations=3, visual_min_votes=1,
              visual_minimal_track_length=1, visual_minimal_quality_use=0.2, visual_minimal_quality_collect=0.3)
    kw.update(over)
    return default_options(**kw)


def _frames(n_scenes, n_objects, dim, n_frames, seed, degenerate=True):
    """Workload frames with a has_feature column (about 10 % absent), a quality column and, in scene 0, rows of zeros
    and rows of one large constant next to the clean unit vectors of the other scenes."""
    from similari_b200.workload import CONFIGS, Workload

    cfg = dataclasses.replace(CONFIGS["cfg5"], n_scenes=n_scenes, n_objects=n_objects, feature_dim=dim,
                              canvas=(900.0, 600.0), drop_frac=0.2, fresh_frac=0.1, seed=seed)
    wl = Workload(cfg)
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n_frames):
        f = wl.next_frame()
        total = int(f["det_offsets"][-1])
        if degenerate and n_objects >= 8:
            m0 = int(f["det_offsets"][1])
            f["features"][: min(3, m0)] = 0.0
            f["features"][3: min(6, m0)] = 1000.0
        f["has_feature"] = (rng.random(total) >= 0.1).astype(np.uint8)
        f["quality"] = rng.uniform(0.0, 1.0, total).astype(np.float32)
        out.append(f)
    return out


def _narrow(feats, t):
    """(the column as sent, its exact f32 widening).  bf16 goes through torch and is sent as its uint16 bits."""
    if t == "f16":
        h = np.ascontiguousarray(feats.astype(np.float16))
        return h, h.astype(np.float32)
    import torch

    tb = torch.from_numpy(np.ascontiguousarray(feats, dtype=np.float32)).to(torch.bfloat16)
    return tb.view(torch.int16).numpy().view(np.uint16).copy(), tb.float().numpy().copy()


def _counters(t):
    w = t.work_counters()
    return (w["pair_associations"], w["visual_dot_products"], w["frames"], w["dense_fallback_scenes"], w["tc_frames"])


def _same_wasted(a, b):
    """wasted_visual() of both trackers, record by record.  Scenes append to the wasted buffer concurrently, so the
    records are matched by (scene, id), not by position."""
    wa, wb = a.wasted_visual(), b.wasted_visual()
    oa, ob = (np.lexsort((w["ids"], w["scene_ids"])) for w in (wa, wb))
    for k in ("ids", "scene_ids", "epochs", "lengths", "predicted", "observed"):
        _same(wa[k][oa], wb[k][ob], k)
    for k in ("features", "feature_present", "predicted_history", "observed_history"):
        assert len(wa[k]) == len(wb[k])
        for i, j in zip(oa, ob):
            _same(wa[k][i], wb[k][j], k)
    return len(wa["ids"])


def _pair(eng, opts, frames, t, scenes_checked=(0, 1), history=True):
    """Tracker A fed the narrow column, tracker B the widened copy; everything compared frame by frame."""
    a, b = eng.Tracker(opts), eng.Tracker(_copy(opts))
    if history:
        a.set_feature_history(True)
        b.set_feature_history(True)
    for fr, f in enumerate(frames):
        h, w = _narrow(f["features"], t)
        kw = dict(has_feature=f["has_feature"], quality=f["quality"])
        ra = a.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=h, feature_type=t, **kw)
        rb = b.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=w, **kw)
        for k in COLS:
            _same(ra[k], rb[k], f"frame {fr}: {k}")
        for s in scenes_checked:
            if s < len(f["scene_ids"]):
                _same(a.last_costs(int(f["scene_ids"][s])), b.last_costs(int(f["scene_ids"][s])), f"frame {fr}: costs")
    assert a.feature_type == t and b.feature_type == "f32"
    assert _counters(a) == _counters(b)
    return a, b


def _copy(opts):
    import ctypes as C

    o = type(opts)()
    C.memmove(C.byref(o), C.byref(opts), C.sizeof(opts))
    return o


PATHS = {   # visual cost path -> (SB200_VIS_KERNEL, euclidean threshold, cosine threshold)
    "screen": ("tc", 0.7, 0.2),
    "dense": ("dense", F32MAX, -1.0),
    "simt": ("simt", 0.7, 0.2),
}


@pytest.mark.parametrize("t", ["f16", "bf16"])
@pytest.mark.parametrize("dim", [512, 100, 129])
@pytest.mark.parametrize("metric", [0, 1], ids=["euclidean", "cosine"])
@pytest.mark.parametrize("path", list(PATHS))
def test_batch_visual_sort_matches_widened_f32(eng, monkeypatch, path, metric, dim, t):
    env, thr_e, thr_c = PATHS[path]
    monkeypatch.setenv("SB200_VIS_KERNEL", env)
    n_obj = 24 if path == "simt" else 96
    frames = _frames(4, n_obj, dim, 6, seed=0xF16 + dim + 7 * metric)
    a, b = _pair(eng, _opts(3, metric, thr_e if metric == 0 else thr_c, dim), frames, t)
    if path != "simt":
        assert _counters(a)[4] > 0   # the tensor-core path ran
    for s in range(4):
        a.skip_epochs(5, s)
        b.skip_epochs(5, s)
    assert _same_wasted(a, b) > 0


@pytest.mark.parametrize("t", ["f16", "bf16"])
@pytest.mark.parametrize("metric", [0, 1], ids=["euclidean", "cosine"])
def test_visual_sort_single_scene_and_blob(eng, monkeypatch, metric, t):
    """VisualSort on one scene, screen path: the results and the saved blobs are identical.  (Without the feature
    history: its pool hands out blocks in the order the detections' threads reach it, which no two runs share.)"""
    monkeypatch.setenv("SB200_VIS_KERNEL", "tc")
    frames = _frames(1, 200, 129, 6, seed=0xB10B + metric)
    a, b = _pair(eng, _opts(2, metric, 0.7 if metric == 0 else 0.2, 129), frames, t, scenes_checked=(0,), history=False)
    _same(a.save(), b.save(), "blob")


def _special_rows(total, dim, t, rng):
    """Rows of +-0, subnormals, +-Inf, NaN with payloads and the largest finite value in every lane."""
    f = rng.standard_normal((total, dim)).astype(np.float32)
    f /= np.linalg.norm(f, axis=1, keepdims=True)
    if t == "f16":
        h = f.astype(np.float16)
        u = h.view(np.uint16)
        specials = [0x0000, 0x8000, 0x0001, 0x83FF, 0x7C00, 0xFC00, 0x7E01, 0xFE55, 0x7BFF]
        for i, v in enumerate(specials):
            u[i] = v
        u[len(specials)][::2] = 0x0001
        return h, h.astype(np.float32)
    import torch

    bits = torch.from_numpy(f).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16).copy()
    specials = [0x0000, 0x8000, 0x0001, 0x807F, 0x7F80, 0xFF80, 0x7FC1, 0xFFE5, 0x7F7F]
    for i, v in enumerate(specials):
        bits[i] = v
    wide = (bits.astype(np.uint32) << 16).view(np.float32)
    return bits, wide


@pytest.mark.parametrize("t", ["f16", "bf16"])
@pytest.mark.parametrize("path", ["screen", "simt"])
def test_special_values(eng, monkeypatch, t, path):
    monkeypatch.setenv("SB200_VIS_KERNEL", PATHS[path][0])
    dim = 64
    rng = np.random.default_rng(7)
    frames = _frames(2, 80, dim, 4, seed=0x5BEC, degenerate=False)
    a = eng.Tracker(_opts(3, 1, 0.2, dim))
    b = eng.Tracker(_opts(3, 1, 0.2, dim))
    a.set_feature_history(True)
    b.set_feature_history(True)
    for f in frames:
        h, w = _special_rows(int(f["det_offsets"][-1]), dim, t, rng)
        ra = a.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=h, feature_type=t)
        rb = b.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=w)
        for k in COLS:
            _same(ra[k], rb[k], k)
    for s in range(2):
        a.skip_epochs(5, s)
        b.skip_epochs(5, s)
    assert _same_wasted(a, b) > 0


def test_async_and_prefetched_host_paths(eng):
    from similari_b200._lib import pinned_empty

    dim = 128
    frames = _frames(3, 64, dim, 8, seed=0xA5C)
    a, p, b = (eng.Tracker(_opts(3, 0, 0.7, dim)) for _ in range(3))
    outs = []
    for f in frames:
        h, w = _narrow(f["features"], "f16")
        total = int(f["det_offsets"][-1])
        out = {"ids": pinned_empty(total, np.uint64), "lengths": pinned_empty(total, np.uint32)}
        a.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=h, out=out, wait=False)
        p.prefetch_inputs(f["boxes"], features=h)
        rp = p.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=h)
        rb = b.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=w)
        outs.append((out, rb))
        _same(rp["ids"], rb["ids"])
        _same(rp["predicted"], rb["predicted"])
    a.sync()
    for out, rb in outs:
        _same(out["ids"], rb["ids"])
        _same(out["lengths"], rb["lengths"])
    assert a.feature_type == "f16" and p.feature_type == "f16"


def test_prefetch_under_another_type_is_not_used(eng):
    """A prefetch of a 2-byte column is not consumed by a predict that reads the same pointer as f32."""
    dim = 64
    frames = _frames(2, 50, dim, 4, seed=0x9EF)
    a, b = eng.Tracker(_opts(3, 0, 0.7, dim)), eng.Tracker(_opts(3, 0, 0.7, dim))
    for f in frames:
        x = np.ascontiguousarray(f["features"], dtype=np.float32)
        total = len(x)
        h = x.reshape(-1).view(np.float16)[: total * dim].reshape(total, dim)   # same base pointer, half the bytes
        a.prefetch_inputs(f["boxes"], features=h)
        ra = a.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=x)
        rb = b.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=x)
        for k in COLS:
            _same(ra[k], rb[k], k)


@pytest.mark.parametrize("misaligned", [False, True], ids=["aligned", "offset2"])
@pytest.mark.parametrize("t", ["f16", "bf16"])
def test_device_path_torch_tensors(eng, monkeypatch, t, misaligned):
    import torch

    monkeypatch.setenv("SB200_VIS_KERNEL", "tc")
    dim = 256
    tdt = torch.float16 if t == "f16" else torch.bfloat16
    frames = _frames(3, 96, dim, 5, seed=0xDE7 + misaligned)
    a, b = eng.Tracker(_opts(3, 1, 0.2, dim)), eng.Tracker(_opts(3, 1, 0.2, dim))
    a.set_feature_history(True)
    b.set_feature_history(True)
    for f in frames:
        total = int(f["det_offsets"][-1])
        ft = torch.from_numpy(f["features"]).cuda().to(tdt)
        base = torch.zeros(total * dim + 8, dtype=tdt, device="cuda")
        off = 1 if misaligned else 0
        base[off: off + total * dim] = ft.reshape(-1)
        db = torch.from_numpy(f["boxes"]).cuda()
        dhf = torch.from_numpy(f["has_feature"]).cuda()
        dq = torch.from_numpy(f["quality"]).cuda()
        ids = torch.zeros(total, dtype=torch.int64, device="cuda")
        vt = torch.zeros(total, dtype=torch.uint8, device="cuda")
        pred = torch.zeros((total, 6), dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        a.predict_batch_device(f["scene_ids"], f["det_offsets"], db.data_ptr(), base.data_ptr() + 2 * off, dhf.data_ptr(),
                               dq.data_ptr(), d_ids=ids.data_ptr(), d_voting_types=vt.data_ptr(),
                               d_predicted=pred.data_ptr(), feature_type=t)
        a.sync()
        rb = b.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=ft.float().cpu().numpy(),
                             has_feature=f["has_feature"], quality=f["quality"])
        _same(ids.cpu().numpy().view(np.uint64), rb["ids"])
        _same(vt.cpu().numpy(), rb["voting_types"])
        _same(pred.cpu().numpy(), rb["predicted"])
        _same(a.last_costs(0), b.last_costs(0))
    assert _counters(a) == _counters(b)
    for s in range(3):
        a.skip_epochs(5, s)
        b.skip_epochs(5, s)
    assert _same_wasted(a, b) > 0


def test_switching_types_between_frames(eng, monkeypatch):
    """f32 -> f16 -> bf16 -> f32 ... on one tracker, with frames in flight, against an all-f32 tracker."""
    from similari_b200._lib import pinned_empty

    monkeypatch.setenv("SB200_VIS_KERNEL", "tc")
    dim = 100
    frames = _frames(3, 96, dim, 9, seed=0x5317)
    a, b = eng.Tracker(_opts(3, 0, 0.7, dim)), eng.Tracker(_opts(3, 0, 0.7, dim))
    kept = []
    for fr, f in enumerate(frames):
        t = ("f32", "f16", "bf16")[fr % 3]
        if t == "f32":
            h = w = np.ascontiguousarray(f["features"], dtype=np.float32)
        else:
            h, w = _narrow(f["features"], t)
        total = int(f["det_offsets"][-1])
        out = {k: pinned_empty(total, np.uint64 if k == "ids" else np.uint32) for k in ("ids", "lengths")}
        a.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=h, out=out, wait=False,
                        feature_type=None if t != "bf16" else "bf16")
        assert a.feature_type == t
        rb = b.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=w)
        kept.append((out, rb, h))
    a.sync()
    for out, rb, _ in kept:
        _same(out["ids"], rb["ids"])
        _same(out["lengths"], rb["lengths"])
    assert _counters(a) == _counters(b)


def test_set_feature_type_refusals(eng):
    from similari_b200._lib import Sb200Error, default_options

    for kind in (0, 1):
        t = eng.Tracker(default_options(kind=kind))
        assert t._L.sb200_set_feature_type(t._h, 1) == -1
        # the wrapper never asks a Sort / BatchSort tracker to switch (it ignores the column)
        t.predict_batch([0], [0, 1], np.array([[10, 10, np.nan, 0.5, 40, 0.9]], np.float32),
                        features=np.zeros((1, 8), np.float16))
    v = eng.Tracker(_opts(2, 0, 0.7, 16))
    for bad in (3, -1, 255):
        assert v._L.sb200_set_feature_type(v._h, bad) == -1
    with pytest.raises(ValueError):
        v.set_feature_type("f64")
    with pytest.raises(Sb200Error):
        eng.Tracker(default_options(kind=1)).set_feature_type("f16")
    for good in (2, 1, 0):
        assert v._L.sb200_set_feature_type(v._h, good) == 0


def test_loaded_tracker_reads_f32(eng, monkeypatch):
    """A tracker saved while it ran on f16 loads as an f32 reader; fed the widened copies it continues exactly like the
    saved tracker fed f16."""
    monkeypatch.setenv("SB200_VIS_KERNEL", "tc")
    dim = 129
    frames = _frames(3, 96, dim, 8, seed=0x10AD)
    a = eng.Tracker(_opts(3, 1, 0.2, dim))
    a.set_feature_history(True)
    for f in frames[:4]:
        a.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=_narrow(f["features"], "f16")[0],
                        has_feature=f["has_feature"], quality=f["quality"])
    c = eng.Tracker.load(a.save())
    assert c.feature_type == "f32"
    for f in frames[4:]:
        h, w = _narrow(f["features"], "f16")
        kw = dict(has_feature=f["has_feature"], quality=f["quality"])
        ra = a.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=h, **kw)
        # an f32 array: the wrapper sends no type switch, so this relies on the loaded tracker reading f32
        rc = c.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=w, **kw)
        for k in COLS:
            _same(ra[k], rc[k], k)
    for s in range(3):
        a.skip_epochs(5, s)
        c.skip_epochs(5, s)
    assert _same_wasted(a, c) > 0
