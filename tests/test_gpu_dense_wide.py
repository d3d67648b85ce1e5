"""The dense tensor-core visual path (kernels_feat_dense.cu) on wide features, against the oracle.

ReID features of 1024 or 2048 components are common.  At those widths the weight-sum kernel runs its TMA ring over
many k-steps (32 at D = 2048 against 4 stages), D = 2000 ends on a partial 64-column chunk, the error terms of the
selection grow with D (dense_f32_err, dense_sample_margin) and the metadata, sample and select kernels see wide rows.
Every case forces the path (SB200_VIS_KERNEL=dense), compares every frame with the oracle and checks how many
scene-frames the path handed to the exact kernels.  The constructions are those of test_gpu_visual_bounds.py."""
import dataclasses
import os
import time

import numpy as np
import pytest

from test_gpu_visual_bounds import (F32MAX, ROW_TIE_SEEDS, VIS_KW, _check_column_tie, _drive, _far_box, _frame,
                                    _grid_boxes, _tie_scenes, bf16, dense_row_interval, row_tie_features, screen_pair,
                                    unit)


@pytest.fixture(scope="module")
def eng():
    import similari_b200.engine as e
    from similari_b200._lib import lib

    if lib().sb200_device_count() <= 0:
        pytest.fail("no CUDA device: the gpu-marked tests must run on an H100")
    return e


def _dense(monkeypatch, generic=False):
    monkeypatch.setenv("SB200_VIS_KERNEL", "dense")
    if generic:
        monkeypatch.setenv("SB200_DENSE_GENERIC", "1")


def _opts(vis, d, kobs, **over):
    kw = dict(kind=3, visual_kind=vis, visual_threshold=F32MAX if vis == 0 else -1.0, feature_dim=d,
              visual_max_observations=kobs, visual_min_votes=2, **VIS_KW)
    kw.update(over)
    return kw


# ------------------------------------------------------------------------------------------------------------ row tie
@pytest.mark.gpu
@pytest.mark.parametrize("kobs,generic", [(3, False), (6, True)])
@pytest.mark.parametrize("vis", [0, 1])
@pytest.mark.parametrize("d", [1024, 2000, 2048, 4096])
def test_row_tie_wide(eng, oracle, d, vis, kobs, generic, monkeypatch):
    """row_tie_features at wide D (2000: the last 64-column k-chunk is partial): BF16 orders q's two tracks the wrong
    way, so only the error interval keeps t1.  Tracks hold kobs identical observations; in the last frame q replaces
    t2's detection far from both, and no scene may leave the path."""
    _dense(monkeypatch, generic)
    n = 40
    q, t1, t2 = row_tie_features(ROW_TIE_SEEDS[vis] + d, d)
    rng = np.random.default_rng(7 + d)
    base = np.stack([unit(rng, d) for _ in range(n)]).astype(np.float32) * np.float32(np.linalg.norm(q))
    base[0], base[1] = t1, t2
    frames = []
    for fr in range(kobs + 1):
        scenes = []
        for _ in range(3):
            boxes, feats = _grid_boxes(n), base.copy()
            if fr == kobs:
                feats[1] = q
                boxes[1] = _far_box(0)
            scenes.append((boxes, feats))
        frames.append(_frame(scenes))
    g = _drive(eng, oracle, _opts(vis, d, kobs), frames)
    wc = g.work_counters()
    assert wc["tc_frames"] >= kobs and wc["dense_fallback_scenes"] == 0


# --------------------------------------------------------------------------------------------------------- column tie
COLUMN_CASES = [(vis, kobs, generic, scale) for vis in (0, 1) for kobs, generic in [(3, False), (6, True)]
                for scale in ((1.0, 3.0e4, 1.0e-6) if vis == 0 else (1.0,))]


@pytest.mark.gpu
@pytest.mark.parametrize("vis,kobs,generic,scale", COLUMN_CASES)
def test_column_tie_2048(eng, oracle, vis, kobs, generic, scale, monkeypatch):
    """The column near-tie of tie_scene_frames at D = 2048 in six scenes, one full of identical features.  At 3e4 the
    fp16 weight sums overflow, at 1e-6 they are subnormal; there the pair lists overflow to the exact kernels, so only
    the assignments are checked."""
    _dense(monkeypatch, generic)
    d, n = 2048, 70
    per_scene = _tie_scenes(d, n, kobs, 300 + kobs, [(None, None)] * 6, scale=scale, identical=(5,))
    frames = [_frame([sc[fr] for sc in per_scene]) for fr in range(kobs + 1)]
    g = _drive(eng, oracle, _opts(vis, d, kobs), frames)
    wc = g.work_counters()
    assert wc["tc_frames"] >= kobs
    if scale == 1.0:   # only the tied scene may fall back
        assert wc["dense_fallback_scenes"] <= kobs
    else:              # the overflowing pair lists send scenes to the exact kernels, never more than every scene-frame
        assert 1 <= wc["dense_fallback_scenes"] <= 6 * kobs


@pytest.mark.gpu
@pytest.mark.parametrize("vis", [0, 1])
def test_column_tie_k25_1024(eng, oracle, vis, monkeypatch):
    """25 observations per track at D = 1024: the warp-per-block metadata kernel, the any-K epilogue and the wide
    selection kernel, with the column near-tie in three scenes."""
    _dense(monkeypatch)
    d, n, kobs = 1024, 40, 25
    per_scene = _tie_scenes(d, n, kobs, 500 + vis, [(None, None)] * 3)
    frames = [_frame([sc[fr] for sc in per_scene]) for fr in range(kobs + 1)]
    g = _drive(eng, oracle, _opts(vis, d, kobs), frames)
    wc = g.work_counters()
    assert wc["tc_frames"] >= kobs and wc["dense_fallback_scenes"] == 0


# ------------------------------------------------------------------------------------------------ dense_norm_ok edge
def edge_feature(d, above):
    """A feature whose f32 squared norm, summed as cand_norm_kernel does, is exactly FLT_MAX / 4 = 2^126 - 2^102 (the
    largest value dense_norm_ok accepts), or 2^126 (the smallest above it)."""
    f = np.zeros(d, np.float32)
    if above:
        f[0] = np.float32(2.0 ** 63)
    else:
        f[0] = np.float32(2.0 ** 63 * (1 - 2.0 ** -24))   # square rounds to 2^126 - 2^103
        f[1] = np.float32(2.0 ** 51)                     # + 2^102, exactly
    return f


def test_edge_feature_norms():
    quarter = np.float32(np.finfo(np.float32).max) * np.float32(0.25)
    for above, want in ((False, quarter), (True, np.float32(2.0 ** 126))):
        f = edge_feature(64, above)
        sq = f[:8] * f[:8]                               # one block holds the whole norm: reduce_add8 adds it exactly
        n2 = ((sq[0] + sq[4]) + (sq[2] + sq[6])) + ((sq[1] + sq[5]) + (sq[3] + sq[7]))
        assert n2 == want and np.isfinite(n2)
    assert edge_feature(64, True)[0] * edge_feature(64, True)[0] > quarter


@pytest.mark.gpu
def test_dense_norm_edge(eng, oracle, monkeypatch):
    """Three scenes of features with norms near 2^62 (their fp16 weight sums overflow: every group is refined, which
    the small scenes' pair lists hold).  In the last frame scene 1 gets a detection whose squared norm is exactly the
    largest dense_norm_ok accepts, scene 2 one just above it.  Only that scene-frame of scene 2 may go to the exact
    kernels, and every assignment is the oracle's."""
    _dense(monkeypatch)
    d, n, kobs = 2048, 12, 3
    per_scene = _tie_scenes(d, n, kobs, 900, [(None, None)] * 3, scale=2.0 ** 62)
    for s, above in ((1, False), (2, True)):
        boxes, feats = per_scene[s][kobs]
        per_scene[s][kobs] = (np.concatenate([boxes, _far_box(1)[None]]),
                              np.concatenate([feats, edge_feature(d, above)[None]]))
    frames = [_frame([sc[fr] for sc in per_scene]) for fr in range(kobs + 1)]
    g = _drive(eng, oracle, _opts(0, d, kobs), frames)
    wc = g.work_counters()
    assert wc["tc_frames"] >= kobs and wc["dense_fallback_scenes"] == 1


# ----------------------------------------------------------------------------------------------------- feature types
@pytest.mark.gpu
@pytest.mark.parametrize("t", ["f16", "bf16"])
@pytest.mark.parametrize("metric", [0, 1], ids=["euclidean", "cosine"])
def test_narrow_columns_2048(eng, monkeypatch, metric, t):
    """FP16 and BF16 request columns at D = 2048 on the dense path (the sample kernel is templated on the element
    type) give exactly what the widened f32 column gives."""
    from test_gpu_feature_types import _opts as ft_opts, _frames, _pair, _counters

    _dense(monkeypatch)
    frames = _frames(4, 96, 2048, 5, seed=0xD2048 + metric)
    a, _ = _pair(eng, ft_opts(3, metric, F32MAX if metric == 0 else -1.0, 2048), frames, t, history=False)
    assert _counters(a)[4] > 0


# --------------------------------------------------------------------------------------------------- realistic run
@pytest.mark.gpu
def test_batch_visual_sort_2048(eng, oracle, monkeypatch):
    """BatchVisualSort, 3 scenes x 120 objects with D = 2048 ReID-like features (unit centroids plus noise), the
    reference's default metric Euclidean(f32::MAX), 5 observations per track, 6 frames: every frame the oracle's."""
    from similari_b200.workload import CONFIGS, Workload

    from test_gpu_tracker import both

    _dense(monkeypatch)
    cfg = dataclasses.replace(CONFIGS["cfg5"], n_scenes=3, n_objects=120, feature_dim=2048, canvas=(1920.0, 1080.0),
                              seed=0x5EED2048)
    wl = Workload(cfg)
    g, o = both(eng, oracle, kind=3, positional_kind=1, iou_threshold=0.3, max_idle_epochs=5, visual_kind=0,
                visual_threshold=F32MAX, feature_dim=2048, visual_max_observations=5, visual_min_votes=2,
                visual_minimal_track_length=1, min_confidence=0.1)
    t_oracle = 0.0
    for fr in range(6):
        f = wl.next_frame()
        args = (f["scene_ids"], f["det_offsets"], f["boxes"])
        rg = g.predict_batch(*args, features=f["features"])
        t0 = time.perf_counter()
        ro = o.predict_batch(*args, features=f["features"])
        t_oracle += time.perf_counter() - t0
        for key in ("ids", "epochs", "lengths", "voting_types"):
            assert np.array_equal(rg[key], ro[key]), (fr, key)
    assert g.active_tracks() == o.active_tracks()
    wc = g.work_counters()
    assert wc["tc_frames"] >= 4 and wc["dense_fallback_scenes"] == 0
    print(f"oracle CPU time, 6 frames: {t_oracle:.2f} s on {os.cpu_count()} threads")


# ------------------------------------------------------------------------------------------------- maximal distance
# Small scenes: at most 32 candidates and 32 feature rows, so vis_dense_sample_kernel samples every candidate
# floor(i m / 32) and every row floor(i rows / 32) -- the scene's maximal pair among them.
MAXD_CASES = [(d, vis, generic) for d in (2048, 4096) for vis in (0, 1) for generic in (False, True)]
N_FILL = 4


def _dist(oracle, vis):
    return (lambda x, y: float(oracle.euclidean(x, y))) if vis == 0 else (lambda x, y: 1.0 - float(oracle.cosine(x, y)))


def maxdist_features(oracle, d, vis, seed):
    """Features of one scene.  The maximal pair is (q, t) = (a, -b) with a ~ b from screen_pair: every component sits
    just below a BF16 rounding midpoint, so |dot~| is ~2^-7 low and the approximate maximal distance is pulled down by
    almost all the BF16 bound allows.  A runner-up candidate r lies 0.3 % below the maximum (in x = d^2 or in 1 - cos).
    Candidate c is nearer to track B (2 observations) than to track A (3 observations), yet A's group outweighs B's by
    g = (maxd - d(r, t)) / 3: an exact max_dist gives c track A, a max_dist that missed (q, t) and fell to the runner-up
    gives it B.  Fillers are unit vectors in general position.  Returns a dict of named f32 features."""
    a, b = screen_pair(seed, d, 1.0, "cos+")
    s = float(np.linalg.norm(a.astype(np.float64)))
    rng = np.random.default_rng(seed + 1)
    ah = a.astype(np.float64) / s
    e = np.linalg.qr(rng.standard_normal((d, 4)))[0].T
    e0 = e[0] - (e[0] @ ah) * ah
    e0 /= np.linalg.norm(e0)
    cphi = 1.0 - 0.006
    r = s * (cphi * ah + np.sqrt(1.0 - cphi * cphi) * e0)
    dist = _dist(oracle, vis)
    t = (-b).astype(np.float32)
    unit_of = (lambda x: x / s) if vis == 0 else (lambda x: x)          # cosine distances are scale-free
    maxd, d2 = unit_of(dist(a, t)), unit_of(dist(r.astype(np.float32), t))
    g = (maxd - d2) / 3.0
    cos_of = (lambda dd: 1.0 - dd * dd / 2.0) if vis == 0 else (lambda dd: 1.0 - dd)
    d_b = 0.1
    d_a = maxd - (2.0 * (maxd - d_b) + g) / 3.0                         # 3 (maxd - d_a) = 2 (maxd - d_b) + g
    fb = e[1]
    c = cos_of(d_b) * e[1] + np.sqrt(1.0 - cos_of(d_b) ** 2) * e[2]
    fa = cos_of(d_a) * c + np.sqrt(1.0 - cos_of(d_a) ** 2) * e[3]
    fill = [unit(rng, d) for _ in range(N_FILL)]
    out = dict(q=a, t=t, r=r, c=s * c, A=s * fa, B=s * fb)
    out.update({f"f{i}": s * f for i, f in enumerate(fill)})
    return {k: np.asarray(v, np.float32) for k, v in out.items()}


def maxdist_frames(f):
    """Frames 0-2: tracks A (frames 0-2: 3 observations), t (0-2), B (1-2: 2 observations) and the fillers; frame 3:
    c, q and r far from every box, the fillers where they were."""
    order = ["A", "t", "B"] + [f"f{i}" for i in range(N_FILL)]
    grid = _grid_boxes(len(order))
    frames = []
    for fr in range(3):
        keep = [i for i, k in enumerate(order) if not (k == "B" and fr == 0)]
        frames.append((grid[keep], np.stack([f[order[i]] for i in keep])))
    last = ["c", "q", "r"]
    boxes = np.concatenate([np.stack([_far_box(j) for j in range(3)]), grid[3:]])
    frames.append((boxes, np.stack([f[k] for k in last] + [f[k] for k in order[3:]])))
    return frames


def _maxd_seed(d, vis):
    return 4000 + d + vis


@pytest.mark.parametrize("vis", [0, 1])
@pytest.mark.parametrize("d", [2048, 4096])
def test_maxdist_construction(oracle, d, vis):
    """(q, t) is the scene's unique maximum, its BF16 estimate is low by at least 1.9 * 2^-8 of |q||t|, the runner-up
    sits within the keep window the bound allows below it, and BestFit gives c track A under the exact max_dist but
    track B under the runner-up's."""
    f = maxdist_features(oracle, d, vis, _maxd_seed(d, vis))
    dist = _dist(oracle, vis)
    frames = maxdist_frames(f)
    tracks = {"A": [f["A"]] * 3, "t": [f["t"]] * 3, "B": [f["B"]] * 2}
    tracks.update({f"f{i}": [f[f"f{i}"]] * 3 for i in range(N_FILL)})
    cands = frames[3][1]
    elems = {(i, k): [dist(x, o) for o in obs] for i, x in enumerate(cands) for k, obs in tracks.items()}
    maxd = max(max(v) for v in elems.values())
    assert max(elems[(1, "t")]) == maxd                                  # q (row 1) against t
    others = sorted({v for key, vs in elems.items() if key != (1, "t") for v in vs}, reverse=True)
    d2 = others[0]
    assert elems[(2, "t")][0] == d2                                      # the runner-up is (r, t)
    ratio = (d2 / maxd) ** 2 if vis == 0 else d2 / maxd
    assert 0.996 < ratio < 0.998
    q64, t64 = f["q"].astype(np.float64), f["t"].astype(np.float64)
    low = (bf16(f["q"]).astype(np.float64) @ bf16(f["t"]).astype(np.float64)) - q64 @ t64
    assert low >= 1.9 * 2.0 ** -8 * np.linalg.norm(q64) * np.linalg.norm(t64)
    assert low <= (2.0 ** -7 + 2.0 ** -16) * np.linalg.norm(q64) * np.linalg.norm(t64)

    def choice(md):   # c (row 0): the track of its best group W = sum (md - d)
        w = {k: sum(md - v for v in elems[(0, k)]) for k in tracks}
        return max(w, key=w.get), w

    best, w = choice(maxd)
    assert best == "A" and w["A"] - w["B"] > 0.2 * (maxd - d2)
    assert choice(d2)[0] == "B"


@pytest.mark.gpu
@pytest.mark.parametrize("d,vis,generic", MAXD_CASES)
def test_maximal_distance_at_the_sample(eng, oracle, d, vis, generic, monkeypatch):
    """Two scenes of maxdist_features on the dense path, every frame the oracle's and no scene-frame handed to the
    exact kernels.  A sampled lower bound above the true maximal distance would either drop (q, t) from the
    max-candidate list -- max_dist falls to the runner-up and c takes track B instead of A -- or leave the list
    empty and send the scene to the exact kernels; both fail here."""
    _dense(monkeypatch, generic)
    per_scene = [maxdist_frames(maxdist_features(oracle, d, vis, _maxd_seed(d, vis) + 10 * s)) for s in range(2)]
    frames = [_frame([sc[fr] for sc in per_scene]) for fr in range(4)]
    g = _drive(eng, oracle, _opts(vis, d, 3, visual_min_votes=1), frames)
    wc = g.work_counters()
    assert wc["tc_frames"] >= 3 and wc["dense_fallback_scenes"] == 0


# ------------------------------------------------------------------------------------- the constructions at these widths
@pytest.mark.parametrize("vis", [0, 1])
@pytest.mark.parametrize("d", [1024, 2000, 2048, 4096])
def test_row_tie_construction_wide(oracle, d, vis):
    """The row tie of test_row_tie_wide holds at its widths and seeds: exactly t1 beats t2, BF16 orders them the other
    way, and the selection's interval reaches t1."""
    q, t1, t2 = row_tie_features(ROW_TIE_SEEDS[vis] + d, d)
    dist = _dist(oracle, vis)
    d1, d2 = dist(q, t1), dist(q, t2)
    assert 0.0 < d2 - d1 < 1e-3
    a1, w1 = dense_row_interval(q, t1, vis, d)
    a2, w2 = dense_row_interval(q, t2, vis, d)
    assert a1 > a2
    assert a1 - a2 < w1 + w2 - 1e-4
    assert d2 - d1 < 0.1 * (w1 + w2)


@pytest.mark.parametrize("vis", [0, 1])
def test_column_tie_construction_wide(oracle, vis):
    """The column near-tie in the clean scenes of test_column_tie_2048 and test_column_tie_k25_1024."""
    for kobs in (3, 6):
        for sc in _tie_scenes(2048, 70, kobs, 300 + kobs, [(None, None)] * 5):
            _check_column_tie(oracle, sc, kobs, vis)
    for sc in _tie_scenes(1024, 40, 25, 500 + vis, [(None, None)] * 3):
        _check_column_tie(oracle, sc, 25, vis)
