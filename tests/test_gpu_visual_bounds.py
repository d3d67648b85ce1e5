"""The tensor-core visual kernels at the edges of their error bounds, and on degenerate features.

The BF16 screen (kernels_feat_tc.cu) drops a pair only when the BF16 dot product is below the threshold by more than the
slack E = screen_rel_err(D) of sb_engine.cuh; the dense selection (kernels_feat_dense.cu) refines only the groups whose
weight interval reaches a row or column bound.  If a bound were too tight, a kernel would silently drop what the reference
keeps.  The tests here build inputs on the host whose BF16 rounding error is one-sided and close to the worst case the
bound assumes, put the reference value exactly on the threshold, and compare every value or assignment with the CPU
oracle.  The CPU tests check the constructions themselves, so the file documents how adversarial its inputs are.

Degenerate features (an all-zero vector, a NaN or +inf component, components whose squares overflow) reach the reference
as they are: its distances are NaN or infinite there, `is_ok` turns them into None (src/trackers/visual_sort/metric.rs
visual_metric, src/distance.rs), and nothing sorts or unwraps them.  None of these inputs makes the reference panic.
"""
import os

import numpy as np
import pytest

F32MAX = float(np.finfo(np.float32).max)
U8 = 2.0 ** -8


# ----------------------------------------------------------------------------------------------- host-side constructions
def bf16(x):
    """Round-to-nearest-even f32 -> BF16, returned as f32 (what launch_to_bf16 / cand_norm_kernel store)."""
    u = np.ascontiguousarray(x, np.float32).view(np.uint32).astype(np.uint64)
    u = (u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000
    return u.astype(np.uint32).view(np.float32)


def midpoint_vector(rng, d, above, exps, signs):
    """Components sgn * 2^e * (1 + 2^-8 -/+ k 2^-23): just below (above) a BF16 rounding midpoint, so every component
    rounds down (up) by almost 2^-8 relative."""
    k = rng.integers(1, 9, d).astype(np.float64)
    mant = 1.0 + U8 + (k if above else -k) * 2.0 ** -23
    return (signs * mant * np.exp2(exps)).astype(np.float32)


def screen_pair(seed, d, norm, kind):
    """(a, b) with a ~ b ('euclid', 'cos+': both below the midpoints, dot~ ~ dot (1 - 2^-7)) or a ~ -b ('cos-': both above
    the midpoints, |dot~| ~ |dot| (1 + 2^-7), dot~ below dot).  `norm` is reached by a power of two, which keeps every
    mantissa."""
    rng = np.random.default_rng(seed)
    exps = rng.integers(-3, 4, d).astype(np.float64)
    signs = rng.choice([-1.0, 1.0], d)
    above = kind == "cos-"
    a = midpoint_vector(rng, d, above, exps, signs)
    b = midpoint_vector(rng, d, above, exps, signs)
    s = np.exp2(np.round(np.log2(norm / np.linalg.norm(a.astype(np.float64)))))
    a, b = (a * s).astype(np.float32), (b * s).astype(np.float32)
    return (a, -b) if kind == "cos-" else (a, b)


def screen_rel_err(d):
    """The slack of sb_engine.cuh."""
    e = 2.0 ** -7 + 2.0 ** -16 + d * 2.0 ** -23
    fl = float(np.float32(2.1) / np.float32(256.0))
    return fl if e <= fl else e * (1 + 2.0 ** -20)


def operand_error(a, b):
    """(dot - dot_bf16) / (||a|| ||b||) in f64: how much of the operand part of the bound the pair uses."""
    a64, b64 = a.astype(np.float64), b.astype(np.float64)
    dot = a64 @ b64
    dot_bf = bf16(a).astype(np.float64) @ bf16(b).astype(np.float64)
    return (dot - dot_bf) / (np.linalg.norm(a64) * np.linalg.norm(b64))


SCREEN_D = [64, 200, 512, 640, 2048]
WIDE_D = [4096, 8192]
NORMS = [2.0 ** -10, 1.0, 2.0 ** 10]
KINDS = ["euclid", "cos+", "cos-"]


def screen_seed(d):
    return 2000 + d


TRACKER_PAIRS = [(77, "euclid"), (78, "cos+")]   # (seed, kind) of the tracker test, D = 512, per metric


@pytest.mark.parametrize("seed,d,norm,kind",
                         [(screen_seed(d), d, norm, kind) for d in SCREEN_D for norm in NORMS for kind in KINDS] +
                         [(screen_seed(d), d, 1.0, kind) for d in WIDE_D for kind in KINDS] +
                         [(seed, 512, 1.0, kind) for seed, kind in TRACKER_PAIRS])
def test_screen_construction_reaches_the_operand_bound(seed, d, norm, kind):
    """Every pair the screen tests use spends at least 1.95 * 2^-8 of ||a|| ||b|| on BF16 operand rounding, in the
    direction that lowers dot~ -- within 0.15 * 2^-8 of the slack the screen allows -- and stays inside the bound."""
    a, b = screen_pair(seed, d, norm, kind)
    assert np.all(np.isfinite(a)) and np.all(np.isfinite(b))
    assert np.all(np.sign(a) == (-np.sign(b) if kind == "cos-" else np.sign(b)))
    err = operand_error(a, b)
    assert 1.95 * U8 <= err <= 2.0 ** -7 + 2.0 ** -16
    assert err < screen_rel_err(d)
    assert 0.5 * norm <= np.linalg.norm(a.astype(np.float64)) <= 2.0 * norm


# rows of a 300-candidate operator call: both halves of each 128-row CTA tile, the cluster's second CTA, the last ragged row
A_ROWS = [0, 63, 64, 127, 128, 191, 255, 256, 299]
# columns of a 600-track call: both ends of the 128-column tiles, and the last column
B_COLS = [0, 127, 128, 255, 256, 511, 599]


def screen_matrix(seed, d, norm, kind):
    """300 x 600 features: the pair (a, b) at every (A_ROWS, B_COLS) crossing, random fillers of the same norm elsewhere."""
    rng = np.random.default_rng(seed)
    a, b = screen_pair(seed, d, norm, kind)
    cand = rng.standard_normal((300, d)).astype(np.float32)
    trk = rng.standard_normal((600, d)).astype(np.float32)
    cand *= np.float32(norm) / np.linalg.norm(cand, axis=1, keepdims=True)
    trk *= np.float32(norm) / np.linalg.norm(trk, axis=1, keepdims=True)
    cand[A_ROWS] = a
    trk[B_COLS] = b
    return cand.astype(np.float32), trk.astype(np.float32), a, b


# ---------------------------------------------------------------------------------------------------------- GPU tests
@pytest.fixture(scope="module")
def eng():
    import similari_b200.engine as e
    from similari_b200._lib import lib

    if lib().sb200_device_count() <= 0:
        pytest.fail("no CUDA device: the gpu-marked tests must run on an H100")
    return e


def _screen_at_threshold(eng, oracle, d, norm, kind, monkeypatch):
    from test_gpu_parity import assert_bits_equal

    monkeypatch.setenv("SB200_VIS_KERNEL", "tc")
    cand, trk, a, b = screen_matrix(screen_seed(d), d, norm, kind)
    if kind == "euclid":
        vk_o, vk_g = oracle.VIS_EUCLIDEAN, eng._lib.VIS_EUCLIDEAN
        thr = np.float32(oracle.euclidean(a, b))
        cut = np.nextafter(thr, np.float32(0))
    else:
        vk_o, vk_g = oracle.VIS_COSINE, eng._lib.VIS_COSINE
        thr = np.float32(oracle.cosine(a, b))
        cut = np.nextafter(thr, np.float32(2))
        if kind == "cos-":   # every filler pair passes a threshold near -1: the list must hold all pairs
            monkeypatch.setenv("SB200_VIS_PAIR_CAP", str(cand.shape[0] * trk.shape[0]))
    for t, kept in ((thr, True), (cut, False)):
        ref = oracle.visual_cost_matrix(vk_o, float(t), cand, trk, threads=os.cpu_count() or 1)
        got = eng.visual_cost_matrix(vk_g, float(t), cand, trk)
        pairs = ref[np.ix_(A_ROWS, B_COLS)]
        assert np.isfinite(pairs).all() if kept else np.isnan(pairs).all()   # the oracle's decision has zero margin
        assert_bits_equal(ref, got)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("d", SCREEN_D)
@pytest.mark.parametrize("norm", NORMS)
def test_screen_keeps_pairs_on_the_threshold(eng, oracle, d, norm, kind, monkeypatch):
    """The operator's BF16 screen on pairs at the worst-case BF16 error, with the threshold exactly at the oracle's value
    (kept) and one ulp past it (dropped), at the tile edges of both screen kernels (D <= 512 A-stationary, 640 and 2048
    streaming, 200 a TMA tail)."""
    _screen_at_threshold(eng, oracle, d, norm, kind, monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("d", WIDE_D)
def test_screen_keeps_pairs_on_the_threshold_wide(eng, oracle, d, kind, monkeypatch):
    """The same at D = 4096 and 8192, where the slack grows with the fp32 accumulation term."""
    _screen_at_threshold(eng, oracle, d, 1.0, kind, monkeypatch)


def _frame(scenes):
    """scenes: list of (boxes [n, 6], features [n, d]) -> flat request."""
    offs = np.concatenate([[0], np.cumsum([len(b) for b, _ in scenes])]).astype(np.int32)
    return (np.arange(len(scenes), dtype=np.uint64), offs, np.concatenate([b for b, _ in scenes]).astype(np.float32),
            np.concatenate([f for _, f in scenes]).astype(np.float32))


def _grid_boxes(n, x0=100.0):
    i = np.arange(n)
    b = np.zeros((n, 6), np.float32)
    b[:, 0] = x0 + 150.0 * (i % 12)
    b[:, 1] = 100.0 + 150.0 * (i // 12)
    b[:, 2] = np.nan
    b[:, 3] = 0.5
    b[:, 4] = 60.0
    b[:, 5] = 0.9
    return b


def _far_box(j):
    """A box that overlaps nothing of the grid (the positional stage cannot match it)."""
    b = _grid_boxes(1)[0].copy()
    b[0], b[1] = 5000.0 + 200.0 * j, 5000.0
    return b


def _drive(eng, oracle, kw, frames):
    from test_gpu_tracker import both

    g, o = both(eng, oracle, **kw)
    for fr, (sid, offs, boxes, feats) in enumerate(frames):
        rg = g.predict_batch(sid, offs, boxes, features=feats)
        ro = o.predict_batch(sid, offs, boxes, features=feats)
        for key in ("ids", "epochs", "lengths", "voting_types"):
            assert np.array_equal(rg[key], ro[key]), (fr, key, np.flatnonzero(rg[key] != ro[key])[:8])
    assert g.active_tracks() == o.active_tracks()
    return g


VIS_KW = dict(positional_kind=1, iou_threshold=0.3, max_idle_epochs=5, visual_minimal_track_length=1, min_confidence=0.1)


@pytest.mark.gpu
@pytest.mark.parametrize("vis", [0, 1])
def test_tracker_screen_keeps_pairs_on_the_threshold(eng, oracle, vis, monkeypatch):
    """The tracker's BF16 rows come from cand_norm_kernel and feat_store, not from the operator's conversion.  Each of four
    scenes holds a track whose three observations are b and, one frame later, a detection a far from it: the threshold is
    the oracle's value for (a, b), so only a visual match keeps the track's id.  The tracker screens D = 512 on e4m3 by
    default; tc16 keeps every frame on the BF16 screen this pair is built for (test_gpu_screen_fp8_bounds.py covers the
    e4m3 rows)."""
    monkeypatch.setenv("SB200_VIS_KERNEL", "tc16")
    d, n = 512, 130
    seed, kind = TRACKER_PAIRS[vis]
    a, b = screen_pair(seed, d, 1.0, kind)
    thr = float(oracle.euclidean(a, b)) if vis == 0 else float(oracle.cosine(a, b))
    assert vis == 0 or -1.0 <= thr <= 1.0   # VisualSortMetricType::cosine accepts [-1, 1]
    rng = np.random.default_rng(5)
    slots = [0, 63, 64, 129]                        # the adversarial detection's row inside its scene
    fill = [rng.standard_normal((n, d)).astype(np.float32) for _ in slots]
    for f in fill:
        f /= np.linalg.norm(f, axis=1, keepdims=True)
    frames = []
    for fr in range(4):
        scenes = []
        for s, slot in enumerate(slots):
            boxes, feats = _grid_boxes(n), fill[s].copy()
            feats[slot] = b
            if fr == 3:                             # a, far from b's track
                boxes[slot] = _far_box(s)
                feats[slot] = a
            scenes.append((boxes, feats))
        frames.append(_frame(scenes))
    g = _drive(eng, oracle, dict(kind=3, visual_kind=vis, visual_threshold=thr, feature_dim=d, visual_max_observations=3,
                                 visual_min_votes=1, **VIS_KW), frames)
    assert g.work_counters()["tc_frames"] >= 3
    sc = g.screen_counters()
    assert sc["bf16_frames"] >= 3 and sc["fp8_frames"] == 0, sc


# ------------------------------------------------------------------------------------ degenerate features, dense selection
def unit(rng, d):
    v = rng.standard_normal(d)
    return v / np.linalg.norm(v)


def column_tie_features(rng, d):
    """Features of track t, track t', and candidates q1, q2 (BestFit, best.rs): q2 is nearer to t than q1 is, but nearer
    still to t'.  The reference gives t' to q2 and nothing to q1 -- (q2, t) is t's column maximum though it is not q2's
    row maximum -- so a selection that only emits row maxima gives t to q1."""
    u, v, w = np.linalg.qr(rng.standard_normal((d, 3)))[0].T   # orthonormal
    q2 = 0.68 * u + 0.73 * v
    q1 = 0.55 * u + 0.835 * w
    return [x.astype(np.float32) for x in (u, v, q2 / np.linalg.norm(q2), q1 / np.linalg.norm(q1))]


def degenerate_feature(kind, d, rng):
    f = unit(rng, d).astype(np.float32)
    if kind == "zero":
        f[:] = 0.0
    elif kind == "nan":
        f[d // 3] = np.nan
    elif kind == "inf":
        f[d // 2] = np.inf
    elif kind == "huge":   # ||a||^2 overflows f32; a - a' stays finite
        f[:2] = np.float32(1.5e19)
    return f


def tie_scene_frames(rng, d, n, kobs, scale=1.0, degenerate=None, placement=None, identical=False):
    """One scene over kobs + 1 frames.  Frames 0..kobs-1: n static, well-separated objects (objects 0 and 1 are the tracks
    t and t'), each frame's feature its own plus a little noise.  Last frame: t and t' are gone, q2 sits on t', q1 far
    from everything (only a visual match could give it an id).  `degenerate` puts a degenerate feature on an extra
    detection in the last frame ('cand') or on an extra object present from frame 0 on ('track').  `identical`: every
    other object carries the same feature (a scene full of tied maxima)."""
    t, tp, q2, q1 = column_tie_features(rng, d)
    base = [unit(rng, d).astype(np.float32) for _ in range(n)]
    if identical:
        base[2:] = [base[2]] * (n - 2)
    base[0], base[1] = t, tp
    deg = degenerate_feature(degenerate, d, rng) if degenerate else None
    out = []
    for fr in range(kobs + 1):
        feats = np.stack(base) + (0.0 if identical else 0.01) * rng.standard_normal((n, d))
        feats[:2] = (t, tp)
        boxes = _grid_boxes(n)
        if fr == kobs:
            feats[0], feats[1] = q1, q2
            boxes[0] = _far_box(0)
        feats = (feats * scale).astype(np.float32)
        if deg is not None and (placement == "track" or fr == kobs):
            boxes = np.concatenate([boxes, _far_box(1)[None]])
            feats = np.concatenate([feats, deg[None]])
        out.append((boxes, feats))
    return out


def _tie_scenes(d, n, kobs, seed, specs, scale=1.0, identical=()):
    rng = np.random.default_rng(seed)
    return [tie_scene_frames(rng, d, n, kobs, scale=scale, degenerate=k, placement=pl, identical=s in identical)
            for s, (k, pl) in enumerate(specs)]


def _check_column_tie(oracle, scene, kobs, vis):
    """q1 (row 0 of the last frame) has row maximum t (track 0), q2 (row 1) has row maximum t' (track 1), and q2's
    group for t outweighs q1's, in the oracle's distances against every track's stored observations."""
    last = scene[kobs][1]
    q1, q2 = last[0], last[1]
    n = scene[0][1].shape[0]
    dist = (lambda x, y: float(oracle.euclidean(x, y))) if vis == 0 else (lambda x, y: 1.0 - float(oracle.cosine(x, y)))
    def group(q, j):   # the track's observations: its features over frames 0..kobs-1
        return sum(dist(q, scene[fr][1][j]) for fr in range(kobs))
    s1 = [group(q1, j) for j in range(n)]
    s2 = [group(q2, j) for j in range(n)]
    assert int(np.argmin(s1)) == 0 and int(np.argmin(s2)) == 1
    assert s2[0] + 0.05 * kobs < s1[0]
    # the gap is far wider than the selection's per-observation bound, so only the column criterion emits (q2, t)
    e = screen_rel_err(d=last.shape[1]) + 2e-4
    assert (s2[0] - s2[1]) / kobs > 4 * (e if vis else 0.536 * e * 2.0 / (s2[1] / kobs))


DEGENERATE = ["zero", "nan", "inf", "huge"]
DEGENERATE_SPECS = [(None, None)] + [(k, "cand") for k in DEGENERATE] + [(None, None)] + [(k, "track") for k in DEGENERATE]
DEGENERATE_KOBS = [3, 6]   # fused epilogue, and the any-K one with its selection pass A
COLUMN_TIE_CASES = [(vis, kobs, generic, scale) for vis in (0, 1)
                    for kobs, generic in [(3, False), (5, False), (6, True), (8, True), (3, True)]
                    for scale in ((1.0, 3.0e4, 1.0e-6) if vis == 0 else (1.0,))]


@pytest.mark.parametrize("vis", [0, 1])
def test_column_tie_construction(oracle, vis):
    """The column near-tie in every scene the GPU tests build (the degenerate scenes' clean part included)."""
    for kobs in DEGENERATE_KOBS:
        for sc in _tie_scenes(128, 60, kobs, 11 + vis + 10 * kobs, DEGENERATE_SPECS):
            _check_column_tie(oracle, [(b[:60], f[:60]) for b, f in sc], kobs, vis)
    for v, kobs, generic, scale in COLUMN_TIE_CASES:
        if v == vis and scale == 1.0:
            for sc in _tie_scenes(128, 70, kobs, 100 + kobs, [(None, None)] * 5):
                _check_column_tie(oracle, sc, kobs, vis)


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["simt", "tc", "dense"])
@pytest.mark.parametrize("vis", [0, 1])
@pytest.mark.parametrize("kobs", DEGENERATE_KOBS)
def test_degenerate_features_match_oracle(eng, oracle, path, vis, kobs, monkeypatch):
    """A batch of ten scenes: two clean ones, and each degenerate feature once on a candidate and once on a stored track,
    every scene with the column near-tie of tie_scene_frames.  Every frame must be the oracle's.  On the dense path, only
    the scene-frames that hold a degenerate feature may fall back to the exact kernels.  K = 6 runs the any-K epilogue
    and the selection's pass A."""
    monkeypatch.setenv("SB200_VIS_KERNEL", path)
    d, n = 128, 60
    specs = DEGENERATE_SPECS
    per_scene = _tie_scenes(d, n, kobs, 11 + vis + 10 * kobs, specs)
    frames = [_frame([sc[fr] for sc in per_scene]) for fr in range(kobs + 1)]
    if path == "dense":
        thr = F32MAX if vis == 0 else -1.0
    else:
        thr = 1.2 if vis == 0 else 0.1
    g = _drive(eng, oracle, dict(kind=3, visual_kind=vis, visual_threshold=thr, feature_dim=d, visual_max_observations=kobs,
                                 visual_min_votes=2, **VIS_KW), frames)
    if path == "dense":
        degenerate_scene_frames = sum(1 if pl == "cand" else kobs for k, pl in specs if k)
        wc = g.work_counters()
        assert wc["tc_frames"] >= kobs and wc["dense_fallback_scenes"] <= degenerate_scene_frames


@pytest.mark.gpu
@pytest.mark.parametrize("vis,kobs,generic,scale", COLUMN_TIE_CASES)
def test_dense_selection_column_tie_matches_oracle(eng, oracle, vis, kobs, generic, scale, monkeypatch):
    """The column near-tie on the dense path (Euclidean(f32::MAX), cosine(-1)) with both epilogues (fused K <= 5, any-K),
    in six scenes, one of them full of identical features (tied maxima: the path holds, or the max-candidate list
    overflows to the exact kernels).  Euclidean features scaled by 3e4 make the fp16 weight sums overflow 65504, by 1e-6
    make them fp16-subnormal; at both scales the selection rules no group out (the overflow rule, the absolute terms of
    the bound) and the pair lists overflow to the exact kernels, so only the assignments are checked there."""
    monkeypatch.setenv("SB200_VIS_KERNEL", "dense")
    if generic:
        monkeypatch.setenv("SB200_DENSE_GENERIC", "1")
    d, n = 128, 70
    per_scene = _tie_scenes(d, n, kobs, 100 + kobs, [(None, None)] * 6, scale=scale, identical=(5,))
    frames = [_frame([sc[fr] for sc in per_scene]) for fr in range(kobs + 1)]
    g = _drive(eng, oracle, dict(kind=3, visual_kind=vis, visual_threshold=F32MAX if vis == 0 else -1.0, feature_dim=d,
                                 visual_max_observations=kobs, visual_min_votes=2, **VIS_KW), frames)
    wc = g.work_counters()
    assert wc["tc_frames"] >= kobs
    if scale == 1.0:   # only the tied scene may fall back
        assert wc["dense_fallback_scenes"] <= kobs


# ------------------------------------------------------------------------------------ dense selection at its row bound
def row_tie_features(seed, d):
    """q = (x, y) with x's components just below BF16 midpoints and y's just above; t1 = (x, 0), t2 = (0, y).  Exactly,
    |x| > |y| by a hair, so t1 is q's best track under both metrics (d(q, t1) = |y|, cos(q, t1) = |x| / |q|).  In BF16,
    dot(q, t1) rounds down and dot(q, t2) rounds up by almost 2^-7 relative each, so the approximate distances order the
    two tracks the other way: the selection must keep t1 on its error interval alone."""
    rng = np.random.default_rng(seed)
    h = d // 2
    for _ in range(100000):   # seeded search for |x| / |y| - 1 in (1e-4, 4e-4)
        x = midpoint_vector(rng, h, False, rng.integers(-3, 4, h).astype(np.float64), rng.choice([-1.0, 1.0], h))
        y = midpoint_vector(rng, h, True, rng.integers(-3, 4, h).astype(np.float64), rng.choice([-1.0, 1.0], h))
        nx, ny = np.linalg.norm(x.astype(np.float64)), np.linalg.norm(y.astype(np.float64))
        if 1e-4 < nx / ny - 1.0 < 4e-4:
            break
    else:
        raise AssertionError("no row tie found")
    s = np.float32(np.exp2(-np.round(np.log2(nx))))
    x, y = x * s, y * s
    z = np.zeros(h, np.float32)
    return np.concatenate([x, y]), np.concatenate([x, z]), np.concatenate([z, y])


def dense_row_interval(q, t, vis, d, halved=False):
    """(approximate per-observation distance, selection half-width per observation) of the dense path for the pair,
    from the BF16 operands and f32 norms as vis_wsum_kernel / vis_dense_select_kernel form them (one observation)."""
    e_rel = screen_rel_err(d) + 2e-4
    dot = bf16(q).astype(np.float64) @ bf16(t).astype(np.float64)
    na, nb = float(np.float32(q @ q)), float(np.float32(t @ t))
    if vis == 1:
        dt, dl = 1.0 - dot / np.sqrt(na * nb), e_rel
    else:
        dt = np.sqrt(max(na + nb - 2.0 * dot, 1e-30))
        e = e_rel * (na + nb)
        qq = e / dt
        dl = (0.536 * qq if dt * dt >= 4.0 * e else min(qq, np.sqrt(e))) * 1.0001 + 1e-6 * (na + nb + 1.0)
    if halved:
        dl *= 0.5
    return dt, dl + dt * 4.9e-4 + float(np.spacing(np.float16(dt)))   # fp16 storage of the sum and of the bound


ROW_TIE_SEEDS = {0: 41, 1: 42}


@pytest.mark.parametrize("vis", [0, 1])
def test_row_tie_construction(oracle, vis):
    """Exactly t1 beats t2; the BF16 approximations order them the other way; the selection's interval still reaches t1
    (it must refine it), and for cosine, an interval half as wide would not: |W1 - W2| is far below the interval width."""
    d = 128
    q, t1, t2 = row_tie_features(ROW_TIE_SEEDS[vis], d)
    dist = (lambda x, y: float(oracle.euclidean(x, y))) if vis == 0 else (lambda x, y: 1.0 - float(oracle.cosine(x, y)))
    d1, d2 = dist(q, t1), dist(q, t2)
    assert 0.0 < d2 - d1 < 1e-3                                     # W1 - W2 = k (d2 - d1) > 0: the reference picks t1
    a1, w1 = dense_row_interval(q, t1, vis, d)
    a2, w2 = dense_row_interval(q, t2, vis, d)
    assert a1 > a2                                                  # BF16 orders the two tracks the other way
    assert a1 - a2 < w1 + w2 - 1e-4                                 # the interval reaches t1: it is refined
    h1, h2 = dense_row_interval(q, t1, vis, d, True)[1], dense_row_interval(q, t2, vis, d, True)[1]
    if vis == 1:
        assert a1 - a2 > h1 + h2 + 1e-4                             # a half-width bound would drop t1
    assert d2 - d1 < 0.1 * (w1 + w2)


@pytest.mark.gpu
@pytest.mark.parametrize("vis", [0, 1])
@pytest.mark.parametrize("kobs,generic", [(3, False), (6, True)])
def test_dense_selection_row_tie_matches_oracle(eng, oracle, vis, kobs, generic, monkeypatch):
    """The row near-tie of row_tie_features on the dense path.  Tracks t1 and t2 hold kobs identical observations; in
    the last frame q arrives far from both, and a candidate equal to t1 takes t1's place, so t1's column maximum is not
    q.  The reference gives q nothing visual (its best group, t1, is taken); a selection that dropped (q, t1) would give
    q the track t2."""
    monkeypatch.setenv("SB200_VIS_KERNEL", "dense")
    if generic:
        monkeypatch.setenv("SB200_DENSE_GENERIC", "1")
    d, n = 128, 40
    q, t1, t2 = row_tie_features(ROW_TIE_SEEDS[vis], d)
    rng = np.random.default_rng(7)
    base = np.stack([unit(rng, d) for _ in range(n)]).astype(np.float32) * np.float32(np.linalg.norm(q))
    base[0], base[1] = t1, t2
    frames = []
    for fr in range(kobs + 1):
        scenes = []
        for s in range(3):
            boxes, feats = _grid_boxes(n), base.copy()
            if fr == kobs:
                feats[1] = q            # q replaces t2's detection, far from both tracks
                boxes[1] = _far_box(0)
            scenes.append((boxes, feats))
        frames.append(_frame(scenes))
    g = _drive(eng, oracle, dict(kind=3, visual_kind=vis, visual_threshold=F32MAX if vis == 0 else -1.0, feature_dim=d,
                                 visual_max_observations=kobs, visual_min_votes=2, **VIS_KW), frames)
    wc = g.work_counters()
    assert wc["tc_frames"] >= kobs and wc["dense_fallback_scenes"] == 0
