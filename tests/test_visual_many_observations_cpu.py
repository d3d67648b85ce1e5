"""CPU checks for trackers that keep 9 to 32 observations per track.

1. The oracle's observation pruning (VisualMetric::optimize with is_merge, visual_sort/metric.rs:297-374, and
   optimize_observations, :129-154) at K = 9, 16, 25 and 32, against the rule written out in test_oracle_observations_cpu:
   quality ties, detections without a feature, merges below, on and one ulp under the collect threshold, and lists that
   fill up to K and drop their lowest-quality entry.
2. The dense selection's weight interval (kernels_feat_dense.cu, vis_dense_select_kernel; DESIGN section 4b) evaluated in
   f32 exactly as the kernel evaluates it, on worst-case inputs at K = 32: sums that lose close to half an ulp per f32
   addition, groups whose observations all sit at the scene's maximal distance, approximate distances at either end of
   their error bound, fp16 sums near overflow and in the fp16 subnormal range.  Every interval must contain the
   reference's f64 weight sum_k (max_dist - d_k)."""
import numpy as np
import pytest

from test_oracle_observations_cpu import D, D8, Q_COLLECT, _merge, _norm2

F32, F16 = np.float32, np.float16


# ------------------------------------------------------------------------------------------------ oracle pruning
def _script(K, seed):
    """(quality, has_feature) of the new track and 2 K + 10 merges: a few qualities (ties are the rule), the collect
    threshold and the f32 value one ulp under it, one detection in seven without a feature."""
    rng = np.random.default_rng(seed)
    qs = np.array([0.2, 0.5, 0.5, 0.9, 0.7, Q_COLLECT, np.nextafter(F32(Q_COLLECT), F32(0)), 0.9, 1.0], F32)
    return [(F32(rng.choice(qs)), bool(rng.random() >= 1 / 7)) for _ in range(2 * K + 11)]


@pytest.mark.parametrize("K", [9, 16, 25, 32])
def test_oracle_pruning_follows_the_merge_rule(oracle, K):
    rng = np.random.default_rng(0x0B5E0 + K)
    o = oracle.Tracker(oracle.make_options(kind=oracle.KIND_VISUAL_SORT, positional_kind=oracle.POS_IOU,
                                           iou_threshold=0.3, max_idle_epochs=3, feature_dim=D,
                                           visual_max_observations=K, visual_minimal_track_length=1,
                                           visual_minimal_quality_collect=Q_COLLECT))
    box = oracle.box(100.0, 80.0, None, 0.5, 60.0, 0.9)
    want, tid, full = [], None, 0
    for i, (q, hf) in enumerate(_script(K, K)):
        feat = rng.standard_normal(D).astype(F32)
        r = o.predict_batch([0], [0, 1], box[None], features=feat[None], has_feature=[hf], quality=[q])
        if i == 0:
            tid = int(r["ids"][0])
            want = [(q, feat if hf else None)]
        else:
            assert int(r["ids"][0]) == tid, i
            kept = feat if (hf and q >= F32(Q_COLLECT)) else None
            want = _merge(want, (q, kept), K)
        full = max(full, len(want))
        got = o.scene_observations(0)
        assert got["n_obs"].tolist() == [len(want)], i
        assert got["feats"].shape == (1, K, D8)
        for k in range(K):
            if k < len(want):
                wq, wf = want[k]
                assert got["quality"][0, k].view(np.uint32) == F32(wq).view(np.uint32), (i, k)
                assert got["has_feat"][0, k] == (wf is not None), (i, k)
                row = np.zeros(D8, F32)
                if wf is not None:
                    row[:D] = wf
                assert np.array_equal(got["feats"][0, k], row), (i, k)
                assert got["norm2"][0, k].view(np.uint32) == (_norm2(row) if wf is not None else F32(0)).view(np.uint32)
            else:
                assert got["has_feat"][0, k] == 0 and got["quality"][0, k] == 0 and not got["feats"][0, k].any()
        assert int(o.scene_tracks(0)["feat_counts"][0]) == sum(f is not None for _, f in want), i
    assert full == K   # the list filled, so the drop of the lowest quality ran


# ------------------------------------------------------------------------------------------------ dense interval
K_HALF_REL = F32(4.9e-4)


def half_ru(x):
    """__float2half_ru: the fp16 value at or above x."""
    h = F16(x)
    if float(h) < float(x):
        h = np.nextafter(h, F16(np.inf))
    return h


def f32_sum(v):
    """The weight-sum epilogue's block sum: f32 additions in observation order, from 0."""
    s = F32(0)
    for x in v:
        s = F32(s + F32(x))
    return s


def interval(d_approx, delta, maxd):
    """[W_lo, W_hi] of one group as vis_dense_select_kernel forms it (any-K selection, pass A and pass B), from the
    approximate distances of its k observations, their per-observation bound and the scene's exact max_dist."""
    k = len(d_approx)
    s32 = f32_sum(d_approx)
    with np.errstate(over="ignore", invalid="ignore"):   # an fp16 sum past 65504 is inf, as on the device
        s16, del16 = F16(s32), half_ru(delta)            # the half2 {S~, delta} of the weight-sum matrix
        ex, ey = F32(s16), F32(del16)
        ey = F32(ey + F32(F32(ex * K_HALF_REL) / F32(k)))   # the fp16 rounding of the sum, per observation
        fk = F32(k)
        a = F32(fk * F32(maxd))
        wlo = F32(F32(F32(a * F32(F32(1) - F32(2e-6))) - F32(1e-7)) - F32(F32(ex * F32(F32(1) + F32(2e-6))) + F32(fk * ey)))
        whi = F32(F32(F32(a * F32(F32(1) + F32(2e-6))) + F32(1e-7)) - F32(F32(ex * F32(F32(1) - F32(2e-6))) - F32(fk * ey)))
    if not ex < F32(6.0e4):
        whi = F32(3.0e38)
    return float(wlo), float(whi)


def weight(d, maxd):
    """BestFit's weight as the voting kernels compute it (best.rs:97): f32 max_dist - d_k, summed in f64."""
    w = 0.0
    for x in d:
        w += float(F32(F32(maxd) - F32(x)))
    return w


def half_ulp_losers(k, s0):
    """s0, then k - 1 terms just under half an ulp of the running f32 sum: every addition rounds down by almost half an
    ulp, the largest relative loss a sequential f32 sum can take."""
    v, s = [F32(s0)], F32(s0)
    for _ in range(k - 1):
        h = F32(np.spacing(s) / 2)
        x = np.nextafter(h, F32(0))
        v.append(x)
        s = F32(s + x)
    return np.array(v, F32)


def half_ulp_gainers(k, s0):
    """The same upwards: terms just over half an ulp round the running sum up by almost half an ulp."""
    v, s = [F32(s0)], F32(s0)
    for _ in range(k - 1):
        x = np.nextafter(F32(np.spacing(s) / 2), F32(np.inf))
        v.append(x)
        s = F32(s + x)
    return np.array(v, F32)


def near_max(k, maxd, rng):
    """k approximate distances within a few ulps of max_dist: S ~ k max_dist, where the bound has the least slack."""
    steps = rng.integers(-6, 1, k)
    return np.array([F32(maxd) + F32(s) * F32(np.spacing(F32(maxd))) for s in steps], F32)


def _check(d_approx, delta, maxd, sign):
    """The reference's distances at one end of the epilogue's bound: d = d~ + sign * delta (clamped to [0, max_dist],
    which every real distance of the scene respects)."""
    d = np.clip(d_approx.astype(np.float64) + sign * float(delta), 0.0, float(maxd)).astype(F32)
    lo, hi = interval(d_approx, delta, maxd)
    w = weight(d, maxd)
    assert lo <= w <= hi, (lo, w, hi)
    return w - lo, hi - w


CASES_K = [32, 25, 9]


@pytest.mark.parametrize("k", CASES_K)
@pytest.mark.parametrize("scale", [1.0, 2.0 ** -20, 1.0e3])
def test_interval_holds_on_adversarial_sums(k, scale):
    rng = np.random.default_rng(k)
    for s0 in (1.0, 1.5, 1.9999999):
        for build in (half_ulp_losers, half_ulp_gainers):
            v = build(k, F32(s0 * scale))
            maxd = F32(v.max())
            # the sum's rounding error is a real share of the (k - 1) u bound the derivation allows
            exact = float(np.sum(v.astype(np.float64)))
            assert abs(float(f32_sum(v)) - exact) >= 0.45 * (k - 1) * 2.0 ** -24 * float(v[0]) - 1e-300
            for delta in (F32(0), F32(1e-3) * maxd):
                for sign in (-1.0, 1.0):
                    _check(v, delta, maxd, sign)
    for _ in range(50):
        maxd = F32(scale * rng.uniform(0.5, 2.0))
        v = near_max(k, maxd, rng)
        for delta in (F32(0), np.spacing(maxd), F32(1e-4) * maxd):
            for sign in (-1.0, 1.0):
                _check(v, delta, maxd, sign)


@pytest.mark.parametrize("k", CASES_K)
def test_interval_at_fp16_overflow_and_underflow(k):
    """Sums on either side of the fp16 overflow (65520 rounds to inf, 6e4 <= S~ <= 65504 stays finite) and sums in
    the fp16 subnormal range: the escape and the absolute 1e-7 keep the true weight inside."""
    rng = np.random.default_rng(100 + k)
    for total in (5.9e4, 6.0e4, 65504.0, 65519.0, 65520.0, 1.0e5, 1.0e-5, 3.0e-7, 6.0e-8):
        for _ in range(20):
            p = rng.dirichlet(np.ones(k))
            v = (p * total).astype(F32)
            maxd = F32(v.max() * F32(rng.uniform(1.0, 1.5)))
            for sign in (-1.0, 1.0):
                _check(v, F32(1e-6) * maxd, maxd, sign)


def test_derivation_constants_at_32():
    """The numbers of DESIGN section 4b: at K = 32 the epilogue's f32 sum may be off by gamma_31 = 31 u / (1 - 31 u)
    of S, more than the 2e-6 S the interval gives it alone, and the k max_dist slack covers the rest because no
    observation of the group lies above max_dist (S <= k max_dist)."""
    u = 2.0 ** -24
    gamma = 31 * u / (1 - 31 * u)
    select = 6 * u + 3.0e-8     # f32 roundings of the interval's own evaluation and of the (1 -+ 2e-6) constants
    ref = u                     # the reference's f32 subtraction max_dist - d_k
    assert gamma > 2e-6 - select
    # needed: (gamma + select) S + (select + ref) k maxd <= 2e-6 (k maxd + S) for every 0 <= S <= k maxd
    for s_over_kmax in np.linspace(0.0, 1.0, 101):
        assert (gamma + select) * s_over_kmax + (select + ref) <= 2e-6 * (1.0 + s_over_kmax)
    # the margin left at the worst point (S = k max_dist), as a share of the slack
    worst = 2e-6 * 2.0 - ((gamma + select) + (select + ref))
    assert worst > 0.3e-6
