"""The e4m3 tensor-core screen (SB200_VIS_KERNEL=tc8) against the CPU oracle.  The screen only filters: every value that
reaches the output is recomputed exactly, so the matrices must be bit-identical to the oracle's whatever the operand
precision -- as long as the screen never drops a pair the exact metric keeps.  The thresholds below sit exactly at oracle
values, so that pairs at the edge of the bound are kept by the oracle and must survive the screen."""
import numpy as np
import pytest

from test_gpu_parity import assert_bits_equal
from test_gpu_tracker import run_frames, small

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    import similari_b200.engine as e
    from similari_b200._lib import lib

    if lib().sb200_device_count() <= 0:
        pytest.fail("no CUDA device: the gpu-marked tests must run on an H100")
    return e


def _both(eng, oracle, kind, thr, cf, tf):
    if kind == "euclid":
        return (oracle.visual_cost_matrix(oracle.VIS_EUCLIDEAN, thr, cf, tf),
                eng.visual_cost_matrix(eng._lib.VIS_EUCLIDEAN, thr, cf, tf))
    return (oracle.visual_cost_matrix(oracle.VIS_COSINE, thr, cf, tf),
            eng.visual_cost_matrix(eng._lib.VIS_COSINE, thr, cf, tf))


def _edge_threshold(oracle, kind, cf, tf, q):
    """an oracle distance (Euclidean) / cosine at quantile q: the pair that has it is kept exactly at the threshold"""
    if kind == "euclid":
        d = oracle.visual_cost_matrix(oracle.VIS_EUCLIDEAN, 3.0e38, cf, tf)
        return float(np.quantile(d[np.isfinite(d)], q, method="nearest"))
    w = oracle.visual_cost_matrix(oracle.VIS_COSINE, -2.0, cf, tf)   # 1 - cos
    c = (1.0 - w[np.isfinite(w)].astype(np.float64)).astype(np.float32)
    return float(np.quantile(c, 1.0 - q, method="nearest"))


@pytest.mark.parametrize("kind", ["euclid", "cosine"])
@pytest.mark.parametrize("m,n,d", [(300, 600, 512), (130, 260, 64), (257, 300, 200), (40, 1100, 136)])
@pytest.mark.parametrize("scale_exp", [-10, 0, 10])
def test_fp8_screen_at_oracle_threshold(eng, oracle, kind, m, n, d, scale_exp, monkeypatch):
    monkeypatch.setenv("SB200_VIS_KERNEL", "tc8")
    rng = np.random.default_rng(900 + d + scale_exp)
    cent = rng.standard_normal((n, d)).astype(np.float32)
    cent /= np.linalg.norm(cent, axis=1, keepdims=True)
    cf = cent[rng.integers(0, n, m)] + 0.05 * rng.standard_normal((m, d)).astype(np.float32)
    # rows of very different norms on both sides (2^-10 .. 2^10 around the case's scale)
    cf *= np.exp2(scale_exp + rng.integers(-3, 4, (m, 1))).astype(np.float32)
    tf = (cent * np.exp2(scale_exp + rng.integers(-3, 4, (n, 1)))).astype(np.float32)
    cf = cf.astype(np.float32)
    for q in (0.002, 0.02):
        thr = _edge_threshold(oracle, kind, cf, tf, q)
        ref, got = _both(eng, oracle, kind, thr, cf, tf)
        assert_bits_equal(got, ref)
        # one ulp past the edge: the edge pair is cut by the exact test, nothing else changes
        thr2 = float(np.nextafter(np.float32(thr), np.float32(-1.0 if kind == "euclid" else 2.0)))
        ref, got = _both(eng, oracle, kind, thr2, cf, tf)
        assert_bits_equal(got, ref)


@pytest.mark.parametrize("kind", ["euclid", "cosine"])
def test_fp8_screen_rounding_one_sided(eng, oracle, kind, monkeypatch):
    """Components that all round the same way in e4m3 (9/16 of a binade step above a representable value), and rows with
    components near the subnormal floor of the scaled copy: the operand error is as large and as one-sided as it gets."""
    monkeypatch.setenv("SB200_VIS_KERNEL", "tc8")
    rng = np.random.default_rng(17)
    m, n, d = 256, 384, 512
    mag = np.exp2(rng.integers(-3, 3, (1, d))).astype(np.float32) * np.float32(1.0 + 9.0 / 256.0)
    sgn = np.where(rng.random((n, d)) < 0.5, -1.0, 1.0).astype(np.float32)
    tf = (sgn * mag).astype(np.float32)
    tf[: n // 4, d // 2:] *= np.float32(2.0 ** -14)   # half of the row near e4m3's subnormal floor after scaling
    cf = tf[rng.integers(0, n, m)].copy()
    flip = rng.random((m, d)) < 0.1
    cf[flip] = -cf[flip]
    for q in (0.01, 0.1):
        thr = _edge_threshold(oracle, kind, cf, tf, q)
        ref, got = _both(eng, oracle, kind, thr, cf, tf)
        assert_bits_equal(got, ref)


def test_fp8_screen_accumulation_probe(eng, oracle, monkeypatch):
    """Large products that cancel, then small terms: what a short accumulator loses, the bound must cover."""
    monkeypatch.setenv("SB200_VIS_KERNEL", "tc8")
    rng = np.random.default_rng(5)
    m, n, d = 256, 256, 512
    big = np.float32(400.0)
    cf = np.zeros((m, d), np.float32)
    tf = np.zeros((n, d), np.float32)
    cf[:, :32] = big
    tf[:, :16] = big
    tf[:, 16:32] = -big                                  # the first k32 step sums to exactly zero
    cf[:, 32:] = rng.uniform(0.5, 1.0, (m, d - 32)).astype(np.float32)
    tf[:, 32:] = rng.uniform(0.5, 1.0, (n, d - 32)).astype(np.float32)
    for kind in ("euclid", "cosine"):
        for q in (0.05, 0.5):
            thr = _edge_threshold(oracle, kind, cf, tf, q)
            ref, got = _both(eng, oracle, kind, thr, cf, tf)
            assert_bits_equal(got, ref)


@pytest.mark.parametrize("kind", ["euclid", "cosine"])
def test_fp8_screen_degenerate_features(eng, oracle, kind, monkeypatch):
    monkeypatch.setenv("SB200_VIS_KERNEL", "tc8")
    rng = np.random.default_rng(23)
    m, n, d = 260, 300, 128
    tf = rng.standard_normal((n, d)).astype(np.float32)
    cf = tf[rng.integers(0, n, m)] + 0.1 * rng.standard_normal((m, d)).astype(np.float32)
    for side in (cf, tf):
        side[0] = 0.0
        side[1, 3] = np.nan
        side[2, 5] = np.inf
        side[3, 7] = -np.inf
        side[4] *= np.float32(1e18)       # squared norm overflows
        side[5] *= np.float32(1e-30)      # squared norm underflows
        side[6, :] = np.float32(3e-39)    # subnormal components
    thr = 1.5 if kind == "euclid" else 0.0
    ref, got = _both(eng, oracle, kind, thr, cf, tf)
    assert_bits_equal(got, ref)


@pytest.mark.parametrize("vis", [0, 1])
@pytest.mark.parametrize("mode", ["tc8", "tc16"])
def test_screen_precisions_match_oracle_in_tracker(eng, oracle, vis, mode, monkeypatch):
    monkeypatch.setenv("SB200_VIS_KERNEL", mode)
    cfg = small("cfg5", n_scenes=4, n_objects=300, oriented=False, canvas=(1400.0, 900.0), feature_dim=256)
    run_frames(eng, oracle, cfg, 6,
               dict(kind=3, positional_kind=0, iou_threshold=0.3, max_idle_epochs=3, visual_kind=vis, feature_dim=256,
                    visual_threshold=0.7 if vis == 0 else 0.2, visual_minimal_track_length=1, visual_max_observations=3, visual_min_votes=2),
               check_costs=False)


def test_screen_precision_switch(eng, oracle, monkeypatch):
    """Cosine 0.2 (the threshold in the bulk of the distribution) leaves the e4m3 screen after its first frame; a
    Euclidean 0.7 on clustered features stays on it.  Both match the oracle."""
    from similari_b200.workload import Workload

    monkeypatch.delenv("SB200_VIS_KERNEL", raising=False)
    for vis, thr, expect_fp8 in ((1, 0.2, False), (0, 0.7, True)):
        cfg = small("cfg5", n_scenes=8, n_objects=400, oriented=False, canvas=(1400.0, 900.0), feature_dim=512)
        kw = dict(kind=3, positional_kind=0, iou_threshold=0.3, max_idle_epochs=3, visual_kind=vis, visual_threshold=thr,
                  visual_minimal_track_length=1, feature_dim=512,
                  visual_max_observations=3, visual_min_votes=2)
        from test_gpu_tracker import both

        g, o = both(eng, oracle, **kw)
        wl = Workload(cfg)
        for _ in range(6):
            f = wl.next_frame()
            rg = g.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=f["features"])
            ro = o.predict_batch(f["scene_ids"], f["det_offsets"], f["boxes"], features=f["features"])
            assert np.array_equal(np.asarray(rg["ids"]), np.asarray(ro["ids"]))
        sc = g.screen_counters()   # the first frame has no tracks to screen
        assert sc["fp8_frames"] + sc["bf16_frames"] >= 4, sc
        if expect_fp8:
            assert sc["bf16_frames"] == 0, sc
        else:
            assert sc["fp8_frames"] == 1, sc
