"""GPU parity tests: the CUDA kernels (called through the C ABI) against the CPU oracle on the same seeded inputs.

Bit-exact for integer / index work (assignments, ids, epochs, lengths, voting types) and for every f32 value that
does not pass through sin/cos; oriented-box IoU (f64 sin/cos of device libm vs glibc) within 1e-6, far inside
north_star's 1e-5."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

NAN = float("nan")


@pytest.fixture(scope="module")
def eng():
    import similari_b200.engine as e
    from similari_b200._lib import lib

    if lib().sb200_device_count() <= 0:
        pytest.fail("no CUDA device: the gpu-marked tests must run on an H100")
    return e


def pack30(st110):
    st110 = np.asarray(st110, np.float32).reshape(-1, 110)
    out = np.zeros((len(st110), 30), np.float32)
    out[:, :10] = st110[:, :10]
    cov = st110[:, 10:].reshape(-1, 10, 10)
    for i in range(5):
        out[:, 10 + 4 * i] = cov[:, i, i]
        out[:, 11 + 4 * i] = cov[:, i, i + 5]
        out[:, 12 + 4 * i] = cov[:, i + 5, i]
        out[:, 13 + 4 * i] = cov[:, i + 5, i + 5]
    return out


def rand_boxes(rng, n, oriented, canvas=(600.0, 400.0)):
    b = np.empty((n, 6), np.float32)
    b[:, 0] = rng.uniform(0, canvas[0], n)
    b[:, 1] = rng.uniform(0, canvas[1], n)
    b[:, 2] = rng.uniform(-1.5, 1.5, n) if oriented else np.nan
    b[:, 3] = rng.uniform(0.3, 0.8, n)
    b[:, 4] = rng.uniform(40, 160, n)
    b[:, 5] = rng.uniform(0.02, 1.0, n)
    return b


def same_nan_pattern(a, b):
    return np.array_equal(np.isnan(a), np.isnan(b))


def assert_bits_equal(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    assert a.shape == b.shape
    assert np.array_equal(a.view(np.uint32) | (np.isnan(a) * np.uint32(0x7fffffff)),
                          b.view(np.uint32) | (np.isnan(b) * np.uint32(0x7fffffff)))


# --------------------------------------------------------------------------------------------- Kalman operators
@pytest.mark.parametrize("oriented", [False, True])
def test_kalman_ops_bit_exact(eng, oracle, oriented):
    rng = np.random.default_rng(5)
    boxes = rand_boxes(rng, 300, oriented)
    ref = np.stack([oracle.kalman_initiate(b) for b in boxes])
    got = eng.kalman_initiate(boxes)
    assert_bits_equal(pack30(ref), got)
    for step in range(4):
        ref = np.stack([oracle.kalman_predict(s) for s in ref])
        got = eng.kalman_predict(got)
        assert_bits_equal(pack30(ref), got)
        z = boxes.copy()
        z[:, :2] += rng.normal(0, 2, (300, 2)).astype(np.float32)
        ref = np.stack([oracle.kalman_update(s, b) for s, b in zip(ref, z)])
        got = eng.kalman_update(got, z)
        assert_bits_equal(pack30(ref), got)
        boxes = z


# --------------------------------------------------------------------------------------------- positional cost
def track_states(oracle, rng, boxes, steps=3):
    st = np.stack([oracle.kalman_initiate(b) for b in boxes])
    cur = boxes.copy()
    for _ in range(steps):
        st = np.stack([oracle.kalman_predict(s) for s in st])
        cur[:, :2] += rng.normal(0, 2, (len(cur), 2)).astype(np.float32)
        st = np.stack([oracle.kalman_update(s, b) for s, b in zip(st, cur)])
    post = np.stack([oracle.kalman_state_box(s) for s in st])
    post[:, 5] = cur[:, 5]
    return st, post


@pytest.mark.parametrize("oriented", [False, True])
@pytest.mark.parametrize("m,n", [(1, 1), (37, 129), (200, 333)])
def test_maha_cost_matrix_bit_exact(eng, oracle, oriented, m, n):
    rng = np.random.default_rng(100 + m + n)
    tb = rand_boxes(rng, n, oriented)
    st, post = track_states(oracle, rng, tb)
    cb = post[rng.integers(0, n, m)].copy()
    cb[:, :2] += rng.normal(0, 3, (m, 2)).astype(np.float32)
    cb[:, 5] = rng.uniform(0.01, 1.0, m)
    ref = oracle.sort_cost_matrix(oracle.POS_MAHA, cb, post, st)
    got = eng.sort_cost_matrix(eng._lib.POS_MAHA, cb, post, pack30(st))
    assert_bits_equal(ref, got)
    assert np.isfinite(got).sum() > 0


@pytest.mark.parametrize("m,n", [(1, 1), (33, 130), (150, 260)])
def test_iou_cost_matrix_axis_aligned_bit_exact(eng, oracle, m, n):
    rng = np.random.default_rng(200 + m)
    tb = rand_boxes(rng, n, False)
    cb = tb[rng.integers(0, n, m)].copy()
    cb[:, :2] += rng.normal(0, 8, (m, 2)).astype(np.float32)
    cb[:, 3:5] *= rng.uniform(0.9, 1.1, (m, 2)).astype(np.float32)
    ref = oracle.sort_cost_matrix(oracle.POS_IOU, cb, tb, iou_threshold=0.3)
    got = eng.sort_cost_matrix(eng._lib.POS_IOU, cb, tb, iou_threshold=0.3)
    assert_bits_equal(ref, got)
    assert np.isfinite(got).sum() >= m // 2


def test_iou_cost_matrix_oriented_within_tolerance(eng, oracle):
    rng = np.random.default_rng(7)
    n, m = 300, 200
    tb = rand_boxes(rng, n, True)
    cb = tb[rng.integers(0, n, m)].copy()
    cb[:, :2] += rng.normal(0, 8, (m, 2)).astype(np.float32)
    cb[:, 2] += rng.normal(0, 0.1, m).astype(np.float32)
    ref = oracle.sort_cost_matrix(oracle.POS_IOU, cb, tb, iou_threshold=0.05)
    got = eng.sort_cost_matrix(eng._lib.POS_IOU, cb, tb, iou_threshold=0.05)
    # None pattern may only differ where the value sits on the threshold
    mism = np.isnan(ref) != np.isnan(got)
    vals = np.where(np.isnan(ref), got, ref)
    assert np.all(np.abs(vals[mism] - 0.05) < 1e-6)
    both = ~np.isnan(ref) & ~np.isnan(got)
    assert both.sum() > 100
    assert np.max(np.abs(ref[both] - got[both])) <= 1e-6


def test_iou_github84_boxes_no_nan(eng, oracle):
    # python/bugfixes/github-84.py regression: near-identical oriented boxes must not crash / produce NaN IoU
    x = np.array([[8044.315, 8011.0454, 2.6787748, 1.00801, 49.8073, 1.0]], np.float32)
    y = np.array([[8044.455, 8011.338, 2.6787748, 1.0083783, 49.79979, 1.0]], np.float32)
    ref = oracle.sort_cost_matrix(oracle.POS_IOU, x, y, iou_threshold=0.3)
    got = eng.sort_cost_matrix(eng._lib.POS_IOU, x, y, iou_threshold=0.3)
    assert np.isfinite(got[0, 0]) and abs(ref[0, 0] - got[0, 0]) <= 1e-6


# --------------------------------------------------------------------------------------------- visual cost
@pytest.mark.parametrize("kind", ["euclid", "cosine"])
@pytest.mark.parametrize("m,n,d", [(1, 1, 8), (70, 130, 512), (65, 64, 13), (5, 200, 2048)])
def test_visual_cost_matrix_bit_exact(eng, oracle, kind, m, n, d):
    rng = np.random.default_rng(300 + d)
    cent = rng.standard_normal((n, d)).astype(np.float32)
    cent /= np.linalg.norm(cent, axis=1, keepdims=True)
    tf = cent
    cf = cent[rng.integers(0, n, m)] + 0.02 * rng.standard_normal((m, d)).astype(np.float32)
    cf = (cf / np.linalg.norm(cf, axis=1, keepdims=True)).astype(np.float32)
    if kind == "euclid":
        ref = oracle.visual_cost_matrix(oracle.VIS_EUCLIDEAN, 1.2, cf, tf)
        got = eng.visual_cost_matrix(eng._lib.VIS_EUCLIDEAN, 1.2, cf, tf)
    else:
        ref = oracle.visual_cost_matrix(oracle.VIS_COSINE, 0.1, cf, tf)
        got = eng.visual_cost_matrix(eng._lib.VIS_COSINE, 0.1, cf, tf)
    assert_bits_equal(ref, got)
    assert np.isfinite(got).sum() >= m


# --------------------------------------------------------------------------------------------- voting
def ents_from_matrix(cost, cand_base=1000, trk_base=1):
    m, n = cost.shape
    return [(cand_base + i, trk_base + j, float(cost[i, j]), None) for i in range(m) for j in range(n)
            if not np.isnan(cost[i, j])]


def oracle_sort_winners(oracle, thr, cost):
    m, n = cost.shape
    w = oracle.sort_voting(thr, m, n, ents_from_matrix(cost))
    out = np.full(m, -1, np.int32)
    for i in range(m):
        t = w.get(1000 + i)
        if t is not None and t[0] != 1000 + i:
            out[i] = t[0] - 1
    return out


@pytest.mark.parametrize("seed", range(6))
def test_sort_voting_matches_kuhn_munkres(eng, oracle, seed):
    rng = np.random.default_rng(seed)
    m, n = int(rng.integers(1, 90)), int(rng.integers(1, 90))
    cost = rng.uniform(0.0, 1.0, (m, n)).astype(np.float32)
    cost[rng.random((m, n)) < 0.6] = np.nan
    if seed % 2 == 0:  # heavy ties: quantised weights
        cost = np.round(cost * 4) / 4
    got = eng.sort_voting(0.3, cost)
    ref = oracle_sort_winners(oracle, 0.3, cost)
    assert np.array_equal(ref, got)


def test_sort_voting_edge_cases(eng, oracle):
    # no tracks, empty rows, all None
    assert list(eng.sort_voting(0.3, np.zeros((3, 0), np.float32))) == [-1, -1, -1]
    allnan = np.full((4, 5), np.nan, np.float32)
    assert list(eng.sort_voting(0.3, allnan)) == [-1] * 4
    # the reference's own test matrix (sort/voting.rs:110-174)
    c = np.array([[0.6, 0.4, 0.4], [0.5, 0.69, 0.4], [0.2, 0.27, 0.28]], np.float32)
    assert list(eng.sort_voting(0.3, c)) == [0, 1, -1]
    # diagonal-dominant 512 x 512 (typical tracking frame)
    rng = np.random.default_rng(1)
    big = np.full((512, 512), np.nan, np.float32)
    perm = rng.permutation(512)
    for i in range(512):
        big[i, perm[i]] = rng.uniform(0.5, 1.0)
        for j in rng.integers(0, 512, 4):
            if np.isnan(big[i, j]):
                big[i, j] = rng.uniform(0.3, 0.6)
    got = eng.sort_voting(0.3, big)
    ref = oracle_sort_winners(oracle, 0.3, big)
    assert np.array_equal(ref, got)


@pytest.mark.parametrize("seed", range(5))
def test_visual_voting_matches_oracle(eng, oracle, seed):
    rng = np.random.default_rng(50 + seed)
    m, n, k = int(rng.integers(1, 60)), int(rng.integers(1, 60)), 3
    pos = rng.uniform(0.3, 1.0, (m, n)).astype(np.float32)
    pos[rng.random((m, n)) < 0.7] = np.nan
    vis = rng.uniform(0.0, 0.7, (m, n, k)).astype(np.float32)
    vis[rng.random((m, n, k)) < 0.75] = np.nan
    if seed % 2 == 0:
        vis = (np.round(vis * 8) / 8).astype(np.float32)  # ties in the f64 weights
    ents = []
    for i in range(m):
        for j in range(n):
            for kk in range(k):
                a = pos[i, j] if kk == 0 else np.nan
                f = vis[i, j, kk]
                if not (np.isnan(a) and np.isnan(f)):
                    ents.append((1000 + i, 1 + j, None if np.isnan(a) else float(a), None if np.isnan(f) else float(f)))
    ref = oracle.visual_voting(0.3, np.finfo(np.float32).max, 2, ents)
    w, vt = eng.visual_voting(0.3, 2, pos, vis)
    for i in range(m):
        r = ref.get(1000 + i)
        if r is None or r[0][0] == 1000 + i:
            assert w[i] == -1, (i, r, w[i])
            if r is not None:
                assert vt[i] == r[0][1]
        else:
            assert (w[i], vt[i]) == (r[0][0] - 1, r[0][1]), (i, r, w[i], vt[i])


# --------------------------------------------------------------------------------------------- NMS
@pytest.mark.parametrize("oriented", [False, True])
def test_nms_matches_oracle(eng, oracle, oriented):
    rng = np.random.default_rng(9)
    base = rand_boxes(rng, 120, oriented)
    boxes = np.repeat(base, 4, axis=0)
    boxes[:, :2] += rng.normal(0, 3, (len(boxes), 2)).astype(np.float32)
    if oriented:
        boxes[:, 2] += rng.normal(0, 0.03, len(boxes)).astype(np.float32)
    scores = rng.uniform(0, 1, len(boxes)).astype(np.float32)
    for sc, st in [(scores, None), (scores, 0.2), (None, None)]:
        ref = oracle.nms(boxes, sc, 0.6, st)
        got = eng.nms_indices(boxes, sc, 0.6, st)
        assert list(ref) == list(got)
    assert len(eng.nms_indices(np.zeros((0, 6), np.float32), None, 0.5)) == 0


# --------------------------------------------------------------------------------------------- tensor-core visual cost
def _tc_inputs(m, n, d, seed):
    rng = np.random.default_rng(seed)
    cent = rng.standard_normal((n, d)).astype(np.float32)
    cent /= np.linalg.norm(cent, axis=1, keepdims=True)
    tf = cent.copy()
    src = rng.integers(1, n, m) if n > 1 else np.zeros(m, dtype=np.int64)  # row 0 of the tracks is special below
    cf = cent[src] + (0.3 / np.sqrt(d)) * rng.standard_normal((m, d)).astype(np.float32)
    cf = (cf / np.linalg.norm(cf, axis=1, keepdims=True)).astype(np.float32)
    cf[0] = tf[src[0]]                       # exact duplicate: euclidean 0, cosine 1
    cf[1] = tf[src[1]] * np.float32(1.0001)  # near duplicate
    if m > 2:
        cf[2] = 0.0
        cf[2, 0] = 1.0                       # one-hot: a single product carries the whole dot
        tf[0] = 0.0
        tf[0, 0] = 0.95
    return cf, tf


@pytest.mark.parametrize("kind", ["euclid", "cosine"])
@pytest.mark.parametrize("m,n,d", [(64, 64, 64), (129, 257, 72), (300, 700, 512), (130, 1000, 2048), (500, 1536, 512)])
def test_visual_cost_matrix_tensor_core_bit_exact(eng, oracle, kind, m, n, d, monkeypatch):
    """Tensor-core BF16 screen + exact f32 refinement: every emitted value is bit-identical to the oracle and no pair
    that passes the threshold is lost by the screen."""
    monkeypatch.setenv("SB200_VIS_KERNEL", "tc")
    cf, tf = _tc_inputs(m, n, d, 400 + d + m)
    if kind == "euclid":
        ref = oracle.visual_cost_matrix(oracle.VIS_EUCLIDEAN, 0.7, cf, tf)
        got = eng.visual_cost_matrix(eng._lib.VIS_EUCLIDEAN, 0.7, cf, tf)
    else:
        ref = oracle.visual_cost_matrix(oracle.VIS_COSINE, 0.3, cf, tf)
        got = eng.visual_cost_matrix(eng._lib.VIS_COSINE, 0.3, cf, tf)
    assert_bits_equal(ref, got)
    assert np.isfinite(got).sum() >= m - 1


def test_visual_cost_matrix_tensor_core_unnormalised_and_overflow(eng, oracle, monkeypatch):
    """Unnormalised features (the error bound scales with the norms) and the survivor-list overflow fallback."""
    rng = np.random.default_rng(78)
    m, n, d = 200, 300, 256
    tf = (rng.standard_normal((n, d)) * 7.0).astype(np.float32)
    cf = tf[rng.integers(0, n, m)] + rng.standard_normal((m, d)).astype(np.float32)
    monkeypatch.setenv("SB200_VIS_KERNEL", "tc")
    for thr in (20.0, 200.0):   # 200: every pair passes -> dense result
        ref = oracle.visual_cost_matrix(oracle.VIS_EUCLIDEAN, thr, cf, tf)
        got = eng.visual_cost_matrix(eng._lib.VIS_EUCLIDEAN, thr, cf, tf)
        assert_bits_equal(ref, got)
    monkeypatch.setenv("SB200_VIS_PAIR_CAP", "16")   # force the overflow -> device-side dense fallback
    ref = oracle.visual_cost_matrix(oracle.VIS_EUCLIDEAN, 20.0, cf, tf)
    got = eng.visual_cost_matrix(eng._lib.VIS_EUCLIDEAN, 20.0, cf, tf)
    assert_bits_equal(ref, got)
