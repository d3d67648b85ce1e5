"""The positional cost kernels (csrc/kernels_cost.cu) against the CPU oracle at their branch boundaries.

pos_scan_kernel (culled: scenes of up to 4096 tracks, sorted by x in shared memory, gated pairs queued 4096 per
512-candidate chunk, a full scan when a track or candidate x or radius is not finite) and pos_cost_kernel (dense tiled:
more than 4096 tracks), through sb200_sort_cost_matrix: Mahalanobis and axis-aligned IoU bit-exact, oriented IoU within
1e-6 (the None pattern may differ only on the threshold).  Then the trackers on frames with a NaN-centre detection, and
a visual tracker across the 96-open-candidate switch of the lazy scan.  Every input is built from a seed."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

NAN, INF = float("nan"), float("inf")


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


def assert_bits_equal(a, b, msg=""):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    assert a.shape == b.shape
    # None is a NaN of any sign or payload (the host and the device produce different ones from NaN inputs)
    ua = np.where(np.isnan(a), np.uint32(0x7fffffff), a.view(np.uint32))
    ub = np.where(np.isnan(b), np.uint32(0x7fffffff), b.view(np.uint32))
    bad = np.argwhere(ua != ub)
    assert len(bad) == 0, (msg, len(bad), [(tuple(i), a[tuple(i)], b[tuple(i)]) for i in bad[:5]])


def assert_oriented_close(ref, got, thr):
    mism = np.isnan(ref) != np.isnan(got)
    vals = np.where(np.isnan(ref), got, ref)
    assert np.all(np.abs(vals[mism] - thr) < 1e-6)
    both = ~np.isnan(ref) & ~np.isnan(got)
    r, g = ref[both], got[both]
    with np.errstate(invalid="ignore"):   # inf - inf where both are inf
        assert np.all((r == g) | (np.abs(r - g) <= 1e-6))


def states(oracle, boxes):
    """Track states: initiate + one predict (pw 1/20, vw 1/160)."""
    return np.stack([oracle.kalman_predict(oracle.kalman_initiate(b)) for b in boxes])


def cost(eng, oracle, pos, cb, tb, thr=0.3, min_conf=0.05, oriented=False, st=None):
    """Oracle and product matrices, compared; returns the oracle's."""
    cb, tb = np.ascontiguousarray(cb, np.float32), np.ascontiguousarray(tb, np.float32)
    if pos == 0:
        st = states(oracle, tb) if st is None else st
        ref = oracle.sort_cost_matrix(oracle.POS_MAHA, cb, tb, st, min_confidence=min_conf, threads=8)
        got = eng.sort_cost_matrix(eng._lib.POS_MAHA, cb, tb, pack30(st), min_confidence=min_conf)
    else:
        ref = oracle.sort_cost_matrix(oracle.POS_IOU, cb, tb, iou_threshold=thr, min_confidence=min_conf, threads=8)
        got = eng.sort_cost_matrix(eng._lib.POS_IOU, cb, tb, iou_threshold=thr, min_confidence=min_conf)
    if oriented and pos == 1:
        assert_oriented_close(ref, got, thr)
    else:
        assert_bits_equal(ref, got)
    return ref


def scene(rng, m, n, oriented=False):
    """n tracks on a canvas that keeps ~6 neighbours per track; m candidates near random tracks."""
    side = 60.0 * np.sqrt(max(n, 1))
    tb = np.empty((n, 6), np.float32)
    tb[:, 0] = rng.uniform(0, side, n)
    tb[:, 1] = rng.uniform(0, side, n)
    tb[:, 2] = rng.uniform(-1.5, 1.5, n) if oriented else NAN
    tb[:, 3] = rng.uniform(0.3, 0.8, n)
    tb[:, 4] = rng.uniform(40, 120, n)
    tb[:, 5] = 1.0
    cb = tb[rng.integers(0, n, m)].copy()
    cb[:, :2] += rng.normal(0, 5, (m, 2)).astype(np.float32)
    cb[:, 3:5] *= rng.uniform(0.9, 1.1, (m, 2)).astype(np.float32)
    if oriented:
        cb[:, 2] += rng.normal(0, 0.1, m).astype(np.float32)
    cb[:, 5] = rng.uniform(0.6, 1.0, m)
    return cb, tb


# ------------------------------------------------------------------------------------------------------- sizes
SMALL_N = [1, 2, 3, 63, 64, 65, 255, 256, 257]
SMALL_M = [1, 16, 17, 64, 65, 512, 513, 1024]


@pytest.mark.parametrize("pos", [0, 1])
@pytest.mark.parametrize("n", SMALL_N)
def test_culled_kernel_sizes(eng, oracle, pos, n):
    """N on both sides of the powers of two the sort pads to; M across TM, the nsplit steps and the 512-candidate chunk."""
    for m in SMALL_M:
        rng = np.random.default_rng(1000 * n + m + pos)
        cb, tb = scene(rng, m, n)
        ref = cost(eng, oracle, pos, cb, tb)
        assert np.isfinite(ref).sum() >= min(m, n) // 4


@pytest.mark.parametrize("pos", [0, 1])
@pytest.mark.parametrize("n", [4095, 4096, 4097, 5000])
def test_large_scenes_culled_and_dense_kernels(eng, oracle, pos, n):
    """4095 / 4096: the culled kernel at Np = 4096; 4097 / 5000: the dense tiled kernel."""
    kept = 0
    for m in [1, 16, 17]:
        rng = np.random.default_rng(7 * n + m + pos)
        cb, tb = scene(rng, m, n)
        kept += np.isfinite(cost(eng, oracle, pos, cb, tb)).sum()
    assert kept >= 8


def test_oriented_iou_sizes(eng, oracle):
    for m, n in [(17, 65), (513, 257), (16, 4096), (17, 4097)]:
        rng = np.random.default_rng(m + n)
        cb, tb = scene(rng, m, n, oriented=True)
        cost(eng, oracle, 1, cb, tb, thr=0.05, oriented=True)


# ------------------------------------------------------------------------------------------------------- queue
@pytest.mark.parametrize("pos", [0, 1])
@pytest.mark.parametrize("m", [64, 65])
def test_gated_pair_queue_boundary(eng, oracle, pos, m):
    """Every box on one spot: 64 x 64 = 4096 gated pairs fill the queue of one chunk exactly; 65 x 64 overflow it and
    the last pairs are evaluated in place."""
    rng = np.random.default_rng(m)
    tb = np.tile(np.array([[300.0, 200.0, NAN, 0.5, 80.0, 1.0]], np.float32), (64, 1))
    tb[:, :2] += rng.normal(0, 0.5, (64, 2)).astype(np.float32)
    cb = np.tile(np.array([[300.0, 200.0, NAN, 0.5, 80.0, 0.9]], np.float32), (m, 1))
    cb[:, :2] += rng.normal(0, 0.5, (m, 2)).astype(np.float32)
    ref = cost(eng, oracle, pos, cb, tb)
    assert np.isfinite(ref).all()


# ------------------------------------------------------------------------------------------------------- too_far
@pytest.mark.parametrize("origin", [0.0, 1e5, -1e5, 1e6, -1e6])
def test_too_far_boundary_and_window_padding(eng, oracle, origin):
    """Aspect 0.75, height 8: radius exactly 5.  Candidates at (dx, dy) = (+-6, +-8) of a track are exactly 2R away and
    kept (Mahalanobis is finite there); their f32 neighbours one ulp further out are too far, up to x = +-1e6."""
    ntr = 40
    tb = np.zeros((ntr, 6), np.float32)
    tb[:, 0] = np.float32(origin) + np.arange(ntr, dtype=np.float32) * np.float32(64.0)
    tb[:, 1] = np.float32(origin / 2) + (np.arange(ntr) % 3).astype(np.float32) * np.float32(128.0)
    tb[:, 2], tb[:, 3], tb[:, 4], tb[:, 5] = NAN, 0.75, 8.0, 1.0
    cands = []
    for t in tb:
        for sx, sy in [(1, 1), (-1, 1), (1, -1), (-1, -1)]:
            for dx, dy in [(6.0, 8.0), (8.0, 6.0), (10.0, 0.0), (0.0, 10.0)]:
                x = np.float32(t[0] + np.float32(sx * dx))
                y = np.float32(t[1] + np.float32(sy * dy))
                cands.append([x, y])
                cands.append([np.nextafter(x, np.float32(sx * INF)), y])
                cands.append([x, np.nextafter(y, np.float32(sy * INF))])
                cands.append([np.nextafter(x, np.float32(-sx * INF)), y])
    cands = np.array(cands, np.float32)
    cb = np.zeros((len(cands), 6), np.float32)
    cb[:, :2] = cands
    cb[:, 2], cb[:, 3], cb[:, 4], cb[:, 5] = NAN, 0.75, 8.0, 1.0
    st = np.stack([oracle.kalman_initiate(b) for b in tb])   # project = the track box itself
    ref = cost(eng, oracle, 0, cb, tb, st=st)
    assert np.isfinite(ref).sum() >= ntr * 16       # the exact-2R pairs are kept ...
    assert np.isnan(ref).sum() > ntr * 16           # ... and their outer neighbours are not


def f32_radius(a, h):
    f = np.float32
    hw, hh = f(f(a) * f(h)) / f(2), f(h) / f(2)
    return f(np.sqrt(f(f(hw * hw) + f(hh * hh))))


@pytest.mark.parametrize("seed", range(4))
def test_window_padding_keeps_every_pair_too_far_keeps(eng, oracle, seed):
    """Radii that are not exactly representable, and candidate / track centres on opposite sides of x = 0, where
    x_c - x_t rounds: too_far keeps pairs whose track lies just outside the unpadded window [x_c - R, x_c + R] in f32.
    The input is checked to hold such pairs, so the test fails if the window's 1e-5 padding is removed."""
    f = np.float32
    rng = np.random.default_rng(900 + seed)
    rows, needy = 40, 0
    for scene_no in range(6):
        a, h = f(rng.uniform(0.3, 1.0)), f(rng.uniform(3, 30))
        md = f(f32_radius(a, h) + f32_radius(a, h))
        tb, cb, need = [], [], []
        for k in range(rows):
            y = f(1024 * k)                     # rows far apart: only a row's own pairs pass too_far
            cx = f(rng.uniform(-1, 1) * md)
            side = f(1 if k % 2 else -1)
            t = f(cx + side * md)
            for _ in range(3):
                t = np.nextafter(t, f(-side * INF))
            for _ in range(7):                  # the f32 neighbours of the 2R point, inside to outside
                x = f(cx - t)
                kept = not (f(x * x) > f(md * md))
                if kept and not (f(cx - md) <= t <= f(cx + md)):
                    need.append((k, len(tb)))
                tb.append([t, y, NAN, a, h, 1.0])
                t = np.nextafter(t, f(side * INF))
            cb.append([cx, y, NAN, a, h, 1.0])
        tb, cb = np.array(tb, np.float32), np.array(cb, np.float32)
        st = np.stack([oracle.kalman_initiate(b) for b in tb])
        ref = cost(eng, oracle, 0, cb, tb, st=st)
        for k, j in need:
            assert np.isfinite(ref[k, j]), (k, j)   # the oracle keeps it, and the kernel matched the oracle above
        needy += len(need)
    assert needy >= 5


# ------------------------------------------------------------------------------------------------------- geometry
def geometry_boxes():
    b = []
    base = [100.0, 100.0, NAN, 0.5, 40.0, 1.0]
    b.append(base)                                          # identical
    b.append([110.0, 100.0, NAN, 0.5, 40.0, 1.0])           # overlap
    b.append([120.0, 100.0, NAN, 0.5, 40.0, 1.0])           # shares an edge (width 20)
    b.append([120.0, 140.0, NAN, 0.5, 40.0, 1.0])           # shares a corner
    b.append([100.0, 100.0, NAN, 0.5, 20.0, 1.0])           # nested
    b.append([100.0, 100.0, 0.0, 0.5, 40.0, 1.0])           # angle exactly 0 == None
    b.append([100.0, 100.0, np.pi / 2, 0.5, 40.0, 1.0])     # +-pi/2
    b.append([100.0, 100.0, -np.pi / 2, 0.5, 40.0, 1.0])
    b.append([100.0, 100.0, NAN, 0.5, 0.0, 1.0])            # zero height
    b.append([100.0, 100.0, NAN, 0.0, 40.0, 1.0])           # zero aspect
    b.append([100.0, 100.0, NAN, 0.5, 1e-40, 1.0])          # subnormal sizes
    b.append([100.0, 100.0, NAN, 1e-40, 40.0, 1.0])
    b.append([100.0, 100.0, NAN, 0.5, 1e20, 1.0])           # f32 area overflows
    b.append([100.0, 100.0, NAN, 3e38, 1e20, 1.0])          # f32 radius overflows
    return np.array(b, np.float32)


@pytest.mark.parametrize("pos", [0, 1])
def test_degenerate_geometry(eng, oracle, pos):
    """Every degenerate box against every other.  The last two boxes overflow the f32 radius: too_far cannot cull them,
    and their whitened Mahalanobis residual overflows, which the reference's forward substitution turns into None
    (NaN) when it is one of x, y, angle, aspect.  The extra candidates overflow only the height residual (cost 0) or
    only the aspect residual (None); as tracks their Kalman covariance would overflow too."""
    g = geometry_boxes()
    extra = np.array([[100.0, 100.0, NAN, 0.5, 3e38, 1.0], [100.0, 100.0, NAN, 3e38, 40.0, 1.0]], np.float32)
    c = np.concatenate([g, extra])
    axis = ~np.isin(np.arange(len(c)), [6, 7])
    # axis aligned pairs bit-exact, then every pair (+-pi/2 goes through sin / cos) within the oriented tolerance
    ref = cost(eng, oracle, pos, c[axis], g[axis[:len(g)]], thr=1e-5)
    cost(eng, oracle, pos, c, g, thr=1e-5, oriented=True)
    if pos == 0:
        assert np.isnan(ref[-1, :-1]).all() and np.isnan(ref[:-3, -1]).all()   # residual overflow -> None
        assert (ref[-2] == 0).sum() >= 8                                       # height-only overflow -> cost 0


# ------------------------------------------------------------------------------------------------------- thresholds
def test_iou_thresholds_and_confidence(eng, oracle):
    rng = np.random.default_rng(5)
    cb, tb = scene(rng, 200, 150)
    cb[0::7, 5] = 0.0
    cb[1::7, 5] = 0.01       # below min_confidence 0.05
    cb[2::7, 5] = NAN
    cb[3::7, 5] = 1.5
    ref0 = cost(eng, oracle, 1, cb, tb, thr=0.0)
    vals = ref0[np.isfinite(ref0) & (ref0 > 0.1)]
    assert len(vals) > 20
    for thr in [1e-5, 1e-4, 0.3, float(vals[len(vals) // 2]), float(vals.max())]:
        ref = cost(eng, oracle, 1, cb, tb, thr=thr)
        if thr == float(vals.max()):
            assert np.isfinite(ref).sum() >= 1       # a value equal to the threshold is kept
    cost(eng, oracle, 0, cb, tb)


def test_mahalanobis_gate_crossing(eng, oracle):
    """Bisect (on f32 values, with the oracle) to the candidate x where the distance crosses chi2(0.95, 4) = 11.07, then
    place candidates on the f32 neighbours of the crossing: cost 100 - d on one side, 0 on the other."""
    rng = np.random.default_rng(11)
    tb = np.array([[200.0 + 300.0 * i, 150.0, NAN, 0.5, 60.0 + 10 * i, 1.0] for i in range(6)], np.float32)
    st = states(oracle, tb)
    cands = []
    for i, t in enumerate(tb):
        dy = np.float32(rng.uniform(-3, 3))

        def d_at(x):
            return oracle.kalman_distance(st[i], np.array([x, t[1] + dy, NAN, t[3], t[4], 1.0], np.float32))
        lo, hi = np.float32(t[0]), np.float32(t[0] + t[4])
        assert d_at(lo) < 11.07 < d_at(hi)
        while np.nextafter(lo, hi) != hi:
            mid = np.float32((float(lo) + float(hi)) / 2)
            if mid in (lo, hi):
                break
            lo, hi = (mid, hi) if d_at(mid) <= np.float32(11.07) else (lo, mid)
        x = lo
        for _ in range(3):
            x = np.nextafter(x, np.float32(-INF))
        for _ in range(7):
            cands.append([x, t[1] + dy, NAN, t[3], t[4], 0.8])
            x = np.nextafter(x, np.float32(INF))
    cb = np.array(cands, np.float32)
    ref = cost(eng, oracle, 0, cb, tb, st=st)
    diag = np.array([ref[k, k // 7] for k in range(len(cb))])
    assert (diag == 0).any() and (diag > 0).any()     # both sides of the gate are present


# ------------------------------------------------------------------------------------------------------- non-finite
@pytest.mark.parametrize("pos", [0, 1])
@pytest.mark.parametrize("n", [3, 7, 100, 300, 1000, 4095])
def test_non_finite_boxes(eng, oracle, pos, n):
    """NaN / +-inf in a track's x, y, height or aspect and in a candidate's x or y: every other track must still score
    exactly as in the oracle (a NaN x used to let the sort drop tracks and read index -1)."""
    rng = np.random.default_rng(n + 17 * pos)
    cb, tb = scene(rng, 60, n)
    if n == 7:
        tb[:, 0] = [78, 10, 86, 55, 43, 0, 54]
        tb[:, 1] = 50.0
        cb[:, 0] = rng.uniform(0, 100, len(cb))
        cb[:, 1] = 50.0
    specials = [NAN, INF, -INF]
    k = max(1, n // 50)
    for col in (0, 1, 3, 4):
        for s in specials:
            idx = rng.integers(0, n, k)
            if n == 7 and col == 0 and s != s:
                idx = np.array([5])
            tb_s = tb.copy()
            tb_s[idx, col] = s
            cost(eng, oracle, pos, cb, tb_s)
    for col in (0, 1):
        for s in specials:
            cb_s = cb.copy()
            cb_s[rng.integers(0, len(cb), 5), col] = s
            tb_s = tb.copy()
            tb_s[rng.integers(0, n, k), 0] = NAN
            cost(eng, oracle, pos, cb_s, tb)
            cost(eng, oracle, pos, cb_s, tb_s)


# ------------------------------------------------------------------------------------------------------- trackers
def both(eng, oracle, **kw):
    from similari_b200._lib import default_options

    return eng.Tracker(default_options(**kw)), oracle.Tracker(oracle.make_options(**kw))


def run_sequence(eng, oracle, frames, kw, full_costs=False, check_costs=True, after=None):
    """frames: list of (scene_ids, det_offsets, boxes, features, has_feature).  Ids, epochs, lengths, voting types, boxes
    and (for the first scene) last_costs identical to the oracle, frame by frame."""
    g, o = both(eng, oracle, **kw)
    for fr, (sids, offs, boxes, feats, hasf) in enumerate(frames):
        sid = int(sids[0])
        ids_g = [int(x) for x in g.scene_tracks(sid)["ids"]]
        ids_o = [int(x) for x in o.scene_tracks(sid)["ids"]]
        if full_costs:
            os.environ["SB200_FULL_COSTS"] = "1"
        try:
            rg = g.predict_batch(sids, offs, boxes, features=feats, has_feature=hasf)
        finally:
            os.environ.pop("SB200_FULL_COSTS", None)
        ro = o.predict_batch(sids, offs, boxes, features=feats, has_feature=hasf)
        for key in ("ids", "epochs", "lengths", "voting_types"):
            assert np.array_equal(rg[key], ro[key]), (fr, key)
        for key in ("predicted", "observed"):
            # Rows of real objects only: the oracle's Kalman step (full 10 x 10 products, 0 * NaN = NaN) spreads a NaN
            # centre over the whole state, the product's block form keeps it in the one coordinate.
            real = np.isfinite(ro[key][:, [0, 1, 3, 4]]).all(axis=1)
            assert np.array_equal(rg[key][real], ro[key][real]) or np.array_equal(
                np.nan_to_num(rg[key][real], nan=-7.0), np.nan_to_num(ro[key][real], nan=-7.0)), (fr, key)
            # rows of a NaN track: every coordinate the product reports NaN is NaN in the oracle, and every coordinate
            # the oracle keeps finite is the product's, bit for bit (DESIGN.md, known divergence of the Kalman state)
            pg, po = rg[key][~real], ro[key][~real]
            assert np.all(~np.isnan(pg) | np.isnan(po)), (fr, key)
            assert np.all(np.isnan(po) | (pg == po)), (fr, key)
        if check_costs:
            # the device store drops an expired track at the end of the frame in which it expires, the oracle at its
            # next collection point (its column is all None until then): compare columns by track id
            assert [i for i in ids_o if i in set(ids_g)] == ids_g, fr
            cg, co = g.last_costs(sid), o.last_costs(sid)
            if co.size:
                col_of = {i: c for c, i in enumerate(ids_o)}
                live = [col_of[i] for i in ids_g]
                if cg.size:
                    assert np.array_equal(np.nan_to_num(cg, nan=-7.0), np.nan_to_num(co[:, live], nan=-7.0)), fr
                assert np.all(np.isnan(co[:, np.setdiff1d(np.arange(len(ids_o)), live)])), fr
        assert g.active_tracks() == o.active_tracks()
        if after is not None:
            after(fr, g)
    return g, o


def grid_objects(rng, n, spacing=90.0):
    side = int(np.ceil(np.sqrt(n)))
    b = np.empty((n, 6), np.float32)
    b[:, 0] = (np.arange(n) % side) * spacing + 50
    b[:, 1] = (np.arange(n) // side) * spacing + 50
    b[:, 2] = NAN
    b[:, 3] = rng.uniform(0.4, 0.6, n)
    b[:, 4] = rng.uniform(40, 60, n)
    b[:, 5] = rng.uniform(0.5, 1.0, n)
    return b


@pytest.mark.parametrize("kind", [0, 1])
@pytest.mark.parametrize("pos", [0, 1])
def test_trackers_with_a_nan_centre_detection(eng, oracle, kind, pos):
    """Frame 1 has one detection with a NaN centre beside finite ones: it becomes a NaN track, and the finite frames after
    it must keep matching every real object exactly as the oracle does."""
    rng = np.random.default_rng(3 + 2 * kind + pos)
    n_scenes = 1 if kind == 0 else 3
    objs = [grid_objects(rng, 37 + 5 * s) for s in range(n_scenes)]
    frames = []
    for fr in range(6):
        boxes, offs = [], [0]
        for s in range(n_scenes):
            b = objs[s].copy()
            b[:, :2] += np.float32(2.0 * fr) + rng.normal(0, 1.0, (len(b), 2)).astype(np.float32)
            if fr == 0:
                bad = b[:1].copy()
                bad[0, 0 if s % 2 == 0 else 1] = NAN
                b = np.concatenate([b[:5], bad, b[5:]])
            boxes.append(b)
            offs.append(offs[-1] + len(b))
        frames.append((np.arange(n_scenes, dtype=np.uint64), np.array(offs, np.int32), np.concatenate(boxes), None, None))
    run_sequence(eng, oracle, frames, dict(kind=kind, positional_kind=pos, iou_threshold=0.3, max_idle_epochs=3))


@pytest.mark.parametrize("full_costs", [False, True])
def test_visual_tracker_across_the_unsorted_scan_limit(eng, oracle, full_costs, monkeypatch):
    """VisualSort on the tensor-core path, whose positional stage is the lazy scan: one scene of 1552 objects with
    features, then a frame in which the first 96 detections carry no feature (the visual pass cannot decide them: 96
    open candidates, the unsorted scan), then one with 97 (the sorted scan, with every claimed track on the 3.0e38 key).
    The other detections repeat their track's feature and are decided visually.  With SB200_FULL_COSTS every pair is
    scanned instead (no lazy scan): that run checks the whole cost matrix."""
    from similari_b200._lib import lib

    monkeypatch.setenv("SB200_VIS_KERNEL", "tc")
    rng = np.random.default_rng(96)
    n, d = 1552, 128
    # pos_scan_impl gives a scene min(16, ceil(M / 64), 2 * 132 SMs / scenes) CTAs, each counting the open candidates of
    # its own ceil(M / nsplit) slice: 16 slices of 97 here, and the open detections are the first rows (slice 0)
    nsplit = max(1, min(16, (n + 63) // 64, 2 * 132 // 1))
    assert nsplit == 16 and -(-n // nsplit) == 97 and lib().sb200_device_count() > 0
    objs = grid_objects(rng, n)
    feats = rng.standard_normal((n, d)).astype(np.float32)
    feats /= np.linalg.norm(feats, axis=1, keepdims=True)
    frames = []
    for fr, n_open in enumerate([0, 0, 0, 96, 97, 0]):
        b = objs.copy()
        b[:, :2] += np.float32(1.5 * fr) + rng.normal(0, 0.5, (n, 2)).astype(np.float32)
        hasf = np.ones(n, np.uint8)
        hasf[:n_open] = 0
        frames.append((np.zeros(1, np.uint64), np.array([0, n], np.int32), b, feats.copy(), hasf))
    # two observations per track keep the visual survivor list (<= 2 per track and detection) under the 4096 entries of
    # the sparse voting kernel, so the scene stays in the lazy (sparse) mode
    kw = dict(kind=2, positional_kind=1, iou_threshold=0.3, max_idle_epochs=3, visual_kind=0, visual_threshold=0.7,
              feature_dim=d, visual_max_observations=2, visual_min_votes=1, visual_minimal_track_length=1,
              min_confidence=0.1)
    # the lazy scan's cost matrix is partial by design: costs are compared on the full-cost run only
    dense = []
    run_sequence(eng, oracle, frames, kw, full_costs=full_costs, check_costs=full_costs,
                 after=lambda fr, g: dense.append(g.work_counters()["dense_fallback_scenes"]))
    # from the second frame on (the first has no tracks to screen) the scene never falls back to the dense kernels, so
    # frames 3 and 4 ran the lazy scan
    if not full_costs:
        assert dense[-1] == dense[0], dense
