"""GPU parity of the point Kalman filter, the box filter's distance and the geometry operators (kernels_state.cu,
kernels_geom.cu) with full restatements: the point filter's 4x4 matrices (tests/host_shim/point_kalman_full.cpp), the
oracle's box filter, clip and area.  Everything is bit-exact.  The API part replays the reference's example scripts
python/kalman_bbox.py, kalman_2d_point.py, kalman_2d_vec.py and clipping_intersection.py (their calls are copied here)."""
import numpy as np
import pytest

from test_geometry_kalman_cpu import PointRef, build_geom_shim, pack12
from test_product_math_cpu import pack30

pytestmark = pytest.mark.gpu
F32 = np.float32


@pytest.fixture(scope="module")
def eng():
    import similari_b200.engine as e
    from similari_b200._lib import lib

    if lib().sb200_device_count() <= 0:
        pytest.fail("no CUDA device: the product has no CPU path")
    return e


@pytest.fixture(scope="module")
def geom(tmp_path_factory):
    return build_geom_shim(tmp_path_factory.mktemp("geomshim_gpu"))


def ref_chain_full(L, pw, vw, p0, steps):
    """Full-matrix states after initiate, then per step (predict, distance to z, update with z)."""
    ref = PointRef(L, pw, vw)
    a = ref.initiate(*p0)
    out = [("initiate", pack12(a))]
    for z in steps:
        a = ref.predict(a)
        out.append(("predict", pack12(a)))
        out.append(("distance", ref.distance(a, *z)))
        a = ref.update(a, *z)
        out.append(("update", pack12(a)))
    return out


@pytest.mark.parametrize("n", [1, 300, (1 << 20) + 17])
def test_point_filter_bit_exact(eng, geom, n):
    r = np.random.default_rng(n)
    pw, vw = (F32(1 / 20), F32(1 / 160)) if n != 300 else (F32(0.3), F32(0.02))
    scale = np.where(r.random(n) < 0.5, 1e2, 1e5)[:, None]
    p0 = (r.uniform(-1, 1, (n, 2)) * scale).astype(F32)
    zs = [(p0 + r.normal(0, 1, (n, 2)) * scale * 1e-2 * (k + 1)).astype(F32) for k in range(4)]
    st = eng.point_kalman_initiate(p0, pw, vw)
    got = [st]
    for z in zs:
        st = eng.point_kalman_predict(st, pw, vw)
        got += [st, eng.point_kalman_distance(st, z, pw, vw)]
        st = eng.point_kalman_update(st, z, pw, vw)
        got.append(st)
    rows = np.unique(np.r_[0, n - 1, n // 2, r.integers(0, n, min(n, 400))])
    for i in rows:
        ref = ref_chain_full(geom, pw, vw, p0[i], [z[i] for z in zs])
        for k, (what, want) in enumerate(ref):
            g = got[k][i]
            assert np.array_equal(g, want), (i, k, what, g, want)


@pytest.mark.parametrize("oriented", [False, True])
def test_box_filter_distance_bit_exact(eng, oracle, oriented):
    r = np.random.default_rng(9 + oriented)
    n = 2000
    pw, vw = F32(1 / 20), F32(1 / 160)
    boxes = np.stack([np.array([r.uniform(0, 1920), r.uniform(0, 1080), r.uniform(-1.5, 1.5) if oriented else np.nan,
                                r.uniform(0.3, 0.8), r.uniform(40, 160), 1.0], F32) for _ in range(n)])
    full = [oracle.kalman_predict(oracle.kalman_update(oracle.kalman_predict(oracle.kalman_initiate(b, pw, vw), pw, vw),
                                                       b, pw, vw), pw, vw) for b in boxes]
    z = boxes.copy()
    z[:, :2] += r.normal(0, 4, (n, 2)).astype(F32)
    got = eng.kalman_distance(np.stack([pack30(s) for s in full]), z, pw, vw)
    want = np.array([oracle.kalman_distance(s, zz, pw, vw) for s, zz in zip(full, z)], F32)
    assert np.array_equal(got, want)


def random_boxes(r, n, oriented, span=400.0):
    b = np.zeros((n, 6), F32)
    b[:, 0] = r.uniform(0, span, n)
    b[:, 1] = r.uniform(0, span, n)
    b[:, 2] = r.uniform(-1.6, 1.6, n) if oriented else np.nan
    b[:, 3] = r.uniform(0.3, 0.8, n)
    b[:, 4] = r.uniform(40, 160, n)
    b[:, 5] = 1.0
    return b


def ref_area(oracle, vertices, a, b):
    """intersection_area_py: polygon_area(sh_clip(...)) on the product's vertices (not oracle.intersection: no too_far)."""
    return oracle.polygon_area(oracle.sh_clip(vertices(a), vertices(b)))


def test_box_vertices(eng, oracle):
    r = np.random.default_rng(1)
    b = np.r_[random_boxes(r, 500, False), random_boxes(r, 500, True)]
    got = eng.box_vertices(b)
    assert np.array_equal(got[:500], np.stack([oracle.vertices(x) for x in b[:500]]))
    # oriented: the product's sin / cos are correctly rounded, the oracle's are the C library's (test_product_math_cpu)
    np.testing.assert_allclose(got[500:], np.stack([oracle.vertices(x) for x in b[500:]]), rtol=0, atol=2e-13)


def test_clip_polygons_bit_exact(eng, oracle):
    r = np.random.default_rng(2)
    n = 10_000
    s = np.r_[random_boxes(r, n // 2, False), random_boxes(r, n // 2, True)]
    c = s.copy()
    c[:, :2] += r.normal(0, 50, (n, 2)).astype(F32)
    c[:, 3:5] *= r.uniform(0.6, 1.4, (n, 2)).astype(F32)
    c[n // 2:, 2] += r.normal(0, 0.7, n // 2).astype(F32)
    v, cnt, area = eng.clip_polygons(s, c)
    verts = eng.box_vertices(np.r_[s, c])
    nonempty = 0
    for i in range(n):
        ref = oracle.sh_clip(verts[i], verts[n + i])
        assert cnt[i] == len(ref), i
        assert np.array_equal(v[i, : cnt[i]], ref), i
        assert not v[i, cnt[i]:].any()
        assert area[i] == oracle.polygon_area(ref), i
        nonempty += cnt[i] >= 3
    assert nonempty > n // 4


@pytest.mark.parametrize("m,n", [(700, 900), (1, 900), (700, 1), (1, 1)])
def test_intersection_areas_bit_exact(eng, oracle, m, n):
    r = np.random.default_rng(m * 7 + n)
    a = np.r_[random_boxes(r, m - m // 2, False), random_boxes(r, m // 2, True)]
    b = np.r_[random_boxes(r, n - n // 2, True), random_boxes(r, n // 2, False)]
    got = eng.intersection_areas(a, b)
    assert got.shape == (m, n)
    va, vb = eng.box_vertices(a), eng.box_vertices(b)
    idx = [(i, j) for i in range(m) for j in range(n)]
    if len(idx) > 60_000:
        sel = r.choice(len(idx), 60_000, replace=False)
        idx = [idx[k] for k in sel] + [(m - 1, n - 1), (0, n - 1), (m - 1, 0)]
    for i, j in idx:
        assert got[i, j] == oracle.polygon_area(oracle.sh_clip(va[i], vb[j])), (i, j)
    if m * n > 100:
        assert (got > 0).any() and (got == 0).any()
    # each row equals the one-pair clip operator
    _, _, area = eng.clip_polygons(np.repeat(a[:1], n, 0), b)
    assert np.array_equal(got[0], area)


def test_degenerate_rows_leave_clean_rows_exact(eng, oracle, geom):
    nan = np.nan
    r = np.random.default_rng(4)
    clean = random_boxes(r, 6, True)
    bad = np.array([[10, 10, nan, 0.5, 0.0, 1],       # zero height
                    [10, 10, nan, 0.0, 50.0, 1],      # zero aspect
                    [nan, 10, nan, 0.5, 50.0, 1],     # NaN coordinate
                    [10, 10, nan, 0.5, 50.0, 1]], F32)
    bad[3, 2] = np.float32(nan)                        # NaN angle == None
    mixed = np.r_[clean[:3], bad, clean[3:]]
    finite = np.isfinite(mixed[:, [0, 1, 3, 4]]).all(1)
    got = eng.intersection_areas(mixed, mixed)
    alone = eng.intersection_areas(clean, clean)
    ci = [0, 1, 2, 7, 8, 9]
    assert np.array_equal(got[np.ix_(ci, ci)], alone)
    va = eng.box_vertices(mixed)
    for i in np.flatnonzero(finite):
        for j in np.flatnonzero(finite):
            assert got[i, j] == oracle.polygon_area(oracle.sh_clip(va[i], va[j]))
    v, cnt, area = eng.clip_polygons(mixed, mixed[::-1].copy())
    assert (cnt >= 0).all()
    # Kalman filters: degenerate rows next to clean ones
    pw, vw = F32(1 / 20), F32(1 / 160)
    pts = np.array([[1, 2], [nan, 3], [1e30, -1e30], [4, 5]], F32)
    st = eng.point_kalman_predict(eng.point_kalman_initiate(pts, pw, vw), pw, vw)
    st2 = eng.point_kalman_update(st, pts, pw, vw)
    d = eng.point_kalman_distance(st2, pts, pw, vw)
    for i in (0, 2, 3):
        ref = ref_chain_full(geom, pw, vw, pts[i], [pts[i]])
        assert np.array_equal(st[i], ref[1][1]) and np.array_equal(st2[i], ref[3][1])
        assert np.array_equal(d[i], PointRef(geom, pw, vw).distance(
            PointRef(geom, pw, vw).update(PointRef(geom, pw, vw).predict(PointRef(geom, pw, vw).initiate(*pts[i])), *pts[i]),
            *pts[i]))
    assert np.isnan(st2[1, [0, 2]]).all() and not np.isnan(st2[1, [1, 3]]).any()
    kb = np.r_[clean[:2], bad, clean[2:]]
    ks = eng.kalman_predict(eng.kalman_initiate(kb, pw, vw), pw, vw)
    kd = eng.kalman_distance(ks, kb, pw, vw)
    alone = eng.kalman_distance(eng.kalman_predict(eng.kalman_initiate(clean, pw, vw), pw, vw), clean, pw, vw)
    assert np.array_equal(kd[[0, 1, 6, 7, 8, 9]], alone)


# ------------------------------------------------------------------------------------ the reference's example scripts
def test_example_kalman_bbox(eng, oracle):
    import similari_b200.api as similari

    pw, vw = F32(0.05), F32(0.00625)
    f = similari.Universal2DBoxKalmanFilter()
    ref = oracle.kalman_initiate(oracle.ltwh(0.0, 0.0, 5.0, 10.0), pw, vw)

    def same(state, ref):
        ub, rb = state.universal_bbox(), oracle.kalman_state_box(ref)
        assert np.array_equal(state._st, pack30(ref))
        assert (ub.xc, ub.yc, ub.aspect, ub.height) == tuple(rb[[0, 1, 3, 4]])
        assert (ub.angle is None) == bool(np.isnan(rb[2])) and ub.confidence == F32(1.0)

    state = f.initiate(similari.BoundingBox(0.0, 0.0, 5.0, 10.0).as_xyaah())
    state = f.predict(state)
    ref = oracle.kalman_predict(ref, pw, vw)
    same(state, ref)
    box_ltwh = state.bbox()
    rb = oracle.kalman_state_box(ref)
    assert box_ltwh.width == rb[4] * rb[3] and box_ltwh.height == rb[4]
    state = f.update(state, similari.BoundingBox(0.2, 0.2, 5.1, 9.9).as_xyaah())
    ref = oracle.kalman_update(ref, oracle.ltwh(0.2, 0.2, 5.1, 9.9), pw, vw)
    state = f.predict(state)
    ref = oracle.kalman_predict(ref, pw, vw)
    same(state, ref)
    for i in range(1, 21):
        state = f.predict(state)
        ref = oracle.kalman_predict(ref, pw, vw)
        same(state, ref)
        obs = similari.BoundingBox(0.2 + i * 0.2, 0.2 + i * 0.2, 5.0, 10.0).as_xyaah()
        d = f.distance(state, obs)
        assert F32(d) == F32(oracle.kalman_distance(ref, np.array(obs._row(), F32), pw, vw))
        assert F32(f.calculate_cost(d, True)) == F32(oracle.kalman_calculate_cost(d, True))
        state = f.update(state, obs)
        ref = oracle.kalman_update(ref, np.array(obs._row(), F32), pw, vw)
    same(state, ref)


def test_example_kalman_2d_point(eng, geom):
    import similari_b200.api as similari

    ref = PointRef(geom, 0.05, 0.00625)
    f = similari.Point2DKalmanFilter()
    state = f.initiate(1.0, 2.0)
    a = ref.initiate(1.0, 2.0)
    for i in range(1, 21):
        state = f.predict(state)
        a = ref.predict(a)
        assert (state.x(), state.y()) == (float(a[0]), float(a[1]))
        assert np.array_equal(state._st, pack12(a))
        pt = (1.0 + i * 0.1, 2.0 + i * 0.1)
        assert F32(f.distance(state, pt[0], pt[1])) == ref.distance(a, *pt)
        state = f.update(state, pt[0], pt[1])
        a = ref.update(a, *pt)
    assert np.array_equal(state._st, pack12(a))


def test_example_kalman_2d_vec(eng, geom):
    import similari_b200.api as similari

    ref = PointRef(geom, 0.05, 0.00625)
    f = similari.Vec2DKalmanFilter()
    state = f.initiate([(1.0, 2.0), (3.0, 4.0)])
    a = [ref.initiate(1.0, 2.0), ref.initiate(3.0, 4.0)]
    for i in range(1, 21):
        state = f.predict(state)
        a = [ref.predict(s) for s in a]
        assert len(state) == 2
        for k in range(2):
            assert (state[k].x(), state[k].y()) == (float(a[k][0]), float(a[k][1]))
        pt1 = (1.0 + i * 0.1, 2.0 + i * 0.1)
        pt2 = (3.0 + i * 0.05, 4.0 + i * 0.05)
        d = f.distance(state, [pt1, pt2])
        assert [F32(x) for x in d] == [ref.distance(a[0], *pt1), ref.distance(a[1], *pt2)]
        state = f.update(state, [pt1, pt2])
        a = [ref.update(a[0], *pt1), ref.update(a[1], *pt2)]
    assert np.array_equal(np.stack([s._st for s in state]), np.stack([pack12(x) for x in a]))
    # a plain list of states is accepted as well
    again = f.predict(list(state))
    assert np.array_equal(np.stack([s._st for s in again]), np.stack([pack12(ref.predict(x)) for x in a]))
    with pytest.raises(AssertionError, match="Lengths of state and points must match"):
        f.update(state, [pt1])


def test_example_clipping_intersection(eng, oracle):
    import similari_b200.api as similari

    def ring(p):
        pts = [tuple(map(float, q)) for q in p]
        return pts + [pts[0]] if pts and pts[0] != pts[-1] else pts

    bbox1 = similari.BoundingBox(0.0, 0.0, 5.0, 10.0).as_xyaah()
    bbox2 = similari.BoundingBox(0.0, 0.0, 10.0, 5.0).as_xyaah()
    clip = similari.sutherland_hodgman_clip(bbox1, bbox2)
    ref = oracle.sh_clip(oracle.vertices(bbox1._row()), oracle.vertices(bbox2._row()))
    assert clip.get_points() == ring(ref)
    area = similari.intersection_area(bbox1, bbox2)
    assert area == oracle.polygon_area(ref) == 25.0
    assert similari.intersection_area(similari.Universal2DBox.ltwh(0, 0, 5, 10), similari.Universal2DBox.ltwh(0, 0, 10, 5)) == 25.0

    bbox1 = similari.BoundingBox(0.0, 0.0, 5.0, 10.0).as_xyaah()
    bbox2 = similari.BoundingBox(0.0, 0.0, 5.0, 10.0).as_xyaah()
    bbox2.rotate(0.5)
    clip = similari.sutherland_hodgman_clip(bbox1, bbox2)
    v1, v2 = eng.box_vertices([bbox1._row(), bbox2._row()])
    ref = oracle.sh_clip(v1, v2)
    assert clip.get_points() == ring(ref)
    assert similari.intersection_area(bbox1, bbox2) == oracle.polygon_area(ref)
    bbox2.gen_vertices()
    assert similari.intersection_area(bbox1, bbox2) == oracle.polygon_area(ref)
    assert bbox1.get_vertices().get_points() == ring(v1)
    assert similari.intersection_areas([bbox1, bbox2], [bbox2])[0, 0] == oracle.polygon_area(ref)
    far = similari.Universal2DBox.ltwh(100.0, 100.0, 1.0, 1.0)
    assert similari.sutherland_hodgman_clip(bbox1, far).get_points() == [] and similari.intersection_area(bbox1, far) == 0.0
