"""CPU checks of the point Kalman filter, the box filter's distance and the vertex-emitting clip (sb_math.cuh,
host-compiled by tests/host_shim/geom_shim.cpp) against full restatements: the point filter's 4x4 matrices
(tests/host_shim/point_kalman_full.cpp) and the oracle's clip and area.  Also the API surface, argument checks and the
no-GPU failure of the new entry points.  No GPU needed."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
F32 = np.float32
WEIGHTS = [(F32(1 / 20), F32(1 / 160)), (F32(0.3), F32(0.02))]


def build_geom_shim(outdir):
    """Compiles the block forms and the full-matrix restatement into one library (flags as test_product_math_cpu)."""
    d = os.path.join(HERE, "host_shim")
    so = os.path.join(str(outdir), "libgeomshim.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-shared", "-x", "c++",
                           os.path.join(d, "geom_shim.cpp"), os.path.join(d, "point_kalman_full.cpp"), "-o", so])
    L = C.CDLL(so)
    f, f32p, f64p, i32p = C.c_float, C.POINTER(C.c_float), C.POINTER(C.c_double), C.POINTER(C.c_int32)
    sig = {
        "gshim_point_initiate": (None, [f, f, f, f, f32p]),
        "gshim_point_predict": (None, [f, f, f32p, f32p]),
        "gshim_point_update": (None, [f, f32p, f, f, f32p]),
        "gshim_point_distance": (f, [f, f32p, f, f]),
        "gshim_box_distance": (f, [f, f32p, f32p]),
        "gshim_clip_ring": (C.c_double, [f64p, f64p, f64p, i32p]),
        "gshim_clip_count": (C.c_double, [f64p, f64p, i32p]),
        "gshim_clip_area": (C.c_double, [f64p, f64p]),
        "pref_initiate": (None, [f, f, f, f, f32p]),
        "pref_predict": (None, [f, f, f32p, f32p]),
        "pref_update": (None, [f, f, f32p, f, f, f32p]),
        "pref_distance": (f, [f, f, f32p, f, f]),
        "pref_calculate_cost": (f, [f, C.c_int]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(L, name)
        fn.restype, fn.argtypes = res, args
    return L


class PointRef:
    """The full-matrix point filter (state = mean[4] + cov[16]) over numpy rows."""

    def __init__(self, L, pw, vw):
        self.L, self.pw, self.vw = L, F32(pw), F32(vw)

    def initiate(self, x, y):
        out = np.zeros(20, F32)
        self.L.pref_initiate(self.pw, self.vw, F32(x), F32(y), fp(out))
        return out

    def predict(self, st):
        out = np.zeros(20, F32)
        self.L.pref_predict(self.pw, self.vw, fp(np.ascontiguousarray(st, F32)), fp(out))
        return out

    def update(self, st, x, y):
        out = np.zeros(20, F32)
        self.L.pref_update(self.pw, self.vw, fp(np.ascontiguousarray(st, F32)), F32(x), F32(y), fp(out))
        return out

    def distance(self, st, x, y):
        return F32(self.L.pref_distance(self.pw, self.vw, fp(np.ascontiguousarray(st, F32)), F32(x), F32(y)))


def fp(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def pack12(st20):
    """full mean[4] + cov[4x4] -> product mean[4] + 2 x (Pii, Pi,i+2, Pi+2,i, Pi+2,i+2)."""
    mean, cov = st20[:4], st20[4:].reshape(4, 4)
    out = np.zeros(12, F32)
    out[:4] = mean
    for i in range(2):
        out[4 + 4 * i: 8 + 4 * i] = [cov[i, i], cov[i, i + 2], cov[i + 2, i], cov[i + 2, i + 2]]
    return out


def offblock_zero(st20):
    cov = st20[4:].reshape(4, 4).copy()
    for i in range(2):
        cov[i, i] = cov[i, i + 2] = cov[i + 2, i] = cov[i + 2, i + 2] = 0
    return not cov.any()


def random_point_chain(r, k):
    """A start point and k measurements: small, negative and large coordinates, smooth and jumpy motion."""
    scale = r.choice([1.0, 100.0, 1e4, 1e6])
    p0 = r.uniform(-scale, scale, 2).astype(F32)
    v = r.normal(0, scale * 1e-2, 2)
    pts = [p0 + (v * (s + 1) + r.normal(0, scale * 1e-3, 2)).astype(F32) for s in range(k)]
    return p0, [p.astype(F32) for p in pts]


REFERENCE_TEST_POINTS = [(1.1, 0.1), (1.2, 0.2), (1.3, 0.3), (1.4, 0.4), (1.5, 0.5), (1.6, 0.6), (1.7, 0.7), (1.8, 0.67),
                         (1.9, 0.60)]   # kalman_2d_point.rs:166-220, then distance to (2.0, 0.57)


@pytest.fixture(scope="module")
def geom(tmp_path_factory):
    return build_geom_shim(tmp_path_factory.mktemp("geomshim"))


class Block:
    def __init__(self, L, pw, vw):
        self.L, self.pw, self.vw = L, F32(pw), F32(vw)

    def initiate(self, x, y):
        out = np.zeros(12, F32)
        self.L.gshim_point_initiate(self.pw, self.vw, F32(x), F32(y), fp(out))
        return out

    def predict(self, st):
        out = np.zeros(12, F32)
        self.L.gshim_point_predict(self.pw, self.vw, fp(st), fp(out))
        return out

    def update(self, st, x, y):
        out = np.zeros(12, F32)
        self.L.gshim_point_update(self.pw, fp(st), F32(x), F32(y), fp(out))
        return out

    def distance(self, st, x, y):
        return F32(self.L.gshim_point_distance(self.pw, fp(st), F32(x), F32(y)))


@pytest.mark.parametrize("weights", WEIGHTS, ids=["default", "heavy"])
def test_point_filter_block_form_bit_exact(geom, weights):
    pw, vw = weights
    ref, mine = PointRef(geom, pw, vw), Block(geom, pw, vw)
    r = np.random.default_rng(5 + int(pw * 100))
    for trial in range(200):
        p0, pts = random_point_chain(r, 8)
        a, b = ref.initiate(*p0), mine.initiate(*p0)
        assert np.array_equal(pack12(a), b) and offblock_zero(a)
        for step, z in enumerate(pts):
            a, b = ref.predict(a), mine.predict(b)
            assert offblock_zero(a)
            assert np.array_equal(pack12(a), b), (trial, step, "predict")
            assert ref.distance(a, *z) == mine.distance(b, *z), (trial, step, "distance")
            a, b = ref.update(a, *z), mine.update(b, *z)
            assert offblock_zero(a)
            assert np.array_equal(pack12(a), b), (trial, step, "update")


def test_point_filter_reference_test_sequence(geom):
    """The exact calls of the reference's kalman_2d_point::tests::test, each state compared in full."""
    ref, mine = PointRef(geom, 1 / 20, 1 / 160), Block(geom, 1 / 20, 1 / 160)
    a, b = ref.initiate(1.0, 0.0), mine.initiate(1.0, 0.0)
    a, b = ref.predict(a), mine.predict(b)
    assert np.array_equal(pack12(a), b)
    for x, y in REFERENCE_TEST_POINTS:
        a, b = ref.update(a, x, y), mine.update(b, x, y)
        a, b = ref.predict(a), mine.predict(b)
        assert np.array_equal(pack12(a), b), (x, y)
    assert ref.distance(a, 2.0, 0.57) == mine.distance(b, 2.0, 0.57)
    assert 1.0 < b[0] < 2.5 and 0.0 < b[1] < 1.0


def rand_box(r, oriented):
    return np.array([r.uniform(0, 400), r.uniform(0, 400), r.uniform(-1.6, 1.6) if oriented else np.nan,
                     r.uniform(0.3, 0.8), r.uniform(40, 160), 1.0], F32)


def check_clip(geom, oracle, l, q):
    """The ring, its count and its area against oracle.sh_clip / oracle.polygon_area on the oracle's vertices."""
    vl = np.ascontiguousarray(oracle.vertices(l), np.float64)
    vq = np.ascontiguousarray(oracle.vertices(q), np.float64)
    ring = np.zeros(32, np.float64)
    cnt = C.c_int32(0)
    area = geom.gshim_clip_ring(dp(vl), dp(vq), dp(ring), C.byref(cnt))
    ref = oracle.sh_clip(vl, vq)
    assert cnt.value == len(ref)
    assert np.array_equal(ring[: 2 * cnt.value].reshape(-1, 2), ref)
    assert area == oracle.polygon_area(ref)
    assert area == geom.gshim_clip_area(dp(vl), dp(vq))
    cnt2 = C.c_int32(0)
    assert geom.gshim_clip_count(dp(vl), dp(vq), C.byref(cnt2)) == area and cnt2.value == cnt.value
    return cnt.value, area


@pytest.mark.parametrize("oriented", [False, True])
def test_vertex_clip_bit_exact(geom, oracle, oriented):
    r = np.random.default_rng(21 + oriented)
    nonempty = 0
    for i in range(3000):
        l = rand_box(r, oriented)
        q = l.copy()
        q[:2] += r.normal(0, 40, 2).astype(F32)
        q[3:5] *= r.uniform(0.6, 1.4, 2).astype(F32)
        if oriented:
            q[2] += F32(r.normal(0, 0.6))
        n, _ = check_clip(geom, oracle, l, q)
        nonempty += n >= 3
    assert nonempty > 1000


def test_vertex_clip_special_pairs(geom, oracle):
    lt = oracle.ltwh
    b = lt(0.0, 0.0, 4.0, 8.0)   # aspects exact in f32: the areas below are exact
    cases = [
        (b, b),                                        # identical
        (b, lt(1.0, 1.0, 2.0, 2.0)),                   # contained
        (lt(1.0, 1.0, 2.0, 2.0), b),                   # containing
        (b, lt(4.0, 0.0, 4.0, 8.0)),                   # shares an edge
        (b, lt(4.0, 8.0, 2.0, 2.0)),                   # shares a corner
        (b, lt(10.0, 10.0, 2.0, 2.0)),                 # disjoint
        (lt(0.0, 0.0, 5.0, 10.0), lt(0.0, 0.0, 10.0, 5.0)),
        (oracle.box(2.5, 5.0, 0.5, 0.5, 10.0), lt(0.0, 0.0, 5.0, 10.0)),
        (oracle.box(0.0, 0.0, 0.7853982, 1.0, 2.0), oracle.box(0.0, 0.0, None, 1.0, 2.0)),
    ]
    got = [check_clip(geom, oracle, l, q) for l, q in cases]
    assert got[0][1] == 32.0 and got[1][1] == 4.0 and got[2][1] == 4.0 and got[5] == (0, 0.0)
    assert got[6][1] == 25.0


def test_box_filter_distance_bit_exact(geom, oracle):
    """sb_math's kalman_distance (the l5 of the positional cost kernel) against the oracle's Cholesky restatement."""
    from test_product_math_cpu import pack30, rand_box as track_box

    r = np.random.default_rng(3)
    pw, vw = F32(1 / 20), F32(1 / 160)
    for trial in range(300):
        b = track_box(r, trial % 2 == 1)
        st = oracle.kalman_predict(oracle.kalman_initiate(b, pw, vw), pw, vw)
        z = b.copy()
        z[:2] += r.normal(0, 5, 2).astype(F32)
        assert F32(oracle.kalman_distance(st, z, pw, vw)) == F32(geom.gshim_box_distance(pw, fp(pack30(st)), fp(z)))


def test_calculate_cost_both_filters(geom, oracle):
    import similari_b200.api as api

    for thr in (F32(5.9915), F32(11.070)):
        for d in (np.nextafter(thr, F32(0)), thr, np.nextafter(thr, F32(1e9)), F32(0.0), F32(50.0), F32(np.nan)):
            for inverted in (False, True):
                want_box = F32(oracle.kalman_calculate_cost(d, inverted))
                want_pt = F32(geom.pref_calculate_cost(d, int(inverted)))
                got_box = F32(api.Universal2DBoxKalmanFilter.calculate_cost(d, inverted))
                got_pt = F32(api.Point2DKalmanFilter.calculate_cost(d, inverted))
                assert np.array_equal(got_box, want_box, equal_nan=True), (d, inverted)
                assert np.array_equal(got_pt, want_pt, equal_nan=True), (d, inverted)
                assert np.array_equal(F32(api.Vec2DKalmanFilter.calculate_cost([d], inverted)[0]), want_pt, equal_nan=True)
    # the two filters differ only in the non-inverted threshold: CHI2INV95[1] for the point, CHI2INV95[4] for the box
    assert api.Point2DKalmanFilter.calculate_cost(8.0, False) == 100.0
    assert api.Universal2DBoxKalmanFilter.calculate_cost(8.0, False) == 8.0


NEW_NAMES = ["Universal2DBoxKalmanFilter", "Universal2DBoxKalmanFilterState", "Point2DKalmanFilter",
             "Point2DKalmanFilterState", "Vec2DKalmanFilter", "Polygon", "sutherland_hodgman_clip", "intersection_area"]


def test_api_names():
    import similari_b200.api as api

    for name in NEW_NAMES + ["intersection_areas"]:
        assert hasattr(api, name), name
    for cls in ("Universal2DBoxKalmanFilter", "Point2DKalmanFilter", "Vec2DKalmanFilter"):
        f = getattr(api, cls)()
        assert (f._pw, f._vw) == (float(F32(0.05)), float(F32(0.00625)))
    b = api.Universal2DBox.ltwh(0.0, 0.0, 5.0, 10.0)
    assert hasattr(b, "get_vertices") and b.gen_vertices() is None
    assert api.Polygon._from_ring([(0, 0), (1, 0), (1, 1)]).get_points() == [(0, 0), (1, 0), (1, 1), (0, 0)]
    assert api.Polygon._from_ring([]).get_points() == []
    st = api.Universal2DBoxKalmanFilterState(np.array([1, 2, 0, 0.5, 10] + [0] * 25, F32))
    assert st.universal_bbox().angle is None and st.bbox().width == F32(5.0)
    st = api.Universal2DBoxKalmanFilterState(np.array([1, 2, 0.1, 0.5, 10] + [0] * 25, F32))
    assert st.universal_bbox().angle == F32(0.1) and st.universal_bbox().confidence == F32(1.0)
    with pytest.raises(AttributeError):
        st.bbox()
    with pytest.raises(AssertionError, match="Lengths of state and points must match"):
        api.Vec2DKalmanFilter().update([], [(1.0, 2.0)])


@pytest.fixture(scope="module")
def L():
    from similari_b200 import _build, _lib

    _build.build()
    return _lib.lib()


def _calls(L, bad):
    """Every new entry point with n = 1; bad=True passes NULL for a required pointer (or a negative size)."""
    from similari_b200._lib import ptr

    s30, s12, b6, p2 = (np.zeros((1, k), F32) for k in (30, 12, 6, 2))
    of, od, oi = np.zeros(16, F32), np.zeros(64, np.float64), np.zeros(4, np.int32)
    nul = None if bad else 1
    pick = (lambda a: None) if bad else ptr
    return [
        L.sb200_kalman_distance(0.05, 0.00625, pick(s30), ptr(b6), 1, ptr(of), 0),
        L.sb200_point_kalman_initiate(0.05, 0.00625, pick(p2), 1, ptr(s12), 0),
        L.sb200_point_kalman_predict(0.05, 0.00625, pick(s12), 1, ptr(s12), 0),
        L.sb200_point_kalman_update(0.05, 0.00625, ptr(s12), pick(p2), 1, ptr(s12), 0),
        L.sb200_point_kalman_distance(0.05, 0.00625, ptr(s12), pick(p2), 1, ptr(of), 0),
        L.sb200_box_vertices(pick(b6), 1, ptr(od), 0),
        L.sb200_clip_polygons(ptr(b6), pick(b6), 1, ptr(od), ptr(oi), ptr(od), 0),
        L.sb200_intersection_areas(ptr(b6), 1, pick(b6), 1, ptr(od), 0),
        L.sb200_box_vertices(ptr(b6), -1 if nul is None else 1, ptr(od), 0),
    ]


def test_bad_arguments_are_invalid(L):
    assert _calls(L, bad=True) == [-1] * 9
    assert L.sb200_intersection_areas(None, -1, None, 0, None, 0) == -1


def test_no_cpu_fallback_for_new_entries(L):
    from similari_b200 import _lib
    import similari_b200.api as api
    import similari_b200.engine as eng

    if L.sb200_device_count() > 0:
        pytest.skip("a GPU is present; the loud-failure path is for CPU-only machines")
    assert _calls(L, bad=False) == [-2] * 9
    b = api.Universal2DBox.ltwh(0.0, 0.0, 5.0, 10.0)
    st = api.Universal2DBoxKalmanFilterState(np.zeros(30, F32))
    ps = api.Point2DKalmanFilterState(np.zeros(12, F32))
    for call in (lambda: api.Universal2DBoxKalmanFilter().initiate(b), lambda: api.Universal2DBoxKalmanFilter().distance(st, b),
                 lambda: api.Point2DKalmanFilter().initiate(1.0, 2.0), lambda: api.Point2DKalmanFilter().predict(ps),
                 lambda: api.Vec2DKalmanFilter().initiate([(1.0, 2.0)]), lambda: b.get_vertices(),
                 lambda: api.sutherland_hodgman_clip(b, b), lambda: api.intersection_area(b, b),
                 lambda: api.intersection_areas([b], [b]), lambda: eng.point_kalman_distance(np.zeros((1, 12)), [[0, 0]])):
        with pytest.raises(_lib.Sb200Error):
            call()
