"""CPU checks behind the positional cost kernels (similari_b200/csrc/kernels_cost.cu), no GPU needed.

1. The culled kernel's bitonic sort of the track centres (pos_sort_swap in sb_math.cuh, driven serially by
   tests/host_shim/shim.cpp exactly as the kernel drives it): whatever the keys -- NaN with any payload, +-inf,
   FLT_MAX, the 3.0e38 key of claimed tracks, +-0 -- positions [0, N) hold every track exactly once, and finite keys
   come out ascending.
2. The oracle that every GPU parity test trusts, pinned to exact arithmetic: the f64 Sutherland-Hodgman clip area
   against the exact (rational) intersection area of the same vertices, and the f32 Mahalanobis distance against the
   same formula in f64."""
import ctypes as C
import os
import subprocess
from fractions import Fraction

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
FLT_MAX = float(np.finfo(np.float32).max)


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("shim") / "libshim_sort.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-shared", "-x", "c++",
                           os.path.join(HERE, "host_shim", "shim.cpp"), "-o", so])
    L = C.CDLL(so)
    f32p, f64p, i32p = C.POINTER(C.c_float), C.POINTER(C.c_double), C.POINTER(C.c_int)
    L.shim_pos_sort.argtypes = [f32p, C.c_int, f32p, i32p]
    L.shim_clip_area.argtypes = [f64p, f64p]
    L.shim_clip_area.restype = C.c_double
    L.shim_maha.argtypes = [C.c_float, f32p, f32p]
    L.shim_maha.restype = C.c_float
    return L


def pos_sort(shim, x):
    x = np.ascontiguousarray(x, np.float32)
    n = len(x)
    np2 = 1
    while np2 < n:
        np2 <<= 1
    kx, kidx = np.empty(np2, np.float32), np.empty(np2, np.int32)
    shim.shim_pos_sort(x.ctypes.data_as(C.POINTER(C.c_float)), n, kx.ctypes.data_as(C.POINTER(C.c_float)),
                       kidx.ctypes.data_as(C.POINTER(C.c_int)))
    return kx, kidx


def nan_with_payload(rng, k):
    bits = rng.integers(1, 1 << 22, k, dtype=np.uint32) | np.uint32(0x7f800000) | \
        (rng.integers(0, 2, k, dtype=np.uint32) << np.uint32(31))
    return bits.view(np.float32)


def check_sorted(x, kx, kidx):
    n = len(x)
    head = kidx[:n]
    assert np.array_equal(np.sort(head), np.arange(n)), "[0, N) is not a permutation of the tracks"
    assert np.all(kidx[n:] == -1)
    assert np.array_equal(kx[:n].view(np.uint32), x[head].view(np.uint32)), "keys and indices separated"
    if not np.isnan(x).any():
        k = kx[:n].astype(np.float64)
        assert np.all(k[:-1] <= k[1:]), "keys are not ascending"
        fin = np.isfinite(k)
        assert np.all(np.diff(np.flatnonzero(fin)) == 1) or fin.sum() == 0


def mixed_keys(rng, n):
    x = rng.uniform(-1e3, 1e3, n).astype(np.float32)
    specials = np.array([np.inf, -np.inf, FLT_MAX, -FLT_MAX, 3.0e38, 0.0, -0.0], np.float32)
    k = int(rng.integers(0, max(2, n // 4)))
    pos = rng.integers(0, n, k)
    x[pos] = rng.choice(specials, k)
    if rng.random() < 0.5:     # duplicates
        d = rng.integers(0, n, n // 3)
        x[d] = x[rng.integers(0, n, len(d))]
    return x


@pytest.mark.parametrize("n", range(1, 601))
def test_pos_sort_finite_and_special_keys(shim, n):
    rng = np.random.default_rng(n)
    for trial in range(3):
        x = mixed_keys(rng, n)
        check_sorted(x, *pos_sort(shim, x))


@pytest.mark.parametrize("n", range(1, 601))
def test_pos_sort_with_nan_keys(shim, n):
    rng = np.random.default_rng(10_000 + n)
    if n <= 40:   # one NaN at every position
        for p in range(n):
            x = rng.uniform(0, 100, n).astype(np.float32)
            x[p] = nan_with_payload(rng, 1)[0]
            check_sorted(x, *pos_sort(shim, x))
    for trial in range(2):
        x = mixed_keys(rng, n)
        k = int(rng.integers(1, max(2, n // 8) + 1))
        x[rng.integers(0, n, k)] = nan_with_payload(rng, k)
        check_sorted(x, *pos_sort(shim, x))


@pytest.mark.parametrize("n", [4095, 4096])
def test_pos_sort_full_scene(shim, n):
    rng = np.random.default_rng(n)
    x = mixed_keys(rng, n)
    check_sorted(x, *pos_sort(shim, x))
    x[rng.integers(0, n, 9)] = nan_with_payload(rng, 9)
    check_sorted(x, *pos_sort(shim, x))
    x[:] = np.float32(3.0e38)    # every track claimed by the visual pass
    check_sorted(x, *pos_sort(shim, x))


def test_pos_sort_cases_that_broke_the_float_compare(shim):
    """A float compare (a > b) == up moves padding into [0, N) (and tracks out of it) once a key is NaN or +inf."""
    for x in ([10, 20, np.nan], [78, 10, 86, 55, 43, np.nan, 54], [10, np.inf, 20]):
        x = np.array(x, np.float32)
        check_sorted(x, *pos_sort(shim, x))


# ------------------------------------------------------------------------------------ oracle vs exact arithmetic
def exact_clip_area(subj, clip):
    """Exact area of the intersection of two convex quadrilaterals (f64 vertices taken as exact rationals), by
    half-plane clipping in rational arithmetic."""
    P = [(Fraction(float(subj[2 * i])), Fraction(float(subj[2 * i + 1]))) for i in range(4)]
    Q = [(Fraction(float(clip[2 * i])), Fraction(float(clip[2 * i + 1]))) for i in range(4)]

    def signed(poly):
        return sum(a[0] * b[1] - a[1] * b[0] for a, b in zip(poly, poly[1:] + poly[:1])) / 2

    orient = 1 if signed(Q) > 0 else -1
    if signed(Q) == 0 or signed(P) == 0:
        return Fraction(0)
    poly = P
    for a, b in zip(Q, Q[1:] + Q[:1]):
        if not poly:
            break

        def side(p):
            return orient * ((b[0] - a[0]) * (p[1] - a[1]) - (b[1] - a[1]) * (p[0] - a[0]))
        out = []
        for s, e in zip(poly[-1:] + poly[:-1], poly):
            ss, se = side(s), side(e)
            if se >= 0:
                if ss < 0:
                    t = ss / (ss - se)
                    out.append((s[0] + t * (e[0] - s[0]), s[1] + t * (e[1] - s[1])))
                out.append(e)
            elif ss >= 0:
                t = ss / (ss - se)
                out.append((s[0] + t * (e[0] - s[0]), s[1] + t * (e[1] - s[1])))
        poly = out
    if len(poly) < 3:
        return Fraction(0)
    return abs(signed(poly))


def pair_cases(rng, scale):
    """(kind, box_l, box_r) at coordinates ~scale: random, near-duplicate, nested, touching and rotated pairs."""
    out = []
    for kind in ("random", "near_dup", "nested", "rotated", "touching"):
        for _ in range(12):
            c = rng.uniform(-scale, scale, 2)
            h = rng.uniform(5, 200)
            a = rng.uniform(0.3, 1.5)
            ang = rng.uniform(-1.5, 1.5) if kind != "touching" else np.nan
            l = np.array([c[0], c[1], ang, a, h, 1], np.float32)
            r = l.copy()
            if kind == "random":
                r[:2] += rng.normal(0, h / 3, 2).astype(np.float32)
                r[2] = rng.uniform(-1.5, 1.5)
                r[3:5] *= rng.uniform(0.6, 1.4, 2).astype(np.float32)
            elif kind == "near_dup":
                r[:2] += rng.normal(0, 1e-3 * h, 2).astype(np.float32)
                r[2] += np.float32(rng.choice([-1e-4, 1e-4]))
            elif kind == "nested":
                r[4] *= np.float32(0.5)
                r[:2] += rng.normal(0, h / 20, 2).astype(np.float32)
            elif kind == "rotated":
                r[2] = np.float32(l[2] + rng.choice([np.pi / 4, np.pi / 2, np.pi / 3]))
            else:   # shares an edge with l (axis aligned): x shifted by exactly its width in f64
                r[0] = np.float32(float(l[0]) + float(l[3]) * float(l[4]))
            out.append((kind, l, r))
    return out


@pytest.mark.parametrize("scale", [1.0, 1e2, 1e4, 1e6])
def test_oracle_and_product_clip_area_against_exact(oracle, shim, scale):
    """The oracle and the product clip bit for bit, and |f64 clip - exact| <= 8 * 2^-52 * (S^2 + S * L * kappa).
    S is the largest coordinate magnitude of the pair (the intersection points are formed from products of absolute
    coordinates), L the largest box side.  kappa = 1 / |sin 2(a_l - a_r)| is the conditioning of an intersection of two
    nearly parallel edges: 0 for exactly parallel edges (never intersected), at most 5e3 here (the near-duplicates are
    turned by exactly 1e-4) and capped at 1e4.  At S ~ 1e4 and L ~ 100 that is ~1e-10 relative to the box area.  Degenerate
    pairs where Sutherland-Hodgman legitimately returns a rounding sliver instead of 0 -- boxes that share an edge, or
    whose exact intersection is a segment or a point -- are held to the same absolute bound."""
    rng = np.random.default_rng(int(scale))
    eps = 2.0 ** -52
    for kind, l, r in pair_cases(rng, scale):
        vl = np.ascontiguousarray(oracle.vertices(l), np.float64).ravel()
        vr = np.ascontiguousarray(oracle.vertices(r), np.float64).ravel()
        exact = exact_clip_area(vl, vr)
        a_orc = oracle.polygon_area(oracle.sh_clip(oracle.vertices(l), oracle.vertices(r)))
        a_prod = shim.shim_clip_area(vl.ctypes.data_as(C.POINTER(C.c_double)), vr.ctypes.data_as(C.POINTER(C.c_double)))
        assert a_orc == a_prod, (kind, a_orc, a_prod)
        S = max(np.abs(vl).max(), np.abs(vr).max(), 1.0)
        L = float(max(l[4], r[4], l[3] * l[4], r[3] * r[4]))
        d = (0.0 if np.isnan(l[2]) else float(l[2])) - (0.0 if np.isnan(r[2]) else float(r[2]))
        s2 = abs(np.sin(2 * d))
        kappa = 0.0 if s2 < 1e-12 else min(1.0 / s2, 1e4)
        bound = 8 * eps * (S * S + S * L * kappa)
        err = abs(Fraction(a_orc) - exact)
        assert err <= Fraction(bound), (kind, float(exact), a_orc, float(err) / bound)
        if kind in ("nested", "near_dup"):
            assert exact > 0


def mahalanobis_f64(st110, box, pw):
    """The reference's Mahalanobis distance evaluated in f64: r^T S^-1 r, S = H P H^T + diag(std_position(1, 0.1)^2)."""
    st = np.asarray(st110, np.float64)
    mean, cov = st[:10], st[10:].reshape(10, 10)
    h = mean[4]
    w = float(np.float32(pw)) * h
    std = np.array([w, w, w, 0.1, w])
    S = cov[:5, :5] + np.diag(std * std)
    ang = 0.0 if np.isnan(box[2]) else float(box[2])
    r = np.array([box[0], box[1], ang, box[3], box[4]], np.float64) - mean[:5]
    return float(r @ np.linalg.solve(S, r))


@pytest.mark.parametrize("oriented", [False, True])
def test_oracle_mahalanobis_against_f64(oracle, oriented):
    """The oracle's f32 distance agrees with the f64 evaluation to 2e-5 relative (plus 1e-6 absolute for distances
    near 0): the projected covariance is diagonal, so the f32 error is a few roundings per term, each 2^-24."""
    rng = np.random.default_rng(3 + oriented)
    pw, vw = 1 / 20, 1 / 160
    for trial in range(400):
        scale = [1.0, 1e2, 1e4, 1e5][trial % 4]
        b = np.array([rng.uniform(-scale, scale), rng.uniform(-scale, scale),
                      rng.uniform(-1.5, 1.5) if oriented else np.nan, rng.uniform(0.3, 1.2), rng.uniform(5, 300), 1],
                     np.float32)
        st = oracle.kalman_initiate(b, pw, vw)
        for _ in range(int(rng.integers(0, 4))):
            st = oracle.kalman_predict(st, pw, vw)
            z = b.copy()
            z[:2] += rng.normal(0, 2, 2).astype(np.float32)
            st = oracle.kalman_update(st, z, pw, vw)
        st = oracle.kalman_predict(st, pw, vw)
        z = b.copy()
        z[:2] += rng.normal(0, float(b[4]) / 10, 2).astype(np.float32)
        z[3:5] *= rng.uniform(0.9, 1.1, 2).astype(np.float32)
        if oriented:
            z[2] += np.float32(rng.normal(0, 0.05))
        d32 = oracle.kalman_distance(st, z, pw, vw)
        d64 = mahalanobis_f64(st, z, pw)
        err = abs(d32 - d64)
        assert err <= 2e-5 * d64 + 1e-6, (trial, d32, d64)


def test_product_mahalanobis_matches_oracle_when_residuals_overflow(oracle, shim):
    """Finite boxes whose whitened residual overflows f32: the reference's forward substitution makes the distance NaN
    (None) when the overflow is in x, y, angle or aspect, and +inf (cost 0) when it is in the height alone.  The
    product's diagonal form (sb_math.cuh maha_distance) must give the same, bit for bit."""
    pw = np.float32(1 / 20)
    tracks = [np.array([100, 100, np.nan, 0.5, 40, 1], np.float32), np.array([100, 100, 0.3, 3e38, 1e20, 1], np.float32),
              np.array([-5e37, 2e37, np.nan, 1.0, 1e3, 1], np.float32)]
    cands = [[100, 100, np.nan, 0.5, 40, 1], [3e38, 100, np.nan, 0.5, 40, 1], [100, -3e38, np.nan, 0.5, 40, 1],
             [100, 100, 3e38, 0.5, 40, 1], [100, 100, np.nan, 3e38, 40, 1], [100, 100, np.nan, 0.5, 3e38, 1],
             [100, 100, np.nan, 3e38, 1e20, 1], [3e38, 3e38, np.nan, 3e38, 3e38, 1], [2e37, 1e37, np.nan, 1.0, 1e3, 1]]
    n_nan = n_inf = 0
    for t in tracks:
        st = oracle.kalman_predict(oracle.kalman_initiate(t))
        mean, cov = st[:10], st[10:].reshape(10, 10)
        st30 = np.zeros(30, np.float32)
        st30[:10] = mean
        for i in range(5):
            st30[10 + 4 * i: 14 + 4 * i] = [cov[i, i], cov[i, i + 5], cov[i + 5, i], cov[i + 5, i + 5]]
        for c in cands:
            c = np.array(c, np.float32)
            ref = np.float32(oracle.kalman_distance(st, c))
            got = np.float32(shim.shim_maha(pw, st30.ctypes.data_as(C.POINTER(C.c_float)),
                                             c.ctypes.data_as(C.POINTER(C.c_float))))
            assert (np.isnan(ref) and np.isnan(got)) or ref == got, (t, c, ref, got)
            n_nan += bool(np.isnan(ref))
            n_inf += bool(np.isinf(ref))
    assert n_nan >= 6 and n_inf >= 1
