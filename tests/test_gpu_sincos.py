"""The device build of the product's sin / cos (sb::sc::sincos_cr, sb_sincos.cuh) and of everything oriented built on it,
bit for bit against the host build of the same headers and against mpmath.

Every oriented box the GPU handles goes through sincos_cr (box_vertices, sb_math.cuh): the IoU cost, NMS, own-area
shares and the box_vertices / clip_polygons / intersection_areas operators.  The header promises correctly rounded
results, the same bits on the host and on the device; the tests against the C library's oracle (test_gpu_parity,
test_gpu_geometry_kalman) only allow a tolerance, so a device build one ulp off would pass them.  Here:
  * the device and the host agree on sin and cos of every f32 angle (tests/gpu_probe/sincos_probe.cu, 2^32 patterns);
  * the device is correctly rounded (mpmath, 200 bits) on the hard cases: next to k pi/2, zero, subnormals, the ends of
    the Cody-Waite domain, huge angles up to FLT_MAX, and inf / NaN;
  * device box vertices, clipped polygons, intersection areas and the oriented IoU cost matrix equal the host build of
    sb_math.cuh (tests/host_shim) on vertices the host computed, bit for bit;
  * for nearly parallel edges, the clipped area is within a stated bound of the exact rational intersection area."""
import ctypes as C
import os
import subprocess
from fractions import Fraction

import numpy as np
import pytest

from own_area_exact import own_area_rational
from test_geometry_kalman_cpu import build_geom_shim
from test_sincos_cpu import near_half_pi_multiples_f32

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "similari_b200", "csrc")
F32 = np.float32
QNAN = 0x7ff8000000000000


@pytest.fixture(scope="module")
def eng():
    import similari_b200.engine as e
    from similari_b200._lib import lib

    if lib().sb200_device_count() <= 0:
        pytest.fail("no CUDA device: the product has no CPU path")
    return e


@pytest.fixture(scope="module")
def probe(tmp_path_factory):
    from similari_b200._build import NVCC_FLAGS, nvcc

    exe = str(tmp_path_factory.mktemp("sincos_probe") / "sincos_probe")
    subprocess.check_call([nvcc(), *NVCC_FLAGS, "-Xcompiler", "-ffp-contract=off", "-Xcompiler", "-pthread", "-I", CSRC,
                           os.path.join(HERE, "gpu_probe", "sincos_probe.cu"), "-o", exe],
                          stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    return exe


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    """tests/host_shim/shim.cpp (flags as test_product_math_cpu): host sin / cos, vertices and IoU."""
    so = str(tmp_path_factory.mktemp("sincos_shim") / "libshim.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-shared", "-x", "c++",
                           os.path.join(HERE, "host_shim", "shim.cpp"), "-o", so])
    L = C.CDLL(so)
    f32p, f64p = C.POINTER(C.c_float), C.POINTER(C.c_double)
    L.shim_sincos.restype = None
    L.shim_sincos.argtypes = [f32p, C.c_longlong, f64p, f64p]
    L.shim_vertices.argtypes = [f32p, f64p]
    L.shim_iou.argtypes = [f32p, f32p]
    L.shim_iou.restype = C.c_float
    return L


@pytest.fixture(scope="module")
def geom(tmp_path_factory):
    return build_geom_shim(tmp_path_factory.mktemp("geomshim_sincos"))


def fp(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def host_sincos(L, a):
    a = np.ascontiguousarray(a, F32)
    s, c = np.empty(len(a)), np.empty(len(a))
    L.shim_sincos(fp(a), len(a), dp(s), dp(c))
    return s, c


def device_sincos(probe, a):
    a = np.ascontiguousarray(a, F32)
    out = subprocess.run([probe, "args"], input=np.int64(len(a)).tobytes() + a.tobytes(), capture_output=True, check=True)
    r = np.frombuffer(out.stdout, np.float64)
    assert len(r) == 2 * len(a)
    return r[:len(a)], r[len(a):]


def host_vertices(L, boxes):
    out = np.empty((len(boxes), 8))
    for i, b in enumerate(np.ascontiguousarray(boxes, F32)):
        L.shim_vertices(fp(b), dp(out[i]))
    return out


def device_vertices(probe, boxes):
    b = np.ascontiguousarray(np.asarray(boxes, F32)[:, :5])
    out = subprocess.run([probe, "vertices"], input=np.int64(len(b)).tobytes() + b.tobytes(), capture_output=True,
                         check=True)
    return np.frombuffer(out.stdout, np.float64).reshape(len(b), 8)


def bits(x):
    return np.ascontiguousarray(x, np.float64).view(np.uint64)


# ------------------------------------------------------------------------------------------------ device vs host
@pytest.fixture(scope="module")
def sweep(probe):
    """The probe's sweep over every f32 bit pattern: count, mismatches (and the first 64 of them), threads, seconds."""
    out = subprocess.run([probe, "sweep", "0", str(1 << 32), "1"], capture_output=True, text=True,
                         check=True).stdout
    res = {"mismatch": []}
    for line in out.splitlines():
        k, v = line.split()
        if k == "mismatch":
            res[k].append(int(v, 16))
        else:
            res[k] = float(v) if k == "seconds" else int(v)
    return res


def test_device_matches_host_for_every_f32(sweep):
    """sin and cos of all 2^32 f32 bit patterns (finite, inf and NaN) widened to f64: the device build of sincos_cr
    against the host build, bit for bit.  The host's share dominates (about 200 ns per argument and thread): the whole
    sweep took 107 s on an H100 machine's 8 threads, so every pattern is swept rather than a strided sample."""
    print(f"\nsincos sweep: {sweep['count']} f32 patterns, {sweep['mismatches']} device / host mismatches, "
          f"{sweep['seconds']:.1f} s on {sweep['threads']} threads")
    assert sweep["count"] == 1 << 32
    assert sweep["mismatches"] == 0, [hex(b) for b in sweep["mismatch"]]


def hard_angles():
    """The arguments where sin / cos implementations go wrong, as f32."""
    vals = []
    for k in range(-2000, 2001):              # +-6 ulps around k pi/2: the reduction cancels most
        c = F32(k * np.pi / 2)
        vals.append(c)
        x = c
        for _ in range(6):
            x = np.nextafter(x, F32(np.inf), dtype=F32)
            vals.append(x)
        x = c
        for _ in range(6):
            x = np.nextafter(x, F32(-np.inf), dtype=F32)
            vals.append(x)
    u = np.uint32
    sub = np.r_[np.arange(0, 300, dtype=u), np.arange(0x007fff00, 0x00800100, dtype=u),
                np.random.default_rng(3).integers(0, 0x00800000, 2000).astype(u)]           # +0, subnormals, FLT_MIN
    edge = np.arange(F32(2e5).view(u) - 64, F32(2e5).view(u) + 64, dtype=u)                  # the 2e5 switch
    top = np.arange(0x7f7fffff - 500, 0x7f800000, dtype=u)                                   # up to FLT_MAX
    rnd = np.random.default_rng(4).integers(0, 0x7f800000, 20_000).astype(u)                 # every binade
    a = np.r_[np.array(vals, F32), sub.view(F32), edge.view(F32), top.view(F32), rnd.view(F32)]
    return np.r_[a, -a[len(vals):], near_half_pi_multiples_f32()]


def test_device_correctly_rounded(probe, shim, sweep):
    """The device's sin / cos equal mpmath's 200-bit values rounded to nearest: on the device / host mismatches the sweep
    reports (its first 64), the hard cases and a random sample (hard_angles); inf and NaN give the host's quiet NaN."""
    import mpmath as mp

    mp.mp.prec = 200
    a = np.r_[hard_angles(), np.array(sweep["mismatch"], np.uint32).view(F32)]
    a = a[np.isfinite(a)]
    s, c = device_sincos(probe, a)
    hs, hc = host_sincos(shim, a)
    assert np.array_equal(bits(s), bits(hs)) and np.array_equal(bits(c), bits(hc))
    wrong = []
    for x, si, ci in zip(a.astype(np.float64).tolist(), s.tolist(), c.tolist()):
        xm = mp.mpf(x)
        if float(mp.sin(xm)) != si or float(mp.cos(xm)) != ci:
            wrong.append(x)
    assert not wrong, (len(wrong), wrong[:10])
    special = np.r_[np.array([np.inf, -np.inf, np.nan], F32), np.array([0x7f800001, 0xffc01234, 0x7fffffff], np.uint32).view(F32)]
    s, c = device_sincos(probe, special)
    assert (bits(s) == QNAN).all() and (bits(c) == QNAN).all()


# --------------------------------------------------------------------------------------------------- oriented boxes
def oriented_boxes(r, n, centre=400.0):
    """n boxes in the angle families that matter: typical angles, one or two ulps from k pi/2 (nearly axis-aligned
    edges), centres up to `centre`, and huge angles (Payne-Hanek reduction)."""
    b = np.zeros((n, 6), F32)
    b[:, 0] = r.uniform(-centre, centre, n)
    b[:, 1] = r.uniform(-centre, centre, n)
    fam = np.arange(n) % 4
    ang = r.uniform(-np.pi, np.pi, n).astype(F32)
    k = F32(r.integers(-8, 9, n) * np.pi / 2)
    step = r.integers(-2, 3, n)
    near = k.copy()
    for i in range(n):
        for _ in range(abs(step[i])):
            near[i] = np.nextafter(near[i], F32(np.inf) if step[i] > 0 else F32(-np.inf), dtype=F32)
    huge = (10.0 ** r.uniform(5.4, 38.5, n)).astype(F32) * np.where(r.random(n) < 0.5, F32(-1), F32(1))
    hard = near_half_pi_multiples_f32()
    b[:, 2] = np.select([fam == 0, fam == 1, fam == 2], [ang, near, huge], hard[r.integers(0, len(hard), n)])
    b[:, 3] = r.uniform(0.3, 0.8, n)
    b[:, 4] = r.uniform(40, 160, n)
    b[:, 5] = 1.0
    return b


@pytest.mark.parametrize("centre", [400.0, 1e4, 1e6])
def test_box_vertices_device_vs_host(eng, probe, shim, centre):
    """sb::box_vertices on the device (in the probe and in the product's own box_vertices operator) against its host
    build, bit for bit, in every angle family and at centres up to 1e6."""
    r = np.random.default_rng(int(centre))
    b = oriented_boxes(r, 4000, centre)
    b[:200, 2] = np.nan                                       # axis-aligned rows too
    want = host_vertices(shim, b)
    assert np.array_equal(bits(device_vertices(probe, b)), bits(want))
    assert np.array_equal(bits(eng.box_vertices(b).reshape(-1, 8)), bits(want))


def near_parallel_pairs(r, n, centre):
    """(subject, clipping) rows whose edges are nearly parallel: the clipping box is the subject turned by 0 to 2 ulps of
    its angle (or by a multiple of pi/2 and an ulp), shifted by up to a third of its size, rescaled a little."""
    s = oriented_boxes(r, n, centre)
    c = s.copy()
    for i in range(n):
        a = c[i, 2]
        if i % 3 == 0:
            a = F32(a + F32(r.integers(-2, 3) * np.pi / 2))
        for _ in range(r.integers(0, 3)):
            a = np.nextafter(a, F32(np.inf) if r.random() < 0.5 else F32(-np.inf), dtype=F32)
        c[i, 2] = a
    c[:, :2] += (r.uniform(-0.33, 0.33, (n, 2)) * s[:, 4:5]).astype(F32)
    c[:, 3:5] *= r.uniform(0.8, 1.25, (n, 2)).astype(F32)
    return s, c


def mixed_pairs(r, n, centre):
    s = oriented_boxes(r, n, centre)
    c = s.copy()
    c[:, :2] += r.normal(0, 40, (n, 2)).astype(F32)
    c[:, 3:5] *= r.uniform(0.6, 1.4, (n, 2)).astype(F32)
    c[::2, 2] = oriented_boxes(r, n, centre)[::2, 2]
    return s, c


@pytest.mark.parametrize("centre", [400.0, 1e5])
def test_clip_polygons_on_host_vertices(eng, shim, geom, centre):
    """engine.clip_polygons of oriented boxes against sb_math's clip_poly run on the host on host-built vertices: ring,
    vertex count and area bit for bit (the existing parity test clips the GPU's own vertices)."""
    r = np.random.default_rng(40 + int(centre))
    s1, c1 = near_parallel_pairs(r, 1500, centre)
    s2, c2 = mixed_pairs(r, 1500, centre)
    s, c = np.r_[s1, s2], np.r_[c1, c2]
    v, cnt, area = eng.clip_polygons(s, c)
    vs, vc = host_vertices(shim, s), host_vertices(shim, c)
    nonempty = 0
    for i in range(len(s)):
        ring = np.zeros(32)
        n = C.c_int(0)
        a = geom.gshim_clip_ring(dp(vs[i]), dp(vc[i]), dp(ring), C.byref(n))
        assert cnt[i] == n.value, i
        k = max(n.value, 0)
        assert np.array_equal(bits(v[i, :k].ravel()), bits(ring[:2 * k])), i
        assert bits(np.array([area[i]]))[0] == bits(np.array([a]))[0], (i, area[i], a)
        nonempty += n.value >= 3
    assert nonempty > len(s) // 2


def test_intersection_areas_on_host_vertices(eng, shim, geom):
    """engine.intersection_areas of oriented boxes (every angle family, near-parallel rows) against the host clip on
    host-built vertices, bit for bit."""
    r = np.random.default_rng(50)
    s, c = near_parallel_pairs(r, 150, 300.0)
    a = np.r_[s, oriented_boxes(r, 150, 300.0)]
    b = np.r_[c, oriented_boxes(r, 150, 300.0)]
    got = eng.intersection_areas(a, b)
    va, vb = host_vertices(shim, a), host_vertices(shim, b)
    want = np.array([[geom.gshim_clip_area(dp(va[i]), dp(vb[j])) for j in range(len(b))] for i in range(len(a))])
    assert np.array_equal(bits(got.ravel()), bits(want.ravel()))
    assert (got > 0).sum() > len(a)


@pytest.mark.parametrize("thr", [0.05, 0.3])
def test_oriented_iou_cost_matrix_vs_host(eng, shim, thr):
    """sort_cost_matrix(POS_IOU) of oriented boxes against shim_iou (sb_math's IoU built on the host): the same None
    pattern and the same f32 values (candidate confidence 1, so the cost is the IoU itself)."""
    r = np.random.default_rng(60 + int(thr * 100))
    tb = oriented_boxes(r, 240, 300.0)
    cb = np.r_[near_parallel_pairs(r, 120, 300.0)[1], oriented_boxes(r, 80, 300.0)]
    cb[120:, :2] = tb[r.integers(0, 240, 80), :2] + r.normal(0, 10, (80, 2)).astype(F32)
    cb[:, 5] = 1.0
    got = eng.sort_cost_matrix(eng._lib.POS_IOU, cb, tb, iou_threshold=thr)
    want = np.full(got.shape, np.nan, F32)
    for i in range(len(cb)):
        for j in range(len(tb)):
            v = shim.shim_iou(fp(cb[i]), fp(tb[j]))
            if not np.isnan(v) and v >= F32(thr):
                want[i, j] = v
    assert np.array_equal(np.isnan(got), np.isnan(want))
    assert np.array_equal(got[~np.isnan(got)], want[~np.isnan(want)])
    assert (~np.isnan(got)).sum() > 100


def shoelace_exact(v):
    q = [(Fraction(float(v[2 * k])), Fraction(float(v[2 * k + 1]))) for k in range(4)]
    return abs(sum(q[k][0] * q[(k + 1) % 4][1] - q[(k + 1) % 4][0] * q[k][1] for k in range(4))) / 2


def test_near_parallel_clip_area_vs_exact(eng, shim):
    """For nearly parallel edges (Sutherland-Hodgman's fragile case) the clipped area of the GPU is within
    CLIP_AREA_BOUND of the exact area of the intersection of the two f64 quadrilaterals, area(A) - own_area_rational(A,
    [B]).  The bound is 2^-40 of the sum of the magnitudes of the shoelace terms of the clipped ring (|x_k y_k+1| +
    |x_k+1 y_k| after the shift by its first vertex), i.e. of the scale of the cancelling sum, generous for rings of at
    most 8 vertices whose intersection points may move along an edge by u R / (angle between the edges)."""
    r = np.random.default_rng(70)
    s, c = near_parallel_pairs(r, 400, 400.0)
    v, cnt, area = eng.clip_polygons(s, c)
    vs, vc = host_vertices(shim, s), host_vertices(shim, c)
    checked = 0
    for i in range(len(s)):
        k = cnt[i]
        if k < 3:
            continue
        ring = v[i, :k] - v[i, 0]
        terms = np.abs(ring[:, 0] * np.roll(ring[:, 1], -1)) + np.abs(np.roll(ring[:, 0], -1) * ring[:, 1])
        bound = 2.0 ** -40 * float(terms.sum())
        exact = shoelace_exact(vs[i]) - own_area_rational(vs[i].reshape(4, 2), [vc[i].reshape(4, 2)])
        assert abs(Fraction(float(area[i])) - exact) <= Fraction(bound), (i, float(area[i]), float(exact), bound)
        checked += 1
    assert checked > 300
