"""sb_sincos.cuh -- the product's f64 sin / cos, one instruction sequence for host and device -- checked on the arguments a
box angle can take (f32 values widened to f64, src/utils/bbox.rs:287-330):

* it is CORRECTLY ROUNDED: every result equals mpmath's 200-bit value rounded to nearest (sampled), so the vertices of an
  oriented box are a pure function of the box on every platform and on the GPU;
* against this platform's C library (what the Rust reference calls here): identical bits for > 99 % of the angles; where
  they differ it is by one ulp and it is the C library that is not correctly rounded (glibc documents < 0.55 ulp).
  (CUDA's own sin / cos, used in round 1, are 1-2 ulp functions.)
* beyond the Cody-Waite domain (|x| >= 2e5) the Payne-Hanek path is checked against mpmath directly: correctly rounded on
  random f32 and f64 arguments, dense slabs and the f32 angles closest to multiples of pi/2 in every binade.
* inf and NaN give the quiet NaN 0x7ff8000000000000."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def shim():
    d = os.path.join(HERE, "host_shim")
    so = os.path.join(d, "libshim_sc.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-shared", "-x", "c++",
                           os.path.join(d, "shim.cpp"), "-o", so])
    L = C.CDLL(so)
    for fn in (L.shim_sincos, L.shim_libm_sincos):
        fn.restype = None
        fn.argtypes = [C.POINTER(C.c_float), C.c_longlong, C.POINTER(C.c_double), C.POINTER(C.c_double)]
    L.shim_sincos_f64.restype = None
    L.shim_sincos_f64.argtypes = [C.POINTER(C.c_double), C.c_longlong, C.POINTER(C.c_double), C.POINTER(C.c_double)]
    return L


def both(L, a):
    a = np.ascontiguousarray(a, dtype=np.float32)
    out = [np.empty(len(a), np.float64) for _ in range(4)]
    p = lambda x: x.ctypes.data_as(C.POINTER(C.c_double))  # noqa: E731
    L.shim_sincos(a.ctypes.data_as(C.POINTER(C.c_float)), len(a), p(out[0]), p(out[1]))
    L.shim_libm_sincos(a.ctypes.data_as(C.POINTER(C.c_float)), len(a), p(out[2]), p(out[3]))
    return a, out


def check(L, angles, max_rate, n_verify=120):
    import mpmath as mp

    mp.mp.prec = 200
    a, (s, c, ls, lc) = both(L, angles)
    diff = (s.view(np.int64) != ls.view(np.int64)) | (c.view(np.int64) != lc.view(np.int64))
    rate = float(diff.mean()) if len(a) else 0.0
    assert rate <= max_rate, rate
    # differences from the C library are one ulp wide
    for ours, lib in ((s, ls), (c, lc)):
        d = np.abs(ours.view(np.int64) - lib.view(np.int64))
        assert d.max() <= 1
    # ours is the correctly rounded one: where the two differ (all of those, up to n_verify) and on a random sample
    idx = np.flatnonzero(diff)[:n_verify]
    rng = np.random.default_rng(1)
    idx = np.concatenate([idx, rng.integers(0, len(a), min(n_verify, len(a)))])
    for i in idx:
        x = mp.mpf(float(a[i]))
        assert float(mp.sin(x)) == s[i] and float(mp.cos(x)) == c[i], (float(a[i]), s[i], ls[i], c[i], lc[i])
    return rate


def test_ten_million_random_angles(shim):
    rng = np.random.default_rng(2024)
    worst = 0.0
    for lo, hi, n in ((-np.pi, np.pi, 6_000_000), (-1.6, 1.6, 2_000_000), (-100.0, 100.0, 1_500_000),
                      (-1e-3, 1e-3, 500_000)):
        worst = max(worst, check(shim, rng.uniform(lo, hi, n), 0.01))
    assert worst < 0.01


def test_neighbourhoods_of_multiples_of_half_pi_and_special_values(shim):
    """Arguments next to k * pi/2 (massive cancellation in the reduction), tiny, subnormal, zero, large."""
    vals = []
    for k in range(-2000, 2001):
        c = np.float32(k * np.pi / 2)
        x = c
        for _ in range(6):
            vals.append(x)
            x = np.nextafter(x, np.float32(np.inf), dtype=np.float32)
        x = c
        for _ in range(6):
            x = np.nextafter(x, np.float32(-np.inf), dtype=np.float32)
            vals.append(x)
    vals += [0.0, -0.0, 1e-45, -1e-45, 1e-30, 1.17549435e-38, 0.5, 1.0, 2.0, 3.0, 1e3, 12345.678, 1e5, 1.9e5]
    check(shim, np.array(vals, np.float32), 0.02, n_verify=400)


def near_half_pi_multiples_f32(lo_exp=17, hi_exp=127, spread=2):
    """The f32 values of binades 2^lo_exp .. 2^hi_exp closest to multiples of pi/2, where the large-argument reduction
    cancels most: in the binade [2^e, 2^(e+1)), x = m 2^(e-23) and x 2/pi = m a with a = 2^(e-23) 2/pi; the m in
    [2^23, 2^24) with m a nearest an integer are the continued-fraction denominators of a and their multiples.  Returns
    those m (and +-spread ulps around each), both signs, as f32."""
    import mpmath as mp

    out = []
    with mp.workprec(400):
        for e in range(lo_exp, hi_exp + 1):
            a = mp.mpf(2) ** (e - 23) * 2 / mp.pi
            a -= mp.floor(a)
            q_prev, q = 0, 1
            t = a
            while q < (1 << 24) and t != 0:
                t = 1 / t
                k = int(mp.floor(t))
                t -= k
                q_prev, q = q, k * q + q_prev
                for qq in (q, q + q_prev, q - q_prev):
                    if 0 < qq < (1 << 24):
                        m = qq * -(-(1 << 23) // qq)
                        if m < (1 << 24):
                            out += [(m + d) * 2.0 ** (e - 23) for d in range(-spread, spread + 1) if (1 << 23) <= m + d < (1 << 24)]
    v = np.unique(np.array(out, np.float32))
    return np.r_[v, -v]


def check_mpmath(s, c, a):
    """s, c == sin, cos of the f64 arguments a, correctly rounded (mpmath, 200 bits)."""
    import mpmath as mp

    mp.mp.prec = 200
    for x, si, ci in zip(a.tolist(), s.tolist(), c.tolist()):
        xm = mp.mpf(x)
        assert float(mp.sin(xm)) == si and float(mp.cos(xm)) == ci, (x, si, float(mp.sin(xm)), ci, float(mp.cos(xm)))


def test_large_angles_correctly_rounded(shim):
    """|x| >= 2e5, where the reduction is Payne-Hanek's: every result equals mpmath's, on a random sample of all such f32,
    the f32 angles closest to multiples of pi/2 in every binade, dense slabs at 2e5, 2^24, 1e10 and FLT_MAX, and random
    doubles up to DBL_MAX (the header's domain is every finite double)."""
    rng = np.random.default_rng(5)
    lo = np.float32(2e5).view(np.uint32)
    big = rng.integers(lo, np.float32(np.finfo(np.float32).max).view(np.uint32), 6000, endpoint=True).astype(np.uint32)
    slabs = [np.arange(s0, s0 + 1500, dtype=np.uint32) for s0 in
             (lo, np.float32(2.0**24).view(np.uint32), np.float32(1e10).view(np.uint32),
              np.float32(np.finfo(np.float32).max).view(np.uint32) - 1499)]
    a = np.concatenate([big] + slabs).view(np.float32)
    a = np.r_[a, -a[::7], near_half_pi_multiples_f32()]
    a, (s, c, _, _) = both(shim, a)
    check_mpmath(s, c, a.astype(np.float64))
    # f64 arguments (not reachable from a box angle, but in the function's domain): through shim_sincos_f64
    d = np.r_[rng.uniform(2e5, 1e6, 300), 10.0 ** rng.uniform(6, 308, 600), [1e22, 1.7976931348623157e308]]
    d = np.r_[d, -d[::5]]
    s, c = np.empty_like(d), np.empty_like(d)
    shim.shim_sincos_f64(d.ctypes.data_as(C.POINTER(C.c_double)), len(d), s.ctypes.data_as(C.POINTER(C.c_double)),
                         c.ctypes.data_as(C.POINTER(C.c_double)))
    check_mpmath(s, c, d)


def test_inf_and_nan_give_one_quiet_nan(shim):
    a = np.array([np.inf, -np.inf, np.nan, -np.nan], np.float32)
    a = np.r_[a, np.array([0x7f800001, 0xffc01234, 0x7fffffff], np.uint32).view(np.float32)]
    _, (s, c, _, _) = both(shim, a)
    assert (s.view(np.uint64) == 0x7ff8000000000000).all() and (c.view(np.uint64) == 0x7ff8000000000000).all()


def test_every_f32_in_a_dense_slab_around_typical_angles(shim):
    """All ~4 million consecutive f32 values of [0.5, 0.75): no gaps for a sampled test to miss."""
    lo = np.float32(0.5).view(np.uint32)
    bits = np.arange(lo, lo + (1 << 22), dtype=np.uint32)
    check(shim, bits.view(np.float32), 0.01)
