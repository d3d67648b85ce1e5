// sb_sincos.cuh -- correctly rounded f64 sine / cosine, the same instruction sequence on the host and on the device.
//
// Why: the reference turns a box into its four vertices with f64 `cos` / `sin` of the f32 angle (src/utils/bbox.rs:287-330),
// i.e. with the C library's functions, which are correctly rounded for practically every argument.  CUDA's `sin` / `cos` are
// within 1-2 ulp but not correctly rounded, so a vertex could differ from the reference's in the last bit, the clipped area
// with it, and a 1-ulp IoU difference can flip `(v * 1e6) as i64` and with it a near-tie of the assignment.  Bit-exact
// oriented IoU needs bit-exact vertices; this header provides them by construction instead of by tolerance:
//   * |x| < 2e5: Cody-Waite reduction by pi/2 held as three doubles (exact products through fma), valid for
//     |x| < 2^17 * pi/2;
//   * larger finite x: Payne-Hanek reduction with 320 bits of 2/pi in integer arithmetic (reduce_large), exact to
//     2^-200 of the quadrant for every finite double;
//   * table lookup at c = i/64 (sin c, cos c as double-doubles, generated with mpmath: sb_sincos_table.inc);
//   * Taylor series of sin t, cos t for |t| <= 1/128 in double-double arithmetic (error < 2^-95);
//   * angle addition in double-double, one final rounding.
// The result is the correctly rounded value unless the exact one lies within ~2^-42 ulp of a rounding boundary -- for the
// 2^32 possible f32 angles that does not happen in practice (tests/test_sincos_cpu.py compares them with mpmath and the C
// library; tests/test_gpu_sincos.py compares every f32 on the device with this header's host build, bit for bit).
// inf and NaN give the quiet NaN 0x7ff8000000000000 for both results.
#pragma once
#include <math.h>
#include <string.h>

#ifndef SB_HD
#ifdef __CUDACC__
#define SB_HD __host__ __device__ __forceinline__
#else
#define SB_HD inline
#endif
#endif

namespace sb {
namespace sc {

struct dd { double h, l; };

SB_HD dd two_sum(double a, double b) {
  const double s = a + b;
  const double bb = s - a;
  return dd{s, (a - (s - bb)) + (b - bb)};
}
SB_HD dd fast_two_sum(double a, double b) {   // |a| >= |b|
  const double s = a + b;
  return dd{s, b - (s - a)};
}
SB_HD dd two_prod(double a, double b) {
  const double p = a * b;
  return dd{p, fma(a, b, -p)};
}
SB_HD dd dd_add(dd a, dd b) {
  dd s = two_sum(a.h, b.h);
  const dd t = two_sum(a.l, b.l);
  s.l += t.h;
  s = fast_two_sum(s.h, s.l);
  s.l += t.l;
  return fast_two_sum(s.h, s.l);
}
SB_HD dd dd_mul(dd a, dd b) {
  dd p = two_prod(a.h, b.h);
  p.l += a.h * b.l;
  p.l += a.l * b.h;
  return fast_two_sum(p.h, p.l);
}
SB_HD dd dd_mul_d(dd a, double b) {
  dd p = two_prod(a.h, b);
  p.l += a.l * b;
  return fast_two_sum(p.h, p.l);
}
SB_HD dd dd_neg(dd a) { return dd{-a.h, -a.l}; }

struct reduced { double h, l; int n; };   // x = (4 m + n) * pi/2 + r, r = h + l as a double-double, |r| <= pi/4

SB_HD void mul64(unsigned long long a, unsigned long long b, unsigned long long* hi, unsigned long long* lo) {
#ifdef __CUDA_ARCH__
  *hi = __umul64hi(a, b);
#else
  *hi = (unsigned long long)(((unsigned __int128)a * b) >> 64);
#endif
  *lo = a * b;
}

// Payne-Hanek reduction of a finite |x| >= 2e5 (any finite double).  x = M 2^E with M < 2^53 an integer, and
// x * 2/pi = M * sum_j kTwoOverPiBits[j] 2^(E - 64 (j + 1)): the words j < j0 only add multiples of 4 (nothing to the
// quadrant or to r), the five words from j0 on give y = x * 2/pi mod 4 with 255 or more fraction bits, off by less than
// M 2^(E - 64 (j0 + 5)) <= 2^-202.  The reduction is integer arithmetic and its product by pi/2 the same double-double
// code as everywhere else here, so the host and the device get the same bits.  Out of line:
// angles this large are rare, and the inlined common path of the IoU, NMS and own-area kernels keeps its code.
#ifdef __CUDACC__
inline __host__ __device__ __noinline__
#else
inline
#endif
reduced reduce_large(double x) {
#define SB_SC_CONST [[maybe_unused]] static const
#include "sb_sincos_table.inc"
#undef SB_SC_CONST
  typedef unsigned long long u64;
  u64 bits;
  memcpy(&bits, &x, 8);
  const int E = (int)((bits >> 52) & 0x7ff) - 1075;            // |x| >= 2e5: a normal number
  const u64 M = (bits & ((1ull << 52) - 1)) | (1ull << 52);
  const int j0 = E >= 2 ? (E - 2) / 64 : 0;
  // p[0..5] (p[0] most significant) = M * words j0 .. j0 + 4; y's bit of weight 2^k sits at bit 320 - sh + k of p
  const int sh = E - 64 * j0;                                  // -35 .. 65
  u64 p[6];
  u64 carry = 0;
#pragma unroll
  for (int k = 4; k >= 0; --k) {
    u64 hi, lo;
    mul64(M, kTwoOverPiBits[j0 + k], &hi, &lo);
    p[k + 1] = lo + carry;
    carry = hi + (p[k + 1] < lo);
  }
  p[0] = carry;
  // shift left by 62 + sh (27 .. 127): weight 2^1 to the top bit, the multiples of 4 out
  int s = 62 + sh;
  if (s >= 64) {
#pragma unroll
    for (int k = 0; k < 5; ++k) p[k] = p[k + 1];
    p[5] = 0;
    s -= 64;
  }
  if (s > 0) {
#pragma unroll
    for (int k = 0; k < 5; ++k) p[k] = (p[k] << s) | (p[k + 1] >> (64 - s));
    p[5] <<= s;
  }
  int n = (int)(p[0] >> 62);
  p[0] &= ~(3ull << 62);
  // fraction f = p * 2^-382 in [0, 1); f >= 1/2: one quadrant up and r = -(1 - f) * pi/2
  const bool up = (p[0] >> 61) & 1;
  if (up) {
    n = (n + 1) & 3;
    u64 c = 1;
#pragma unroll
    for (int k = 5; k >= 0; --k) {
      p[k] = ~p[k] + c;
      c = c && p[k] == 0;
    }
    p[0] &= ~(3ull << 62);
  }
  // normalize: the leading one to bit 63 of p[0] (p != 0: x * 2/pi is never an integer), then 106 bits as a double-double
  int z = 0;
#pragma unroll
  for (int w = 0; w < 5; ++w) {
    if (p[0] != 0) break;
#pragma unroll
    for (int k = 0; k < 5; ++k) p[k] = p[k + 1];
    p[5] = 0;
    z += 64;
  }
#ifdef __CUDA_ARCH__
  const int c = __clzll((long long)p[0]);
#else
  const int c = __builtin_clzll(p[0]);
#endif
  z += c;
  const u64 g0 = c ? (p[0] << c) | (p[1] >> (64 - c)) : p[0];
  const u64 g1 = c ? (p[1] << c) | (p[2] >> (64 - c)) : p[1];
  // f = g0 2^(-62 - z) + g1 2^(-126 - z) + more; the top 106 of these bits are exact in two doubles
  const dd f = dd{ldexp((double)(g0 >> 11), -51 - z), ldexp((double)(((g0 & 0x7ff) << 42) | (g1 >> 22)), -104 - z)};
  dd r = dd_mul(f, dd{kPio2[0], kPio2[1]});
  if (up) r = dd_neg(r);
  if (x < 0.0) {
    r = dd_neg(r);
    n = (4 - n) & 3;
  }
  return reduced{r.h, r.l, n};
}

// sin and cos of x, both correctly rounded (see the header comment)
SB_HD void sincos_cr(double x, double* sn, double* cs) {
  // constant tables (function-local so that one definition serves the host and the device compilation)
#define SB_SC_CONST [[maybe_unused]] static const
#include "sb_sincos_table.inc"
#undef SB_SC_CONST
  dd r;
  int n;
  if (fabs(x) < 2.0e5) {
    // ---- x = k * pi/2 + r, |r| <= pi/4 (+ a hair), r as a double-double
    const double kd = rint(x * kTwoOverPi);
    if (kd == 0.0) r = dd{x, 0.0};
    else {
      const dd p0 = two_prod(kd, kPio2[0]);
      const double r1 = x - p0.h;                 // exact (Sterbenz: p0.h is within a factor 2 of x)
      r = two_sum(r1, -p0.l);
      const dd p1 = two_prod(kd, kPio2[1]);
      r = dd_add(r, dd{-p1.h, -p1.l});
      r.l -= kd * kPio2[2];
      r = fast_two_sum(r.h, r.l);
    }
    const long long k = (long long)kd;
    n = (int)(((k % 4) + 4) % 4);
  } else if (fabs(x) <= 1.7976931348623157e308) {
    const reduced q = reduce_large(x);
    r = dd{q.h, q.l};
    n = q.n;
  } else {   // inf or NaN
    const unsigned long long qnan = 0x7ff8000000000000ull;
    memcpy(sn, &qnan, 8);
    memcpy(cs, &qnan, 8);
    return;
  }
  const bool neg = r.h < 0.0;
  if (neg) r = dd_neg(r);
  // ---- r = c + t, c = i / 64
  int i = (int)rint(r.h * 64.0);
  if (i > 51) i = 51;
  const double c = (double)i * 0.015625;
  dd t = two_sum(r.h - c, r.l);                 // r.h - c is exact (both are multiples of ulp(r.h), same binade or below)
  const dd t2 = dd_mul(t, t);
  // sin t = t + t * t2 * (-1/3! + t2 * (1/5! + t2 * (-1/7! + t2 * (1/9! - t2 / 11!))))
  double u = kSinCoef[3][0] - t2.h * kSinCoef[4][0];
  u = -kSinCoef[2][0] + t2.h * u;
  dd q = dd_add(dd{kSinCoef[1][0], kSinCoef[1][1]}, dd_mul_d(t2, u));
  q = dd_add(dd{-kSinCoef[0][0], -kSinCoef[0][1]}, dd_mul(t2, q));
  q = dd_mul(t2, q);
  const dd st = dd_add(t, dd_mul(t, q));
  // cos t = 1 + t2 * (-1/2! + t2 * (1/4! + t2 * (-1/6! + t2 * (1/8! - t2 / 10!))))
  double v = kCosCoef[3][0] - t2.h * kCosCoef[4][0];
  v = -kCosCoef[2][0] + t2.h * v;
  dd w = dd_add(dd{kCosCoef[1][0], kCosCoef[1][1]}, dd_mul_d(t2, v));
  w = dd_add(dd{-kCosCoef[0][0], -kCosCoef[0][1]}, dd_mul(t2, w));
  w = dd_mul(t2, w);
  const dd ct = dd_add(dd{1.0, 0.0}, w);
  // ---- sin(c + t), cos(c + t)
  const dd sc_ = dd{kSinTab[i][0], kSinTab[i][1]}, cc_ = dd{kCosTab[i][0], kCosTab[i][1]};
  dd s = dd_add(dd_mul(sc_, ct), dd_mul(cc_, st));
  dd co = dd_add(dd_mul(cc_, ct), dd_neg(dd_mul(sc_, st)));
  if (neg) s = dd_neg(s);
  // ---- quadrant
  dd rs, rc;
  if (n == 0) { rs = s; rc = co; }
  else if (n == 1) { rs = co; rc = dd_neg(s); }
  else if (n == 2) { rs = dd_neg(s); rc = dd_neg(co); }
  else { rs = dd_neg(co); rc = s; }
  *sn = rs.h + rs.l;
  *cs = rc.h + rc.l;
}

}  // namespace sc
}  // namespace sb
