// sb_math.cuh -- per-pair / per-track arithmetic of the association engine.
//
// Everything here is written against the *semantics* of the reference (file:line cited per function) but in the
// shape a GPU wants: no heap, fixed-size polygons, the Kalman covariance kept as five 2x2 (position, velocity)
// blocks instead of a 10x10 matrix (the reference's matrix never couples two different box coordinates, so the
// 10x10 products in src/utils/kalman/kalman_2d_box.rs reduce exactly -- bit for bit in f32 -- to these block forms).
// Compiled with --fmad=false: Rust never contracts a*b+c, so neither may we.
//
// The functions are `__host__ __device__` so the CPU test-suite can check them against the oracle without a GPU
// (tests/host_shim); the product only ever calls them from device code.
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#ifndef __CUDACC__
#ifndef __host__
#define __host__
#endif
#ifndef __device__
#define __device__
#endif
#ifndef __forceinline__
#define __forceinline__ inline
#endif
#endif
#define SB_HD __host__ __device__ __forceinline__

#include "sb_sincos.cuh"

namespace sb {

constexpr float kEps = 0.00001f;            // EPS, src/lib.rs:80
constexpr float kChi2Inv95_4 = 11.070f;     // CHI2INV95[4], src/utils/kalman.rs:18
constexpr float kChi2Upper = 100.0f;        // CHI2_UPPER_BOUND, src/utils/kalman.rs:16
constexpr float kWeightMult = 1000000.0f;   // F32_U64_MULT, src/trackers/sort/voting.rs:9
constexpr int kMaxPoly = 16;                // clipped quad-by-quad polygon: <= 8 vertices in exact arithmetic

struct Box {
  float xc, yc, angle, aspect, height, conf;  // angle NaN == None
};

SB_HD bool is_nan(float v) { return v != v; }

// wide::f32x8::reduce_add of one 8-lane block (src/distance.rs:9-47): lo + hi quads, then pairs, then the last add
SB_HD float reduce_add8(const float* t) {
  float q0 = t[0] + t[4], q1 = t[1] + t[5], q2 = t[2] + t[6], q3 = t[3] + t[7];
  float d0 = q0 + q2, d1 = q1 + q3;
  return d0 + d1;
}
SB_HD float angle_or0(float a) { return is_nan(a) ? 0.0f : a; }

// Universal2DBox::get_radius, src/utils/bbox.rs:157-161
SB_HD float box_radius(float aspect, float height) {
  float hw = aspect * height / 2.0f;
  float hh = height / 2.0f;
  return sqrtf(hw * hw + hh * hh);
}
// Universal2DBox::area, src/utils/bbox.rs:163-166
SB_HD float box_area(float aspect, float height) {
  float w = height * aspect;
  return w * height;
}
// Universal2DBox::too_far, src/utils/bbox.rs:452-462 (radii precomputed per box)
SB_HD bool too_far(float xl, float yl, float rl, float xr, float yr, float rr) {
  float max_distance = rl + rr;
  float x = xl - xr;
  float y = yl - yr;
  return x * x + y * y > max_distance * max_distance;
}
// Sort key of the culled positional scan (pos_scan_kernel): a total order on (x, track index) with the padding
// (idx < 0) after every track.  x in IEEE order (-0 before +0), every NaN after +inf, ties by index.  The float
// compare `a > b` is not an order once a key is NaN (the network then moves padding into [0, N) and tracks out of it).
SB_HD uint64_t pos_sort_key(float x, int idx) {
  if (idx < 0) return ~0ull;
  uint32_t u;
  memcpy(&u, &x, 4);
  u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  if (is_nan(x)) u = 0xffffffffu;
  return ((uint64_t)u << 32) | (uint32_t)idx;
}
// One compare-exchange of the bitonic network on (x, idx) entries: true when entries i and i ^ j swap, `up` the
// direction of the i-th block of the current merge size.
SB_HD bool pos_sort_swap(float xi, int ii, float xj, int ij, bool up) {
  return (pos_sort_key(xi, ii) > pos_sort_key(xj, ij)) == up;
}
// Universal2DBox::dist_in_2r, src/utils/bbox.rs:464-474
SB_HD float dist_in_2r(float xl, float yl, float rl, float xr, float yr, float rr) {
  float radial_distance = rl + rr;
  float x = xl - xr;
  float y = yl - yr;
  return sqrtf(x * x + y * y) / sqrtf(radial_distance * radial_distance + kEps);
}

// From<&Universal2DBox> for Polygon<f64>, src/utils/bbox.rs:287-330. out = 4 vertices (x0,y0,...,x3,y3).
SB_HD void box_vertices(float xc, float yc, float angle, float aspect_f, float height_f, double* out) {
  double a = (double)angle_or0(angle);
  double height = (double)height_f;
  double aspect = (double)aspect_f;
  // correctly rounded, identical on host and device: the reference's vertices bit for bit (sb_sincos.cuh)
  double c, s;
  sc::sincos_cr(a, &s, &c);
  double half_width = height * aspect / 2.0;
  double half_height = height / 2.0;
  double r1x = -half_width * c - half_height * s;
  double r1y = -half_width * s + half_height * c;
  double r2x = half_width * c - half_height * s;
  double r2y = half_width * s + half_height * c;
  double x = (double)xc, y = (double)yc;
  out[0] = x + r1x; out[1] = y + r1y;
  out[2] = x + r2x; out[3] = y + r2y;
  out[4] = x - r1x; out[5] = y - r1y;
  out[6] = x - r2x; out[7] = y - r2y;
}

// sutherland_hodgman_clip(subject, clip) (src/utils/clipping.rs:12-91) followed by geo's Area::unsigned_area (shoelace
// on coordinates shifted by the first vertex).  Ping-pong buffers, no heap.  What else it reports is chosen at compile
// time, so the area-only instantiation (clip_area) carries none of it:
//   kClipArea   the area only;
//   kClipCount  also *out_n = number of vertices of the clipped ring, or -1 when the reference's unbounded Vec would have
//               held more than kMaxPoly vertices at some step (the area is then that of a truncated ring: not the
//               reference's);
//   kClipRing   also the ring itself, out_xy = (x, y) pairs of the first *out_n vertices, in the reference's order and
//               without the closing repeat that geo::Polygon::new adds.
enum ClipOut { kClipArea = 0, kClipCount = 1, kClipRing = 2 };

template <int kOut>
SB_HD double clip_poly(const double* subj, const double* clp, double* out_xy, int* out_n) {
  double ax[kMaxPoly], ay[kMaxPoly], bx[kMaxPoly], by[kMaxPoly];
  [[maybe_unused]] bool over = false;
  int na = 4;
#pragma unroll
  for (int i = 0; i < 4; ++i) { ax[i] = subj[2 * i]; ay[i] = subj[2 * i + 1]; }
  double* sx = ax; double* sy = ay; double* dx = bx; double* dy = by;
#pragma unroll 1
  for (int i = 0; i < 4; ++i) {
    const int ii = (i == 0) ? 3 : i - 1;
    const double c1x = clp[2 * ii], c1y = clp[2 * ii + 1];  // c_edge_start
    const double c2x = clp[2 * i], c2y = clp[2 * i + 1];    // c_edge_end
    const double ex = c2x - c1x, ey = c2y - c1y;
    int nd = 0;
    if (na > 0) {
      double psx = sx[na - 1], psy = sy[na - 1];
      bool p_in = (ex * (psy - c1y) - ey * (psx - c1x)) <= 0.0;  // is_inside(s_edge_start)
      for (int j = 0; j < na; ++j) {
        const double qx = sx[j], qy = sy[j];
        const bool q_in = (ex * (qy - c1y) - ey * (qx - c1x)) <= 0.0;  // is_inside(s_edge_end)
        if (q_in != p_in) {
          // compute_intersection(cp1 = s_edge_start, cp2 = s_edge_end, s = c_edge_start, e = c_edge_end)
          const double dcx = psx - qx, dcy = psy - qy;
          const double dpx = c1x - c2x, dpy = c1y - c2y;
          const double n1 = psx * qy - psy * qx;
          const double n2 = c1x * c2y - c1y * c2x;
          const double n3 = 1.0 / (dcx * dpy - dcy * dpx);
          if constexpr (kOut != kClipArea) over = over || nd >= kMaxPoly;
          if (nd < kMaxPoly) { dx[nd] = (n1 * dpx - n2 * dcx) * n3; dy[nd] = (n1 * dpy - n2 * dcy) * n3; ++nd; }
        }
        if constexpr (kOut != kClipArea) over = over || (q_in && nd >= kMaxPoly);
        if (q_in && nd < kMaxPoly) { dx[nd] = qx; dy[nd] = qy; ++nd; }
        psx = qx; psy = qy; p_in = q_in;
      }
    }
    double* t;
    t = sx; sx = dx; dx = t;
    t = sy; sy = dy; dy = t;
    na = nd;
  }
  if constexpr (kOut != kClipArea) *out_n = over ? -1 : na;
  if constexpr (kOut == kClipRing) {
    for (int j = 0; j < na; ++j) { out_xy[2 * j] = sx[j]; out_xy[2 * j + 1] = sy[j]; }
  }
  if (na < 3) return 0.0;
  // geo: ring closed by Polygon::new; shift by first coord; sum of determinants over ring lines; |sum / 2|
  const double shx = sx[0], shy = sy[0];
  double tmp = 0.0;
  double pax = 0.0, pay = 0.0;  // first vertex shifted == (0,0)
  for (int j = 1; j <= na; ++j) {
    const int jj = (j == na) ? 0 : j;
    const double qx = sx[jj] - shx, qy = sy[jj] - shy;
    tmp += pax * qy - pay * qx;
    pax = qx; pay = qy;
  }
  return fabs(tmp / 2.0);
}
SB_HD double clip_area(const double* subj, const double* clp) { return clip_poly<kClipArea>(subj, clp, nullptr, nullptr); }

// Conservative pre-gates of the IoU metric: they decide "certainly None" for any threshold above ~1e-6, so that the f64
// clip can be skipped.  Pairs they cannot decide go through clip_area unchanged.
//   * rect_overlap_bound: both quadrilaterals are projected on the edge directions of each of them (f64, the very
//     vertices the clip uses).  A gap on any axis (with a margin nine orders of magnitude above the rounding of a dot
//     product) separates them: the intersection is empty and Sutherland-Hodgman returns either nothing or a rounding
//     sliver whose IoU (~1e-12) no positive threshold accepts -> the bound is 0.  Otherwise the intersection lies inside
//     the axis-aligned (in that rectangle's frame) box spanned by the overlap intervals, whose area bounds it from
//     above; the smaller of the two frames' bounds is returned (1e300: no bound, e.g. a degenerate edge).
//   * iou_bound_fails: intersection <= min(area), union >= max(area)  =>  IoU <= min / max.
SB_HD double rect_overlap_bound(const double* a, const double* b) {
  double scale = 0.0;
#pragma unroll
  for (int i = 0; i < 8; ++i) { scale = fmax(scale, fabs(a[i])); scale = fmax(scale, fabs(b[i])); }
  double bound = 1e300;
#pragma unroll
  for (int pass = 0; pass < 2; ++pass) {
    const double* q = pass == 0 ? a : b;
    double area = 1.0;
    bool usable = true;
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      // edge e of the quadrilateral: vertices e -> e + 1 (the two edge directions of a rectangle are its two axes)
      const double ux = q[2 * (e + 1)] - q[2 * e], uy = q[2 * (e + 1) + 1] - q[2 * e + 1];
      double amin = 1e300, amax = -1e300, bmin = 1e300, bmax = -1e300;
#pragma unroll
      for (int v = 0; v < 4; ++v) {
        const double pa = a[2 * v] * ux + a[2 * v + 1] * uy;
        const double pb = b[2 * v] * ux + b[2 * v + 1] * uy;
        amin = fmin(amin, pa); amax = fmax(amax, pa);
        bmin = fmin(bmin, pb); bmax = fmax(bmax, pb);
      }
      const double tol = 1e-7 * (fabs(ux) + fabs(uy)) * (scale + 1.0);
      if (bmin - amax > tol || amin - bmax > tol) return 0.0;
      const double len2 = ux * ux + uy * uy;
      if (!(len2 > 0.0)) { usable = false; continue; }
      const double ov = fmin(amax, bmax) - fmax(amin, bmin) + tol;   // in units of |u| * length
      area *= fmax(ov, 0.0) / len2 * sqrt(len2);                      // -> length along this axis
    }
    if (usable) bound = fmin(bound, area);
  }
  return bound;
}
SB_HD bool iou_bound_fails(float h_l, float a_l, float h_r, float a_r, float conf, float threshold) {
  const float al = h_l * h_l * a_l, ar = h_r * h_r * a_r;
  if (!(al > 0.0f) || !(ar > 0.0f) || !(conf == conf)) return false;   // degenerate / NaN boxes: let the exact path decide
  const float lo = fminf(al, ar), hi = fmaxf(al, ar);
  return lo * conf * 1.0001f < threshold * hi;
}

// Universal2DBox::calculate_metric_object (src/utils/bbox.rs:512-535) given the clipped area.
// Returns NaN for None (intersection == 0).
SB_HD float iou_from_area(double inter, float h_l, float a_l, float h_r, float a_r) {
  if (inter == 0.0) return nanf("");
  double uni = (double)(h_l * h_l * a_l + h_r * h_r * a_r) - inter;
  return (float)(inter / uni);
}

// ---------------------------------------------------------------------------------------------------------
// Kalman filter, src/utils/kalman/kalman_2d_box.rs.  State = mean[10] + cov[20] where
// cov[4*i + {0,1,2,3}] = P[i][i], P[i][i+5], P[i+5][i], P[i+5][i+5]  (i = xc, yc, angle, aspect, height).
constexpr int kStateFloats = 30;

SB_HD void kalman_initiate(float pw, float vw, const Box& b, float* st) {  // initiate, :58-84
  st[0] = b.xc; st[1] = b.yc; st[2] = angle_or0(b.angle); st[3] = b.aspect; st[4] = b.height;
#pragma unroll
  for (int i = 5; i < 10; ++i) st[i] = 0.0f;
  const float sp = 2.0f * pw * b.height;   // std_position(2.0, 1e-2, h): k * w * p, left to right
  const float sv = 10.0f * vw * b.height;  // std_velocity(10.0, 1e-5, h)
#pragma unroll
  for (int i = 0; i < 5; ++i) {
    const float p = (i == 3) ? 1e-2f : sp;
    const float v = (i == 3) ? 1e-5f : sv;
    st[10 + 4 * i + 0] = p * p;
    st[10 + 4 * i + 1] = 0.0f;
    st[10 + 4 * i + 2] = 0.0f;
    st[10 + 4 * i + 3] = v * v;
  }
}

SB_HD void kalman_predict(float pw, float vw, const float* in, float* out) {  // predict, :86-102
  const float h = in[4];
  const float sp = 1.0f * pw * h;
  const float sv = 1.0f * vw * h;
#pragma unroll
  for (int i = 0; i < 5; ++i) {
    const float m = in[i], v = in[5 + i];
    const float a = in[10 + 4 * i], b = in[10 + 4 * i + 1], c = in[10 + 4 * i + 2], d = in[10 + 4 * i + 3];
    const float p = (i == 3) ? 1e-2f : sp;
    const float q = (i == 3) ? 1e-5f : sv;
    out[i] = m + v;      // F * mean
    out[5 + i] = v;
    const float fa = a + c, fb = b + d;        // (F P) rows i
    out[10 + 4 * i + 0] = (fa + fb) + p * p;   // (F P F^T)[i][i] + motion_cov
    out[10 + 4 * i + 1] = fb;                  // [i][i+5]
    out[10 + 4 * i + 2] = c + d;               // [i+5][i]
    out[10 + 4 * i + 3] = d + q * q;           // [i+5][i+5]
  }
}

// project (:104-120): S_ii = P_ii + std_i^2 (S is exactly diagonal)
SB_HD float kalman_proj_var(float pw, float h, float pii, int i) {
  const float sp = 1.0f * pw * h;
  const float p = (i == 3) ? 1e-1f : sp;
  return pii + p * p;
}

SB_HD void kalman_update(float pw, const float* in, const Box& z, float* out) {  // update, :124-148
  const float h = in[4];
  const float meas[5] = {z.xc, z.yc, angle_or0(z.angle), z.aspect, z.height};
#pragma unroll
  for (int i = 0; i < 5; ++i) {
    const float m = in[i], v = in[5 + i];
    const float a = in[10 + 4 * i], b = in[10 + 4 * i + 1], c = in[10 + 4 * i + 2], d = in[10 + 4 * i + 3];
    const float s = kalman_proj_var(pw, h, a, i);
    const float kp = a / s;   // kalman_gain[i][i]   = P[i][i]   / S_ii
    const float kv = c / s;   // kalman_gain[i][i+5] = P[i+5][i] / S_ii
    const float innov = meas[i] - m;
    out[i] = m + innov * kp;
    out[5 + i] = v + innov * kv;
    const float kps = kp * s, kvs = kv * s;  // (K^T S)
    out[10 + 4 * i + 0] = a - kps * kp;
    out[10 + 4 * i + 1] = b - kps * kv;
    out[10 + 4 * i + 2] = c - kvs * kp;
    out[10 + 4 * i + 3] = d - kvs * kv;
  }
}

// distance (:150-170) with the diagonal S: sum_i ((z_i - mean_i) / sqrt(S_ii))^2, accumulated in index order.
// mean5 / lsq5 = per-track precomputed means and sqrt(S_ii).
SB_HD float maha_distance(const float* mean5, const float* l5, float xc, float yc, float angle0, float aspect,
                          float height) {
  const float y0 = (xc - mean5[0]) / l5[0];
  const float y1 = (yc - mean5[1]) / l5[1];
  const float y2 = (angle0 - mean5[2]) / l5[2];
  const float y3 = (aspect - mean5[3]) / l5[3];
  const float y4 = (height - mean5[4]) / l5[4];
  // The reference's forward substitution adds (-y_i) * L_ri (L_ri == 0) to every later row, so an infinite y0..y3 (a
  // finite box whose whitened residual overflows f32) makes its distance NaN -- None -- not +inf (cost 0).
  if (isinf(y0) || isinf(y1) || isinf(y2) || isinf(y3)) return nanf("");
  float s = y0 * y0;
  s = s + y1 * y1;
  s = s + y2 * y2;
  s = s + y3 * y3;
  s = s + y4 * y4;
  return s;
}
// calculate_cost(d, inverted = true), :172-184
SB_HD float maha_cost(float d) { return d > kChi2Inv95_4 ? 0.0f : kChi2Upper - d; }

// TryFrom<KalmanState> for Universal2DBox, src/utils/kalman.rs:72-92
SB_HD Box state_box(const float* st, float conf) {
  Box b;
  b.xc = st[0]; b.yc = st[1];
  b.angle = (st[2] == 0.0f) ? nanf("") : st[2];
  b.aspect = st[3]; b.height = st[4]; b.conf = conf;
  return b;
}

// ---------------------------------------------------------------------------------------------------------
// Kalman filter of a 2-D point, src/utils/kalman/kalman_2d_point.rs.  State = mean[4] + cov[8] where
// mean = (x, y, vx, vy) and cov[4*i + {0,1,2,3}] = P[i][i], P[i][i+2], P[i+2][i], P[i+2][i+2]  (i = x, y): the box
// state's layout with two blocks.  The reference's 4x4 matrices never couple x with y either, so the same argument
// holds: S is exactly diagonal and every entry of the full products has at most two non-zero terms.
constexpr int kPointStateFloats = 12;

SB_HD void point_kalman_initiate(float pw, float vw, float x, float y, float* st) {  // initiate, :51-65
  st[0] = x; st[1] = y; st[2] = 0.0f; st[3] = 0.0f;
  const float sp = 2.0f * pw;   // std_position(2.0) = k * w, :41-44 (no height factor, unlike the box filter)
  const float sv = 10.0f * vw;  // std_velocity(10.0), :46-49
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    st[4 + 4 * i + 0] = sp * sp;
    st[4 + 4 * i + 1] = 0.0f;
    st[4 + 4 * i + 2] = 0.0f;
    st[4 + 4 * i + 3] = sv * sv;
  }
}

SB_HD void point_kalman_predict(float pw, float vw, const float* in, float* out) {  // predict, :67-84
  const float p = 1.0f * pw;  // std_position(1.0)
  const float q = 1.0f * vw;  // std_velocity(1.0)
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const float m = in[i], v = in[2 + i];
    const float a = in[4 + 4 * i], b = in[4 + 4 * i + 1], c = in[4 + 4 * i + 2], d = in[4 + 4 * i + 3];
    out[i] = m + v;      // F * mean, F = [[I, I], [0, I]] (DT = 1)
    out[2 + i] = v;
    const float fa = a + c, fb = b + d;      // (F P) row i
    out[4 + 4 * i + 0] = (fa + fb) + p * p;  // (F P F^T)[i][i] + motion_cov
    out[4 + 4 * i + 1] = fb;                 // [i][i+2]
    out[4 + 4 * i + 2] = c + d;              // [i+2][i]
    out[4 + 4 * i + 3] = d + q * q;          // [i+2][i+2]
  }
}

// project (:86-101): S_ii = P_ii + std_position(1.0)^2 (S is exactly diagonal)
SB_HD float point_kalman_proj_var(float pw, float pii) {
  const float p = 1.0f * pw;
  return pii + p * p;
}

SB_HD void point_kalman_update(float pw, const float* in, float x, float y, float* out) {  // update, :103-121
  const float meas[2] = {x, y};
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const float m = in[i], v = in[2 + i];
    const float a = in[4 + 4 * i], b = in[4 + 4 * i + 1], c = in[4 + 4 * i + 2], d = in[4 + 4 * i + 3];
    const float s = point_kalman_proj_var(pw, a);
    const float kp = a / s;   // kalman_gain[i][i]   = P[i][i]   / S_ii  (solve_lower_triangular on the diagonal S)
    const float kv = c / s;   // kalman_gain[i][i+2] = P[i+2][i] / S_ii
    const float innov = meas[i] - m;
    out[i] = m + innov * kp;
    out[2 + i] = v + innov * kv;
    const float kps = kp * s, kvs = kv * s;  // (K^T S)
    out[4 + 4 * i + 0] = a - kps * kp;
    out[4 + 4 * i + 1] = b - kps * kv;
    out[4 + 4 * i + 2] = c - kvs * kp;
    out[4 + 4 * i + 3] = d - kvs * kv;
  }
}

// distance (:123-137): the Cholesky factor of the diagonal S is diag(sqrt(S_ii)); sum of squares in index order
SB_HD float point_kalman_distance(float pw, const float* st, float x, float y) {
  const float l0 = sqrtf(point_kalman_proj_var(pw, st[4]));
  const float l1 = sqrtf(point_kalman_proj_var(pw, st[8]));
  const float y0 = (x - st[0]) / l0;
  const float y1 = (y - st[1]) / l1;
  float s = y0 * y0;
  s = s + y1 * y1;
  return s;
}

// Universal2DBoxKalmanFilter::distance (src/utils/kalman/kalman_2d_box.rs:150-170) of a packed 30-float state: the
// same l5 as the positional cost kernel's Mahalanobis pair (kernels_cost.cu, pos_eval_pair)
SB_HD float kalman_distance(float pw, const float* st, const Box& z) {
  float l5[5];
  const float hh = st[4];
#pragma unroll
  for (int q = 0; q < 5; ++q) l5[q] = sqrtf(kalman_proj_var(pw, hh, st[10 + 4 * q], q));
  return maha_distance(st, l5, z.xc, z.yc, angle_or0(z.angle), z.aspect, z.height);
}

// Rust `f32 as i64` (saturating, NaN -> 0) of value * 1e6, src/trackers/sort/voting.rs:20,59
SB_HD long long weight_i64(float v) {
  float w = v * kWeightMult;
  if (w != w) return 0;
  if (w >= 9223372036854775807.0f) return 9223372036854775807LL;
  if (w <= -9223372036854775808.0f) return (-9223372036854775807LL - 1);
  return (long long)w;
}

}  // namespace sb
