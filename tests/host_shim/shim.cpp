// Host build of the product's per-pair arithmetic (similari_b200/csrc/sb_math.cuh) so that the CPU test-suite can
// compare it bit-for-bit with the oracle before any GPU time is spent.  TEST INFRASTRUCTURE: the product never
// loads this library and has no CPU execution path.
#include <string.h>
#include <vector>
#include "../../similari_b200/csrc/sb_math.cuh"
#include "../../similari_b200/csrc/sb_own_area.cuh"
extern "C" {
void shim_vertices(const float* b, double* out8) { sb::box_vertices(b[0], b[1], b[2], b[3], b[4], out8); }
double shim_clip_area(const double* s8, const double* c8) { return sb::clip_area(s8, c8); }
float shim_iou(const float* l, const float* r) {
  if (sb::too_far(l[0], l[1], sb::box_radius(l[3], l[4]), r[0], r[1], sb::box_radius(r[3], r[4]))) return nanf("");
  double vl[8], vr[8];
  sb::box_vertices(l[0], l[1], l[2], l[3], l[4], vl);
  sb::box_vertices(r[0], r[1], r[2], r[3], r[4], vr);
  return sb::iou_from_area(sb::clip_area(vl, vr), l[4], l[3], r[4], r[3]);
}
void shim_kalman_initiate(float pw, float vw, const float* b, float* st) {
  sb::Box bx{b[0], b[1], b[2], b[3], b[4], b[5]};
  sb::kalman_initiate(pw, vw, bx, st);
}
void shim_kalman_predict(float pw, float vw, const float* in, float* out) { sb::kalman_predict(pw, vw, in, out); }
void shim_kalman_update(float pw, const float* in, const float* b, float* out) {
  sb::Box bx{b[0], b[1], b[2], b[3], b[4], b[5]};
  sb::kalman_update(pw, in, bx, out);
}
float shim_maha(float pw, const float* st, const float* b) {
  float l5[5];
  for (int i = 0; i < 5; ++i) l5[i] = sqrtf(sb::kalman_proj_var(pw, st[4], st[10 + 4 * i], i));
  return sb::maha_distance(st, l5, b[0], b[1], sb::angle_or0(b[2]), b[3], b[4]);
}
long long shim_weight(float v) { return sb::weight_i64(v); }
float shim_box_radius(float aspect, float height) { return sb::box_radius(aspect, height); }
float shim_dist_in_2r(float xl, float yl, float rl, float xr, float yr, float rr) {
  return sb::dist_in_2r(xl, yl, rl, xr, yr, rr);
}
void shim_own_area_shares(const float* boxes, int n, float* out) {
  for (int i = 0; i < n; ++i) out[i] = sb::own_area_share_seq(boxes, n, i);
}
// own_area_big_kernel's arithmetic for box i, run serially: the same gather in index order as own_area_share_seq, without
// its kOwnMaxNb cap (the kernel's cap is kOwnBigNb: -1 above it), and own_edge_term_big summed in edge order.
float shim_own_area_share_big(const float* boxes, int n, int i) {
  const float* bi = boxes + (size_t)i * 6;
  std::vector<double> quads(8);
  sb::box_vertices(bi[0], bi[1], bi[2], bi[3], bi[4], quads.data());
  const double s = sb::quad_area_signed(quads.data()) < 0.0 ? -1.0 : 1.0;
  const float ri = sb::box_radius(bi[3], bi[4]);
  int k = 0;
  for (int j = 0; j < n; ++j) {
    if (j == i) continue;
    const float* bj = boxes + (size_t)j * 6;
    if (sb::too_far(bi[0], bi[1], ri, bj[0], bj[1], sb::box_radius(bj[3], bj[4]))) continue;
    double vj[8];
    sb::box_vertices(bj[0], bj[1], bj[2], bj[3], bj[4], vj);
    if (!sb::own_can_cover(quads.data(), vj)) continue;
    if (k >= sb::kOwnBigNb) return -1.0f;
    ++k;
    quads.insert(quads.end(), vj, vj + 8);
  }
  double sum = 0.0;
  for (int js = 0; js <= k; ++js)
    for (int e = 0; e < 4; ++e) sum += sb::own_edge_term_big(quads.data(), k, js, e, s);
  return sb::own_share(s * sum / 2.0, bi[3], bi[4]);
}
double shim_overlap_bound(const double* a8, const double* b8) { return sb::rect_overlap_bound(a8, b8); }
int shim_iou_bound_fails(const float* l, const float* r, float conf, float thr) {
  return sb::iou_bound_fails(l[4], l[3], r[4], r[3], conf, thr) ? 1 : 0;
}
// pos_scan_kernel's sort of the track centres, run serially: the same padding to Np (a power of two) and the same
// (k2, j) network.  Within one (k2, j) step the exchanges touch disjoint pairs, so the serial order gives the kernel's
// result exactly.  kx, kidx: Np entries out.
void shim_pos_sort(const float* x, int n, float* kx, int* kidx) {
  int np = 1;
  while (np < n) np <<= 1;
  for (int i = 0; i < np; ++i) {
    kx[i] = i < n ? x[i] : 3.402823466e+38f;
    kidx[i] = i < n ? i : -1;
  }
  for (int k2 = 2; k2 <= np; k2 <<= 1)
    for (int j = k2 >> 1; j > 0; j >>= 1)
      for (int i = 0; i < np; ++i) {
        const int ixj = i ^ j;
        if (ixj > i && sb::pos_sort_swap(kx[i], kidx[i], kx[ixj], kidx[ixj], (i & k2) == 0)) {
          const float a = kx[i]; kx[i] = kx[ixj]; kx[ixj] = a;
          const int t = kidx[i]; kidx[i] = kidx[ixj]; kidx[ixj] = t;
        }
      }
}
}
// sincos_cr (sb_sincos.cuh) and the C library's sin / cos over an array of f32 angles
extern "C" void shim_sincos(const float* angles, long long n, double* s, double* c) {
  for (long long i = 0; i < n; ++i) sb::sc::sincos_cr((double)angles[i], &s[i], &c[i]);
}
extern "C" void shim_sincos_f64(const double* x, long long n, double* s, double* c) {
  for (long long i = 0; i < n; ++i) sb::sc::sincos_cr(x[i], &s[i], &c[i]);
}
extern "C" void shim_libm_sincos(const float* angles, long long n, double* s, double* c) {
  for (long long i = 0; i < n; ++i) { s[i] = sin((double)angles[i]); c[i] = cos((double)angles[i]); }
}
