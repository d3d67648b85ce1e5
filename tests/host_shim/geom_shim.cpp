// Host build of the point Kalman filter's block form, the box filter's distance and the vertex-emitting clip
// (similari_b200/csrc/sb_math.cuh), so that the CPU test-suite can compare them bit-for-bit with full-matrix
// restatements before any GPU time is spent.  TEST INFRASTRUCTURE: the product never loads this library.
#include "../../similari_b200/csrc/sb_math.cuh"
extern "C" {
void gshim_point_initiate(float pw, float vw, float x, float y, float* st12) { sb::point_kalman_initiate(pw, vw, x, y, st12); }
void gshim_point_predict(float pw, float vw, const float* in12, float* out12) { sb::point_kalman_predict(pw, vw, in12, out12); }
void gshim_point_update(float pw, const float* in12, float x, float y, float* out12) {
  sb::point_kalman_update(pw, in12, x, y, out12);
}
float gshim_point_distance(float pw, const float* st12, float x, float y) { return sb::point_kalman_distance(pw, st12, x, y); }
float gshim_box_distance(float pw, const float* st30, const float* b) {
  return sb::kalman_distance(pw, st30, sb::Box{b[0], b[1], b[2], b[3], b[4], b[5]});
}
// ring = (x, y) pairs, kMaxPoly of them; returns the area, *count = vertices or -1 past kMaxPoly
double gshim_clip_ring(const double* s8, const double* c8, double* ring, int* count) {
  return sb::clip_poly<sb::kClipRing>(s8, c8, ring, count);
}
double gshim_clip_count(const double* s8, const double* c8, int* count) {
  return sb::clip_poly<sb::kClipCount>(s8, c8, nullptr, count);
}
double gshim_clip_area(const double* s8, const double* c8) { return sb::clip_area(s8, c8); }
}
