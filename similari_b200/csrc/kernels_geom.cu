// kernels_geom.cu -- stateless oriented-box geometry: vertices, clipped polygons and intersection-area matrices.
//
// Replaces Universal2DBox::get_vertices (From<&Universal2DBox> for Polygon<f64>, src/utils/bbox.rs:287-330),
// sutherland_hodgman_clip_py and intersection_area_py (src/utils/clipping/clipping_py.rs:29-46) for many boxes at once.
// The arithmetic is sb_math.cuh's box_vertices and clip_poly, the same code the IoU, NMS and own-area kernels run, so a
// pair's area here is bit for bit the area those kernels clip.  Unlike the IoU metric there is no too_far pre-gate and no
// IoU gate: intersection_area_py has neither.
#include "sb_engine.cuh"

namespace sb {

__global__ void box_vertices_kernel(const float* __restrict__ boxes, int n, double* __restrict__ out8) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* b = boxes + (size_t)i * 6;
  box_vertices(b[0], b[1], b[2], b[3], b[4], out8 + (size_t)i * 8);
}

void launch_box_vertices(const float* boxes6, int n, double* out8, cudaStream_t st) {
  if (n == 0) return;
  box_vertices_kernel<<<(n + 127) / 128, 128, 0, st>>>(boxes6, n, out8);
  note_launch();
}

// one thread per (subject, clipping) pair; the ring goes straight to its [kMaxPoly][2] slot
__global__ void clip_polygons_kernel(const float* __restrict__ subj6, const float* __restrict__ clip6, int n,
                                     double* __restrict__ out_xy, int* __restrict__ out_counts,
                                     double* __restrict__ out_areas, int* status) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* s = subj6 + (size_t)i * 6;
  const float* c = clip6 + (size_t)i * 6;
  double sv[8], cv[8];
  box_vertices(s[0], s[1], s[2], s[3], s[4], sv);
  box_vertices(c[0], c[1], c[2], c[3], c[4], cv);
  int cnt = 0;
  const double area = clip_poly<kClipRing>(sv, cv, out_xy + (size_t)i * kMaxPoly * 2, &cnt);
  out_counts[i] = cnt;
  out_areas[i] = area;
  if (cnt < 0) atomicOr(status, 1);
}

void launch_clip_polygons(const float* subjects6, const float* clippings6, int n, double* out_xy, int* out_counts,
                          double* out_areas, int* d_status, cudaStream_t st) {
  if (n == 0) return;
  clip_polygons_kernel<<<(n + 127) / 128, 128, 0, st>>>(subjects6, clippings6, n, out_xy, out_counts, out_areas, d_status);
  note_launch();
}

// m x n areas.  A CTA covers IA_ROWS subjects x 32 clipping boxes; both tiles' vertices are staged in shared memory once.
// Lane = clipping box (its vertices then live in registers), warp = a row stride, so every store of a warp is 32
// consecutive doubles of one output row and every subject read is a shared-memory broadcast.
constexpr int IA_COLS = 32, IA_WARPS = 8, IA_ROWS = 64;

__global__ void __launch_bounds__(IA_COLS * IA_WARPS) intersection_areas_kernel(
    const double* __restrict__ a_vert, int m, const double* __restrict__ b_vert, int n, double* __restrict__ out,
    int* status) {
  __shared__ double s_a[IA_ROWS * 8];
  __shared__ double s_b[IA_COLS * 8];
  const int tx = threadIdx.x, ty = threadIdx.y, t = ty * IA_COLS + tx;
  const int j0 = blockIdx.x * IA_COLS, i0 = blockIdx.y * IA_ROWS;
  const int rows = min(IA_ROWS, m - i0), cols = min(IA_COLS, n - j0);
  for (int k = t; k < rows * 8; k += IA_COLS * IA_WARPS) s_a[k] = a_vert[(size_t)i0 * 8 + k];
  for (int k = t; k < cols * 8; k += IA_COLS * IA_WARPS) s_b[k] = b_vert[(size_t)j0 * 8 + k];
  __syncthreads();
  if (tx >= cols) return;
  double cv[8];
#pragma unroll
  for (int q = 0; q < 8; ++q) cv[q] = s_b[tx * 8 + q];
  int bad = 0;
  for (int r = ty; r < rows; r += IA_WARPS) {
    int cnt;
    const double area = clip_poly<kClipCount>(&s_a[r * 8], cv, nullptr, &cnt);
    bad |= cnt < 0;
    out[(size_t)(i0 + r) * n + j0 + tx] = area;
  }
  if (bad) atomicOr(status, 1);
}

void launch_intersection_areas(const double* a_vert, int m, const double* b_vert, int n, double* out_mn, int* d_status,
                               cudaStream_t st) {
  constexpr int kRowsPerLaunch = 65535 * IA_ROWS;   // gridDim.y limit
  for (int r0 = 0; r0 < m && n > 0; r0 += kRowsPerLaunch) {
    const int mr = min(kRowsPerLaunch, m - r0);
    dim3 grid((n + IA_COLS - 1) / IA_COLS, (mr + IA_ROWS - 1) / IA_ROWS);
    intersection_areas_kernel<<<grid, dim3(IA_COLS, IA_WARPS), 0, st>>>(a_vert + (size_t)r0 * 8, mr, b_vert, n,
                                                                        out_mn + (size_t)r0 * n, d_status);
    note_launch();
  }
}

}  // namespace sb
