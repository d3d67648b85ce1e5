// kernels_own.cu -- exclusively owned area shares of a scene's detections (one warp per detection).
//
// Replaces exclusively_owned_areas + exclusively_owned_areas_normalized_shares
// (src/utils/clipping/bbox_own_areas.rs:8-46) as the visual trackers call them when an own-area threshold is set
// (src/trackers/visual_sort/simple_api.rs:110-127, visual_sort/batch_api.rs:236-249).  Arithmetic: sb_own_area.cuh.
// Step 1: the lanes scan the scene's boxes 32 at a time; a box that is not too_far, not certainly disjoint (separating
// axis pre-gate) and not of zero area (own_can_cover) is appended, in index order, to the warp's list in shared memory.  Step 2: the 4 * (k + 1) edges of box_i
// and of the k listed boxes are spread over the lanes; each lane integrates its edges' parts that border the difference
// region; a shuffle tree adds the lanes.  Cost: O(m) cheap gates + O(k^2) half-plane tests per detection.
#include "sb_engine.cuh"
#include "sb_own_area.cuh"

namespace sb {

constexpr int OW_WARPS = 4;

__global__ void __launch_bounds__(OW_WARPS * 32) own_area_kernel(Frame f, const float* __restrict__ boxes, float* __restrict__ out, int* ovf_cnt, int2* ovf) {
  __shared__ double s_quads[OW_WARPS][(kOwnMaxNb + 1) * 8];
  const int scene = blockIdx.y;
  const SceneDesc sc = f.scenes[scene];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m = blockIdx.x * OW_WARPS + w;
  if (m >= sc.m) return;   // warp-uniform
  double* quads = s_quads[w];
  const int g = sc.det_base + m;
  const float* bi = boxes + (size_t)g * 6;
  const float bx = bi[0], by = bi[1], basp = bi[3], bh = bi[4];
  double vi[8];
  box_vertices(bx, by, bi[2], basp, bh, vi);   // every lane: the same eight values
  if (lane < 8) quads[lane] = vi[lane];
  const double s = quad_area_signed(vi) < 0.0 ? -1.0 : 1.0;
  const float ri = box_radius(basp, bh);
  int k = 0;
  for (int j0 = 0; j0 < sc.m; j0 += 32) {
    const int j = j0 + lane;
    bool keep = false;
    double vj[8];
    if (j < sc.m && j != m) {
      const float* bj = boxes + (size_t)(sc.det_base + j) * 6;
      if (!too_far(bx, by, ri, bj[0], bj[1], box_radius(bj[3], bj[4]))) {   // bbox_own_areas.rs:12-14
        box_vertices(bj[0], bj[1], bj[2], bj[3], bj[4], vj);
        keep = own_can_cover(vi, vj);
      }
    }
    const unsigned int mask = __ballot_sync(0xffffffffu, keep);
    if (keep) {
      const int slot = k + __popc(mask & ((1u << lane) - 1u));
      if (slot < kOwnMaxNb) {
#pragma unroll
        for (int q = 0; q < 8; ++q) quads[(slot + 1) * 8 + q] = vj[q];
      }
    }
    k += __popc(mask);
  }
  __syncwarp();
  if (k > kOwnMaxNb) {   // more overlapping boxes than the warp's list holds: the CTA-per-detection second pass takes it
    if (lane == 0) {
      const int slot = atomicAdd(ovf_cnt, 1);
      ovf[slot] = make_int2(scene, m);
      out[g] = 1.0f;
    }
    return;
  }
  double sum = 0.0;
  for (int q = lane; q < 4 * (k + 1); q += 32) sum += own_edge_term(quads, k, q >> 2, q & 3, s);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if (lane == 0) out[g] = own_share(s * sum / 2.0, basp, bh);
}

// Second pass: one CTA per detection that more than kOwnMaxNb boxes overlap (dense crowds).  The overlapping boxes are
// gathered in index order into dynamic shared memory (up to kOwnBigNb), the 4 (k + 1) edges are spread over the threads and
// each edge is integrated without per-thread interval storage (own_edge_term_big).  A fixed grid walks the overflow list, so
// the launch costs a few microseconds when the list is empty (the common case).
constexpr int OB_T = 256;

__global__ void __launch_bounds__(OB_T) own_area_big_kernel(Frame f, const float* __restrict__ boxes, float* __restrict__ out,
                                                            const int* ovf_cnt, const int2* ovf) {
  extern __shared__ double ob_quads[];   // [(kOwnBigNb + 1) * 8]
  __shared__ int s_warp[OB_T / 32];
  __shared__ double s_sum[OB_T / 32];
  __shared__ int s_k;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int cnt = *ovf_cnt;
  for (int it = blockIdx.x; it < cnt; it += gridDim.x) {
    const int2 e = ovf[it];
    const SceneDesc sc = f.scenes[e.x];
    const int m = e.y, g = sc.det_base + m;
    const float* bi = boxes + (size_t)g * 6;
    const float bx = bi[0], by = bi[1], basp = bi[3], bh = bi[4];
    double vi[8];
    box_vertices(bx, by, bi[2], basp, bh, vi);
    if (tid < 8) ob_quads[tid] = vi[tid];
    const double s = quad_area_signed(vi) < 0.0 ? -1.0 : 1.0;
    const float ri = box_radius(basp, bh);
    if (tid == 0) s_k = 0;
    __syncthreads();
    for (int j0 = 0; j0 < sc.m; j0 += OB_T) {
      const int j = j0 + tid;
      bool keep = false;
      double vj[8];
      if (j < sc.m && j != m) {
        const float* bj = boxes + (size_t)(sc.det_base + j) * 6;
        if (!too_far(bx, by, ri, bj[0], bj[1], box_radius(bj[3], bj[4]))) {
          box_vertices(bj[0], bj[1], bj[2], bj[3], bj[4], vj);
          keep = own_can_cover(vi, vj);
        }
      }
      const unsigned int mask = __ballot_sync(0xffffffffu, keep);
      if (lane == 0) s_warp[wid] = __popc(mask);
      __syncthreads();
      int woff = 0, wtot = 0;
      for (int w = 0; w < OB_T / 32; ++w) { if (w < wid) woff += s_warp[w]; wtot += s_warp[w]; }
      const int k0 = s_k;
      if (keep) {
        const int slot = k0 + woff + __popc(mask & ((1u << lane) - 1u));
        if (slot < kOwnBigNb) {
#pragma unroll
          for (int q = 0; q < 8; ++q) ob_quads[(slot + 1) * 8 + q] = vj[q];
        }
      }
      __syncthreads();
      if (tid == 0) s_k = k0 + wtot;
      __syncthreads();
    }
    const int k = s_k;
    if (k > kOwnBigNb) {
      if (tid == 0) { atomicOr(&f.status[e.x], 2); out[g] = 1.0f; }
    } else {
      double sum = 0.0;
      for (int q = tid; q < 4 * (k + 1); q += OB_T) sum += own_edge_term_big(ob_quads, k, q >> 2, q & 3, s);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
      if (lane == 0) s_sum[wid] = sum;
      __syncthreads();
      if (tid == 0) {
        double t = 0.0;
        for (int w = 0; w < OB_T / 32; ++w) t += s_sum[w];
        out[g] = own_share(s * t / 2.0, basp, bh);
      }
    }
    __syncthreads();
  }
}

void launch_own_area(const Frame& f, int n_scenes, int max_m, const float* d_boxes, float* d_out, int* d_ovf_cnt,
                     int2* d_ovf, cudaStream_t st) {
  if (n_scenes == 0 || max_m == 0) return;
  cudaMemsetAsync(d_ovf_cnt, 0, sizeof(int), st);
  dim3 grid((max_m + OW_WARPS - 1) / OW_WARPS, n_scenes);
  own_area_kernel<<<grid, OW_WARPS * 32, 0, st>>>(f, d_boxes, d_out, d_ovf_cnt, d_ovf);
  const size_t smem = (size_t)(kOwnBigNb + 1) * 8 * sizeof(double);
  cudaFuncSetAttribute(own_area_big_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  own_area_big_kernel<<<kNumSms, OB_T, smem, st>>>(f, d_boxes, d_out, d_ovf_cnt, d_ovf);
  note_launch(2);
}

}  // namespace sb
