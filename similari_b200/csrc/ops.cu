// ops.cu -- stateless operators of the C ABI (sb200_sort_cost_matrix, sb200_visual_cost_matrix, sb200_sort_voting,
// sb200_visual_voting, sb200_kalman_*).  They drive the SAME kernels as the tracker's predict path on a one-scene
// scratch store, so a parity test of an operator is a parity test of the product kernel.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/similari_b200.h"
#include "sb_engine.cuh"
#include "sb_host.cuh"

namespace {

using sb::DBuf;
using sb::fail;

// The device memory and stream of one operator call.  The first allocation, upload or memset that fails sets the last
// error and `rc`, and the ones after it are skipped: an operator checks `rc` once, before its first launch.
struct Scratch {
  std::vector<DBuf> bufs;
  cudaStream_t st = nullptr;
  int rc = 0;
  ~Scratch() {
    bufs.clear();
    if (st) cudaStreamDestroy(st);
  }
  void check(cudaError_t e, const char* what) {
    if (e == cudaSuccess || rc) return;
    cudaGetLastError();
    rc = fail(SB200_ERR_CUDA, "%s failed: %s", what, cudaGetErrorString(e));
  }
  template <typename T>
  T* alloc(size_t n, bool zero = false) {
    if (rc) return nullptr;
    const size_t bytes = std::max<size_t>(1, n) * sizeof(T);
    DBuf b;
    if ((rc = b.ensure(bytes))) return nullptr;
    if (zero) check(cudaMemsetAsync(b.p, 0, bytes, st), "cudaMemsetAsync");
    bufs.push_back(std::move(b));
    return bufs.back().as<T>();
  }
  template <typename T>
  T* upload(const T* h, size_t n) {
    T* d = alloc<T>(n);
    if (d && n) check(cudaMemcpyAsync(d, h, n * sizeof(T), cudaMemcpyHostToDevice, st), "cudaMemcpyAsync");
    return d;
  }
};

int begin(Scratch& sc, int device) {
  if (int rc = sb::check_device(device)) return rc;
  CU(cudaSetDevice(device));
  CU(cudaStreamCreateWithFlags(&sc.st, cudaStreamNonBlocking));
  return 0;
}
int finish(Scratch& sc) {
  cudaError_t e = cudaStreamSynchronize(sc.st);
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e != cudaSuccess) return fail(SB200_ERR_CUDA, "CUDA error: %s", cudaGetErrorString(e));
  return 0;
}

sb::Params base_params() {
  sb::Params p;
  memset(&p, 0, sizeof(p));
  p.max_idle_epochs = 1;
  p.max_obs = 1;
  p.d8 = 8;
  return p;
}

__global__ void track_geom_kernel(int iou, const float* boxes, int n, float* radius, double* vert, unsigned int* epoch) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* b = boxes + (size_t)i * 6;
  radius[i] = sb::box_radius(b[3], b[4]);
  epoch[i] = 0;
  if (iou) sb::box_vertices(b[0], b[1], b[2], b[3], b[4], vert + (size_t)i * 8);
}
__global__ void fill_u8_kernel(unsigned char* p, unsigned char v, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

// The voting operators' entry lists: the valid (non-NaN) entries of a dense row-major [rows][cols] matrix in the
// tracker's list format -- PosEntry {row, col, v}, or VisPair {g = row, outcol = col} plus vis_val -- in REVERSE
// row-major order.  The tracker's lists arrive in atomic order, so the sparse voting kernel must not rely on sorted
// input, and the operator does not hand it one.  One CTA walks the matrix from its end in chunks of 1024 with a
// block-wide scan of the valid flags; entries past `cap` are counted but not stored, as in the tracker (the count then
// sends the scene to the dense voting kernel).
constexpr int kListThreads = 1024;
__global__ void __launch_bounds__(kListThreads) vote_list_kernel(const float* a, int rows, int cols, int cap,
                                                                 sb::PosEntry* pos_out, sb::VisPair* vis_out,
                                                                 float* vis_val, int* cnt) {
  __shared__ int s_warp[kListThreads / 32];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const long long total = (long long)rows * cols;
  int carry = 0;
  for (long long base = 0; base < total; base += kListThreads) {
    const long long i = total - 1 - (base + tid);   // position base + tid of the reversed order
    const float v = i >= 0 ? a[i] : 0.0f;
    const bool ok = i >= 0 && v == v;
    const unsigned int bal = __ballot_sync(0xffffffffu, ok);
    if (lane == 0) s_warp[wid] = __popc(bal);
    __syncthreads();
    int woff = 0, chunk = 0;
    for (int w = 0; w < kListThreads / 32; ++w) {
      woff += w < wid ? s_warp[w] : 0;
      chunk += s_warp[w];
    }
    const int slot = carry + woff + __popc(bal & ((1u << lane) - 1u));
    if (ok && slot < cap) {
      const int r = (int)(i / cols), c = (int)(i % cols);
      if (pos_out) pos_out[slot] = sb::PosEntry{(unsigned short)r, (unsigned short)c, v};
      else {
        vis_out[slot] = sb::VisPair{r, -1, 0, c};
        vis_val[slot] = v;
      }
    }
    carry += chunk;
    __syncthreads();
  }
  if (tid == 0) *cnt = carry;
}
}  // namespace

extern "C" {

int sb200_sort_cost_matrix(int32_t positional_kind, float iou_threshold, float min_confidence, float pos_weight,
                           float vel_weight, const float* cand_boxes, int32_t m, const float* track_boxes,
                           const float* track_states30, int32_t n, float* out_mn, int32_t device) {
  if (m < 0 || n < 0 || (m > 0 && !cand_boxes) || (n > 0 && !track_boxes) || (m > 0 && n > 0 && !out_mn))
    return fail(SB200_ERR_INVALID, "bad arguments");
  if (positional_kind == SB200_POS_MAHA && n > 0 && !track_states30)
    return fail(SB200_ERR_INVALID, "track_states30 is required for the Mahalanobis metric");
  Scratch sc;
  int rc = begin(sc, device);
  if (rc) return rc;
  if (m == 0 || n == 0) return 0;
  sb::Params p = base_params();
  p.positional_kind = positional_kind;
  p.iou_threshold = iou_threshold;
  p.min_confidence = min_confidence;
  p.pos_weight = pos_weight;
  p.vel_weight = vel_weight;
  sb::TrackStore ts;
  memset(&ts, 0, sizeof(ts));
  ts.track_cap = n;
  ts.pred = sc.upload(track_boxes, (size_t)n * 6);
  ts.radius = sc.alloc<float>(n);
  ts.epoch = sc.alloc<unsigned int>(n);
  ts.vert = sc.alloc<double>((size_t)n * 8);
  ts.kst_stride = 30;
  ts.kst = track_states30 ? sc.upload(track_states30, (size_t)n * 30) : sc.alloc<float>((size_t)n * 30, true);
  sb::Frame f;
  memset(&f, 0, sizeof(f));
  f.total = m;
  f.in_boxes = sc.upload(cand_boxes, (size_t)m * 6);
  f.c_box = sc.alloc<float>((size_t)m * 6);
  f.c_radius = sc.alloc<float>(m);
  f.c_conf = sc.alloc<float>(m);
  f.c_vert = sc.alloc<double>((size_t)m * 8);
  f.pos = sc.alloc<float>((size_t)m * n);
  f.pos_total = (long long)m * n;
  f.pos_dense_all = true;               // the operator returns the dense matrix
  int* counters = sc.alloc<int>(sb::counter_ints(1), true);
  f.pos_list = sc.alloc<sb::PosEntry>(1);   // sparse list disabled here (capacity 0): only the dense matrix is returned
  sb::SceneDesc d;
  memset(&d, 0, sizeof(d));
  d.m = m; d.n = n; d.epoch = 1;
  f.scenes = sc.upload(&d, 1);
  if (sc.rc) return sc.rc;
  sb::carve_counters(counters, 1, f);
  f.screen_cnt = nullptr;   // the operators count nothing
  track_geom_kernel<<<(n + 127) / 128, 128, 0, sc.st>>>(positional_kind == SB200_POS_IOU, ts.pred, n, ts.radius, ts.vert, ts.epoch);
  sb::launch_prep(p, f, 1, m, sc.st);
  sb::launch_pos_cost(p, ts, f, 1, m, n, sc.st);
  cudaMemcpyAsync(out_mn, f.pos, (size_t)m * n * 4, cudaMemcpyDeviceToHost, sc.st);
  return finish(sc);
}

int sb200_visual_cost_matrix(int32_t visual_kind, float threshold, const float* cand_features, int32_t m,
                             const float* track_features, int32_t n, int32_t d, float* out_mn, int32_t device) {
  if (m < 0 || n < 0 || d <= 0 || (m > 0 && !cand_features) || (n > 0 && !track_features) || (m > 0 && n > 0 && !out_mn))
    return fail(SB200_ERR_INVALID, "bad arguments");
  Scratch sc;
  int rc = begin(sc, device);
  if (rc) return rc;
  if (m == 0 || n == 0) return 0;
  sb::Params p = base_params();
  p.is_visual = true;
  p.visual_kind = visual_kind;
  p.visual_threshold = threshold;
  p.feature_dim = d;
  p.d8 = (d + 7) / 8 * 8;
  p.vis_rel_err = sb::screen_rel_err(d);
  p.vis_rel_err8 = sb::screen_rel_err_fp8(d);
  p.vis_dense_f32 = sb::dense_f32_err(d);
  p.vis_sample_margin = sb::dense_sample_margin(d);
  p.max_obs = 1;
  p.min_track_length = 0;
  // track side: norms through the candidate-norm kernel on a scratch frame
  sb::Frame ft;
  memset(&ft, 0, sizeof(ft));
  ft.total = n;
  ft.in_feat = sc.upload(track_features, (size_t)n * d);
  ft.in_boxes = sc.alloc<float>((size_t)n * 6, true);
  ft.c_box = sc.alloc<float>((size_t)n * 6);
  ft.c_radius = sc.alloc<float>(n);
  ft.c_conf = sc.alloc<float>(n);
  ft.c_flags = sc.alloc<unsigned char>(n);
  ft.c_norm2 = sc.alloc<float>(n, true);
  sb::TrackStore ts;
  memset(&ts, 0, sizeof(ts));
  ts.track_cap = n;
  ts.pred = sc.alloc<float>((size_t)n * 6, true);
  ts.radius = sc.alloc<float>(n, true);
  ts.epoch = sc.alloc<unsigned int>(n, true);
  ts.feat = sc.alloc<float>((size_t)n * p.d8, true);
  ts.obs_phys = sc.alloc<unsigned char>(n, true);
  ts.obs_hasf = sc.alloc<unsigned char>(n);
  ts.obs_n = sc.alloc<unsigned char>(n);
  ts.feat_cnt = sc.alloc<unsigned char>(n);
  sb::Frame f;
  memset(&f, 0, sizeof(f));
  f.total = m;
  f.in_feat = sc.upload(cand_features, (size_t)m * d);
  f.in_boxes = sc.alloc<float>((size_t)m * 6, true);
  f.c_box = sc.alloc<float>((size_t)m * 6);
  f.c_radius = sc.alloc<float>(m);
  f.c_conf = sc.alloc<float>(m);
  f.c_flags = sc.alloc<unsigned char>(m);
  f.c_norm2 = sc.alloc<float>(m, true);
  f.vis = sc.alloc<float>((size_t)m * n);
  ts.fnorm2 = ft.c_norm2;
  // the tracker's path rule (sb_engine.cuh), except that the operator has no dense path, and no frames to learn the e4m3
  // screen's selectivity from: it screens on BF16 unless SB200_VIS_KERNEL=tc8 asks for e4m3 operands (d8 <= 512)
  sb::TcArgs tc;
  memset(&tc, 0, sizeof(tc));
  const sb::VisKernel vk = sb::vis_kernel_env();
  tc.use_tc = vk == sb::kVisTc || vk == sb::kVisTc8 || vk == sb::kVisTc16 ||
              (vk != sb::kVisSimt && sb::vis_selective(visual_kind == SB200_VIS_EUCLIDEAN, threshold) &&
               sb::vis_tc_worth(p.d8, (long long)m * n));
  tc.fp8 = vk == sb::kVisTc8 && p.d8 <= sb::kFp8MaxD8;
  cudaDeviceGetAttribute(&tc.num_sms, cudaDevAttrMultiProcessorCount, device);
  int lcap = std::max(4096, m * 64);
  if (const char* ev = getenv("SB200_VIS_PAIR_CAP")) lcap = std::max(1, atoi(ev));
  sb::SceneDesc sd;
  memset(&sd, 0, sizeof(sd));
  sd.m = m; sd.n = n; sd.nb = n; sd.epoch = 1;   // stateless operator: one observation per track, block == track
  sd.vis_lcap = lcap;
  f.scenes = sc.upload(&sd, 1);
  f.scene_max = sc.alloc<unsigned int>(1);
  f.vis_pairs = sc.alloc<sb::VisPair>((size_t)lcap);
  f.vis_val = sc.alloc<float>((size_t)lcap);
  int* counters = sc.alloc<int>(sb::counter_ints(1), true);
  f.pos_list = sc.alloc<sb::PosEntry>(1);
  // the candidates' operand rows join the frame after its launch_prep: the operator converts them with launch_to_* below,
  // and cand_norm_kernel would write them as well if it saw them
  unsigned char* c_fp8 = nullptr;
  float* c_scale = nullptr;
  unsigned short* c_bf16 = nullptr;
  if (tc.use_tc) {
    std::vector<sb::TcTile> tiles;
    tc.cstep = sb::vis_screen_ucols(p.d8, tc.num_sms, 1, &m, &n, 1);
    for (int m0 = 0; m0 < m; m0 += 256)
      for (int c0 = 0; c0 < n; c0 += tc.cstep) tiles.push_back(sb::TcTile{0, m0, c0, 0});
    tc.n_tiles = (int)tiles.size();
    tc.d_tiles = sc.upload(tiles.data(), tiles.size());
    tc.a_rows = m;
    tc.b_rows = n;
    if (tc.fp8) {
      const int p8 = sb::fp8_pitch(p.d8);
      c_fp8 = sc.alloc<unsigned char>((size_t)m * p8);
      c_scale = sc.alloc<float>(m);
      ts.feat_fp8 = sc.alloc<unsigned char>((size_t)n * p8);
      ts.fscale = sc.alloc<float>(n);
      tc.colsb = sc.alloc<float>(n + 256);
    } else {
      c_bf16 = sc.alloc<unsigned short>((size_t)m * p.d8);
      ts.feat_bf16 = sc.alloc<unsigned short>((size_t)n * p.d8);
    }
    tc.colmeta = sc.alloc<sb::VisColMeta>(n + 256);   // the screen kernel bulk-copies whole 256-column slabs
    tc.colgeo = sc.alloc<sb::VisColGeo>(n);
    tc.colb = sc.alloc<float>(n + 256);
    tc.colvalid = sc.alloc<unsigned int>((n + 256) / 32 + 4);
    tc.rowmeta = sc.alloc<sb::VisRowMeta>(m + 256);
    tc.total_cols = n;
  }
  if (sc.rc) return sc.rc;
  sb::carve_counters(counters, 1, f);
  f.screen_cnt = nullptr;   // the operators count nothing
  sb::launch_prep(p, ft, 1, n, sc.st);
  cudaMemcpy2DAsync(ts.feat, (size_t)p.d8 * 4, ft.in_feat, (size_t)d * 4, (size_t)d * 4, n, cudaMemcpyDeviceToDevice, sc.st);
  fill_u8_kernel<<<(n + 255) / 256, 256, 0, sc.st>>>(ts.obs_hasf, 1, n);
  fill_u8_kernel<<<(n + 255) / 256, 256, 0, sc.st>>>(ts.obs_n, 1, n);
  fill_u8_kernel<<<(n + 255) / 256, 256, 0, sc.st>>>(ts.feat_cnt, 1, n);
  sb::launch_prep(p, f, 1, m, sc.st);
  fill_u8_kernel<<<(m + 255) / 256, 256, 0, sc.st>>>(f.c_flags, 3, m);
  f.c_fp8 = c_fp8;
  f.c_scale = c_scale;
  f.c_bf16 = c_bf16;
  if (tc.use_tc) {
    // (the tracker fuses these into cand_norm_kernel and feat_store_kernel)
    if (tc.fp8) {
      sb::launch_to_fp8(static_cast<const float*>(ft.in_feat), d, d, p.d8, n, ts.feat_fp8, ts.fscale, sc.st);
      sb::launch_to_fp8(static_cast<const float*>(f.in_feat), d, d, p.d8, m, f.c_fp8, f.c_scale, sc.st);
    } else {
      sb::launch_to_bf16(static_cast<const float*>(ft.in_feat), d, d, p.d8, n, ts.feat_bf16, sc.st);
      sb::launch_to_bf16(static_cast<const float*>(f.in_feat), d, d, p.d8, m, f.c_bf16, sc.st);
    }
  }
  int vr = sb::launch_vis_cost(p, ts, f, 1, m, n, tc, sc.st);
  if (vr == 0 && tc.use_tc) sb::launch_vis_densify(p, f, 1, sc.st);
  if (vr != 0) return fail(SB200_ERR_CUDA, "visual cost launch failed");
  cudaMemcpyAsync(out_mn, f.vis, (size_t)m * n * 4, cudaMemcpyDeviceToHost, sc.st);
  return finish(sc);
}

static int run_voting(bool visual, float threshold, int min_votes, const float* pos_mn, const float* vis_mnk, int m, int n,
                      int k, int32_t* winner, uint8_t* voting_type, int device) {
  if (m < 0 || n < 0 || (m > 0 && !winner) || (m > 0 && n > 0 && !pos_mn)) return fail(SB200_ERR_INVALID, "bad arguments");
  if (visual && (k < 1 || k > sb::kMaxObsWide || (m > 0 && n > 0 && !vis_mnk))) return fail(SB200_ERR_INVALID, "bad arguments");
  // Which voting kernel runs: by default the tracker's rule (the sparse kernel on the entry lists unless a list exceeds
  // its capacity); SB200_VOTE_KERNEL=dense|sparse|prepass forces one, so that a test can hand each kernel the matrix of
  // its choosing.  A forced kernel the rule would not allow is an error, never a silent switch to the other one.
  enum { kRule, kDense, kSparse, kPrepass } want = kRule;
  if (const char* ev = getenv("SB200_VOTE_KERNEL")) {
    if (!strcmp(ev, "dense")) want = kDense;
    else if (!strcmp(ev, "sparse")) want = kSparse;
    else if (!strcmp(ev, "prepass")) want = kPrepass;
    else if (*ev) return fail(SB200_ERR_INVALID, "SB200_VOTE_KERNEL must be dense, sparse or prepass");
  }
  if (want == kPrepass && !visual) return fail(SB200_ERR_INVALID, "SB200_VOTE_KERNEL=prepass applies to visual voting only");
  Scratch sc;
  int rc = begin(sc, device);
  if (rc) return rc;
  if (m == 0) return 0;
  sb::Params p = base_params();
  p.positional_kind = SB200_POS_IOU;  // threshold is taken verbatim: (threshold * 1e6) as i64
  p.iou_threshold = threshold;
  p.is_visual = visual;
  p.max_obs = visual ? k : 1;
  p.min_votes = min_votes;
  p.vote_vis_cap = sb::kVoteVisCap;
  sb::TrackStore ts;
  memset(&ts, 0, sizeof(ts));
  ts.track_cap = n;
  sb::Frame f;
  memset(&f, 0, sizeof(f));
  f.total = m;
  f.pos = sc.upload(pos_mn, (size_t)m * n);
  if (visual) f.vis = sc.upload(vis_mnk, (size_t)m * n * k);
  f.winner = sc.alloc<int>(m);
  f.c_vt = sc.alloc<unsigned char>(m);
  f.new_count = sc.alloc<int>(1);
  // the counters, zero but for scene mode 1 until the rule below runs: the scene-maximum reduction skips sparse scenes
  // (the tracker's refinement reduces their maximum), and the operator has no refinement
  std::vector<int> counters(sb::counter_ints(1), 0);
  sb::carve_counters(counters.data(), 1, f);
  *f.scene_mode = *f.vis_mode = 1;
  int* d_counters = sc.upload(counters.data(), counters.size());
  // one scene, list slices sized as the tracker sizes them
  sb::SceneDesc sd;
  memset(&sd, 0, sizeof(sd));
  sd.m = m; sd.n = n; sd.epoch = 1;
  sd.pos_lcap = sb::pos_lcap(m);
  sd.vis_lcap = visual ? sb::vis_lcap(m, sb::kVoteVisCap) : 0;
  f.scenes = sc.upload(&sd, 1);
  f.pos_list = sc.alloc<sb::PosEntry>(sd.pos_lcap);
  if (visual) {
    f.vis_pairs = sc.alloc<sb::VisPair>(sd.vis_lcap);
    f.vis_val = sc.alloc<float>(sd.vis_lcap);
    f.scene_max = sc.alloc<unsigned int>(1);
  }
  if (want == kPrepass) {
    f.decided = sc.alloc<unsigned char>(m);
    f.excl = sc.alloc<unsigned char>(n);
    f.pre_winner = sc.alloc<int>(m);
  }
  if (sc.rc) return sc.rc;
  sb::carve_counters(d_counters, 1, f);
  f.screen_cnt = nullptr;   // the operators count nothing
  f.dense_cnt = nullptr;    // ... and voting has no dense visual kernel that the count would let leave early
  vote_list_kernel<<<1, kListThreads, 0, sc.st>>>(f.pos, m, n, sd.pos_lcap, f.pos_list, nullptr, nullptr, f.pos_cnt);
  if (visual) vote_list_kernel<<<1, kListThreads, 0, sc.st>>>(f.vis, m, n * k, sd.vis_lcap, nullptr, f.vis_pairs, f.vis_val, f.vis_cnt);
  if (visual) {
    sb::launch_scene_max(p, f, 1, /*init_only=*/true, sc.st);
    if (n > 0) sb::launch_scene_max(p, f, 1, /*init_only=*/false, sc.st);
  }
  if (want != kDense) {
    // the tracker's rule, with the list capacities above and the sparse visual lists of its tensor-core path
    sb::launch_vis_mode(p, f, 1, /*tc_used=*/true, sc.st);
    sb::launch_scene_mode(p, f, 1, /*tc_used=*/true, sc.st);
  }
  if (want == kSparse || want == kPrepass) {
    int mode = 1;
    cudaMemcpyAsync(&mode, f.scene_mode, sizeof(int), cudaMemcpyDeviceToHost, sc.st);
    if ((rc = finish(sc))) return rc;
    if (mode != 0)
      return fail(SB200_ERR_CAPACITY, "SB200_VOTE_KERNEL: the entry lists exceed the sparse voting kernel's capacity");
  }
  if (want == kPrepass) {
    // the tracker's lazy positional stage: BestFit pre-pass, then the full pass reuses its decisions
    int vr = sb::launch_vote_masks(p, ts, f, 1, m, n, sc.st);
    if (vr == -3) return fail(SB200_ERR_CAPACITY, "scene too large for the on-chip assignment solver");
    if (vr != 0) return fail(SB200_ERR_CUDA, "voting launch failed: %s", cudaGetErrorString((cudaError_t)vr));
  }
  int vr = sb::launch_voting(p, ts, f, 1, m, n, sc.st);
  if (vr == -3) return fail(SB200_ERR_CAPACITY, "scene too large for the on-chip assignment solver");
  if (vr != 0) return fail(SB200_ERR_CUDA, "voting launch failed: %s", cudaGetErrorString((cudaError_t)vr));
  cudaMemcpyAsync(winner, f.winner, (size_t)m * 4, cudaMemcpyDeviceToHost, sc.st);
  if (voting_type) cudaMemcpyAsync(voting_type, f.c_vt, (size_t)m, cudaMemcpyDeviceToHost, sc.st);
  return finish(sc);
}

int sb200_sort_voting(float threshold, const float* cost_mn, int32_t m, int32_t n, int32_t* winner, int32_t device) {
  return run_voting(false, threshold, 0, cost_mn, nullptr, m, n, 1, winner, nullptr, device);
}

int sb200_visual_voting(float positional_threshold, int32_t min_votes, const float* pos_mn, const float* vis_mnk,
                        int32_t m, int32_t n, int32_t k, int32_t* winner, uint8_t* voting_type, int32_t device) {
  return run_voting(true, positional_threshold, min_votes, pos_mn, vis_mnk, m, n, k, winner, voting_type, device);
}

int sb200_own_area_shares(const float* boxes, int32_t n, float* out, int32_t device) {
  if (n < 0 || (n > 0 && (!boxes || !out))) return fail(SB200_ERR_INVALID, "bad arguments");
  Scratch sc;
  int rc = begin(sc, device);
  if (rc) return rc;
  if (n == 0) return 0;
  sb::Frame f;
  memset(&f, 0, sizeof(f));
  f.total = n;
  sb::SceneDesc sd;
  memset(&sd, 0, sizeof(sd));
  sd.m = n;
  f.scenes = sc.upload(&sd, 1);
  f.status = sc.alloc<int>(1, true);
  float* d_boxes = sc.upload(boxes, (size_t)n * 6);
  float* d_out = sc.alloc<float>(n);
  int* d_ovf_cnt = sc.alloc<int>(1);
  int2* d_ovf = sc.alloc<int2>(n);
  if (sc.rc) return sc.rc;
  sb::launch_own_area(f, 1, n, d_boxes, d_out, d_ovf_cnt, d_ovf, sc.st);
  int status = 0;
  cudaMemcpyAsync(out, d_out, (size_t)n * 4, cudaMemcpyDeviceToHost, sc.st);
  cudaMemcpyAsync(&status, f.status, sizeof(int), cudaMemcpyDeviceToHost, sc.st);
  rc = finish(sc);
  if (rc) return rc;
  if (status & 2) return fail(SB200_ERR_CAPACITY, "more than 2800 boxes overlap one box (own-area shares)");
  return 0;
}

static int kalman_op(int op, float pw, float vw, const float* in30, const float* boxes, int n, float* out30, int device) {
  if (n < 0 || (n > 0 && !out30) || (op != 0 && n > 0 && !in30) || (op != 1 && n > 0 && !boxes)) return fail(SB200_ERR_INVALID, "bad arguments");
  Scratch sc;
  int rc = begin(sc, device);
  if (rc) return rc;
  if (n == 0) return 0;
  float* din = in30 ? sc.upload(in30, (size_t)n * 30) : nullptr;
  float* db = boxes ? sc.upload(boxes, (size_t)n * 6) : nullptr;
  float* dout = sc.alloc<float>((size_t)n * 30);
  if (sc.rc) return sc.rc;
  sb::launch_kalman_ops(op, pw, vw, din, db, n, dout, sc.st);
  cudaMemcpyAsync(out30, dout, (size_t)n * 120, cudaMemcpyDeviceToHost, sc.st);
  return finish(sc);
}
int sb200_kalman_initiate(float pw, float vw, const float* boxes, int32_t n, float* states30, int32_t device) {
  return kalman_op(0, pw, vw, nullptr, boxes, n, states30, device);
}
int sb200_kalman_predict(float pw, float vw, const float* in30, int32_t n, float* out30, int32_t device) {
  return kalman_op(1, pw, vw, in30, nullptr, n, out30, device);
}
int sb200_kalman_update(float pw, float vw, const float* in30, const float* boxes, int32_t n, float* out30, int32_t device) {
  return kalman_op(2, pw, vw, in30, boxes, n, out30, device);
}

// Universal2DBoxKalmanFilter::distance, src/utils/kalman/kalman_2d_box.rs:150-170
int sb200_kalman_distance(float pw, float vw, const float* states30, const float* boxes, int32_t n, float* out,
                          int32_t device) {
  (void)vw;   // the distance reads only the position weight (project, :104-120)
  if (n < 0 || (n > 0 && (!states30 || !boxes || !out))) return fail(SB200_ERR_INVALID, "bad arguments");
  Scratch sc;
  int rc = begin(sc, device);
  if (rc) return rc;
  if (n == 0) return 0;
  float* din = sc.upload(states30, (size_t)n * 30);
  float* db = sc.upload(boxes, (size_t)n * 6);
  float* dout = sc.alloc<float>(n);
  if (sc.rc) return sc.rc;
  sb::launch_kalman_distance(pw, din, db, n, dout, sc.st);
  cudaMemcpyAsync(out, dout, (size_t)n * 4, cudaMemcpyDeviceToHost, sc.st);
  return finish(sc);
}

// op as launch_point_kalman: 0 initiate, 1 predict, 2 update, 3 distance
static int point_kalman_op(int op, float pw, float vw, const float* in12, const float* points, int n, float* out,
                           int device) {
  const bool need_in = op != 0, need_pts = op != 1;
  if (n < 0 || (n > 0 && (!out || (need_in && !in12) || (need_pts && !points))))
    return fail(SB200_ERR_INVALID, "bad arguments");
  Scratch sc;
  int rc = begin(sc, device);
  if (rc) return rc;
  if (n == 0) return 0;
  const size_t out_floats = op == 3 ? (size_t)n : (size_t)n * 12;
  float* din = need_in ? sc.upload(in12, (size_t)n * 12) : nullptr;
  float* dp = need_pts ? sc.upload(points, (size_t)n * 2) : nullptr;
  float* dout = sc.alloc<float>(out_floats);
  if (sc.rc) return sc.rc;
  sb::launch_point_kalman(op, pw, vw, din, dp, n, dout, sc.st);
  cudaMemcpyAsync(out, dout, out_floats * 4, cudaMemcpyDeviceToHost, sc.st);
  return finish(sc);
}
// Point2DKalmanFilter::initiate, src/utils/kalman/kalman_2d_point.rs:51-65
int sb200_point_kalman_initiate(float pw, float vw, const float* points2, int32_t n, float* states12, int32_t device) {
  return point_kalman_op(0, pw, vw, nullptr, points2, n, states12, device);
}
// Point2DKalmanFilter::predict, src/utils/kalman/kalman_2d_point.rs:67-84
int sb200_point_kalman_predict(float pw, float vw, const float* in12, int32_t n, float* out12, int32_t device) {
  return point_kalman_op(1, pw, vw, in12, nullptr, n, out12, device);
}
// Point2DKalmanFilter::update, src/utils/kalman/kalman_2d_point.rs:103-121
int sb200_point_kalman_update(float pw, float vw, const float* in12, const float* points2, int32_t n, float* out12,
                              int32_t device) {
  return point_kalman_op(2, pw, vw, in12, points2, n, out12, device);
}
// Point2DKalmanFilter::distance, src/utils/kalman/kalman_2d_point.rs:123-137
int sb200_point_kalman_distance(float pw, float vw, const float* states12, const float* points2, int32_t n, float* out,
                                int32_t device) {
  return point_kalman_op(3, pw, vw, states12, points2, n, out, device);
}

// Universal2DBox::get_vertices, src/utils/bbox.rs:169-171,287-330
int sb200_box_vertices(const float* boxes, int32_t n, double* out8, int32_t device) {
  if (n < 0 || (n > 0 && (!boxes || !out8))) return fail(SB200_ERR_INVALID, "bad arguments");
  Scratch sc;
  int rc = begin(sc, device);
  if (rc) return rc;
  if (n == 0) return 0;
  float* db = sc.upload(boxes, (size_t)n * 6);
  double* dv = sc.alloc<double>((size_t)n * 8);
  if (sc.rc) return sc.rc;
  sb::launch_box_vertices(db, n, dv, sc.st);
  cudaMemcpyAsync(out8, dv, (size_t)n * 64, cudaMemcpyDeviceToHost, sc.st);
  return finish(sc);
}

// sutherland_hodgman_clip_py + intersection_area_py, src/utils/clipping/clipping_py.rs:29-46
int sb200_clip_polygons(const float* subjects, const float* clippings, int32_t n, double* out_vertices,
                        int32_t* out_counts, double* out_areas, int32_t device) {
  if (n < 0 || (n > 0 && (!subjects || !clippings || !out_vertices || !out_counts || !out_areas)))
    return fail(SB200_ERR_INVALID, "bad arguments");
  Scratch sc;
  int rc = begin(sc, device);
  if (rc) return rc;
  if (n == 0) return 0;
  const size_t nv = (size_t)n * sb::kMaxPoly * 2;
  float* ds = sc.upload(subjects, (size_t)n * 6);
  float* dc = sc.upload(clippings, (size_t)n * 6);
  double* dv = sc.alloc<double>(nv, true);
  int* dn = sc.alloc<int>(n);
  double* da = sc.alloc<double>(n);
  int* dst = sc.alloc<int>(1, true);
  if (sc.rc) return sc.rc;
  sb::launch_clip_polygons(ds, dc, n, dv, dn, da, dst, sc.st);
  int status = 0;
  cudaMemcpyAsync(&status, dst, sizeof(int), cudaMemcpyDeviceToHost, sc.st);
  rc = finish(sc);
  if (rc) return rc;
  if (status & 1) return fail(SB200_ERR_CAPACITY, "a clipped polygon would have more than 16 vertices");
  // outputs are written only when every pair fits
  cudaMemcpy(out_vertices, dv, nv * sizeof(double), cudaMemcpyDeviceToHost);
  cudaMemcpy(out_counts, dn, (size_t)n * 4, cudaMemcpyDeviceToHost);
  cudaMemcpy(out_areas, da, (size_t)n * 8, cudaMemcpyDeviceToHost);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(SB200_ERR_CUDA, "CUDA error: %s", cudaGetErrorString(e));
  return 0;
}

// intersection_area_py (src/utils/clipping/clipping_py.rs:41-46) of every (a[i], b[j]) pair
int sb200_intersection_areas(const float* a, int32_t m, const float* b, int32_t n, double* out_mn, int32_t device) {
  if (m < 0 || n < 0 || (m > 0 && !a) || (n > 0 && !b) || (m > 0 && n > 0 && !out_mn))
    return fail(SB200_ERR_INVALID, "bad arguments");
  Scratch sc;
  int rc = begin(sc, device);
  if (rc) return rc;
  if (m == 0 || n == 0) return 0;
  float* da = sc.upload(a, (size_t)m * 6);
  float* db = sc.upload(b, (size_t)n * 6);
  double* va = sc.alloc<double>((size_t)m * 8);
  double* vb = sc.alloc<double>((size_t)n * 8);
  double* dout = sc.alloc<double>((size_t)m * n);
  int* dst = sc.alloc<int>(1, true);
  if (sc.rc) return sc.rc;
  sb::launch_box_vertices(da, m, va, sc.st);
  sb::launch_box_vertices(db, n, vb, sc.st);
  sb::launch_intersection_areas(va, m, vb, n, dout, dst, sc.st);
  int status = 0;
  cudaMemcpyAsync(&status, dst, sizeof(int), cudaMemcpyDeviceToHost, sc.st);
  rc = finish(sc);
  if (rc) return rc;
  if (status & 1) return fail(SB200_ERR_CAPACITY, "a clipped polygon would have more than 16 vertices");
  cudaError_t e = cudaMemcpy(out_mn, dout, (size_t)m * n * sizeof(double), cudaMemcpyDeviceToHost);
  if (e != cudaSuccess) return fail(SB200_ERR_CUDA, "CUDA error: %s", cudaGetErrorString(e));
  return 0;
}

}  // extern "C"
