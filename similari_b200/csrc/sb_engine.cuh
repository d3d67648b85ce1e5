// sb_engine.cuh -- device data layout and kernel launch interfaces of the association engine.
//
// HBM layout (all arrays allocated once per tracker and grown by doubling):
//   track store   : dense per scene slot, index = slot * track_cap + j, j in [0, n_tracks[slot]) in store order
//                   (insertion order; wasted tracks are removed by a stable compaction).  Array-of-structs rows
//                   of 6 / 30 floats so that a tile of tracks is one contiguous, fully coalesced block copy.
//   features      : [slot][track][physical obs slot][D8] f32, D8 = D rounded up to 8 lanes (Feature::from_vec
//                   zero-padding, src/track/utils.rs:45-71); the logical observation order of
//                   VisualMetric::optimize (src/trackers/visual_sort/metric.rs:297-374) is a per-track
//                   permutation (obs_phys) so feature rows never move.
//   per frame     : candidates in request order; cost matrices packed per scene (row-major m x n, and
//                   m x n x K for visual distances), NaN == None.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <cstdlib>
#include <cstring>

#include "sb_math.cuh"

namespace sb {

constexpr int kMaxConstraints = 8;
constexpr int kNumSms = 132;  // H100 SXM: grid sizes of the launches that do not query the device
// gridDim.y and gridDim.z stop at 65,535, and a request's scene count has no bound: a launch with one scene per y (or z)
// index takes at most this many and its kernel strides over the scenes
constexpr int kMaxGridYZ = 65535;
inline unsigned int scene_grid(int n_scenes) { return (unsigned int)(n_scenes < kMaxGridYZ ? n_scenes : kMaxGridYZ); }
constexpr int kMaxObs = 8;  // visual_max_observations the per-thread kernels keep in registers (reference default 5)
constexpr int kMaxObsWide = 32;  // visual_max_observations supported on device: above kMaxObs, one warp lane per observation
constexpr int kStateStride = 32;   // floats per Kalman state row in the tracker's store (kStateFloats padded to 128 bytes)
constexpr int kMaxHist = 64;  // box history kept per track on the device (history_length above it, or 0 = unlimited, is capped)

// BF16 operand rounding bound on a dot product of width d, relative to ||a|| ||b||.  BF16 keeps 8 significant bits;
// round-to-nearest leaves a relative error of at most u = 2^-8 per operand (a value just above a power of two sits half a
// 2^-7 spacing from its neighbours).  Two rounded operands: |a~ b~ - a b| <= (2u + u^2) |a b|, hence by Cauchy-Schwarz
//   |dot~ - dot| <= (2^-7 + 2^-16) * sum|a_i b_i| <= (2^-7 + 2^-16) * ||a|| ||b||.
// Products of BF16 operands are exact in fp32.  The fp32 accumulation of the tensor cores is modelled as one truncation per
// addition, at most d * 2^-23 relative to sum|a_i b_i|; that model has not been measured on the H100.  The slack is
// 2.1 * 2^-8, which covers 2^-7 + 2^-16 + d * 2^-23 up to d = 3148, and that sum for wider features.  (1.5 * 2^-8 would
// cover the rounding errors of real feature vectors, which average out, but not the adversarial worst case -- the screen
// must never drop a pair the exact metric keeps.)
inline float screen_rel_err(int d) {
  const double e = 0x1p-7 + 0x1p-16 + (double)d * 0x1p-23;
  const float floor_e = 2.1f / 256.0f;
  return e <= (double)floor_e ? floor_e : (float)(e * (1.0 + 0x1p-20));   // rounded up past the f32 conversion
}

// The same bound for the e4m3 screen (FP8 operands, fp32 accumulation), relative to ||a|| ||b|| of the UNSCALED rows.  Each
// row r is stored as x~ = e4m3(2^k_r x) with 2^k_r the power of two that puts max|x| in [224, 448) (fp8_row_scale): the
// scaling is exact and saturation cannot occur, so only the e4m3 rounding and the accumulation add error.
//   1. Operand rounding.  e4m3 keeps 4 significant bits: for a normal value |x~ - x| <= u |x|, u = 2^-4.  As above,
//      sum |a~_i b~_i - a_i b_i| <= (2u + u^2) sum|a_i b_i| for the normal part.
//   2. Subnormal floor.  Below 2^-6 the spacing is 2^-9, so |x~ - x| <= 2^-10 in scaled units.  Its share of the dot product
//      is at most 2^-10 (1 + u) (sum|a_i| + sum|b_i|) + d 2^-20 <= 2^-10 (1 + u) sqrt(d) (||a|| + ||b||) + d 2^-20; both
//      scaled norms are >= max|x| >= 224, so relative to ||a|| ||b|| it is <= 2 (1 + u) sqrt(d) 2^-10 / 224 + d 2^-20 / 224^2.
//   3. Accumulation.  Products of e4m3 values are exact in fp32.  The FP8 tensor cores of the H100 are publicly reported to
//      keep only about 14 bits when they add a k32 group of products to the accumulator.  Model (one bit narrower than
//      the hardware): every k32 step aligns its 32 products and the accumulator to the largest of them and truncates each
//      to 13 significant bits, then rounds the sum.  tests/gpu_probe/fp8_wgmma_probe.cu measures it on an H100 (80 GB): an
//      accumulator of 2^16 keeps a next-step product of 8 and drops one of 4 (14 bits), and on the constructions of
//      tests/screen_fp8_constructions.py the error stays below 10.6 * 2^-12 of the largest step term per k32 step.  Each of
//      those 34 operations errs by less than 2^-12 of the step's largest
//      term, which is at most sum|a~_i b~_i| <= (1 + u)^2 ||a|| ||b|| (plus the floor, covered by the 1.01 below), so
//      ceil(d / 32) steps add at most ceil(d / 32) * 34 * 2^-12 * (1 + u)^2 * 1.01.
// At d = 512 the sum is 0.129 + 0.0003 + 0.150 = 0.280: on unit-norm features the Euclidean screen keeps d <= 0.7 pairs
// up to d~ = sqrt(0.49 + 2 E) ~ 1.04, the cosine screen keeps cos >= thr pairs down to cos~ = thr - 0.28.  Selective enough
// for thresholds in the tail of the distance distribution; where it is not, the tracker goes back to the BF16 screen.
inline float screen_rel_err_fp8(int d) {
  const double u = 0x1p-4;
  const double rnd = 2.0 * u + u * u;
  const double sub = 2.0 * (1.0 + u) * __builtin_sqrt((double)d) * 0x1p-10 / 224.0 + (double)d * 0x1p-20 / (224.0 * 224.0);
  const double acc = (double)((d + 31) / 32) * 34.0 * 0x1p-12 * (1.0 + u) * (1.0 + u) * 1.01;
  return (float)((rnd + sub + acc) * (1.0 + 0x1p-20));   // rounded up past the f32 conversion
}

// The f32 part of the dense path's error bound (kernels_feat_dense.cu dense_err), as a function of the width d.  The dense
// path compares x~ = |a|^2 + |b|^2 - 2 dot~ (f32 norms of cand_norm_kernel, BF16 tensor-core dot) with the reference's f32
// squared distance acc = sum over 8-lane blocks of reduce_add8((a - b)^2), blocks added in order (src/distance.rs), relative
// to N = |a|^2 + |b|^2; under cosine it compares 1 - dot~ rsqrt(|a|^2) rsqrt(|b|^2) with 1 - divided / sqrt(f1 f2)
// absolutely.  The BF16 operands and the tensor-core accumulation are screen_rel_err's; this is everything else.  With
// u = 2^-24, g(k) = k u / (1 - k u) and n8 = ceil(d / 8) blocks, a term that passes k roundings errs by at most g(k) of its
// magnitude (Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed., Lemma 3.1):
//   1. Norms.  A square is rounded once, the block tree adds three roundings, the blocks are added in order (n8 - 1): each
//      term of |a|^2 passes n8 + 3 roundings, |na - |a|^2| <= g(n8 + 3) |a|^2, and the two norms together g(n8 + 3) N.
//   2. The reference.  a - b, its square (twice the first rounding) and the same n8 + 2 additions: n8 + 5 roundings of
//      terms that sum to |a - b|^2 <= 2 N, so |acc - |a - b|^2| <= 2 g(n8 + 5) N.  Cosine: divided errs by g(n8 + 3)
//      sum|a_i b_i| <= g(n8 + 3) |a||b|, its norms f1, f2 by g(n8 + 3) each, and so do the kernel's norms: 3 g(n8 + 3).
//   3. Forming x~ (a sum and an fma on values <= 2.1 N) and the bound (f32 products of the f32 norms, themselves low by up
//      to g(n8 + 3)): 8 u N.  Cosine: two rsqrtf (2 ulp = 4 u each), two products, the subtraction from 1 and the
//      reference's product, square root and division: 15 u.
// Both metrics stay below g(3 n8 + 24) <= (3 n8 + 24) u (1 + 2^-8) for d <= kDenseMaxD = 2^16 (k u <= 2^-9 there).  The
// factor 1 + 2^-5 leaves room for the share of the BF16 term the kernel under-counts because it scales E by the f32
// norms: E g(n8 + 6) N, with E = screen_rel_err(d) <= 2^-6 + 2^-16 up to kDenseMaxD, is below 0.03 (3 n8 + 24) u N.
// That is 1.3e-5 at d = 512 and 1.9e-4 at d = 8192; the path has always budgeted 2e-4, which the function keeps as a
// floor, so it changes the bound only above d ~ 8900.  Wider than kDenseMaxD no bound is proven here: +inf keeps the
// tracker off the dense path (engine.cu).
constexpr int kDenseMaxD = 1 << 16;
inline float dense_f32_err(int d) {
  if (d > kDenseMaxD) return __builtin_inff();
  const double n8 = (double)((d + 7) / 8);
  const double e = (3.0 * n8 + 24.0) * 0x1p-24 * (1.0 + 0x1p-5);
  return e <= 2e-4 ? 2e-4f : (float)(e * (1.0 + 0x1p-20));   // rounded up past the f32 conversion
}

// Margin of the dense path's sampled lower bound of the scene's maximal distance (vis_dense_sample_kernel): a sampled
// pair's distance, computed with a lane-strided f32 FMA dot product, minus margin * N (Euclidean) or margin (cosine) must
// not exceed the reference's value for that pair, or the max-candidate list could miss the true maximum.  The sampled
// value uses the same f32 norms as above (1.: g(n8 + 3) N) against the same reference (2.: 2 g(n8 + 5) N), and its dot
// product: every lane adds ceil(d / 32) products by fma (one rounding each), five butterfly additions join the lanes, so
// |dot_s - dot| <= g(ceil(d / 32) + 5) sum|a_i b_i| and 2 |dot_s - dot| <= g(ceil(d / 32) + 5) N.  Forming the sample and
// subtracting the margin: 8 u N.  Cosine: dot_s, divided and both pairs of norms (g(ceil(d / 32) + 5) + 3 g(n8 + 3)), the
// rsqrtf and the reference's quotient as above, 17 u.  So (3 n8 + ceil(d / 32) + 32) u (1 + 2^-5), about 13 d / 32 u:
// 1.5e-5 at d = 512, 1.04e-4 at d = 4096, 2.1e-4 at d = 8192.  The path has always subtracted 1e-4, kept as the floor.
inline float dense_sample_margin(int d) {
  if (d > kDenseMaxD) return __builtin_inff();
  const double n8 = (double)((d + 7) / 8), n32 = (double)((d + 31) / 32);
  const double e = (3.0 * n8 + n32 + 32.0) * 0x1p-24 * (1.0 + 0x1p-5);
  return e <= 1e-4 ? 1e-4f : (float)(e * (1.0 + 0x1p-20));
}

// Rows whose squared norm lies outside [2^-60, 2^60] (zero, tiny, huge, inf or NaN features) keep every pair in the e4m3
// screen: the exact pass decides.  Inside that range max|x| lies in [2^-35, 2^30], the scale 2^k_r is a normal float and
// the folded screen constants neither overflow nor lose bits to subnormals.
__host__ __device__ __forceinline__ bool fp8_norm_ok(float n2) { return n2 >= 0x1p-60f && n2 <= 0x1p60f; }
// 2^k with max|x| * 2^k in [224, 448), exact; 1 for a row without a usable maximum (such rows fail fp8_norm_ok)
__host__ __device__ __forceinline__ float fp8_row_scale(float amax) {
  if (!(amax >= 0x1p-100f && amax <= 0x1p100f)) return 1.0f;
  int e = 0;
  const float m = frexpf(amax, &e);   // amax = m 2^e, m in [0.5, 1)
  return ldexpf(1.0f, (m >= 0.875f ? 8 : 9) - e);
}
// bytes per row of the e4m3 copies: d8 rounded up to 16 (the tensor maps need 16-byte row pitches)
__host__ __device__ __forceinline__ int fp8_pitch(int d8) { return (d8 + 15) & ~15; }

// 4 consecutive values of a row -> their e4m3 bytes of s x (cvt.rn.satfinite.e4m3x2.f32: round to nearest even)
__device__ __forceinline__ unsigned int fp8_pack4(float a, float b, float c, float d, float s) {
  const unsigned int lo = __nv_cvt_float2_to_fp8x2(make_float2(a * s, b * s), __NV_SATFINITE, __NV_E4M3);
  const unsigned int hi = __nv_cvt_float2_to_fp8x2(make_float2(c * s, d * s), __NV_SATFINITE, __NV_E4M3);
  return lo | (hi << 16);
}
// the same for 8 values
__device__ __forceinline__ uint2 fp8_pack8(const float* x, float s) {
  return make_uint2(fp8_pack4(x[0], x[1], x[2], x[3], s), fp8_pack4(x[4], x[5], x[6], x[7], s));
}
// One warp, a row of d8 <= 512 values held as blocks lane and lane + 32 (x[h], zero past the row): writes the e4m3 copy
// to out (fp8_pitch(d8) bytes) and returns the row's scale.  NaN elements do not enter the maximum; such rows fail
// fp8_norm_ok and keep every pair.
__device__ __forceinline__ float fp8_row_store(const float (&x)[2][8], int d8, unsigned char* out) {
  const int lane = threadIdx.x & 31;
  float amax = 0.0f;
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int l = 0; l < 8; ++l) amax = fmaxf(amax, fabsf(x[h][l]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  const float s = fp8_row_scale(amax);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int blk = h * 32 + lane;
    if (blk * 8 < d8) *reinterpret_cast<uint2*>(out + blk * 8) = fp8_pack8(x[h], s);
  }
  return s;
}
// the same from a f32 row in memory (d values, zero padded to d8)
__device__ __forceinline__ float fp8_row_from(const float* src, int d, int d8, unsigned char* out) {
  const int lane = threadIdx.x & 31;
  float x[2][8];
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int l = 0; l < 8; ++l) {
      const int c = (h * 32 + lane) * 8 + l;
      x[h][l] = c < d ? src[c] : 0.0f;
    }
  return fp8_row_store(x, d8, out);
}

struct Params {  // immutable per tracker, passed by value to kernels
  int kind, positional_kind, visual_kind;
  float iou_threshold, min_confidence, pos_weight, vel_weight;
  int max_idle_epochs;
  int n_constraints;
  int constraint_epochs[kMaxConstraints];
  float constraint_max_dist[kMaxConstraints];
  float visual_threshold;
  float vis_rel_err;  // screen_rel_err(feature_dim): the BF16 slack of the tensor-core visual kernels
  float vis_rel_err8; // screen_rel_err_fp8(feature_dim): the slack of the e4m3 screen
  float vis_dense_f32;      // dense_f32_err(feature_dim): the f32 part of the dense path's bound
  float vis_sample_margin;  // dense_sample_margin(feature_dim): margin of the dense path's sampled maximal distance
  int feature_dim, d8, max_obs, min_votes, min_track_length;
  int vote_vis_cap;   // visual entries per scene the sparse voting kernel keeps in shared memory (0: kVoteVisCap)
  float min_area, min_quality_use, min_quality_collect, min_own_use, min_own_collect;
  bool is_visual, is_batch, use_own_area;
};

struct SceneDesc {  // one per scene of the current request
  int slot;        // scene slot in the track store
  int m;           // detections of this scene
  int n;           // stored tracks of this scene before this frame
  int det_base;    // first detection (row of the request)
  long long pos_off;  // offset of the m x n positional cost matrix
  long long vis_off;  // offset of the m x n x K visual matrix
  unsigned int epoch; // the scene's freshly incremented epoch (candidate epoch)
  int col_off;        // first entry of this scene in the per-frame column metadata (n * K physical feature rows)
  unsigned long long scene_id;
  int pos_lbase, pos_lcap;  // this scene's slice of the sparse positional entry list
  int vis_lbase, vis_lcap;  // this scene's slice of the visual survivor list
  int nb;             // feature blocks of this scene's arena in use (physical rows scanned by the screen = nb * K)
  int pad0;
  // dense tensor-core visual cost (kernels_feat_dense.cu) only:
  long long ws_off;   // first element of this scene's weight-sum matrix ws[block][candidate] (row pitch = m rounded up to 128)
  int blk_off;        // first entry of this scene in the per-block metadata (prefix of nb)
  int slab_off;       // first 256-column metadata slab of this scene (one slab per column tile)
};

// Host-written half of a scene descriptor.  The host knows the request (slot, detections, epoch, list slices) but -- with
// several frames in flight -- not how many tracks the scene's store holds when this frame runs; frame_setup_kernel joins
// the two on the device (n, nb, matrix / column / tile offsets) so that predict never waits for the previous frame.
struct SceneReq {
  int slot, m, det_base;
  unsigned int epoch;
  unsigned long long scene_id;
  int pos_lbase, pos_lcap, vis_lbase, vis_lcap;
};
struct FrameDyn {   // per-frame scalars only the device knows (written by frame_setup_kernel, read by later kernels)
  int n_tiles;            // tiles of the tensor-core visual cost kernel
  int total_cols;         // padded physical feature rows of all scenes (dense kernel: 256 x metadata slabs)
  int max_rows;           // max over the scenes of nb * K
  int max_n;              // max over the scenes of n
  long long pos_total;    // elements of the packed positional matrices
  long long vis_total;    // elements of the packed visual matrices
  unsigned long long units_mn;     // sum over the scenes of m * n   (pair-associations of this frame)
  unsigned long long units_rows;   // sum over the scenes of m * nb * K (dot products the visual cost kernel evaluates)
  long long live_total;   // sum over the scenes of n
  long long ws_total;     // elements of the dense kernel's weight-sum matrices
  int blk_total;          // arena blocks of all scenes
  int dense_scenes;       // scenes the dense exact kernels had to take (written late in the frame by scene_mode_kernel)
};

struct VisPair { int g, row, scene, outcol; };  // screen survivor: detection, feature row, scene, logical column
struct PosEntry { unsigned short m, n; float v; };  // one valid (candidate, track, cost) positional entry
constexpr int kVotePosCap = 3072;   // sparse entries per scene the voting kernel keeps in shared memory
constexpr int kVoteVisCap = 4096;   // power of two: the BestFit bitonic sort pads the list up to the next power of two

// Host side: the slices of a scene of m detections in the sparse entry lists (SceneDesc::pos_lcap / vis_lcap);
// vote_cap is the voting kernel's visual capacity (Params::vote_vis_cap).
inline int pos_lcap(int m) {
  const long long c = (long long)m * 32;
  return (int)(c < 2ll * kVotePosCap ? c : 2ll * kVotePosCap);
}
inline int vis_lcap(int m, int vote_cap) {
  const long long c = (long long)m * 64;
  return (int)(c < 4ll * vote_cap ? c : 4ll * vote_cap);
}
// Visual cost path, shared by the tracker and the operators.  The tensor-core screen and its exact refinement pay off for
// a selective threshold (one that can cut pairs) on rows of d8 >= 64 when the frame's dot products (`work`, pairs of
// candidate and stored feature row) reach 2^28 multiply-adds; smaller frames take the exact SIMT kernel.
inline bool vis_selective(bool euclidean, float threshold) { return euclidean ? threshold < 1e18f : threshold > -1.0f; }
inline bool vis_tc_worth(int d8, long long work) { return d8 >= 64 && work * d8 >= (1ll << 28); }
// SB200_VIS_KERNEL=simt|tc|tc8|tc16|dense forces a path (tc8 / tc16: the screen on e4m3 / BF16 operands); any other
// value, or none, leaves the choice to the rule.  Read on every call: tests switch it between calls.
enum VisKernel { kVisRule, kVisSimt, kVisTc, kVisTc8, kVisTc16, kVisDense };
inline VisKernel vis_kernel_env() {
  const char* e = getenv("SB200_VIS_KERNEL");
  if (!e) return kVisRule;
  if (!strcmp(e, "simt")) return kVisSimt;
  if (!strcmp(e, "tc")) return kVisTc;
  if (!strcmp(e, "tc8")) return kVisTc8;
  if (!strcmp(e, "tc16")) return kVisTc16;
  if (!strcmp(e, "dense")) return kVisDense;
  return kVisRule;
}

struct TrackStore {
  int track_cap;
  unsigned long long* id;
  unsigned int* epoch;
  unsigned int* length;
  long long* custom;
  signed char* vt;       // -1 == None
  float* pred;           // [idx][6] last predicted (posterior) box == observation attr box
  float* obs;            // [idx][6] last observed box
  float* radius;         // [idx]
  float* kst;            // [idx][kst_stride]: 30 state floats per track (8 mean + 8x8 covariance upper part ... see sb_math.cuh)
  int kst_stride;        // floats per row: 32 in the tracker's store (128-byte rows, 16-byte vector access), 30 for caller rows
  double* vert;          // [idx][8] vertex cache (IoU mode)
  // box history (SortAttributes::update_history, src/trackers/sort.rs:157-171): the last hist_len observed / predicted boxes
  // of every track as a ring, observation number j (0-based) in slot j % hist_len; null unless history_length > 1
  int hist_len;
  float* hist_pred;      // [idx][hist_len][6]
  float* hist_obs;       // [idx][hist_len][6]
  // visual
  float* feat;           // [idx][K][d8]
  void* feat_bf16;       // [idx][K][d8] bf16 copy of feat: B operand of the tensor-core screen
  unsigned char* feat_fp8;  // [idx][K][fp8_pitch(d8)] e4m3 copy of 2^k feat (d8 <= 512 only, else null): B operand of the e4m3 screen
  float* fscale;            // [idx][K] the row's 2^k (fp8_row_scale)
  float* fnorm2;         // [idx][K] by physical slot
  unsigned char* obs_phys;  // [idx][K] logical -> physical
  unsigned char* obs_hasf;  // [idx][K] logical: feature present
  float* obs_q;             // [idx][K] logical: quality
  unsigned char* obs_n;     // [idx]
  unsigned char* feat_cnt;  // [idx] visual_features_collected_count
  // Feature arena (tracker stores; null in the stateless operators, where block == track index).  A track owns one block
  // of K feature rows inside its scene's arena, feature row = (slot * track_cap + fblk[idx]) * K + physical slot.  The
  // small per-track arrays above are compacted (stably) whenever tracks expire; the feature rows never move: an expired
  // track's block goes to the scene's free list and is handed to the next new track.
  int* fblk;        // [idx] block of the track
  int* blk_owner;   // [slot * track_cap + block] track index j of the owner in current store order, -1: free
  int* blk_free;    // [slot * track_cap + i] free-list stack
  int* n_free;      // [slot]
  int* arena_top;   // [slot] blocks ever handed out (== live tracks + free blocks)
  // Feature history (VisualAttributes::update_history, src/trackers/visual_sort/track_attributes.rs:73-90): the input
  // feature of each of the last fhist_len observations, kept for the wasted tracks (sb200_wasted_visual).  One
  // tracker-wide pool of history blocks, not indexed by scene slot: block b = fhist_len rings of d8 floats plus a present
  // byte each, observation number j (0-based) in ring slot j % fhist_len.  A live track owns the block in hblk; when it
  // expires only the index moves into its wasted record (WastedBuf::hblk), and the host puts the block back on the free
  // list when the record leaves the wasted buffer.  All null (history off): the kernels take no extra memory traffic.
  int fhist_len;
  int* hblk;                // [idx] history block of the track
  float* hrows;             // [block][fhist_len][d8]
  unsigned char* hpresent;  // [block][fhist_len] the observation had a feature
  int* hfree;               // free-list stack of blocks
  int* hpool;               // [2] free blocks, blocks ever handed out (advanced once per frame by the sweep)
};

// first feature row of track `ti` (absolute store index) of scene slot `slot`, divided by K
__device__ __forceinline__ size_t feat_block(const TrackStore& ts, int slot, size_t ti) {
  return ts.fblk ? (size_t)slot * ts.track_cap + (size_t)ts.fblk[ti] : ti;
}

// Element type of the request's feature column (SB200_FEATURE_*).  The kernels that read the column are instantiated per
// type and widen each element where they load it; widening binary16 / bfloat16 to f32 is exact, so every later step sees
// the values of the widened f32 request.
constexpr int kFeatF32 = 0, kFeatF16 = 1, kFeatBF16 = 2;

// Widening from the bits, so that NaN payloads move as the IEEE widening (and numpy's astype) moves them: a binary16 NaN
// keeps its sign and its 10 payload bits in the top of the f32 payload; a bfloat16 is the top half of its f32.
__device__ __forceinline__ float widen_f16(unsigned int h) {
  if ((h & 0x7c00u) == 0x7c00u) return __uint_as_float(((h & 0x8000u) << 16) | 0x7f800000u | ((h & 0x3ffu) << 13));
  return __half2float(__ushort_as_half((unsigned short)h));   // finite values (subnormals included): exact
}
__device__ __forceinline__ float widen_bf16(unsigned int b) { return __uint_as_float(b << 16); }

__device__ __forceinline__ float feat_elem(const float* p, size_t i) { return p[i]; }
__device__ __forceinline__ float feat_elem(const __half* p, size_t i) {
  return widen_f16(reinterpret_cast<const unsigned short*>(p)[i]);
}
__device__ __forceinline__ float feat_elem(const __nv_bfloat16* p, size_t i) {
  return widen_bf16(reinterpret_cast<const unsigned short*>(p)[i]);
}
// the 8 elements of one 16-byte load of a 2-byte column, widened
__device__ __forceinline__ void feat_widen8(const uint4& r, const __half*, float* x) {
  const unsigned int w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) { x[2 * i] = widen_f16(w[i] & 0xffffu); x[2 * i + 1] = widen_f16(w[i] >> 16); }
}
__device__ __forceinline__ void feat_widen8(const uint4& r, const __nv_bfloat16*, float* x) {
  const unsigned int w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) { x[2 * i] = widen_bf16(w[i] & 0xffffu); x[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u); }
}
// Host side: calls fn(T{}) with T the element type of `type` (float, __half or __nv_bfloat16), so that a launcher can
// start the kernel instance of the frame's type.
template <class Fn>
inline void feat_dispatch(int type, Fn&& fn) {
  if (type == kFeatF16) fn(__half());
  else if (type == kFeatBF16) fn(__nv_bfloat16());
  else fn(float());
}

struct Frame {  // per-request transient device buffers (a request may be processed in scene chunks)
  int total;               // detections of this chunk
  int det0;                // first detection of this chunk (global row of the request)
  int scene0;              // first scene of this chunk (index into the request)
  int feat_type;           // element type of in_feat (kFeatF32 / kFeatF16 / kFeatBF16), fixed when the frame is enqueued
  const int* new_count_all;  // [all scenes of the request] (ids of non-batch trackers need the global prefix)
  long long pos_fill_off;  // offset of this chunk's positional matrices inside `pos`
  const float* in_boxes;   // [total][6] raw request boxes
  const void* in_feat;     // [total][D] elements of type feat_type, or null
  const unsigned char* in_hasf;
  const float* in_quality;
  const long long* in_custom;
  const float* in_own;
  float* c_box;            // [total][6] candidate (Kalman-normalised) boxes
  float* c_radius;
  float* c_conf;           // max(conf, min_confidence)
  double* c_vert;          // [total][8]
  unsigned char* c_flags;  // bit0 has feature, bit1 feature usable (feature_can_be_used with *_use thresholds)
  float* c_norm2;
  void* c_bf16;            // [total][d8] bf16 copy of the candidate features (A operand of the screen)
  unsigned char* c_fp8;    // [total][fp8_pitch(d8)] e4m3 copy of 2^k x (A operand of the e4m3 screen), or null
  float* c_scale;          // [total] the row's 2^k
  int* screen_cnt;         // [3] survivors refined, how many of them the exact test cut, scenes whose survivor list
                           // overflowed (null: not counted)
  unsigned int* scene_max; // [n_scenes] order-preserving encoding of best.rs "max_dist"
  int* winner;             // [total] track index within the scene or -1
  unsigned char* c_vt;     // voting type of the decision
  float* pos;              // packed positional cost matrices
  // The dense positional matrices are only materialised where somebody reads them: the stateless operators and
  // SB200_FULL_COSTS runs (pos_dense_all), and the scenes that fall back to the dense voting kernel (filled and scanned
  // again after scene_mode is known).  Everywhere else the per-scene entry list IS the cost matrix.
  bool pos_dense_all;
  long long pos_total;     // elements in `pos` this frame
  float* vis;              // packed visual matrices
  SceneDesc* scenes;       // [n_scenes]
  int* new_count;          // [n_scenes] new tracks per scene (written by voting)
  int* status;             // [n_scenes] per-scene status flags (capacity overflow etc.)
  int* feat_dst;           // [total] destination feature row (block*K + phys) or -1
  // Frames on the e4m3 screen leave the BF16 arena rows unwritten: only the BF16 screen and the dense path read them, and
  // the tracker converts the skipped rows again, in stream order, before the first frame or blob that does.
  bool skip_bf16;
  int* bf16_log;           // [total] with skip_bf16: feat_dst again, this frame's part of the tracker's dirty-row log
                           // (null: the log is full, every arena row gets converted)
  int* hist_dst;           // [total] destination history row (block*fhist_len + ring slot) or -1 (null: history off)
  int* app_row;            // [scenes][track_cap] apply phase 1: the detection that updates store row j of the scene, or -1
  int4* app_meta;          // [scenes] apply phase 1: (new tracks of earlier scenes, free blocks, arena top) before the frame,
                           // and the scene's store rows after it
  int* frame_out;          // [n_scenes][3] written by the end-of-frame sweep: live tracks, arena blocks, newly expired
  const FrameDyn* dyn;     // device-built frame scalars (null in the stateless operators: host values are used)
  unsigned long long* id_counter;   // device copy of the tracker's id counter (null: the id_base argument is used)
  long long id_add;        // ids this frame consumes when known up front (batch trackers: one per detection), else -1
  // sparse views of the (mostly None) cost matrices, consumed by the voting stage
  PosEntry* pos_list;      // valid positional entries, per-scene slices
  int* pos_cnt;            // [n_scenes]
  VisPair* vis_pairs;      // screen survivors, per-scene slices
  float* vis_val;          // exact value of each survivor (NaN == failed the threshold)
  int* vis_cnt;            // [n_scenes]
  int* scene_mode;         // [n_scenes] 0: voting consumes the sparse lists; 1: dense matrices (a list overflowed)
  int* vis_mode;           // [n_scenes] visual side alone (set right after the screen): 0 = the survivors get refined
  // Lazy positional stage of the visual trackers (null: every pair is evaluated).  VisualVoting (visual_sort/voting.rs:
  // 45-100) only lets the positional metric decide candidates the visual BestFit pass left undecided, against tracks it
  // did not claim; a BestFit pre-pass publishes both sets and the culled scan skips everything else.
  unsigned char* decided;  // [total] candidate was decided by the visual pass
  unsigned char* excl;     // [slot * track_cap + n] track was claimed by the visual pass
  int* pre_winner;         // [total] the pre-pass's decision: track index the candidate won, -1 = decided as a new track
  int* dense_cnt;          // [1] scenes of the request in dense mode (null: unknown); lets the dense kernels leave at once
  int* refine_next;        // [n_scenes] next unclaimed survivor of the scene (the refinement's warps claim 16 at a time)
  const int* dense_bad;    // [n_scenes] dense tensor-core path only: != 0 sends the scene to the exact SIMT kernels
  // outputs (device), any may be null
  unsigned long long* o_ids;
  unsigned int* o_epochs;
  unsigned int* o_lengths;
  unsigned char* o_vt;
  float* o_pred;
  float* o_obs;
};

// The per-scene counters of a frame, zeroed together (the tracker: by frame_setup_kernel): pos_cnt | vis_cnt | scene_mode |
// vis_mode | refine_next | status, [n] ints each, then dense_cnt and screen_cnt[3].
inline size_t counter_ints(int n) { return 6 * (size_t)n + 4; }
inline void carve_counters(int* c, int n, Frame& f) {
  using F = Frame;
  int* F::* const rows[] = {&F::pos_cnt, &F::vis_cnt, &F::scene_mode, &F::vis_mode, &F::refine_next, &F::status, &F::dense_cnt};
  for (int i = 0; i < 7; ++i) f.*rows[i] = c + (size_t)i * n;
  f.screen_cnt = f.dense_cnt + 1;
}

struct TcTile { int scene, m0, c0, pad; };  // pad: column-tile index inside the scene (dense kernel: its metadata slab)  // one 128 x 256 output tile of the tensor-core visual cost kernel
// per-frame metadata of one physical feature row (track n, physical slot p) of a scene, built once per frame
struct VisColMeta {
  float colb;    // column constant of the screen test (copy of TcArgs::colb)
  float colc;    // column part of the screen test
  int outcol;    // logical output column n*K + k (-1: none)
  int row;       // feature row idx*K + phys when the observation takes part in the metric, else -1
};
struct VisColGeo { float tx, ty, tr; unsigned int tep; };  // only read when spatio-temporal constraints exist
// row constant of the screen test, candidate may vote visually, e4m3 Euclidean screen: 2^-k of the candidate row
struct VisRowMeta { float rowk; int ok; float rowi; int pad; };
struct DenseTrackMeta { int n; int kt; float cmax; int pad; };   // arena block: owner (store index, -1: none), valid observations

// ---- kernel launchers (each in its own .cu) ----
void launch_prep(const Params& p, const Frame& f, int n_scenes, int max_m, cudaStream_t st);
// own-area shares of every detection among the detections of its scene (raw request boxes [total][6]) -> d_out[total].
// d_ovf_cnt / d_ovf ([total] (scene, detection) pairs): detections that more than kOwnMaxNb boxes overlap, handled by a
// second, CTA-per-detection pass; bit 1 of Frame::status[scene] is only set beyond kOwnBigNb overlapping boxes.
void launch_own_area(const Frame& f, int n_scenes, int max_m, const float* d_boxes, float* d_out, int* d_ovf_cnt,
                     int2* d_ovf, cudaStream_t st);
// dst (device) <- src (device alias of mapped pinned host memory), bytes a multiple of 4; a kernel instead of a DMA
void launch_pull(void* dst, const void* src, size_t bytes, cudaStream_t st);
// Per-frame tables built on the device: scene descriptors (request half from `req`, a device alias of mapped pinned host
// memory; store half from d_n_tracks / ts.arena_top), the tile list of the tensor-core visual cost kernel (mstep = 256
// candidate rows per entry: a 2-CTA cluster's pair of 128-row tiles; 0: none) and the frame scalars; also zeroes the
// `n_zero` ints at `zero` (list counters, status).
// cstep: feature rows per entry (the screen: vis_screen_ucols(); (256 / K) * K for the dense kernel, which also gets
// ws_off / blk_off / slab_off and one metadata slab per column tile instead of 128-padded columns)
void launch_frame_setup(const Params& p, const TrackStore& ts, const Frame& f, const SceneReq* req, int n_scenes,
                        const int* d_n_tracks, int mstep, int cstep, bool dense, TcTile* tiles, FrameDyn* dyn, int* zero,
                        int n_zero, cudaStream_t st);
// kernels launched by this library since it was loaded (every launch site counts itself)
void note_launch(int n = 1);
unsigned long long launch_count();
void launch_pos_cost(const Params& p, const TrackStore& ts, const Frame& f, int n_scenes, int max_m, int max_n,
                     cudaStream_t st);
// visual cost: fp32 SIMT kernel in the reference's summation order (use_tc == false) or the tensor-core screen
struct TcArgs {
  int max_init_done;   // the frame's setup kernel already reset scene_max
  int colmeta_done;    // the column metadata of the screen was launched by the caller (side stream)  // tensor-core screen resources (all null / 0 when the dense exact kernel is used)
  bool use_tc;
  const TcTile* d_tiles;  // candidate-tile PAIRS (m0 step 256) x column ranges of cstep rows, run by 2-CTA clusters
  int n_tiles;            // tiles (stateless operators) or an upper bound of them (trackers: the count is d_n_tiles[0])
  const int* d_n_tiles;   // device-side tile count (null: n_tiles is exact)
  long long a_rows, b_rows;
  int num_sms;
  cudaEvent_t ev_screen0, ev_screen1, ev_refine1;  // optional per-kernel timing (null: not timed)
  VisColMeta* colmeta;   // [sum n_s*K]
  VisColGeo* colgeo;     // [sum n_s*K]
  float* colb;                // [sum n_s*K (+pad)] column constant of the screen test
  unsigned int* colvalid;     // bit per column: the observation takes part in the metric
  VisRowMeta* rowmeta;   // [total]
  bool fp8;              // the A-stationary screen runs on the e4m3 copies (d8 <= 512)
  float* colsb;          // [like colb] e4m3 Euclidean screen: the column's 2^k
  int total_cols;
  int max_rows;          // max over the scenes of nb * K
  // ---- dense weight-sum path (mode 2)
  bool dense;            // run launch_vis_dense instead of the screen
  // feature rows per entry of d_tiles: dense, (256 / K) * K, so that no track straddles two tiles; screen,
  // vis_screen_ucols()
  int cstep;
  int max_blocks;        // upper bound of nb over the scenes
  int n_slabs_ub;        // upper bound of the 256-column metadata slabs of the frame
  void* ws;              // weight sums {S~, per-observation error bound} per (block, candidate), packed as half2
  unsigned int* d_rowb;  // [total][5] fused row bounds (per candidate and observation count)
  unsigned int* d_colb;  // [blk_ub] fused column bounds (per arena block of the frame)
  long long blk_ub;      // upper bound of the arena blocks of the frame
  float* slab_ktf;       // [slab][256] voting observations of the column's block (0: none)
  DenseTrackMeta* tmeta; // per arena block
  int2* rowinfo;         // per physical feature row: {logical output column, feature row or -1}
  float* slab_colc;      // [slab][256] column constant (|b|^2, or 1/|b| for cosine)
  float* slab_cmax;      // [slab][256] maximum of |b|^2 over the observations of the column's track
  unsigned int* slab_vmask;  // [slab][8] bit per column: observation takes part in the metric
  unsigned int* slab_bmask;  // [slab][8] bit per column: last physical slot of its block (flush the weight sum)
  float* scene_l0;       // [n_scenes] sampled lower bound of the scene's maximal distance (domain of the kernel's x)
  float* scene_cmax;     // [n_scenes] max |b|^2 of the scene
  VisPair* maxc;         // candidates for the maximal distance (same per-scene slices as the pair lists)
  float* maxc_val;
  int* maxc_cnt;         // [n_scenes]
  int* maxc_next;        // [n_scenes]
  int* dense_bad;        // [n_scenes] != 0: the dense result cannot be used for this scene (exact SIMT path takes it)
  int* zeros;            // [n_scenes] all zero (vis_mode view for the max refinement)
  int* dbg_counts;       // [8] per-frame diagnostics: scenes per fallback reason (1, 2, 4), max candidates
};
int launch_vis_cost(const Params& p, const TrackStore& ts, const Frame& f, int n_scenes, int max_m, int max_n,
                    const TcArgs& tc, cudaStream_t st);
// Dense tensor-core visual cost for thresholds that cut nothing (the reference's default Euclidean(f32::MAX), the published
// bench's Euclidean(10.0) on unit vectors): see kernels_feat_dense.cu.  Fills the same per-scene pair lists the screen fills
// (whole (candidate, track) groups that can be a row or column maximum of BestFit's weight matrix), which the exact
// refinement and the sparse voting kernel then consume unchanged.
int launch_vis_dense(const Params& p, const TrackStore& ts, const Frame& f, int n_scenes, int max_m, const TcArgs& tc,
                     cudaStream_t st);
// The same in two halves, so that the positional cost can run on a second stream next to the refinement:
//   _a: metadata, tensor-core screen, vis_mode, exact refinement of the survivors (needs nothing from the positional stage)
//   _b: final scene_mode (needs the positional list counters), dense exact kernel for the scenes in dense mode
int launch_vis_cost_a(const Params& p, const TrackStore& ts, const Frame& f, int n_scenes, int max_m, int max_n,
                      const TcArgs& tc, cudaStream_t st);
int launch_vis_cost_b(const Params& p, const TrackStore& ts, const Frame& f, int n_scenes, int max_m, int max_n,
                      const TcArgs& tc, cudaStream_t st);
// positional cost in two launches (dense None fill, culled scan) for callers that place them on a side stream
void launch_pos_fill(const Params& p, const Frame& f, int n_scenes, int max_m, int max_n, cudaStream_t st);
void launch_pos_scan(const Params& p, const TrackStore& ts, const Frame& f, int n_scenes, int max_m, int max_n,
                     cudaStream_t st);
// pass 0: scenes whose visual lists are complete (vis_mode == 0) skip decided candidates / claimed tracks, the others are
// scanned in full; pass 1 (after scene_mode): full scan of the scenes that fell back to dense voting only then
void launch_pos_scan_lazy(const Params& p, const TrackStore& ts, const Frame& f, int n_scenes, int max_m, int max_n,
                          int pass, cudaStream_t st);
// BestFit pre-pass of the sparse voting kernel: writes Frame::decided / Frame::excl for the scenes with vis_mode == 0
int launch_vote_masks(const Params& p, const TrackStore& ts, const Frame& f, int n_scenes, int max_m, int max_n,
                      cudaStream_t st);
// phase 0: metadata + tensor-core screen; phase 1: exact refinement of the survivors of the sparse scenes
// screen metadata of the stored feature rows (needs the frame tables and the store, not the candidates)
void launch_vis_colmeta(const Params& p, const TrackStore& ts, const Frame& f, int n_scenes, int max_n, const TcArgs& tc,
                        cudaStream_t st);
// feature rows per work unit of the screen (TcArgs::cstep), from each scene's candidates m[s] and (an upper bound of) its
// arena blocks nb[s]
int vis_screen_ucols(int d8, int num_sms, int n_scenes, const int* m, const int* nb, int K);
int launch_vis_cost_tc(const Params& p, const TrackStore& ts, const Frame& f, int n_scenes, int max_n, const TcArgs& tc,
                       int phase, cudaStream_t st);
// materialises the dense visual matrix of the sparse scenes (operators / debugging only)
void launch_vis_densify(const Params& p, const Frame& f, int n_scenes, cudaStream_t st);
void launch_to_bf16(const float* src, int src_pitch, int d, int d8, long long rows, void* dst, cudaStream_t st);
// e4m3 copies of f32 rows (d8 <= 512): dst[r][fp8_pitch(d8)] = e4m3(2^k_r src[r]), scale[r] = 2^k_r; one warp per row
void launch_to_fp8(const float* src, int src_pitch, int d, int d8, long long rows, unsigned char* dst, float* scale,
                   cudaStream_t st);
// largest d8 the e4m3 (A-stationary) screen takes
constexpr int kFp8MaxD8 = 512;
// scene_max init (all scenes) and, unless init_only, the dense reduction for the scenes whose mode has bit1 set
void launch_scene_max(const Params& p, const Frame& f, int n_scenes, bool init_only, cudaStream_t st);
// per-scene voting mode from the list counters (runs after the cost kernels); launch_vis_mode: the visual half of it
void launch_scene_mode(const Params& p, const Frame& f, int n_scenes, bool tc_used, cudaStream_t st);
void launch_vis_mode(const Params& p, const Frame& f, int n_scenes, bool tc_used, cudaStream_t st);
// shared memory the voting kernels need for scenes of up to max_m x max_n (limit: kVotingSmemLimit)
size_t voting_smem_need(int max_m, int max_n, int viscap = 0);
constexpr size_t kVotingSmemLimit = 220 * 1024;
// returns cudaError from configuration (dynamic smem), 0 on success
int launch_voting(const Params& p, const TrackStore& ts, const Frame& f, int n_scenes, int max_m, int max_n,
                  cudaStream_t st);
// max_rows: an upper bound of every scene's stored tracks plus detections
void launch_apply(const Params& p, const TrackStore& ts, const Frame& f, int n_scenes, int max_rows,
                  unsigned long long id_base, int* d_n_tracks, cudaStream_t st);
// the kept features of the frame -> the tracks' feature blocks; false when the frame has none (no launch)
bool launch_feat_store(const Params& p, const TrackStore& ts, const Frame& f, cudaStream_t st);
// BF16 arena rows again from the f32 rows, converted as feat_store_kernel converts them: the n rows listed in `rows`
// (-1: none), or with rows == null every row of the blocks [0, arena_top[slot]) of slots [0, n_slots)
void launch_bf16_regen(const TrackStore& ts, int d8, int K, const int* rows, long long n, int n_slots, cudaStream_t st);
// stable compaction of wasted tracks; appends them to the wasted buffers
struct WastedBuf {
  int cap;
  int* count;  // device counter
  unsigned long long* id;
  unsigned long long* scene;
  unsigned int* epoch;
  unsigned int* length;
  float* pred;
  float* obs;
  float* hist_pred;   // [cap][hist_len][6] rings of the wasted tracks (null unless history_length > 1)
  float* hist_obs;
  int* hblk;          // [cap] feature-history block of the record (null: history off)
};
void launch_waste(const Params& p, const TrackStore& ts, int n_slots, const unsigned int* d_cur_epoch,
                  const unsigned long long* d_scene_ids, int* d_n_tracks, const WastedBuf& wb, int max_n,
                  cudaStream_t st);
// end-of-frame sweep over the scenes of the request: tracks that can never match again (EpochDb::baked,
// src/trackers/epoch_db.rs:51-66, evaluated at the scene's new epoch) leave the device store at once -- their records go
// to the wasted buffer, where the host keeps them hidden until the reference's own collection point -- and
// frame_out[s] = {live tracks, arena blocks, newly expired} is written for the host mirror.
void launch_frame_sweep(const Params& p, const TrackStore& ts, const Frame& f, int n_scenes, int* d_n_tracks,
                        const WastedBuf& wb, cudaStream_t st);
// feature histories of n wasted records (their blocks `blk`, observation counts `lengths`) in the order of
// sb200_wasted_visual: entry c of record i (oldest first, at most hist_cap) -> out_rows[i][c][d8], out_present[i][c];
// entries without a feature, and entries past a record's count, get present 0 and a zero row
void launch_hist_gather(const TrackStore& ts, int d8, const int* blk, const unsigned int* lengths, int n, int hist_cap,
                        float* out_rows, unsigned char* out_present, cudaStream_t st);

// state blob (kernels_xfer.cu): pack / unpack as lists of contiguous segments, each cut into kXferChunk-byte chunks;
// d_cpre[i] = chunks of the segments before i (n_seg + 1 entries)
constexpr int kXferChunk = 32 * 1024;
struct XferSeg { const char* src; char* dst; unsigned long long bytes; };
int launch_xfer_copy(const XferSeg* d_segs, const long long* d_cpre, int n_seg, long long chunks, int num_sms,
                     cudaStream_t st);
// feature-history blocks of the tracks of the listed slots (d_pre: prefix of their live tracks, n + 1 entries) in store
// order: dir 0 gathers them from the pool into rows / pres, dir 1 scatters them to the fresh blocks [base, base + total)
// and points the tracks' hblk there
int launch_xfer_hist(const TrackStore& ts, int d8, const int* d_slots, const int* d_pre, int n, int total, int dir,
                     float* rows, unsigned char* pres, int base, int num_sms, cudaStream_t st);
// per slot: push the history blocks of its first `push` tracks onto the free list at free0 + push_off (a removed scene),
// then set its device counters; once: id counter = max(itself, id_min), pool counters {free, top} += {free_add, top_add}
struct XferSlot { int slot, n_tracks, n_free, arena_top, push, push_off; };
// range checks of index columns of a blob: kind 0 int32 values in [lo, hi); kind 1 uint8 values in [lo, hi); kind 2
// rows of K uint8 (observation permutations) whose first aux[i] entries lie in [lo, hi).  *bad counts the violations.
struct XferCheck { const void* p; const unsigned char* aux; long long n; int lo, hi, kind; };
int launch_xfer_check(const XferCheck* d_ck, int n, int K, int* bad, cudaStream_t st);
int launch_xfer_slots(const XferSlot* d_tab, int n, int* d_n_tracks, int* d_n_free, int* d_arena_top,
                      const TrackStore& ts, int free0, int free_add, int top_add, unsigned long long* id_counter,
                      unsigned long long id_min, cudaStream_t st);

// stateless operators
void launch_kalman_ops(int op, float pw, float vw, const float* in30, const float* boxes, int n, float* out30,
                       cudaStream_t st);
void launch_kalman_distance(float pw, const float* in30, const float* boxes, int n, float* out, cudaStream_t st);
// op: 0 initiate, 1 predict, 2 update (out = 12-float states), 3 distance (out = one float per state); in12 16-byte aligned
void launch_point_kalman(int op, float pw, float vw, const float* in12, const float* points, int n, float* out,
                         cudaStream_t st);
// kernels_geom.cu
void launch_box_vertices(const float* boxes6, int n, double* out8, cudaStream_t st);
// n (subject, clipping) pairs: ring [n][kMaxPoly][2], counts (-1: more than kMaxPoly vertices), areas; *d_status |= 1
// when any count is -1
void launch_clip_polygons(const float* subjects6, const float* clippings6, int n, double* out_xy, int* out_counts,
                          double* out_areas, int* d_status, cudaStream_t st);
// m x n intersection areas from the boxes' vertices (launch_box_vertices); *d_status |= 1 when a pair would need more
// than kMaxPoly vertices
void launch_intersection_areas(const double* a_vert, int m, const double* b_vert, int n, double* out_mn, int* d_status,
                               cudaStream_t st);

// shared device helpers
__device__ __forceinline__ bool compat_ok(const Params& p, unsigned int cand_epoch, unsigned int trk_epoch, float cx,
                                          float cy, float cr, float tx, float ty, float tr) {
  // SortAttributes::compatible, src/trackers/sort.rs:250-270 (scene equality is structural here)
  unsigned int delta = cand_epoch > trk_epoch ? cand_epoch - trk_epoch : trk_epoch - cand_epoch;
  if ((unsigned int)p.max_idle_epochs < delta) return false;
  // SpatioTemporalConstraints::validate, src/trackers/spatio_temporal_constraints.rs:48-59
  for (int i = 0; i < p.n_constraints; ++i) {
    if ((unsigned int)p.constraint_epochs[i] >= delta) {
      float d = dist_in_2r(cx, cy, cr, tx, ty, tr);
      return d <= p.constraint_max_dist[i];
    }
  }
  return true;
}

}  // namespace sb
