// kernels_cost.cu -- candidate preparation and the positional cost matrix (IoU / Mahalanobis).
//
// Replaces, for every (candidate, track) pair of a scene, the reference chain
//   TrackStore::foreign_track_distances -> Track::distances (compatible gate, src/track.rs:604-652)
//   -> SortMetric::metric / VisualMetric::positional_metric (src/trackers/sort/metric.rs:38-77,
//      src/trackers/visual_sort/metric.rs:156-198)
// Roofline: HBM-write bound -- 4 B of cost per pair-association out, (m + n) small per-box records in.
#include <cuda_bf16.h>

#include <algorithm>
#include <cstdlib>
#include <type_traits>

#include "sb_engine.cuh"

namespace sb {

// --------------------------------------------------------------------------------------------------------
// prep: one thread per detection. Candidate track construction (sort/simple_api.rs:125-145): the Kalman
// initiate->predict->update of a fresh state leaves the box unchanged except angle == 0.0 -> None
// (src/utils/kalman.rs:82-86); confidence is preserved (kalman_prediction.rs:28-29).
__global__ void prep_kernel(Params p, Frame f) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= f.total) return;
  i += f.det0;
  if (f.decided) f.decided[i] = 0;   // lazy positional stage: nobody is decided before the BestFit pre-pass
  const float* b = f.in_boxes + (size_t)i * 6;
  float xc = b[0], yc = b[1], ang = b[2], asp = b[3], h = b[4], conf = b[5];
  if (ang == 0.0f) ang = nanf("");
  float* cb = f.c_box + (size_t)i * 6;
  cb[0] = xc; cb[1] = yc; cb[2] = ang; cb[3] = asp; cb[4] = h; cb[5] = conf;
  f.c_radius[i] = box_radius(asp, h);
  f.c_conf[i] = conf < p.min_confidence ? p.min_confidence : conf;
  if (p.positional_kind == 1) box_vertices(xc, yc, ang, asp, h, f.c_vert + (size_t)i * 8);
  if (p.is_visual) {
    bool hasf = f.in_feat != nullptr && (f.in_hasf == nullptr || f.in_hasf[i] != 0);
    float q = f.in_quality ? f.in_quality[i] : 1.0f;
    // VisualMetric::feature_can_be_used with the *_use thresholds, visual_sort/metric.rs:227-249
    bool ok = q >= p.min_quality_use;
    if (p.use_own_area && f.in_own) ok = ok && (f.in_own[i] >= p.min_own_use);
    ok = ok && (box_area(asp, h) >= p.min_area);
    f.c_flags[i] = (unsigned char)((hasf ? 1 : 0) | ((hasf && ok) ? 2 : 0));
  }
}

// One warp per detection: squared norm in the reference's order (per 8-lane block reduce_add, blocks accumulated
// sequentially) and, when the tensor-core screen will run, the BF16 or the e4m3 operand copy of the row (f.c_bf16 /
// f.c_fp8, whichever the frame's screen reads) -- the feature row is read from HBM once for all.  T: element type of the request's feature column (f32, or a 2-byte type widened on load,
// where one 16-byte load is a whole 8-lane block).
template <class T>
__global__ void cand_norm_kernel(Params p, Frame f, __nv_bfloat16* __restrict__ bf16_out) {
  int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  int lane = threadIdx.x & 31;
  if (w >= f.total) return;
  w += f.det0;
  const int nblk = p.d8 / 8;
  const T* __restrict__ row = static_cast<const T*>(f.in_feat) + (size_t)w * p.feature_dim;
  constexpr bool kF32 = std::is_same<T, float>::value;
  const bool vec = (p.feature_dim % (kF32 ? 4 : 8) == 0) && (reinterpret_cast<uintptr_t>(f.in_feat) & 15) == 0;
  float acc = 0.0f;
  // two rounds of 32 blocks per step: the loads of both are issued before anything waits for them (2 KB in flight per warp)
  for (int base = 0; base < nblk; base += 64) {
    float x[2][8];
    bool have[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int blk = base + h * 32 + lane;
      have[h] = blk < nblk;
#pragma unroll
      for (int l = 0; l < 8; ++l) x[h][l] = 0.0f;
      if (have[h]) {
        if (vec && blk * 8 + 8 <= p.feature_dim) {
          if constexpr (kF32) {
            const float4 a = __ldcs(reinterpret_cast<const float4*>(row + blk * 8));
            const float4 b = __ldcs(reinterpret_cast<const float4*>(row + blk * 8 + 4));
            x[h][0] = a.x; x[h][1] = a.y; x[h][2] = a.z; x[h][3] = a.w; x[h][4] = b.x; x[h][5] = b.y; x[h][6] = b.z; x[h][7] = b.w;
          } else {
            feat_widen8(__ldcs(reinterpret_cast<const uint4*>(row + blk * 8)), row, x[h]);
          }
        } else {
#pragma unroll
          for (int l = 0; l < 8; ++l) { int d = blk * 8 + l; x[h][l] = d < p.feature_dim ? feat_elem(row, d) : 0.0f; }
        }
      }
    }
    if (f.c_fp8) {   // d8 <= 512 (kFp8MaxD8): this round holds the whole row
      const float s = fp8_row_store(x, p.d8, f.c_fp8 + (size_t)w * fp8_pitch(p.d8));
      if (lane == 0) f.c_scale[w] = s;
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float bs = 0.0f;
      if (have[h]) {
        const int blk = base + h * 32 + lane;
        float t[8];
#pragma unroll
        for (int l = 0; l < 8; ++l) t[l] = x[h][l] * x[h][l];
        bs = reduce_add8(t);
        if (bf16_out) {
          __nv_bfloat162 hh[4];
#pragma unroll
          for (int l = 0; l < 4; ++l) hh[l] = __floats2bfloat162_rn(x[h][2 * l], x[h][2 * l + 1]);
          *reinterpret_cast<uint4*>(bf16_out + (size_t)w * p.d8 + blk * 8) = *reinterpret_cast<uint4*>(hh);
        }
      }
      const int cnt = min(32, nblk - (base + h * 32));   // <= 0 for a round past the end
      for (int j = 0; j < cnt; ++j) {
        float v = __shfl_sync(0xffffffffu, bs, j);
        acc = acc + v;
      }
    }
  }
  if (lane == 0) f.c_norm2[w] = acc;
}

void launch_prep(const Params& p, const Frame& f, int n_scenes, int max_m, cudaStream_t st) {
  (void)n_scenes; (void)max_m;
  if (f.total == 0) return;
  prep_kernel<<<(f.total + 255) / 256, 256, 0, st>>>(p, f);
  note_launch();
  if (p.is_visual && f.in_feat) {  // squared norms (+ BF16 operand rows when f.c_bf16 is set for this frame)
    long long threads = (long long)f.total * 32;
    feat_dispatch(f.feat_type, [&](auto t) {
      cand_norm_kernel<decltype(t)><<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(p, f, reinterpret_cast<__nv_bfloat16*>(f.c_bf16));
    });
    note_launch();
  }
}

// --------------------------------------------------------------------------------------------------------
// positional cost: tile = TM candidates x TN tracks per CTA of TN threads*TY; thread owns one track column
// (its record lives in registers) and walks TM/TY candidates staged in shared memory (broadcast reads).
constexpr int TN = 128;
constexpr int TM = 16;
constexpr int TY = 2;

struct CandTile {
  float xc[TM], yc[TM], ang0[TM], asp[TM], h[TM], r[TM], conf[TM];
  double vert[TM][8];
};

template <int POS>
__global__ void __launch_bounds__(TN * TY) pos_cost_kernel(Params p, TrackStore ts, Frame f, int n_scenes) {
  __shared__ CandTile ct;
  for (int s = blockIdx.z; s < n_scenes; s += gridDim.z) {
    const SceneDesc sc = f.scenes[s];
    const int n0 = blockIdx.x * TN, m0 = blockIdx.y * TM;
    if (n0 >= sc.n || m0 >= sc.m) continue;   // CTA-uniform
    const int tid = threadIdx.y * TN + threadIdx.x;
    // stage candidates
    for (int i = tid; i < TM; i += TN * TY) {
      int m = m0 + i;
      if (m < sc.m) {
        int g = sc.det_base + m;
        const float* cb = f.c_box + (size_t)g * 6;
        ct.xc[i] = cb[0]; ct.yc[i] = cb[1]; ct.ang0[i] = angle_or0(cb[2]); ct.asp[i] = cb[3]; ct.h[i] = cb[4];
        ct.r[i] = f.c_radius[g]; ct.conf[i] = f.c_conf[g];
      }
    }
    if (POS == 1) {
      for (int i = tid; i < TM * 8; i += TN * TY) {
        int m = m0 + i / 8;
        if (m < sc.m) ct.vert[i / 8][i % 8] = f.c_vert[(size_t)(sc.det_base + m) * 8 + (i % 8)];
      }
    }
    __syncthreads();
    const int n = n0 + threadIdx.x;
    if (n < sc.n) {
      const size_t ti = (size_t)sc.slot * ts.track_cap + n;
      const float* tb = ts.pred + ti * 6;
      const float txc = tb[0], tyc = tb[1], tasp = tb[3], th = tb[4];
      const float tr = ts.radius[ti];
      const unsigned int tep = ts.epoch[ti];
      float mean5[5], l5[5];
      double tv[8];
      if (POS == 0) {
        const float* st = ts.kst + ti * ts.kst_stride;
        const float hh = st[4];
#pragma unroll
        for (int i = 0; i < 5; ++i) {
          mean5[i] = st[i];
          l5[i] = sqrtf(kalman_proj_var(p.pos_weight, hh, st[10 + 4 * i], i));
        }
      } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) tv[i] = ts.vert[ti * 8 + i];
      }
      float* out = f.pos + sc.pos_off;
      const float qnan = nanf("");
#pragma unroll 1
      for (int i = threadIdx.y; i < TM; i += TY) {
        int m = m0 + i;
        if (m >= sc.m) break;
        float v = qnan;
        const float cx = ct.xc[i], cy = ct.yc[i], cr = ct.r[i];
        if (compat_ok(p, sc.epoch, tep, cx, cy, cr, txc, tyc, tr) && !too_far(cx, cy, cr, txc, tyc, tr)) {
          if (POS == 0) {
            float d = maha_distance(mean5, l5, cx, cy, ct.ang0[i], ct.asp[i], ct.h[i]);
            v = maha_cost(d) / ct.conf[i];
          } else {
            double a = clip_area(ct.vert[i], tv);
            float iou = iou_from_area(a, ct.h[i], ct.asp[i], th, tasp);
            if (!is_nan(iou)) {
              iou = iou * ct.conf[i];
              v = iou >= p.iou_threshold ? iou : qnan;
            }
          }
        }
        out[(size_t)m * sc.n + n] = v;
        // sparse view for the voting stage: valid entries are rare (gated by 2R and the threshold), append them
        const bool valid = !is_nan(v);
        const unsigned am = __activemask();
        const unsigned bal = __ballot_sync(am, valid);
        if (bal) {
          const int lane = threadIdx.x & 31;
          const int leader = __ffs(bal) - 1;
          int base = 0;
          if (lane == leader) base = atomicAdd(&f.pos_cnt[s], __popc(bal));
          base = __shfl_sync(am, base, leader);
          if (valid) {
            const int slot = base + __popc(bal & ((1u << lane) - 1));
            if (slot < sc.pos_lcap) {
              PosEntry e; e.m = (unsigned short)m; e.n = (unsigned short)n; e.v = v;
              f.pos_list[sc.pos_lbase + slot] = e;
            }
          }
        }
      }
    }
    __syncthreads();   // every thread is done with ct before the next scene restages it
  }
}

// --------------------------------------------------------------------------------------------------------
// Culled positional cost.  Both metrics return None behind the circumscribed-circle gate (too_far), so a candidate
// can only score against tracks whose centre lies within (r_c + max_t r_t) of its own in x.  One CTA per scene
// sorts the scene's track centres by x in shared memory; each thread then walks one candidate's x-window, runs the
// cheap gates on shared-memory copies (x, y, r, epoch) and only touches the heavy per-track record (Kalman state /
// f64 vertices) for the handful of survivors.  The dense matrix is pre-filled with None by pos_fill_none_kernel.
// The window is padded by 1e-5 relative so that float rounding in too_far can never keep a culled pair.  A scene with
// a non-finite track x or radius, and a candidate with a non-finite x or radius, skip the window: every pair of them
// goes through the gates, which decide it as the reference does (NaN distances are never too far).
constexpr int PS_THREADS = 512;
constexpr int PS_MAXN = 4096;   // tracks per scene the culled kernel sorts in shared memory (else dense kernel)

__global__ void pos_fill_none_kernel(Frame f, long long total4, long long total) {
  const float qnan = nanf("");
  float4 q4 = make_float4(qnan, qnan, qnan, qnan);
  // chunk range [off, off + total): scalar head up to 16-byte alignment, vector body, scalar tail
  float* base = f.pos + f.pos_fill_off;
  if (f.dyn) total = f.dyn->pos_total;   // stream-ordered predict: only the device knows the packed size
  const long long head = min(total, (long long)((4 - (f.pos_fill_off & 3)) & 3));
  float4* o4 = reinterpret_cast<float4*>(base + head);
  const long long n4 = (total - head) / 4;
  (void)total4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) o4[i] = q4;
  if (blockIdx.x == 0) {
    for (long long i = threadIdx.x; i < head; i += blockDim.x) base[i] = qnan;
    for (long long i = head + n4 * 4 + threadIdx.x; i < total; i += blockDim.x) base[i] = qnan;
  }
}

constexpr int PS_QCAP = 4096;
constexpr int PS_UND = 96;     // lazy scan: up to this many open candidates take the unsorted path

// exact metric of one gated (candidate, track) pair; valid results go to the dense matrix and the sparse list
template <int POS>
__device__ __forceinline__ void pos_eval_pair(const Params& p, const TrackStore& ts, const Frame& f, const SceneDesc& sc,
                                              int sidx, size_t tbase, int m, int n, float* out, bool dense, bool list) {
  const int g = sc.det_base + m;
  const float* cb = f.c_box + (size_t)g * 6;
  const float cconf = f.c_conf[g];
  const size_t ti = tbase + n;
  float v = nanf("");
  if (POS == 0) {
    const float* st = ts.kst + ti * ts.kst_stride;
    float mean5[5], l5[5];
    const float hh = st[4];
#pragma unroll
    for (int q = 0; q < 5; ++q) { mean5[q] = st[q]; l5[q] = sqrtf(kalman_proj_var(p.pos_weight, hh, st[10 + 4 * q], q)); }
    v = maha_cost(maha_distance(mean5, l5, cb[0], cb[1], angle_or0(cb[2]), cb[3], cb[4])) / cconf;
  } else {
    const float* tb = ts.pred + ti * 6;
    // cheap certain-None gates first (any threshold a tracker would use; tiny thresholds take the exact path)
    const bool pregate = p.iou_threshold > 1e-4f;
    if (pregate && iou_bound_fails(cb[4], cb[3], tb[4], tb[3], cconf, p.iou_threshold)) return;
    double cv[8], tv[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) { cv[q] = f.c_vert[(size_t)g * 8 + q]; tv[q] = ts.vert[ti * 8 + q]; }
    if (pregate) {
      // upper bound of the intersection area -> upper bound of IoU = ub / (sum - ub), increasing in ub
      const double ub = rect_overlap_bound(cv, tv);
      if (ub == 0.0) return;
      const double sum = (double)(cb[4] * cb[4] * cb[3] + tb[4] * tb[4] * tb[3]);
      if (ub < 0.5 * sum && ub * (double)cconf * 1.0001 < (double)p.iou_threshold * (sum - ub)) return;
    }
    float iou = iou_from_area(clip_area(cv, tv), cb[4], cb[3], tb[4], tb[3]);
    if (!is_nan(iou)) {
      iou = iou * cconf;
      if (iou >= p.iou_threshold) v = iou;
    }
  }
  if (!is_nan(v)) {
    if (dense) out[(size_t)m * sc.n + n] = v;
    if (list) {
      const int slot = atomicAdd(&f.pos_cnt[sidx], 1);
      if (slot < sc.pos_lcap) {
        PosEntry e; e.m = (unsigned short)m; e.n = (unsigned short)n; e.v = v;
        f.pos_list[sc.pos_lbase + slot] = e;
      }
    }
  }
}

// The CTA evaluates its queue of gated pairs, one pair per thread.  All threads of the CTA call this.
template <int POS>
__device__ __forceinline__ void pos_flush_queue(const Params& p, const TrackStore& ts, const Frame& f, const SceneDesc& sc,
                                                int sidx, size_t tbase, const int2* queue, int qn, float* out, bool wdense,
                                                bool wlist) {
  for (int e = threadIdx.x; e < qn; e += blockDim.x) {
    const int2 q = queue[e];
    pos_eval_pair<POS>(p, ts, f, sc, sidx, tbase, q.x, q.y, out, wdense, wlist);
  }
  __syncthreads();
}

// lazy_pass < 0: plain scan.  0: lazy (visual trackers) -- in scenes whose visual lists are complete only candidates the
// visual pass left undecided and tracks it did not claim take part; 1: full scan of the scenes that ended in dense mode
// although their visual lists were complete (their first scan was a lazy one).
template <int POS>
__global__ void __launch_bounds__(PS_THREADS, 2) pos_scan_kernel(Params p, TrackStore ts, Frame f, int lazy_pass) {
  extern __shared__ __align__(16) unsigned char ps_smem[];
  __shared__ float s_rmax[PS_THREADS / 32];
  __shared__ int s_bad;
  __shared__ int s_qn;
  __shared__ int s_nund;
  __shared__ int s_und[PS_UND];
  const int sidx = blockIdx.x;
  const SceneDesc sc = f.scenes[sidx];
  const int N = sc.n, M = sc.m;
  if (N == 0 || M == 0 || N > PS_MAXN) return;   // N > PS_MAXN: the dense kernel handles this scene
  // pass 1: the scenes that ended in dense voting mode get their dense matrix now -- None fill and a full scan (their first
  // scan, if any, was a lazy one and wrote the entry list only)
  if (lazy_pass == 1 && f.scene_mode[sidx] == 0) return;
  const bool lazy = lazy_pass == 0 && f.vis_mode[sidx] == 0;
  const bool wdense = f.pos_dense_all || lazy_pass == 1;
  const bool wlist = lazy_pass != 1;
  const unsigned char* excl = lazy ? f.excl + (size_t)sc.slot * ts.track_cap : nullptr;
  // gridDim.y CTAs share a scene (few scenes, many SMs): each sorts the tracks for itself and takes a slice of candidates
  const int mchunk = (M + (int)gridDim.y - 1) / (int)gridDim.y;
  const int m_begin = (int)blockIdx.y * mchunk, m_end = min(M, m_begin + mchunk);
  if (m_begin >= M) return;
  int Np = 1;
  while (Np < N) Np <<= 1;
  float* kx = reinterpret_cast<float*>(ps_smem);           // [Np] sorted x
  int* kidx = reinterpret_cast<int*>(kx + Np);             // [Np] track index
  float* sy = reinterpret_cast<float*>(kidx + Np);         // [N] by sorted position
  float* sr = sy + N;
  unsigned int* sep = reinterpret_cast<unsigned int*>(sr + N);
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const size_t tbase = (size_t)sc.slot * ts.track_cap;
  if (tid == 0) s_bad = 0;
  float* out = f.pos + sc.pos_off;
  if (lazy) {
    // The visual pass usually leaves a handful of candidates open (new objects, ambiguous votes).  For those the sort
    // costs more than it saves: every (open candidate, track) pair goes through the same cheap gates directly -- the
    // x-window of the sorted path only ever removes pairs these gates reject -- and the survivors are evaluated as below.
    if (tid == 0) { s_nund = 0; s_qn = 0; }
    __syncthreads();
    for (int m = m_begin + tid; m < m_end; m += PS_THREADS)
      if (!f.decided[sc.det_base + m]) {
        const int k = atomicAdd(&s_nund, 1);
        if (k < PS_UND) s_und[k] = m;
      }
    __syncthreads();
    const int nund = s_nund;
    if (nund == 0) return;
    if (nund <= PS_UND) {
      for (int n = tid; n < N; n += PS_THREADS) {
        const float2 xy = *reinterpret_cast<const float2*>(ts.pred + (tbase + n) * 6);
        kx[n] = xy.x; sy[n] = xy.y; sr[n] = ts.radius[tbase + n]; sep[n] = ts.epoch[tbase + n];
        kidx[n] = excl[n];
      }
      __syncthreads();
      int2* queue = reinterpret_cast<int2*>((reinterpret_cast<uintptr_t>(sep + N) + 7) & ~(uintptr_t)7);
      for (int c = wid; c < nund; c += PS_THREADS / 32) {   // a warp per open candidate, lanes over the tracks
        const int m = s_und[c];
        const int g = sc.det_base + m;
        const float cx = f.c_box[(size_t)g * 6], cy = f.c_box[(size_t)g * 6 + 1], cr = f.c_radius[g];
        for (int n = lane; n < N; n += 32) {
          if (kidx[n]) continue;   // claimed by the visual pass
          const float tx = kx[n], ty = sy[n], tr = sr[n];
          if (!compat_ok(p, sc.epoch, sep[n], cx, cy, cr, tx, ty, tr) || too_far(cx, cy, cr, tx, ty, tr)) continue;
          const int slot = atomicAdd(&s_qn, 1);
          if (slot < PS_QCAP) queue[slot] = make_int2(m, n);
          else pos_eval_pair<POS>(p, ts, f, sc, sidx, tbase, m, n, out, wdense, wlist);
        }
      }
      __syncthreads();
      pos_flush_queue<POS>(p, ts, f, sc, sidx, tbase, queue, min(s_qn, PS_QCAP), out, wdense, wlist);
      return;
    }
    __syncthreads();
  }
  float rmax = 0.0f;
  for (int n = tid; n < Np; n += PS_THREADS) {
    if (n < N) {
      const float x = ts.pred[(tbase + n) * 6];
      const float r = ts.radius[tbase + n];
      // a non-finite x or radius makes the window bounds meaningless (inf - inf): every candidate scans [0, N) in full
      if (!isfinite(x) || !isfinite(r)) s_bad = 1;
      // a track the visual pass claimed sorts behind every window; the sort key puts the padding behind every track,
      // whatever its x (pos_sort_key), so that [0, N) holds exactly the N tracks
      kx[n] = (excl && excl[n]) ? 3.0e38f : x; kidx[n] = n;
      rmax = fmaxf(rmax, r);
    } else { kx[n] = 3.402823466e+38f; kidx[n] = -1; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) rmax = fmaxf(rmax, __shfl_xor_sync(0xffffffffu, rmax, o));
  if (lane == 0) s_rmax[wid] = rmax;
  __syncthreads();
  rmax = s_rmax[0];
  for (int w = 1; w < PS_THREADS / 32; ++w) rmax = fmaxf(rmax, s_rmax[w]);
  // bitonic sort of (x, index)
  for (int k2 = 2; k2 <= Np; k2 <<= 1) {
    for (int j = k2 >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < Np; i += PS_THREADS) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const float a = kx[i], b = kx[ixj];
          if (pos_sort_swap(a, kidx[i], b, kidx[ixj], (i & k2) == 0)) {
            kx[i] = b; kx[ixj] = a;
            const int t = kidx[i]; kidx[i] = kidx[ixj]; kidx[ixj] = t;
          }
        }
      }
      __syncthreads();
    }
  }
  for (int i = tid; i < N; i += PS_THREADS) {
    const int n = kidx[i];
    sy[i] = ts.pred[(tbase + n) * 6 + 1];
    sr[i] = ts.radius[tbase + n];
    sep[i] = ts.epoch[tbase + n];
  }
  __syncthreads();
  if (lazy_pass == 1 && !f.pos_dense_all) {   // this CTA's candidate rows of the dense matrix: None everywhere first
    const float qnan = nanf("");
    for (long long i = (long long)m_begin * N + tid; i < (long long)m_end * N; i += PS_THREADS) out[i] = qnan;
    __syncthreads();
  }
  const bool bad = s_bad != 0;
  int2* queue = reinterpret_cast<int2*>((reinterpret_cast<uintptr_t>(sep + N) + 7) & ~(uintptr_t)7);   // [PS_QCAP] gated pairs
  for (int m0 = m_begin; m0 < m_end; m0 += PS_THREADS) {
    if (tid == 0) s_qn = 0;
    __syncthreads();
    // ---- phase 1: cheap gates over the candidate's x-window; survivors go to the work queue
    const int m = m0 + tid;
    if (m < m_end && !(lazy && f.decided[sc.det_base + m])) {
      const int g = sc.det_base + m;
      const float* cb = f.c_box + (size_t)g * 6;
      const float cx = cb[0], cy = cb[1];
      const float cr = f.c_radius[g];
      int lo = 0, hi = N;
      if (!bad && isfinite(cx) && isfinite(cr)) {   // else the full scan: the gates below decide every pair
        const float R = (cr + rmax) * (1.0f + 1e-5f) + 1e-30f;
        const float xlo = cx - R, xhi = cx + R;
        int a = 0, b = N;
        while (a < b) { int mid = (a + b) >> 1; if (kx[mid] < xlo) a = mid + 1; else b = mid; }
        lo = a;
        b = N;
        while (a < b) { int mid = (a + b) >> 1; if (kx[mid] <= xhi) a = mid + 1; else b = mid; }
        hi = a;
      }
      for (int i = lo; i < hi; ++i) {
        if (excl && excl[kidx[i]]) continue;   // (only reachable on the full scan; sorted windows never hold them)
        const float tx = kx[i], ty = sy[i], tr = sr[i];
        if (!compat_ok(p, sc.epoch, sep[i], cx, cy, cr, tx, ty, tr) || too_far(cx, cy, cr, tx, ty, tr)) continue;
        const int slot = atomicAdd(&s_qn, 1);
        if (slot < PS_QCAP) queue[slot] = make_int2(m, kidx[i]);
        else pos_eval_pair<POS>(p, ts, f, sc, sidx, tbase, m, kidx[i], out, wdense, wlist);   // queue full: evaluate in place
      }
    }
    __syncthreads();
    // ---- phase 2: the survivors are evaluated, one per thread
    pos_flush_queue<POS>(p, ts, f, sc, sidx, tbase, queue, min(s_qn, PS_QCAP), out, wdense, wlist);
  }
}

static bool pos_use_dense(int max_n) { return max_n > PS_MAXN; }

void launch_pos_fill(const Params& p, const Frame& f, int n_scenes, int max_m, int max_n, cudaStream_t st) {
  (void)p;
  if (!f.pos_dense_all) return;   // trackers: only the scenes that need the dense matrix fill it (pos_scan pass 1)
  if (n_scenes == 0 || max_m == 0 || max_n == 0 || pos_use_dense(max_n)) return;   // the dense kernel writes every element
  // pos matrices are packed back to back: total elements = last offset + last size (the host passes it via f.pos_total)
  const long long total = f.pos_total;   // exact (operators) or an upper bound (trackers: the kernel reads f.dyn)
  if (total > 0) { pos_fill_none_kernel<<<1184, 256, 0, st>>>(f, total / 4, total); note_launch(); }
}

static void pos_scan_impl(const Params& p, const TrackStore& ts, const Frame& f, int n_scenes, int max_m, int max_n,
                          int lazy_pass, cudaStream_t st) {
  if (n_scenes == 0 || max_m == 0 || max_n == 0) return;
  if (pos_use_dense(max_n)) {
    if (lazy_pass == 1) return;   // the dense kernel has already written every element
    // very large scenes: dense tiled kernel
    dim3 grid((max_n + TN - 1) / TN, (max_m + TM - 1) / TM, scene_grid(n_scenes));
    dim3 block(TN, TY);
    if (p.positional_kind == 0) pos_cost_kernel<0><<<grid, block, 0, st>>>(p, ts, f, n_scenes);
    else pos_cost_kernel<1><<<grid, block, 0, st>>>(p, ts, f, n_scenes);
    note_launch();
    return;
  }
  int Np = 1;
  while (Np < max_n) Np <<= 1;
  size_t smem = (size_t)Np * 8 + (size_t)max_n * 12 + (size_t)PS_QCAP * 8 + 64;
  // two CTAs fit an SM: with fewer scenes than that, several CTAs per scene (each at least 64 candidates)
  int nsplit = std::max(1, std::min(std::min(16, (max_m + 63) / 64), (2 * kNumSms) / std::max(1, n_scenes)));
  dim3 grid(n_scenes, nsplit);
  if (p.positional_kind == 0) {
    cudaFuncSetAttribute(pos_scan_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    pos_scan_kernel<0><<<grid, PS_THREADS, smem, st>>>(p, ts, f, lazy_pass);
  } else {
    cudaFuncSetAttribute(pos_scan_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    pos_scan_kernel<1><<<grid, PS_THREADS, smem, st>>>(p, ts, f, lazy_pass);
  }
  note_launch();
}

void launch_pos_scan(const Params& p, const TrackStore& ts, const Frame& f, int n_scenes, int max_m, int max_n,
                     cudaStream_t st) {
  pos_scan_impl(p, ts, f, n_scenes, max_m, max_n, -1, st);
}
void launch_pos_scan_lazy(const Params& p, const TrackStore& ts, const Frame& f, int n_scenes, int max_m, int max_n,
                          int pass, cudaStream_t st) {
  pos_scan_impl(p, ts, f, n_scenes, max_m, max_n, (f.decided && f.excl) ? pass : (pass == 0 ? -1 : 1), st);
}

void launch_pos_cost(const Params& p, const TrackStore& ts, const Frame& f, int n_scenes, int max_m, int max_n,
                     cudaStream_t st) {
  launch_pos_fill(p, f, n_scenes, max_m, max_n, st);
  launch_pos_scan(p, ts, f, n_scenes, max_m, max_n, st);
}

// --------------------------------------------------------------------------------------------------------
// visual distances, fp32 SIMT in the reference's summation order (src/distance.rs:9-47): per 8-lane block a
// horizontal reduce_add, blocks accumulated sequentially.  One CTA computes a VM x VN tile of
// (candidate, track-observation) pairs; operands are staged through shared memory in chunks of VK floats.
// Output layout vis[m][n][k] (k = logical observation index of the track), NaN == None after the threshold /
// gate logic of VisualMetric::metric (src/trackers/visual_sort/metric.rs:200-225,253-295).
constexpr int VM = 64, VN = 64, VK = 32, VT = 256;  // 4x4 pairs per thread

// tile body; `scene`, `bx`, `by` identify the VM x VN tile
template <class T>
__device__ void vis_cost_tile(const Params& p, const TrackStore& ts, const Frame& f, int scene, int bx, int by);

// Dense kernel over the scenes in dense mode.  The grid is a fixed number of CTAs that walk (scene, tile) pairs, so
// when every scene took the screen + refine path (the common case) the launch costs a few microseconds.
// T: element type of the request's feature column.
template <class T>
__global__ void __launch_bounds__(VT) vis_cost_kernel(Params p, TrackStore ts, Frame f, int n_scenes, int tiles_x, int tiles_y) {
  if (f.dense_cnt && *f.dense_cnt == 0) return;   // the common case: every scene took the screen + refine path
  const long long per_scene = (long long)tiles_x * tiles_y;
  for (int scene = 0; scene < n_scenes; ++scene) {
    if (f.scene_mode[scene] == 0) continue;  // this scene's visual entries come from the screen + refine path
    for (long long t = blockIdx.x; t < per_scene; t += gridDim.x) {
      vis_cost_tile<T>(p, ts, f, scene, (int)(t % tiles_x), (int)(t / tiles_x));
      __syncthreads();
    }
  }
}

template <class T>
__device__ void vis_cost_tile(const Params& p, const TrackStore& ts, const Frame& f, int scene, int bx, int by) {
  const SceneDesc sc = f.scenes[scene];
  const int K = p.max_obs;
  const int ncols = sc.n * K;  // column c = n*K + k (logical obs)
  const int c0 = bx * VN, m0 = by * VM;
  if (c0 >= ncols || m0 >= sc.m) return;
  __shared__ float sa[VM][VK + 1];
  __shared__ float sb_[VN][VK + 1];
  __shared__ int col_row[VN];      // feature row (idx*K + phys) or -1
  __shared__ float col_norm[VN];
  __shared__ unsigned char col_ok[VN];
  __shared__ unsigned char row_ok[VM];
  __shared__ float row_norm[VM];
  const int tid = threadIdx.x;
  const bool cosine = p.visual_kind == 1;
  if (tid < VN) {
    int c = c0 + tid;
    int row = -1; float nrm = 0.0f; unsigned char ok = 0;
    if (c < ncols) {
      int n = c / K, k = c % K;
      size_t ti = (size_t)sc.slot * ts.track_cap + n;
      if (k < ts.obs_n[ti] && ts.obs_hasf[ti * K + k] && ts.feat_cnt[ti] >= p.min_track_length) {
        int phys = ts.obs_phys[ti * K + k];
        row = (int)(feat_block(ts, sc.slot, ti) * K + phys);
        nrm = cosine ? ts.fnorm2[row] : 0.0f;
        ok = 1;
      }
    }
    col_row[tid] = row; col_norm[tid] = nrm; col_ok[tid] = ok;
  }
  if (tid >= 64 && tid < 64 + VM) {
    int i = tid - 64;
    int m = m0 + i;
    unsigned char ok = 0; float nrm = 0.0f;
    if (m < sc.m) {
      int g = sc.det_base + m;
      ok = (f.c_flags[g] & 2) ? 1 : 0;
      nrm = cosine ? f.c_norm2[g] : 0.0f;
    }
    row_ok[i] = ok; row_norm[i] = nrm;
  }
  __syncthreads();
  const int tx = tid % 16, ty = tid / 16;  // thread computes rows ty*4..+3, cols tx*4..+3
  float acc[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) acc[a][b] = 0.0f;
  const int D = p.feature_dim, D8 = p.d8;
  for (int k0 = 0; k0 < D8; k0 += VK) {
    // stage VM x VK candidate floats and VN x VK track floats (zero padded)
    for (int e = tid; e < VM * VK; e += VT) {
      int r = e / VK, c = e % VK;
      int m = m0 + r, d = k0 + c;
      float v = 0.0f;
      if (m < sc.m && d < D && row_ok[r]) v = feat_elem(static_cast<const T*>(f.in_feat), (size_t)(sc.det_base + m) * D + d);
      sa[r][c] = v;
    }
    for (int e = tid; e < VN * VK; e += VT) {
      int r = e / VK, c = e % VK;
      int d = k0 + c;
      float v = 0.0f;
      int row = col_row[r];
      if (row >= 0 && d < D8) v = ts.feat[(size_t)row * D8 + d];
      sb_[r][c] = v;
    }
    __syncthreads();
#pragma unroll
    for (int blk = 0; blk < VK / 8; ++blk) {
      float av[4][8], bv[4][8];
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int l = 0; l < 8; ++l) av[a][l] = sa[ty * 4 + a][blk * 8 + l];
#pragma unroll
      for (int b = 0; b < 4; ++b)
#pragma unroll
        for (int l = 0; l < 8; ++l) bv[b][l] = sb_[tx * 4 + b][blk * 8 + l];
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) {
          float t[8];
          if (cosine) {
#pragma unroll
            for (int l = 0; l < 8; ++l) t[l] = av[a][l] * bv[b][l];
          } else {
#pragma unroll
            for (int l = 0; l < 8; ++l) { float df = av[a][l] - bv[b][l]; t[l] = df * df; }
          }
          acc[a][b] = acc[a][b] + reduce_add8(t);
        }
    }
    __syncthreads();
  }
  float* out = f.vis + sc.vis_off;
  const float qnan = nanf("");
#pragma unroll
  for (int a = 0; a < 4; ++a) {
    int r = ty * 4 + a, m = m0 + r;
    if (m >= sc.m) continue;
    int g = sc.det_base + m;
    const float cx = f.c_box[(size_t)g * 6], cy = f.c_box[(size_t)g * 6 + 1], cr = f.c_radius[g];
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      int cc = tx * 4 + b, c = c0 + cc;
      if (c >= ncols) continue;
      float v = qnan;
      if (row_ok[r] && col_ok[cc]) {
        int n = c / K;
        size_t ti = (size_t)sc.slot * ts.track_cap + n;
        const float* tb = ts.pred + ti * 6;
        if (compat_ok(p, sc.epoch, ts.epoch[ti], cx, cy, cr, tb[0], tb[1], ts.radius[ti])) {
          if (cosine) {
            float d = acc[a][b] / sqrtf(row_norm[r] * col_norm[cc]);
            if (d >= p.visual_threshold) v = 1.0f - d;   // is_ok + distance_to_weight
          } else {
            float d = sqrtf(acc[a][b]);
            if (d <= p.visual_threshold) v = d;
          }
        }
      }
      out[(size_t)m * ncols + c] = v;
    }
  }
}

int launch_vis_cost_a(const Params& p, const TrackStore& ts, const Frame& f, int n_scenes, int max_m, int max_n,
                      const TcArgs& tc, cudaStream_t st) {
  if (n_scenes == 0 || !p.is_visual) return 0;
  const bool any = max_m > 0 && max_n > 0 && f.in_feat != nullptr;
  const bool use_tc = tc.use_tc && any;
  if (!tc.max_init_done) launch_scene_max(p, f, n_scenes, /*init_only=*/true, st);
  if (use_tc && tc.dense) {
    // thresholds that cut nothing: dense weight sums on the tensor cores, groups that can win go to the pair lists
    int rc = launch_vis_dense(p, ts, f, n_scenes, max_m, tc, st);
    if (rc != 0) return rc;
  } else if (use_tc) {
    // tensor-core screen -> per-scene survivor lists
    // (the BF16 operand rows of the candidates were written by cand_norm_kernel in launch_prep)
    int rc = launch_vis_cost_tc(p, ts, f, n_scenes, max_n, tc, /*phase=*/0, st);
    if (rc != 0) return rc;
  }
  launch_vis_mode(p, f, n_scenes, use_tc, st);   // which scenes' survivor lists are complete
  if (use_tc) {
    int rc = launch_vis_cost_tc(p, ts, f, n_scenes, max_n, tc, /*phase=*/1, st);   // exact refinement of the survivors
    if (rc != 0) return rc;
  }
  return 0;
}

int launch_vis_cost_b(const Params& p, const TrackStore& ts, const Frame& f, int n_scenes, int max_m, int max_n,
                      const TcArgs& tc, cudaStream_t st) {
  if (n_scenes == 0) return 0;
  if (!p.is_visual) {
    launch_scene_mode(p, f, n_scenes, false, st);
    return 0;
  }
  const bool any = max_m > 0 && max_n > 0 && f.in_feat != nullptr;
  const bool use_tc = tc.use_tc && any;
  launch_scene_mode(p, f, n_scenes, use_tc, st);   // which scenes stay sparse, which fall back to the dense kernels
  if (max_m > 0 && max_n > 0) {
    // a scene in dense mode is recomputed whole by the exact kernel (whatever the refinement did for it before)
    const int tx = (max_n * p.max_obs + VN - 1) / VN, ty = (max_m + VM - 1) / VM;
    const long long want = (long long)tx * ty * (use_tc ? 1 : n_scenes);
    const int grid = (int)std::min<long long>(want, kNumSms * 8);
    feat_dispatch(f.feat_type, [&](auto t) { vis_cost_kernel<decltype(t)><<<grid, VT, 0, st>>>(p, ts, f, n_scenes, tx, ty); });
    note_launch();
    launch_scene_max(p, f, n_scenes, /*init_only=*/false, st);
  }
  return 0;
}

int launch_vis_cost(const Params& p, const TrackStore& ts, const Frame& f, int n_scenes, int max_m, int max_n,
                    const TcArgs& tc, cudaStream_t st) {
  int rc = launch_vis_cost_a(p, ts, f, n_scenes, max_m, max_n, tc, st);
  if (rc != 0) return rc;
  return launch_vis_cost_b(p, ts, f, n_scenes, max_m, max_n, tc, st);
}

}  // namespace sb
