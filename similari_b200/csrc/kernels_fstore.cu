// kernels_fstore.cu -- the feature track store's call: distances, TopN voting, merge / append; the request rows built
// from a typed or device-resident feature column (fs_stage_kernel); the slot scrub of the store blob, whose index check
// is fs_class_check_kernel for every blob version.
// Every kernel that touches stored rows is a template over their element type Elem (float, __half or __nv_bfloat16,
// FsStore::stype); its launcher picks the instance.  A 2-byte stored element is widened to f32 from its bits where it is
// loaded, which is exact, so every stage after the load sees f32 values; fs_apply_kernel rounds a request row once when
// it stores it.  The f32 instances are the kernels of the f32-only store.
//
// Replaces, for feature-only tracks (benches/feature_tracker.rs),
//   TrackStore::foreign_track_distances -> Track::distances -> euclidean / cosine (src/track/store.rs:199-250,
//   src/track.rs:604-652, src/distance.rs:9-47) + postprocess_distances (d < distance_filter)
//   TopNVoting::winners (src/track/voting/topn.rs:74-138)
//   TrackStore::merge_external / add_track / add (src/track/store.rs:265-277, 510-580, 625-691)
//   TrackStore::owned_track_distances / merge_owned (src/track/store.rs:471-486, 584-611): the owned stage, the
//   distance / TopN instances of the owned modes and the two-launch row move
//   Track::distances' attributes.compatible check and Track::merge's attributes.merge (src/track.rs:604-652, 522-530)
//   with examples/track_merging.rs:218-245's CamTrackingAttributes, for a gated store: the gated distance instances,
//   fs_gate_resolve_kernel and the attribute kernels
//   TrackStore::find_usable (src/track/store.rs:348-374) with examples/track_merging.rs:240-247's `baked`, for a gated
//   store: fs_baked_kernel; and that example's fetch_tracks + merge_external(.., true) / add_track from one store into
//   another: the owned stage reading the source store, fs_qual_stage_kernel and the hq instances of fs_qmerge_kernel
// Every value that reaches the voting stage is the oracle's f32 bit for bit: --fmad=false, 8-lane blocks reduced by
// reduce_add8 and accumulated one after another, then sqrt (euclidean) or the quotient by sqrt(|a|^2 |b|^2) (cosine).
#include <climits>

#include "sb_engine.cuh"
#include "sb_fstore.cuh"

namespace sb {

namespace {

__device__ __forceinline__ float fs_unkey(int k) { return __int_as_float(k >= 0 ? k : (k ^ 0x7fffffff)); }

// ------------------------------------------------------------------------------------------------ stored elements
// 16 bytes hold kPer16<Elem> stored elements, so a stored row is d8 / kPer16<Elem> 16-byte vectors (d8 is a multiple of
// 8, and a 2-byte row of d8 elements keeps 16-byte alignment).
template <typename Elem>
constexpr int kPer16 = 16 / (int)sizeof(Elem);

// 8 elements at p (16-byte aligned) as f32: two float4 loads, or one 16-byte load of a 2-byte type widened from its bits
__device__ __forceinline__ void fs_load8(const float* p, float* x) {
  const float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
  x[0] = a.x; x[1] = a.y; x[2] = a.z; x[3] = a.w; x[4] = b.x; x[5] = b.y; x[6] = b.z; x[7] = b.w;
}
template <typename T>
__device__ __forceinline__ void fs_load8(const T* p, float* x) {
  feat_widen8(*reinterpret_cast<const uint4*>(p), p, x);
}

// The rounding of a stored row: each f32 element once to the storage type, to nearest with ties to even, overflow to
// +-inf, subnormals kept (cvt.rn), two elements per 32-bit word, the lower index in the low half.  A NaN stays a NaN.
__device__ __forceinline__ unsigned int fs_round2(float a, float b, const __half*) {
  return (unsigned int)__half_as_ushort(__float2half_rn(a)) | ((unsigned int)__half_as_ushort(__float2half_rn(b)) << 16);
}
__device__ __forceinline__ unsigned int fs_round2(float a, float b, const __nv_bfloat16*) {
  return (unsigned int)__bfloat16_as_ushort(__float2bfloat16_rn(a)) |
         ((unsigned int)__bfloat16_as_ushort(__float2bfloat16_rn(b)) << 16);
}
template <typename T>
__device__ __forceinline__ uint4 fs_round8(const float4& a, const float4& b) {
  const T* tag = nullptr;
  return make_uint4(fs_round2(a.x, a.y, tag), fs_round2(a.z, a.w, tag), fs_round2(b.x, b.y, tag), fs_round2(b.z, b.w, tag));
}

// ------------------------------------------------------------------------------------------------ squared norms
// One warp per row (query rows first, then every stored slot): per 8-lane block reduce_add, blocks accumulated in
// order (src/distance.rs:36-44).  Lane l takes blocks l, l + 32, ...; lane 0 adds the block sums in block order.
// A stored row of a 2-byte type is widened as it is loaded.
template <typename T>
__device__ __forceinline__ float fs_norm_acc(const T* row, int nblk, int lane) {
  float acc = 0.0f;
  for (int base = 0; base < nblk; base += 32) {
    const int blk = base + lane;
    float bs = 0.0f;
    if (blk < nblk) {
      float x[8];
      fs_load8(row + blk * 8, x);
      float t[8] = {x[0] * x[0], x[1] * x[1], x[2] * x[2], x[3] * x[3], x[4] * x[4], x[5] * x[5], x[6] * x[6], x[7] * x[7]};
      bs = reduce_add8(t);
    }
    const int cntb = min(32, nblk - base);
    for (int j = 0; j < cntb; ++j) acc = acc + __shfl_sync(0xffffffffu, bs, j);
  }
  return acc;
}

template <typename Elem>
__global__ void fs_norm_kernel(FsStore s, FsCall c) {
  const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const long long S = (long long)s.live * s.K;
  if (w >= c.R + S) return;
  const Elem* feat = static_cast<const Elem*>(s.feat);
  const int nblk = s.d8 / 8;
  float acc;
  if constexpr (sizeof(Elem) == 4)   // one row pointer for both kinds of row
    acc = fs_norm_acc(w < c.R ? c.rows + (size_t)w * s.d8 : feat + (size_t)(w - c.R) * s.d8, nblk, lane);
  else   // w is the same across the warp
    acc = w < c.R ? fs_norm_acc(c.rows + (size_t)w * s.d8, nblk, lane)
                  : fs_norm_acc(feat + (size_t)(w - c.R) * s.d8, nblk, lane);
  if (lane == 0) {
    if (w < c.R) c.qnorm[w] = acc;
    else c.snorm[w - c.R] = acc;
  }
}

// ------------------------------------------------------------------------------------------------ distance tiles
// 64 query rows x 64 stored rows per CTA of 256 threads; thread (ty, tx) owns rows ty + 16 i and columns tx + 16 j
// (i, j < 4), so the float4 reads of shared memory are broadcast (A) or conflict-free (B, pitch 36).  Operands are staged
// kDC 8-lane blocks at a time.  Per pair and block: 8 sub + 8 mul + 7 adds of the tree + 1 accumulate (euclidean), or
// 8 mul + 8 adds (cosine), all on the FP32 pipe.
constexpr int kDT = 64;
constexpr int kDC = 4;
constexpr int kDP = kDC * 8 + 4;

// The gate of a gated store: the empty pack (every ungated instance) passes every pair; a gated instance takes one FsGate
// after the existing parameters and drops the pairs that are not compatible, in the epilogue, as filtered entries.
struct FsTriple {
  unsigned long long src;
  long long t0, t1;
};
__device__ __forceinline__ FsTriple fs_stored_triple(int) { return FsTriple{}; }
__device__ __forceinline__ FsTriple fs_stored_triple(int t, const FsGate& g) {
  return FsTriple{g.st.src[t], g.st.t0[t], g.st.t1[t]};
}
__device__ __forceinline__ bool fs_gate_pass(int, const FsTriple&) { return true; }
__device__ __forceinline__ bool fs_gate_pass(int q, const FsTriple& b, const FsGate& g) {
  return fs_compatible(g.rule, g.qsrc[q], g.qt0[q], g.qt1[q], b.src, b.t0, b.t1);
}

// MODE (kFsForeign / kFsOwnedGroup / kFsOwnedEach) changes the epilogue only: the group mode drops every entry of a
// queried track (excl), the each mode folds max_dist per query (per row across its 16 threads, then one atomicMax per row).
// Elem changes the staging of the stored (B) rows only: a 2-byte row block of 8 elements is one 16-byte load, widened
// into the same f32 tile, so 64 rows x kDC blocks are one load per thread; everything after the tile is the same.
static_assert(kDT * kDC == 256, "one 16-byte load of stored 2-byte elements per thread and stage");
template <typename Elem, int METRIC, int MODE, typename... Gate>
__global__ void __launch_bounds__(256) fs_dist_kernel(FsStore s, FsCall c, float filter, int tiles_s,
                                                      const unsigned char* __restrict__ excl, Gate... gate) {
  __shared__ __align__(16) float sa[kDT][kDP];
  __shared__ __align__(16) float sbm[kDT][kDP];
  __shared__ int s_max[8];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int S = s.live * s.K;
  const int r0 = (int)(blockIdx.x / tiles_s) * kDT, c0 = (int)(blockIdx.x % tiles_s) * kDT;
  const int nblk = s.d8 / 8;
  const Elem* feat = static_cast<const Elem*>(s.feat);
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.0f;

  for (int b0 = 0; b0 < nblk; b0 += kDC) {
    if constexpr (sizeof(Elem) == 4) {
#pragma unroll
      for (int k = tid; k < kDT * kDC * 2; k += 256) {
        const int row = k / (kDC * 2), q4 = k % (kDC * 2), blk = b0 + q4 / 2;
        float4 va = make_float4(0.f, 0.f, 0.f, 0.f), vb = va;
        if (blk < nblk) {
          if (r0 + row < c.R) va = *reinterpret_cast<const float4*>(c.rows + (size_t)(r0 + row) * s.d8 + q4 * 4 + b0 * 8);
          if (c0 + row < S) vb = *reinterpret_cast<const float4*>(feat + (size_t)(c0 + row) * s.d8 + q4 * 4 + b0 * 8);
        }
        *reinterpret_cast<float4*>(&sa[row][q4 * 4]) = va;
        *reinterpret_cast<float4*>(&sbm[row][q4 * 4]) = vb;
      }
    } else {
#pragma unroll
      for (int k = tid; k < kDT * kDC * 2; k += 256) {
        const int row = k / (kDC * 2), q4 = k % (kDC * 2), blk = b0 + q4 / 2;
        float4 va = make_float4(0.f, 0.f, 0.f, 0.f);
        if (blk < nblk && r0 + row < c.R)
          va = *reinterpret_cast<const float4*>(c.rows + (size_t)(r0 + row) * s.d8 + q4 * 4 + b0 * 8);
        *reinterpret_cast<float4*>(&sa[row][q4 * 4]) = va;
      }
      const int row = tid / kDC, q8 = tid % kDC, blk = b0 + q8;
      float x[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      if (blk < nblk && c0 + row < S) fs_load8(feat + (size_t)(c0 + row) * s.d8 + blk * 8, x);
      *reinterpret_cast<float4*>(&sbm[row][q8 * 8]) = make_float4(x[0], x[1], x[2], x[3]);
      *reinterpret_cast<float4*>(&sbm[row][q8 * 8 + 4]) = make_float4(x[4], x[5], x[6], x[7]);
    }
    __syncthreads();
    const int nb = min(kDC, nblk - b0);
    for (int bb = 0; bb < nb; ++bb) {
      float a[4][8], b[4][8];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float4 x0 = *reinterpret_cast<const float4*>(&sa[ty + 16 * i][bb * 8]);
        const float4 x1 = *reinterpret_cast<const float4*>(&sa[ty + 16 * i][bb * 8 + 4]);
        a[i][0] = x0.x; a[i][1] = x0.y; a[i][2] = x0.z; a[i][3] = x0.w;
        a[i][4] = x1.x; a[i][5] = x1.y; a[i][6] = x1.z; a[i][7] = x1.w;
        const float4 y0 = *reinterpret_cast<const float4*>(&sbm[tx + 16 * i][bb * 8]);
        const float4 y1 = *reinterpret_cast<const float4*>(&sbm[tx + 16 * i][bb * 8 + 4]);
        b[i][0] = y0.x; b[i][1] = y0.y; b[i][2] = y0.z; b[i][3] = y0.w;
        b[i][4] = y1.x; b[i][5] = y1.y; b[i][6] = y1.z; b[i][7] = y1.w;
      }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float t[8];
#pragma unroll
          for (int l = 0; l < 8; ++l) {
            if (METRIC == 0) {
              const float e = a[i][l] - b[j][l];
              t[l] = e * e;
            } else {
              t[l] = a[i][l] * b[j][l];
            }
          }
          acc[i][j] = acc[i][j] + reduce_add8(t);
        }
    }
    __syncthreads();
  }

  // epilogue: the metric, postprocess_distances (d < filter), the same-id skip and empty ring slots -> NaN
  int kmax = INT_MIN;
  int rmax[4] = {INT_MIN, INT_MIN, INT_MIN, INT_MIN};   // kFsOwnedEach: per row
  const float nan = __int_as_float(0x7fc00000);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int col = c0 + tx + 16 * j;
    if (col >= S) continue;
    const int t = col / s.K, slot = col - t * s.K;
    bool filled = ((slot - s.start[t] + s.K) % s.K) < s.cnt[t];
    if (MODE == kFsOwnedGroup) filled = filled && !excl[t];
    const unsigned long long tid_ = s.ids[t];
    const float sn = METRIC == 1 ? c.snorm[col] : 0.0f;
    const FsTriple tt = fs_stored_triple(t, gate...);   // once per stored track of the column
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int row = r0 + ty + 16 * i;
      if (row >= c.R) continue;
      float d;
      if (METRIC == 0) d = sqrtf(acc[i][j]);
      else d = 1.0f - acc[i][j] / sqrtf(c.qnorm[row] * sn);
      const bool keep = filled && c.qid[c.row_q[row]] != tid_ && d < filter && fs_gate_pass(c.row_q[row], tt, gate...);
      c.dist[(size_t)row * S + col] = keep ? d : nan;
      if (MODE == kFsOwnedEach) {
        if (keep) rmax[i] = max(rmax[i], fs_key(d));
      } else {
        if (keep) kmax = max(kmax, fs_key(d));
      }
    }
  }
  if constexpr (MODE == kFsOwnedEach) {
    // a row's 16 threads (tx) are one half of a warp
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      int m = rmax[i];
#pragma unroll
      for (int off = 8; off > 0; off >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, off));
      const int row = r0 + ty + 16 * i;
      if (tx == 0 && row < c.R && m != INT_MIN) atomicMax(c.maxkey + c.row_q[row], m);
    }
    return;
  }
  kmax = __reduce_max_sync(0xffffffffu, kmax);
  if ((tid & 31) == 0) s_max[tid >> 5] = kmax;
  __syncthreads();
  if (tid == 0) {
    int m = s_max[0];
    for (int w = 1; w < 8; ++w) m = max(m, s_max[w]);
    if (m != INT_MIN) atomicMax(c.maxkey, m);
  }
}

// ------------------------------------------------------------------------------------------------ TopN
// One CTA per query; thread t takes stored tracks t, t + 256, ...  A track's group = its entries with d <= max_distance
// in entry order (query observation outer, track observation inner, both oldest first); its weight is the sum of
// (max_dist - d) computed in f32 and widened to f64 (topn.rs:96-108).  The CTA keeps the best `topn` (weight descending,
// store position ascending) in shared memory; each round only the candidates that beat its last entry are ranked in.
constexpr int kTopnThreads = 256;

__device__ __forceinline__ bool fs_better(double wa, int pa, double wb, int pb) {
  return wa > wb || (wa == wb && pa < pb);
}

// The votes of the group (query rows a0 .. a0 + na, stored track t) and, in *w, its weight: fs_topn_kernel's loop (kept
// inline there, so that its instances keep their code), the same operations in the same order, so a group weighs the
// same bits in TopN and in the BestFit claim passes.
__device__ __forceinline__ int fs_group(const FsStore& s, const FsCall& c, int t, int a0, int na, float maxd,
                                        float max_distance, double* w) {
  const int K = s.K;
  const size_t S = (size_t)s.live * K;
  const int n = s.cnt[t], st = s.start[t];
  int votes = 0;
  double acc = 0.0;
  for (int a = 0; a < na; ++a) {
    const float* dr = c.dist + (size_t)(a0 + a) * S + (size_t)t * K;
    int slot = st;
    for (int b = 0; b < n; ++b) {
      const float d = dr[slot];
      if (d <= max_distance) {   // false for NaN: dropped entries
        ++votes;
        acc = acc + (double)(maxd - d);
      }
      slot = slot + 1 == K ? 0 : slot + 1;
    }
  }
  *w = acc;
  return votes;
}

// PERQ: max_dist is the query's own (maxkey[q], kFsOwnedEach), else the call's (maxkey[0])
template <int PERQ>
__global__ void __launch_bounds__(kTopnThreads) fs_topn_kernel(FsStore s, FsCall c, float max_distance, int min_votes,
                                                                int topn, int want_dest) {
  __shared__ double l_w[kFsMaxTopn], n_w[kFsMaxTopn], b_w[kTopnThreads];
  __shared__ int l_p[kFsMaxTopn], n_p[kFsMaxTopn], b_p[kTopnThreads];
  __shared__ int s_nb;
  const int q = blockIdx.x, tid = threadIdx.x;
  const float maxd = fs_unkey(PERQ ? c.maxkey[q] : *c.maxkey);
  const unsigned long long qid = c.qid[q];
  const int a0 = c.qoff[q], na = c.qoff[q + 1] - a0;
  const int K = s.K;
  const size_t S = (size_t)s.live * K;
  const int need = max(1, min_votes);
  int nl = 0;
  for (int base = 0; base < s.live; base += kTopnThreads) {
    const int t = base + tid;
    bool have = false;
    double w = 0.0;
    if (t < s.live && s.ids[t] != qid) {
      const int n = s.cnt[t], st = s.start[t];
      int votes = 0;
      for (int a = 0; a < na; ++a) {
        const float* dr = c.dist + (size_t)(a0 + a) * S + (size_t)t * K;
        int slot = st;
        for (int b = 0; b < n; ++b) {
          const float d = dr[slot];
          if (d <= max_distance) {   // false for NaN: dropped entries
            ++votes;
            w = w + (double)(maxd - d);
          }
          slot = slot + 1 == K ? 0 : slot + 1;
        }
      }
      have = votes >= need;
    }
    if (tid == 0) s_nb = 0;
    __syncthreads();
    if (have && (nl < topn || fs_better(w, t, l_w[nl - 1], l_p[nl - 1]))) {
      const int k = atomicAdd(&s_nb, 1);
      b_w[k] = w;
      b_p[k] = t;
    }
    __syncthreads();
    const int nb = s_nb;
    if (nb > 0) {
      const int m = nl + nb;
      for (int e = tid; e < m; e += kTopnThreads) {
        const double we = e < nl ? l_w[e] : b_w[e - nl];
        const int pe = e < nl ? l_p[e] : b_p[e - nl];
        int rank = 0;
        for (int f = 0; f < m; ++f) {
          const double wf = f < nl ? l_w[f] : b_w[f - nl];
          const int pf = f < nl ? l_p[f] : b_p[f - nl];
          rank += fs_better(wf, pf, we, pe) ? 1 : 0;
        }
        if (rank < topn) { n_w[rank] = we; n_p[rank] = pe; }
      }
      __syncthreads();
      nl = min(topn, m);
      for (int e = tid; e < nl; e += kTopnThreads) { l_w[e] = n_w[e]; l_p[e] = n_p[e]; }
    }
    __syncthreads();
  }
  for (int e = tid; e < topn; e += kTopnThreads) {
    c.out_pos[(size_t)q * topn + e] = e < nl ? l_p[e] : -1;
    c.out_w[(size_t)q * topn + e] = e < nl ? l_w[e] : 0.0;
  }
  if (tid == 0) {
    c.out_cnt[q] = nl;
    if (want_dest) c.dest[q] = nl > 0 ? l_p[0] : -1;
  }
}

// ------------------------------------------------------------------------------------------------ BestFit claims
// BestFitVoting::winners (src/track/voting/best.rs:52-128) over one call's groups, after TopN: a group (q, t) that
// reaches min_votes wins track t iff it comes first, among all the groups of the call naming t, in the order weight
// descending, then q ascending.  Every group counts, also those past a query's topn cut.  No sort is needed: a group wins
// iff it holds the column maximum.  Each pass is laid out as TopN (one CTA per query, a thread per stored track) and
// recomputes the weights with fs_group.  Weights are >= +0 (every kept d is <= max_dist), so their f64 bits order as
// u64 and one atomicMax folds them.
//   pass 0: wmax[t] = the largest weight of a group naming t (a stale read of wmax only skips an atomic that would
//           not raise it);
//   pass 1: qmin[t] = the lowest q whose group on t weighs wmax[t].
__global__ void __launch_bounds__(kTopnThreads) fs_claim_kernel(FsStore s, FsCall c, float max_distance, int min_votes,
                                                                 int pass, unsigned long long* __restrict__ wmax,
                                                                 int* __restrict__ qmin) {
  const int q = blockIdx.x;
  const float maxd = fs_unkey(*c.maxkey);
  const unsigned long long qid = c.qid[q];
  const int a0 = c.qoff[q], na = c.qoff[q + 1] - a0;
  const int need = max(1, min_votes);
  for (int t = threadIdx.x; t < s.live; t += kTopnThreads) {
    double w;
    if (s.ids[t] == qid || fs_group(s, c, t, a0, na, maxd, max_distance, &w) < need) continue;
    const unsigned long long b = (unsigned long long)__double_as_longlong(w);
    if (pass == 0) {
      if (b > wmax[t]) atomicMax(wmax + t, b);
    } else if (b == wmax[t]) {
      atomicMin(qmin + t, q);
    }
  }
}

// Element e of query q's TopN list keeps its track only if q claimed it; otherwise its position becomes -2, which the
// host reports as the query's own id (best.rs:112-120).  dest[q] (want_dest) = the first element's track when q claimed
// it, else -1.
__global__ void fs_claim_final_kernel(FsCall c, int topn, int want_dest, const int* __restrict__ qmin) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)c.Q * topn) return;
  const int q = (int)(i / topn), e = (int)(i % topn);
  if (e >= c.out_cnt[q]) return;
  const int p = c.out_pos[i];
  const bool won = qmin[p] == q;
  if (!won) c.out_pos[i] = -2;
  if (want_dest && e == 0) c.dest[q] = won ? p : -1;
}

// ------------------------------------------------------------------------------------------------ apply
// Plan (one CTA, items in order): item q goes to position p = dest[q] (a stored track), or, for dest[q] == -1, to a new
// track appended after the tracks that exist and the earlier new ones.  Appending the items of one destination one
// after another and keeping the newest K after each append (Track::merge / add_observation + optimize) keeps the last K
// of the concatenation; so item q's rows take combined indices c0 .. c0 + n - 1 after the track's old observations and
// the rows of the earlier items with the same destination, and a row survives when its index is >= total - K.
constexpr int kOrderThreads = 1024;

__global__ void __launch_bounds__(kOrderThreads) fs_order_kernel(FsStore s, FsCall c) {
  __shared__ int s_p[kOrderThreads], s_n[kOrderThreads], s_warp[kOrderThreads / 32];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  int new_base = 0;
  for (int base = 0; base < c.Q; base += kOrderThreads) {
    const int q = base + tid;
    const bool in = q < c.Q;
    const int d = in ? c.dest[q] : 0;
    const int n = in ? c.qoff[q + 1] - c.qoff[q] : 0;
    const bool isnew = in && d < 0;
    const unsigned int bal = __ballot_sync(0xffffffffu, isnew);
    if (lane == 0) s_warp[wid] = __popc(bal);
    __syncthreads();
    int woff = 0, chunk_new = 0;
    for (int w = 0; w < kOrderThreads / 32; ++w) {
      woff += w < wid ? s_warp[w] : 0;
      chunk_new += s_warp[w];
    }
    const int p = isnew ? s.live + new_base + woff + __popc(bal & ((1u << lane) - 1u)) : d;
    s_p[tid] = in ? p : -1;
    s_n[tid] = n;
    __syncthreads();
    int pre = 0;
    bool last = true;
    for (int j = 0; j < kOrderThreads; ++j) {
      if (s_p[j] != p) continue;
      if (j < tid) pre += s_n[j];
      else if (j > tid) last = false;
    }
    int run = 0;
    if (in) {
      const bool old = p < s.live;
      run = s.run[p];
      c.dest[q] = p;
      c.plan[q] = make_int4(p, (old ? s.cnt[p] : 0) + run + pre, 0, old ? s.start[p] : 0);
    }
    __syncthreads();   // every read of run[] of this chunk precedes its update
    if (in && last) s.run[p] = run + pre + n;
    __syncthreads();
    new_base += chunk_new;
  }
  for (int q = tid; q < c.Q; q += kOrderThreads) {
    int4 pl = c.plan[q];
    pl.z = (pl.x < s.live ? s.cnt[pl.x] : 0) + s.run[pl.x];
    c.plan[q] = pl;
  }
  __syncthreads();   // cnt[] and run[] are read above before they are written below
  for (int q = tid; q < c.Q; q += kOrderThreads) {
    const int4 pl = c.plan[q];
    if (pl.y + (c.qoff[q + 1] - c.qoff[q]) != pl.z) continue;   // not the last item of its destination
    const int K = s.K, T = pl.z;
    s.cnt[pl.x] = min(T, K);
    s.start[pl.x] = (pl.w + max(0, T - K)) % K;
    s.run[pl.x] = 0;
    if (pl.x >= s.live) s.ids[pl.x] = c.qid[q];
  }
}

// ------------------------------------------------------------------------------------------------ gate (associate)
// One CTA, queries in chunks of kOrderThreads.  In each chunk the first query of every destination walks the chunk's
// queries with that destination in order, carrying the window in the stored columns from one chunk to the next.
__global__ void __launch_bounds__(kOrderThreads) fs_gate_resolve_kernel(FsCall c, FsGate g) {
  __shared__ int s_d[kOrderThreads];
  const int tid = threadIdx.x;
  for (int base = 0; base < c.Q; base += kOrderThreads) {
    const int n = min(kOrderThreads, c.Q - base);
    const int d = tid < n ? c.dest[base + tid] : -1;
    s_d[tid] = d;
    __syncthreads();
    bool lead = d >= 0;
    for (int j = 0; j < tid && lead; ++j) lead = s_d[j] != d;
    if (lead) {
      const unsigned long long src = g.st.src[d];
      long long w0 = g.st.t0[d], w1 = g.st.t1[d];
      for (int j = tid; j < n; ++j) {
        if (s_d[j] != d) continue;
        const int q = base + j;
        const long long q0 = g.qt0[q], q1 = g.qt1[q];
        if (fs_compatible(g.rule, g.qsrc[q], q0, q1, src, w0, w1)) {
          w0 = min(w0, q0);
          w1 = max(w1, q1);
        } else {
          c.dest[q] = -1;
        }
      }
      g.st.t0[d] = w0;
      g.st.t1[d] = w1;
    }
    __syncthreads();   // the windows and dest[] of this chunk precede the next chunk's reads
  }
}

__global__ void fs_attr_new_kernel(int live, FsCall c, FsGate g) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= c.Q) return;
  const int p = c.dest[q];
  if (p < live) return;
  g.st.src[p] = g.qsrc[q];
  g.st.t0[p] = g.qt0[q];
  g.st.t1[p] = g.qt1[q];
}

__global__ void fs_attr_gather_kernel(FsAttrCols a, const int* __restrict__ pos, int n, FsAttrCols out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int p = pos[i];
  out.src[i] = p >= 0 ? a.src[p] : 0ull;
  out.t0[i] = p >= 0 ? a.t0[p] : 0ll;
  out.t1[i] = p >= 0 ? a.t1[p] : 0ll;
}

__global__ void fs_attr_scatter_kernel(FsAttrCols a, const int* __restrict__ pos, int n, FsAttrCols in) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int p = pos[i];
  a.src[p] = in.src[i];
  a.t0[p] = in.t0[i];
  a.t1[p] = in.t1[i];
}

__global__ void fs_attr_check_kernel(const long long* __restrict__ t0, const long long* __restrict__ t1, int n, int* bad) {
  int b = 0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) b += t0[i] > t1[i];
  if (b) atomicAdd(bad, b);
}

// One CTA per item: writes the item's surviving rows into their ring slots.  A 2-byte store rounds each f32 element
// once (fs_round8): one thread per 8-element block, one 16-byte store.
template <typename Elem>
__global__ void fs_apply_kernel(FsStore s, FsCall c) {
  const int q = blockIdx.x;
  const int4 pl = c.plan[q];
  const int a0 = c.qoff[q], n = c.qoff[q + 1] - a0, K = s.K, w4 = s.d8 / 4;
  for (int k = 0; k < n; ++k) {
    const int ci = pl.y + k;
    if (ci < pl.z - K) continue;
    const int slot = (pl.w + ci) % K;
    const float4* src = reinterpret_cast<const float4*>(c.rows + (size_t)(a0 + k) * s.d8);
    if constexpr (sizeof(Elem) == 4) {
      float4* dst = reinterpret_cast<float4*>(static_cast<float*>(s.feat) + ((size_t)pl.x * K + slot) * s.d8);
      for (int e = threadIdx.x; e < w4; e += blockDim.x) dst[e] = src[e];
    } else {
      uint4* dst = reinterpret_cast<uint4*>(static_cast<Elem*>(s.feat) + ((size_t)pl.x * K + slot) * s.d8);
      for (int e = threadIdx.x; e < w4 / 2; e += blockDim.x) dst[e] = fs_round8<Elem>(src[2 * e], src[2 * e + 1]);
    }
  }
}

// ------------------------------------------------------------------------------------------------ fetch / remove
// out is f32 whatever the storage type: a 2-byte row is widened, one 8-element block per thread
template <typename Elem>
__global__ void fs_gather_kernel(FsStore s, const int* pos, float* out, int* out_cnt) {
  const int i = blockIdx.x, p = pos[i], K = s.K, w4 = s.d8 / 4;
  const int n = p >= 0 ? s.cnt[p] : 0;
  if (threadIdx.x == 0) out_cnt[i] = n;
  for (int b = 0; b < K; ++b) {
    float4* dst = reinterpret_cast<float4*>(out + ((size_t)i * K + b) * s.d8);
    if (b < n) {
      const Elem* row = static_cast<const Elem*>(s.feat) + ((size_t)p * K + (s.start[p] + b) % K) * s.d8;
      if constexpr (sizeof(Elem) == 4) {
        const float4* src = reinterpret_cast<const float4*>(row);
        for (int e = threadIdx.x; e < w4; e += blockDim.x) dst[e] = src[e];
      } else {
        for (int e = threadIdx.x; e < w4 / 2; e += blockDim.x) {
          float x[8];
          fs_load8(row + 8 * e, x);
          dst[2 * e] = make_float4(x[0], x[1], x[2], x[3]);
          dst[2 * e + 1] = make_float4(x[4], x[5], x[6], x[7]);
        }
      }
    } else {
      for (int e = threadIdx.x; e < w4; e += blockDim.x) dst[e] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
}

// The row movers below copy rows as 16-byte vectors (float4 whatever the element type): d8 / kPer16<Elem> per row.
template <typename Elem>
__global__ void fs_compact_kernel(FsStore src, FsStore dst, const int* from) {
  const int i = blockIdx.x, p = from[i];
  const size_t w4 = (size_t)src.K * src.d8 / kPer16<Elem>;
  const float4* a = reinterpret_cast<const float4*>(static_cast<const Elem*>(src.feat) + (size_t)p * src.K * src.d8);
  float4* b = reinterpret_cast<float4*>(static_cast<Elem*>(dst.feat) + (size_t)i * src.K * src.d8);
  for (size_t e = threadIdx.x; e < w4; e += blockDim.x) b[e] = a[e];
  if (threadIdx.x == 0) {
    dst.cnt[i] = src.cnt[p];
    dst.start[i] = src.start[p];
    dst.ids[i] = src.ids[p];
  }
}

// ------------------------------------------------------------------------------------------------ owned calls
// search_owned: one thread per 16-byte vector of a stored row (a float4, or 8 elements of a 2-byte type, widened); row r
// is observation r - qoff[q] (oldest first) of the stored track at qpos[q], q = row_q[r].  No staging goes through the
// host.
template <typename Elem>
__global__ void __launch_bounds__(256) fs_owned_stage_kernel(FsStore s, FsCall c, const int* __restrict__ qpos,
                                                             float* __restrict__ rows) {
  const int w4 = s.d8 / kPer16<Elem>;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)c.R * w4) return;
  const int r = (int)(i / w4), e = (int)(i - (long long)r * w4);
  const int q = c.row_q[r], p = qpos[q];
  const int slot = (s.start[p] + (r - c.qoff[q])) % s.K;
  const Elem* feat = static_cast<const Elem*>(s.feat);
  if constexpr (sizeof(Elem) == 4) {
    reinterpret_cast<float4*>(rows + (size_t)r * s.d8)[e] =
        reinterpret_cast<const float4*>(feat + ((size_t)p * s.K + slot) * s.d8)[e];
  } else {
    float x[8];
    fs_load8(feat + ((size_t)p * s.K + slot) * s.d8 + 8 * e, x);
    float4* dst = reinterpret_cast<float4*>(rows + (size_t)r * s.d8) + 2 * e;
    dst[0] = make_float4(x[0], x[1], x[2], x[3]);
    dst[1] = make_float4(x[4], x[5], x[6], x[7]);
  }
}

__global__ void fs_peek_kernel(FsStore s, const int* __restrict__ pos, int n, int* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  out[2 * i] = s.cnt[pos[i]];
  out[2 * i + 1] = s.start[pos[i]];
}

// merge_owned in two launches whatever the chain structure: every moving row is read from its pre-call slot into
// scratch first, then written to its final slot, so no row is read after it has been overwritten.  One CTA per row.
// Scratch rows are in the storage type: rows move, they are never converted.
template <typename Elem>
__global__ void fs_move_gather_kernel(FsStore s, const int* __restrict__ src, Elem* __restrict__ scratch) {
  const int m = blockIdx.x, w4 = s.d8 / kPer16<Elem>;
  const float4* a = reinterpret_cast<const float4*>(static_cast<const Elem*>(s.feat) + (size_t)src[m] * s.d8);
  float4* b = reinterpret_cast<float4*>(scratch + (size_t)m * s.d8);
  for (int e = threadIdx.x; e < w4; e += blockDim.x) b[e] = a[e];
}

template <typename Elem>
__global__ void fs_move_scatter_kernel(FsStore s, const int* __restrict__ dst, int n_moves, const int* __restrict__ hdr,
                                       int n_hdr, const Elem* __restrict__ scratch) {
  const int m = blockIdx.x, w4 = s.d8 / kPer16<Elem>;
  if (m < n_moves) {
    const float4* a = reinterpret_cast<const float4*>(scratch + (size_t)m * s.d8);
    float4* b = reinterpret_cast<float4*>(static_cast<Elem*>(s.feat) + (size_t)dst[m] * s.d8);
    for (int e = threadIdx.x; e < w4; e += blockDim.x) b[e] = a[e];
  }
  if (m < n_hdr && threadIdx.x == 0) {
    s.cnt[hdr[3 * m]] = hdr[3 * m + 1];
    s.start[hdr[3 * m]] = hdr[3 * m + 2];
  }
}

// ------------------------------------------------------------------------------------------------ request rows
// Builds FsCall::rows from a feature column that is on the device already (the caller's, or the uploaded raw rows of a
// 2-byte host column): one thread per 8-lane block of a request row.  Widening is exact and done from the bits (sb_engine.cuh),
// so every later stage sees the values of the widened f32 request.  With `vec` (D % 8 == 0 and a 16-byte aligned base) a
// block of a 2-byte column is one 16-byte load, as in cand_norm_kernel; otherwise elements are read one by one and the
// last block is zero-padded from D to d8.
template <typename T>
__global__ void __launch_bounds__(256) fs_stage_kernel(const T* __restrict__ col, const int* __restrict__ row_src, int R,
                                                       int D, int d8, int vec, float* __restrict__ rows) {
  const int nblk = d8 / 8;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)R * nblk) return;
  const int r = (int)(i / nblk), k0 = (int)(i - (long long)r * nblk) * 8;
  const T* src = col + (size_t)row_src[r] * D + k0;
  float x[8];
  if (vec) {
    fs_load8(src, x);
  } else {
#pragma unroll
    for (int l = 0; l < 8; ++l) x[l] = k0 + l < D ? feat_elem(src, l) : 0.0f;
  }
  float4* dst = reinterpret_cast<float4*>(rows + (size_t)r * d8 + k0);
  dst[0] = make_float4(x[0], x[1], x[2], x[3]);
  dst[1] = make_float4(x[4], x[5], x[6], x[7]);
}

// ------------------------------------------------------------------------------------------------ store blob
// one warp per track; a track whose ring is full has nothing to zero
template <typename Elem>
__global__ void fs_blob_scrub_kernel(Elem* feat, const int* __restrict__ cnt, const int* __restrict__ start, int n, int K,
                                     int d8) {
  const int t = (int)(((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (t >= n) return;
  const int c = cnt[t], s0 = start[t], w4 = d8 / kPer16<Elem>;
  for (int j = c; j < K; ++j) {
    float4* d = reinterpret_cast<float4*>(feat + ((size_t)t * K + (s0 + j) % K) * d8);
    for (int e = lane; e < w4; e += 32) d[e] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

// ------------------------------------------------------------------------------------------------ quality store
// A quality store (sb200_fstore_set_retention) keeps each track's observations in the track's order (best first) in ring
// slots 0, 1, ... (its ring start is always 0), so every kernel above walks it in that order unchanged.  qual[cap][K]
// holds the quality of the row in each slot (0 in a slot that holds none) and hlen[cap] each track's history length.
// Associate and add plan and apply on the device (fs_qorder_kernel, then fs_qmerge_kernel); merge_owned plans on the
// host: stored rows move with the two row move kernels above, request rows are written by fs_put_rows_kernel, and
// fs_qual_set_kernel rewrites the qualities and history lengths of every touched track.

// Associate / add on a quality store, after TopN (and the gate): one CTA, items in chunks of kOrderThreads.  Item q with
// dest[q] == -1 becomes a new track after the stored ones and the earlier new ones (fs_order_kernel's rule); dest[q] is
// set to its position p, and run[p] (zero between calls) to the largest Q - q, marking p's first item as its leader.
__global__ void __launch_bounds__(kOrderThreads) fs_qorder_kernel(FsStore s, FsCall c) {
  __shared__ int s_warp[kOrderThreads / 32];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  int new_base = 0;
  for (int base = 0; base < c.Q; base += kOrderThreads) {
    const int q = base + tid;
    const bool in = q < c.Q;
    const int d = in ? c.dest[q] : 0;
    const bool isnew = in && d < 0;
    const unsigned int bal = __ballot_sync(0xffffffffu, isnew);
    if (lane == 0) s_warp[wid] = __popc(bal);
    __syncthreads();
    int woff = 0, chunk_new = 0;
    for (int w = 0; w < kOrderThreads / 32; ++w) {
      woff += w < wid ? s_warp[w] : 0;
      chunk_new += s_warp[w];
    }
    const int p = isnew ? s.live + new_base + woff + __popc(bal & ((1u << lane) - 1u)) : d;
    if (in) {
      c.dest[q] = p;
      atomicMax(s.run + p, c.Q - q);
    }
    __syncthreads();   // s_warp is rewritten by the next chunk
    new_base += chunk_new;
  }
}

// One CTA per item; the leader of each destination p (run[p] == Q - q) plans and applies p's whole call.  Thread 0 walks
// p's items in order (found 128 at a time by the block): associate adds each query's history (length 1) and merges its
// rows; add appends its row (a new track starts with history length 1).  Each step is the stable merge of two lists
// sorted by quality, descending (the stored list, and a query's rows from the row table, are sorted; equal qualities
// keep the stored rows first), truncated to c(h) at the new h (cap_tab), so a row an earlier step dropped never comes
// back.  The surviving stored rows are a prefix of the old list and only move later, so they are moved in place, last
// first; request rows are then rounded into their slots as fs_apply_kernel rounds them.  Every thread handles the same
// 16-byte vectors of every row, so no row is read after another thread has overwritten it.
// The history length after item qi: associate adds a query of history 1 and add starts a new track at 1 (the empty
// pack, every existing instance); associate_store adds the queried stored track's whole history, hq[qi] (Track::merge
// with merge_history = true, src/track.rs:555-560).
__device__ __forceinline__ int fs_qhist(int h, int, const FsQCall& qc) {
  if (qc.assoc) ++h;
  else if (h == 0) h = 1;
  return h;
}
__device__ __forceinline__ int fs_qhist(int h, int qi, const FsQCall&, const int* hq) { return h + hq[qi]; }

template <typename Elem, typename... HQ>
__global__ void __launch_bounds__(128) fs_qmerge_kernel(FsStore s, FsCall c, FsQCall qc, HQ... hq) {
  __shared__ int s_src[kFsMaxObs], t_src[kFsMaxObs];   // >= 0: old slot; < 0: request row -(r + 1)
  __shared__ float s_q[kFsMaxObs], t_q[kFsMaxObs];
  __shared__ unsigned int s_hit[4];
  __shared__ int s_n, s_h;
  const int q = blockIdx.x, tid = threadIdx.x, K = s.K;
  const int p = c.dest[q];
  if (s.run[p] != c.Q - q) return;   // not p's first item (uniform across the CTA)
  const bool old = p < s.live;
  const int n0 = old ? s.cnt[p] : 0;
  for (int j = tid; j < n0; j += blockDim.x) {
    s_src[j] = j;
    s_q[j] = qc.qual[(size_t)p * K + j];
  }
  if (tid == 0) {
    s_n = n0;
    s_h = old ? qc.hlen[p] : 0;
  }
  __syncthreads();
  for (int base = q; base < c.Q; base += blockDim.x) {
    const bool hit = base + tid < c.Q && c.dest[base + tid] == p;
    const unsigned int b = __ballot_sync(0xffffffffu, hit);
    if ((tid & 31) == 0) s_hit[tid >> 5] = b;
    __syncthreads();
    if (tid == 0) {
      int n = s_n, h = s_h;
      for (int w = 0; w < 4; ++w)
        for (unsigned int m = s_hit[w]; m; m &= m - 1) {
          const int qi = base + 32 * w + __ffs(m) - 1;
          h = fs_qhist(h, qi, qc, hq...);
          const int cap = qc.cap_tab[min(h, qc.ntab - 1)];
          const int r0 = c.qoff[qi], r1 = c.qoff[qi + 1];
          int a = 0, r = r0, k = 0;
          while (k < cap && (a < n || r < r1)) {
            if (r == r1 || (a < n && !(qc.rq[r] > s_q[a]))) { t_src[k] = s_src[a]; t_q[k] = s_q[a]; ++a; }
            else { t_src[k] = -(r + 1); t_q[k] = qc.rq[r]; ++r; }
            ++k;
          }
          for (int j = 0; j < k; ++j) { s_src[j] = t_src[j]; s_q[j] = t_q[j]; }
          n = k;
        }
      s_n = n;
      s_h = h;
    }
    __syncthreads();
  }
  const int n = s_n, w16 = s.d8 / kPer16<Elem>;
  Elem* feat = static_cast<Elem*>(s.feat);
  for (int i = n - 1; i >= 0; --i) {   // stored rows, in place: slot s_src[i] <= i
    const int j = s_src[i];
    if (j < 0 || j == i) continue;
    const float4* a = reinterpret_cast<const float4*>(feat + ((size_t)p * K + j) * s.d8);
    float4* d = reinterpret_cast<float4*>(feat + ((size_t)p * K + i) * s.d8);
    for (int e = tid; e < w16; e += blockDim.x) d[e] = a[e];
  }
  for (int i = 0; i < n; ++i) {   // request rows
    if (s_src[i] >= 0) continue;
    const float4* src = reinterpret_cast<const float4*>(c.rows + (size_t)(-s_src[i] - 1) * s.d8);
    if constexpr (sizeof(Elem) == 4) {
      float4* d = reinterpret_cast<float4*>(feat + ((size_t)p * K + i) * s.d8);
      for (int e = tid; e < w16; e += blockDim.x) d[e] = src[e];
    } else {
      uint4* d = reinterpret_cast<uint4*>(feat + ((size_t)p * K + i) * s.d8);
      for (int e = tid; e < w16; e += blockDim.x) d[e] = fs_round8<Elem>(src[2 * e], src[2 * e + 1]);
    }
  }
  for (int i = tid; i < n; i += blockDim.x) qc.qual[(size_t)p * K + i] = s_q[i];
  if (tid == 0) {
    s.cnt[p] = n;
    s.start[p] = 0;
    qc.hlen[p] = s_h;
    if (!old) s.ids[p] = c.qid[q];
    s.run[p] = 0;
  }
}

// associate_store on a quality store: the quality of each request row, read where fs_owned_stage_kernel reads its row
__global__ void fs_qual_stage_kernel(FsStore s, FsCall c, const float* __restrict__ qual, const int* __restrict__ qpos,
                                     float* __restrict__ rq) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= c.R) return;
  const int q = c.row_q[r], p = qpos[q];
  rq[r] = qual[(size_t)p * s.K + (s.start[p] + (r - c.qoff[q])) % s.K];
}

// ------------------------------------------------------------------------------------------------ find_baked
// One CTA of kOrderThreads: warp w scans the contiguous strip [w L, (w + 1) L) of the n tracks, 32 coalesced windows
// at a time.  A first pass counts each strip's baked tracks, the strips' counts are prefix-summed, and a second pass
// writes each baked position at its warp's offset plus its rank in the ballot, so the positions come out in store order.
__global__ void __launch_bounds__(kOrderThreads) fs_baked_kernel(const long long* __restrict__ t_end, int n, long long now,
                                                                 long long period, int* __restrict__ out) {
  constexpr int kWarps = kOrderThreads / 32;
  __shared__ int s_cnt[kWarps];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int L = (n + kOrderThreads - 1) / kOrderThreads * 32;
  const int b = (int)min((long long)n, (long long)wid * L), e = min(n, b + L);
  int cnt = 0;
  for (int i = b + lane; i < e; i += 32) cnt += fs_baked(now, t_end[i], period) ? 1 : 0;
  cnt = __reduce_add_sync(0xffffffffu, cnt);
  if (lane == 0) s_cnt[wid] = cnt;
  __syncthreads();
  int at = 0, total = 0;
  for (int w = 0; w < kWarps; ++w) {
    at += w < wid ? s_cnt[w] : 0;
    total += s_cnt[w];
  }
  if (threadIdx.x == 0) out[0] = total;
  for (int base = b; base < e; base += 32) {
    const int i = base + lane;
    const bool baked = i < e && fs_baked(now, t_end[i], period);
    const unsigned int bal = __ballot_sync(0xffffffffu, baked);
    if (baked) out[1 + at + __popc(bal & ((1u << lane) - 1u))] = i;
    at += __popc(bal);
  }
}

// out[2 i] = cnt, out[2 i + 1] = start of the track at pos[i]; oq[i][j] = the quality of its observation j (0 past cnt)
__global__ void fs_qpeek_kernel(FsStore s, const float* __restrict__ qual, const int* __restrict__ pos, int n,
                                int* __restrict__ out, float* __restrict__ oq) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int p = pos[i], c = s.cnt[p], st = s.start[p], K = s.K;
  out[2 * i] = c;
  out[2 * i + 1] = st;
  for (int j = 0; j < K; ++j) oq[(size_t)i * K + j] = j < c ? qual[(size_t)p * K + (st + j) % K] : 0.0f;
}

// qual[pos[i]][j] = vals[i][j], j < K; hlen[pos[i]] = hl[i]
__global__ void fs_qual_set_kernel(float* __restrict__ qual, int* __restrict__ hlen, const int* __restrict__ pos,
                                   const float* __restrict__ vals, const int* __restrict__ hl, int n, int K) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (long long)n * K) return;
  const int i = (int)(e / K), j = (int)(e - (long long)i * K);
  qual[(size_t)pos[i] * K + j] = vals[e];
  if (j == 0) hlen[pos[i]] = hl[i];
}

// dst[i][.] = src[from[i]][.], w 32-bit words per track: the qualities and history lengths of fs_compact_kernel's kept
// tracks
__global__ void fs_words_compact_kernel(const unsigned int* __restrict__ src, unsigned int* __restrict__ dst,
                                        const int* __restrict__ from, int n, int w) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (long long)n * w) return;
  const int i = (int)(e / w), j = (int)(e - (long long)i * w);
  dst[e] = src[(size_t)from[i] * w + j];
}

// ring slot j of a track with ring start st holds observation (j - st) mod K; filled when that is < c.  Safe for any
// st and c (a blob's, not yet checked).
__device__ __forceinline__ bool fs_slot_filled(int j, int st, int c, int K) {
  return (((j - st) % K) + K) % K < c;
}

// store blob: bad[0] counts the NaN qualities in filled slots, bad[1] the observations whose quality is above the one
// before (a list out of the quality order)
__global__ void fs_qual_check_kernel(const float* __restrict__ qual, const int* __restrict__ cnt,
                                     const int* __restrict__ start, int n, int K, int* bad) {
  int b = 0, o = 0;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < (long long)n * K;
       e += (long long)gridDim.x * blockDim.x) {
    const int t = (int)(e / K), j = (int)(e - (long long)t * K);
    const int st = start[t], i = (((j - st) % K) + K) % K;   // observation index of slot j
    if (i >= cnt[t]) continue;
    b += isnan(qual[e]);
    if (i > 0) o += qual[e] > qual[(size_t)t * K + (((st + i - 1) % K) + K) % K];
  }
  if (b) atomicAdd(bad, b);
  if (o) atomicAdd(bad + 1, o);
}

// store blob, after its sections are copied: zeroes the qualities of the slots that hold no observation
__global__ void fs_qual_scrub_kernel(float* __restrict__ qual, const int* __restrict__ cnt, const int* __restrict__ start,
                                     int n, int K) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (long long)n * K) return;
  const int t = (int)(e / K), j = (int)(e - (long long)t * K);
  if (!fs_slot_filled(j, start[t], cnt[t], K)) qual[e] = 0.0f;
}

// ------------------------------------------------------------------------------------------------ feature classes
__global__ void fs_class_counts_kernel(FsClassCols cc, const int* __restrict__ pos, int n, int* __restrict__ out) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (long long)n * cc.n) return;
  const int i = (int)(e / cc.n), k = (int)(e - (long long)i * cc.n), p = pos[i];
  out[e] = p >= 0 ? cc.cnt[k][p] : 0;
}

__global__ void fs_class_check_kernel(FsClassCols cc, int n, int K, int* bad) {
  int bc = 0, bs = 0, be = 0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    bool rows = false;
    for (int k = 0; k < cc.n; ++k) {
      const int c = cc.cnt[k][i], s0 = cc.start[k][i];
      bc += (c < 0 || c > K);
      bs += (s0 < 0 || s0 >= K);
      rows |= c > 0;
    }
    be += !rows;
  }
  if (bc) atomicAdd(bad, bc);
  if (bs) atomicAdd(bad + 1, bs);
  if (be) atomicAdd(bad + 2, be);
}

}  // namespace

template <typename Elem, int MODE, typename... Gate>
void fs_dist_grid(int metric, float filter, const FsStore& s, const FsCall& c, int tiles_s, unsigned grid,
                  const unsigned char* excl, cudaStream_t st, Gate... gate) {
  if (metric == 0) fs_dist_kernel<Elem, 0, MODE><<<grid, 256, 0, st>>>(s, c, filter, tiles_s, excl, gate...);
  else fs_dist_kernel<Elem, 1, MODE><<<grid, 256, 0, st>>>(s, c, filter, tiles_s, excl, gate...);
}

template <typename Elem, typename... Gate>
void fs_dist_mode(int mode, int metric, float filter, const FsStore& s, const FsCall& c, int tiles_s, unsigned grid,
                  const unsigned char* excl, cudaStream_t st, Gate... gate) {
  if (mode == kFsOwnedGroup) fs_dist_grid<Elem, kFsOwnedGroup>(metric, filter, s, c, tiles_s, grid, excl, st, gate...);
  else if (mode == kFsOwnedEach) fs_dist_grid<Elem, kFsOwnedEach>(metric, filter, s, c, tiles_s, grid, excl, st, gate...);
  else fs_dist_grid<Elem, kFsForeign>(metric, filter, s, c, tiles_s, grid, excl, st, gate...);
}

void fs_launch_dist(int metric, float filter, const FsStore& s, const FsCall& c, cudaStream_t st, int mode,
                    const unsigned char* excl, const FsGate* gate) {
  const long long S = (long long)s.live * s.K;
  if (c.R == 0 || S == 0) return;
  const int tiles_s = (int)((S + kDT - 1) / kDT), tiles_r = (c.R + kDT - 1) / kDT;
  const unsigned grid = (unsigned)((long long)tiles_s * tiles_r);
  feat_dispatch(s.stype, [&](auto tag) {
    using Elem = decltype(tag);
    if (metric == 1) {
      const long long warps = c.R + S;
      fs_norm_kernel<Elem><<<(unsigned)((warps * 32 + 255) / 256), 256, 0, st>>>(s, c);
      note_launch();
    }
    if (gate) fs_dist_mode<Elem>(mode, metric, filter, s, c, tiles_s, grid, excl, st, *gate);
    else fs_dist_mode<Elem>(mode, metric, filter, s, c, tiles_s, grid, excl, st);
  });
  note_launch();
}

void fs_launch_topn(float max_distance, int min_votes, int topn, bool want_dest, const FsStore& s, const FsCall& c,
                    cudaStream_t st, int mode) {
  if (c.Q == 0) return;
  if (mode == kFsOwnedEach)
    fs_topn_kernel<1><<<c.Q, kTopnThreads, 0, st>>>(s, c, max_distance, min_votes, topn, want_dest ? 1 : 0);
  else
    fs_topn_kernel<0><<<c.Q, kTopnThreads, 0, st>>>(s, c, max_distance, min_votes, topn, want_dest ? 1 : 0);
  note_launch();
}

cudaError_t fs_launch_claim(float max_distance, int min_votes, int topn, bool want_dest, const FsStore& s,
                            const FsCall& c, unsigned long long* wmax, int* qmin, cudaStream_t st) {
  if (c.Q == 0 || s.live == 0) return cudaSuccess;
  cudaError_t e = cudaMemsetAsync(wmax, 0, (size_t)s.live * 8, st);
  if (e == cudaSuccess) e = cudaMemsetAsync(qmin, 0x7f, (size_t)s.live * 4, st);   // above every query index
  if (e != cudaSuccess) return e;
  for (int pass = 0; pass < 2; ++pass)
    fs_claim_kernel<<<c.Q, kTopnThreads, 0, st>>>(s, c, max_distance, min_votes, pass, wmax, qmin);
  const long long n = (long long)c.Q * topn;
  fs_claim_final_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(c, topn, want_dest ? 1 : 0, qmin);
  note_launch(3);
  return cudaSuccess;
}

void fs_launch_owned_stage(const FsStore& s, const FsCall& c, const int* qpos, float* rows, cudaStream_t st) {
  if (c.R == 0) return;
  feat_dispatch(s.stype, [&](auto tag) {
    using Elem = decltype(tag);
    const long long threads = (long long)c.R * (s.d8 / kPer16<Elem>);
    fs_owned_stage_kernel<Elem><<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(s, c, qpos, rows);
  });
  note_launch();
}

void fs_launch_peek(const FsStore& s, const int* pos, int n, int* out, cudaStream_t st) {
  if (n == 0) return;
  fs_peek_kernel<<<(n + 255) / 256, 256, 0, st>>>(s, pos, n, out);
  note_launch();
}

void fs_launch_move_rows(const FsStore& s, const int* src, const int* dst, int n_moves, const int* hdr, int n_hdr,
                         void* scratch, cudaStream_t st) {
  feat_dispatch(s.stype, [&](auto tag) {
    using Elem = decltype(tag);
    if (n_moves > 0) {
      fs_move_gather_kernel<Elem><<<n_moves, 128, 0, st>>>(s, src, static_cast<Elem*>(scratch));
      note_launch();
    }
    if (std::max(n_moves, n_hdr) > 0) {
      fs_move_scatter_kernel<Elem><<<std::max(n_moves, n_hdr), 128, 0, st>>>(s, dst, n_moves, hdr, n_hdr,
                                                                             static_cast<const Elem*>(scratch));
      note_launch();
    }
  });
}

void fs_launch_apply(const FsStore& s, const FsCall& c, cudaStream_t st) {
  if (c.Q == 0) return;
  fs_order_kernel<<<1, kOrderThreads, 0, st>>>(s, c);
  feat_dispatch(s.stype, [&](auto tag) { fs_apply_kernel<decltype(tag)><<<c.Q, 128, 0, st>>>(s, c); });
  note_launch(2);
}

void fs_launch_gate_resolve(const FsCall& c, const FsGate& g, cudaStream_t st) {
  if (c.Q == 0) return;
  fs_gate_resolve_kernel<<<1, kOrderThreads, 0, st>>>(c, g);
  note_launch();
}

void fs_launch_attr_new(int live, const FsCall& c, const FsGate& g, cudaStream_t st) {
  if (c.Q == 0) return;
  fs_attr_new_kernel<<<(c.Q + 255) / 256, 256, 0, st>>>(live, c, g);
  note_launch();
}

void fs_launch_attr_gather(const FsAttrCols& a, const int* pos, int n, const FsAttrCols& out, cudaStream_t st) {
  if (n == 0) return;
  fs_attr_gather_kernel<<<(n + 255) / 256, 256, 0, st>>>(a, pos, n, out);
  note_launch();
}

void fs_launch_attr_scatter(const FsAttrCols& a, const int* pos, int n, const FsAttrCols& in, cudaStream_t st) {
  if (n == 0) return;
  fs_attr_scatter_kernel<<<(n + 255) / 256, 256, 0, st>>>(a, pos, n, in);
  note_launch();
}

void fs_launch_attr_check(const long long* t0, const long long* t1, int n, int* bad, cudaStream_t st) {
  if (n == 0) return;
  fs_attr_check_kernel<<<std::min((n + 255) / 256, 1024), 256, 0, st>>>(t0, t1, n, bad);
  note_launch();
}

void fs_launch_gather(const FsStore& s, const int* pos, int n, float* out, int* out_cnt, cudaStream_t st) {
  if (n == 0) return;
  feat_dispatch(s.stype, [&](auto tag) { fs_gather_kernel<decltype(tag)><<<n, 128, 0, st>>>(s, pos, out, out_cnt); });
  note_launch();
}

void fs_launch_compact(const FsStore& src, const FsStore& dst, const int* from, int n, cudaStream_t st) {
  if (n == 0) return;
  feat_dispatch(src.stype, [&](auto tag) { fs_compact_kernel<decltype(tag)><<<n, 128, 0, st>>>(src, dst, from); });
  note_launch();
}

void fs_launch_stage(int type, const void* col, const int* row_src, int R, int D, int d8, float* rows, cudaStream_t st) {
  if (R == 0) return;
  const int vec = D % 8 == 0 && (reinterpret_cast<uintptr_t>(col) & 15) == 0;
  const long long threads = (long long)R * (d8 / 8);
  feat_dispatch(type, [&](auto tag) {
    using T = decltype(tag);
    fs_stage_kernel<T><<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(static_cast<const T*>(col), row_src, R, D, d8, vec,
                                                                         rows);
  });
  note_launch();
}

void fs_launch_blob_scrub(int stype, void* feat, const int* cnt, const int* start, int n, int K, int d8, cudaStream_t st) {
  if (n == 0) return;
  feat_dispatch(stype, [&](auto tag) {
    using Elem = decltype(tag);
    fs_blob_scrub_kernel<Elem><<<(unsigned)(((long long)n * 32 + 255) / 256), 256, 0, st>>>(static_cast<Elem*>(feat), cnt,
                                                                                           start, n, K, d8);
  });
  note_launch();
}

namespace {
unsigned fs_blocks(long long threads) { return (unsigned)((threads + 255) / 256); }
}  // namespace

void fs_launch_qpeek(const FsStore& s, const float* qual, const int* pos, int n, int* out, float* oq, cudaStream_t st) {
  if (n == 0) return;
  fs_qpeek_kernel<<<fs_blocks(n), 256, 0, st>>>(s, qual, pos, n, out, oq);
  note_launch();
}

void fs_launch_qual_set(float* qual, int* hlen, const int* pos, const float* vals, const int* hl, int n, int K,
                        cudaStream_t st) {
  if (n == 0) return;
  fs_qual_set_kernel<<<fs_blocks((long long)n * K), 256, 0, st>>>(qual, hlen, pos, vals, hl, n, K);
  note_launch();
}

void fs_launch_words_compact(const void* src, void* dst, const int* from, int n, int w, cudaStream_t st) {
  if (n == 0) return;
  fs_words_compact_kernel<<<fs_blocks((long long)n * w), 256, 0, st>>>(static_cast<const unsigned int*>(src),
                                                                       static_cast<unsigned int*>(dst), from, n, w);
  note_launch();
}

void fs_launch_qmerge(const FsStore& s, const FsCall& c, const FsQCall& qc, cudaStream_t st, const int* hq) {
  if (c.Q == 0) return;
  fs_qorder_kernel<<<1, kOrderThreads, 0, st>>>(s, c);
  feat_dispatch(s.stype, [&](auto tag) {
    if (hq) fs_qmerge_kernel<decltype(tag)><<<c.Q, 128, 0, st>>>(s, c, qc, hq);
    else fs_qmerge_kernel<decltype(tag)><<<c.Q, 128, 0, st>>>(s, c, qc);
  });
  note_launch(2);
}

void fs_launch_qual_stage(const FsStore& s, const FsCall& c, const float* qual, const int* qpos, float* rq,
                          cudaStream_t st) {
  if (c.R == 0) return;
  fs_qual_stage_kernel<<<fs_blocks(c.R), 256, 0, st>>>(s, c, qual, qpos, rq);
  note_launch();
}

void fs_launch_baked(const long long* t_end, int n, long long now, long long period, int* out, cudaStream_t st) {
  fs_baked_kernel<<<1, kOrderThreads, 0, st>>>(t_end, n, now, period, out);
  note_launch();
}

void fs_launch_class_counts(const FsClassCols& cc, const int* pos, int n, int* out, cudaStream_t st) {
  if (n == 0) return;
  fs_class_counts_kernel<<<fs_blocks((long long)n * cc.n), 256, 0, st>>>(cc, pos, n, out);
  note_launch();
}

void fs_launch_class_check(const FsClassCols& cc, int n, int K, int* bad, cudaStream_t st) {
  if (n == 0) return;
  fs_class_check_kernel<<<std::min((n + 255) / 256, 1024), 256, 0, st>>>(cc, n, K, bad);
  note_launch();
}

void fs_launch_qual_check(const float* qual, const int* cnt, const int* start, int n, int K, int* bad, cudaStream_t st) {
  if (n == 0) return;
  fs_qual_check_kernel<<<(unsigned)std::min<long long>(fs_blocks((long long)n * K), 1024), 256, 0, st>>>(qual, cnt, start,
                                                                                                          n, K, bad);
  note_launch();
}

void fs_launch_qual_scrub(float* qual, const int* cnt, const int* start, int n, int K, cudaStream_t st) {
  if (n == 0) return;
  fs_qual_scrub_kernel<<<fs_blocks((long long)n * K), 256, 0, st>>>(qual, cnt, start, n, K);
  note_launch();
}

}  // namespace sb
