// kernels_assign.cu -- the voting stage: one CTA per scene.
//
// Replaces Voting::winners of the reference on the dense per-scene cost matrices (NaN == None):
//   SortVoting::winners      src/trackers/sort/voting.rs:30-100   (i64 weights, diagonal "new track" columns,
//                            pathfinding::kuhn_munkres maximum-weight assignment)
//   BestFitVoting::winners   src/track/voting/best.rs:52-128      (greedy on sum_k (max_dist - d_k) weights)
//   VisualVoting::winners    src/trackers/visual_sort/voting.rs:45-100 (BestFit cascade, then SortVoting on the rest)
//
// Kuhn-Munkres keeps the exact label/slack formulation of pathfinding (rows in order, lowest-index column of
// minimal slack) so that the assignment -- including ties -- is the one the oracle computes.  The column state
// (slack, ly, alternating, slackx, yx) lives in shared memory; every thread owns a strided set of columns, and a
// root iteration is one pass over the owned columns plus one block-wide lexicographic (slack, column) argmin.
// The weight matrix is never materialised: w(row, col) is derived on the fly from the f32 cost matrix
// (L2-resident: m*n*4 B per scene) and the diagonal / zero columns are implicit.
//
// BestFit needs no sort on a GPU: in the reference's greedy pass over the weight-sorted list an element wins its
// track iff it is the FIRST element naming that track, i.e. the column-wise argmax of the weight matrix, and a
// query's decision is its first element, i.e. its row-wise argmax.  Both are plain reductions.
#include <algorithm>

#include "sb_engine.cuh"

namespace sb {

constexpr int VT_THREADS = 512;
constexpr int NWARPS = VT_THREADS / 32;
constexpr int kNone = -1, kSelf = -2;

struct MinPair { long long v; int y; };

__device__ __forceinline__ MinPair min_pair(MinPair a, MinPair b) {
  return (b.v < a.v || (b.v == a.v && b.y < a.y)) ? b : a;
}
__device__ __forceinline__ MinPair warp_min(MinPair a) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    MinPair b;
    b.v = __shfl_xor_sync(0xffffffffu, a.v, o);
    b.y = __shfl_xor_sync(0xffffffffu, a.y, o);
    a = min_pair(a, b);
  }
  return a;
}

struct BestPair { double w; int i; };  // maximise w, tie -> smaller index
__device__ __forceinline__ BestPair best_pair(BestPair a, BestPair b) {
  if (b.i < 0) return a;
  if (a.i < 0) return b;
  return (b.w > a.w || (b.w == a.w && b.i < a.i)) ? b : a;
}

__device__ __forceinline__ unsigned int enc_f32(float v) {  // order-preserving f32 -> u32
  unsigned int u = __float_as_uint(v);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float dec_f32(unsigned int u) {
  return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

// per-scene maximum over all valid visual entries ("max_dist" of best.rs:58,72-74), init -1.0
__global__ void vis_max_kernel(Params p, Frame f, unsigned int* scene_max, int n_scenes) {
  for (int s = blockIdx.y; s < n_scenes; s += gridDim.y) {
    if (f.scene_mode[s] == 0) continue;  // sparse scenes: the refine kernel already reduced their maximum
    const SceneDesc sc = f.scenes[s];
    const long long cnt = (long long)sc.m * sc.n * p.max_obs;
    const float* v = f.vis + sc.vis_off;
    float mx = -1.0f;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < cnt; i += (long long)gridDim.x * blockDim.x) {
      float e = v[i];
      if (!is_nan(e) && mx < e) mx = e;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      float t = __shfl_xor_sync(0xffffffffu, mx, o);
      if (mx < t) mx = t;
    }
    if ((threadIdx.x & 31) == 0) atomicMax(scene_max + s, enc_f32(mx));
  }
}
__global__ void vis_max_init_kernel(unsigned int* scene_max, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) scene_max[i] = enc_f32(-1.0f);
}

struct VoteSmem {
  long long* slack; long long* ly; long long* lx; long long* rmax;
  int* slackx; int* alt; int* yx; int* xy; int* row_cand; int* col_trk; int* first_m; int* row_of_m;
  int* fw; int* cnt_m;
  unsigned char* inS; unsigned char* excl; unsigned char* seen_m;
};

__host__ __device__ inline size_t vote_smem_bytes(int M, int N) {
  size_t ny = (size_t)M + N;
  size_t b = 0;
  b += ny * 8 * 2;            // slack, ly
  b += (size_t)M * 8 * 2;     // lx, rmax
  b += ny * 4 * 3;            // slackx, alt, yx
  b += (size_t)M * 4 * 5;     // xy, row_cand, row_of_m, fw, cnt_m
  b += (size_t)N * 4 * 2;     // col_trk, first_m
  b += (size_t)M * 2 + N;     // inS, seen_m, excl
  return b + 64;
}

__device__ inline VoteSmem carve(unsigned char* base, int M, int N) {
  VoteSmem s;
  size_t ny = (size_t)M + N;
  long long* p8 = reinterpret_cast<long long*>(base);
  s.slack = p8; p8 += ny;
  s.ly = p8; p8 += ny;
  s.lx = p8; p8 += M;
  s.rmax = p8; p8 += M;
  int* p4 = reinterpret_cast<int*>(p8);
  s.slackx = p4; p4 += ny;
  s.alt = p4; p4 += ny;
  s.yx = p4; p4 += ny;
  s.xy = p4; p4 += M;
  s.row_cand = p4; p4 += M;
  s.row_of_m = p4; p4 += M;
  s.fw = p4; p4 += M;
  s.cnt_m = p4; p4 += M;
  s.col_trk = p4; p4 += N;
  s.first_m = p4; p4 += N;
  unsigned char* p1 = reinterpret_cast<unsigned char*>(p4);
  s.inS = p1; p1 += M;
  s.seen_m = p1; p1 += M;
  s.excl = p1; p1 += N;
  return s;
}

// block-wide exclusive scan of 0/1 flags over `n` items (n arbitrary), result in out[i], returns total.
__device__ int block_scan_flags(const unsigned char* flags, int* out, int n, int* s_warp, int* s_carry) {
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid == 0) *s_carry = 0;
  __syncthreads();
  for (int base = 0; base < n; base += VT_THREADS) {
    int i = base + tid;
    int v = (i < n && flags[i]) ? 1 : 0;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int t = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += t;
    }
    if (lane == 31) s_warp[wid] = x;
    __syncthreads();
    int woff = 0;
    for (int w = 0; w < wid; ++w) woff += s_warp[w];
    int carry = *s_carry;
    if (i < n) out[i] = carry + woff + x - v;
    __syncthreads();
    if (tid == VT_THREADS - 1) *s_carry = carry + woff + x;
    __syncthreads();
  }
  return *s_carry;
}

template <bool VISUAL>
__global__ void __launch_bounds__(VT_THREADS) voting_kernel(Params p, Frame f) {
  const unsigned int* scene_max = f.scene_max;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ MinPair s_red[2][NWARPS];
  __shared__ BestPair s_rowc[32][NWARPS];
  __shared__ int s_warp[NWARPS];
  __shared__ int s_misc[4];
  const int sidx = blockIdx.x;
  if (f.scene_mode[sidx] == 0) return;  // handled by voting_sparse_kernel
  const SceneDesc sc = f.scenes[sidx];
  const int M = sc.m, N = sc.n;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  int* winner = f.winner + sc.det_base;
  unsigned char* cvt = f.c_vt + sc.det_base;
  if (M == 0) {
    if (tid == 0) f.new_count[sidx] = 0;
    return;
  }
  VoteSmem s = carve(smem_raw, M, N);
  const float* pos = f.pos + sc.pos_off;

  for (int m = tid; m < M; m += VT_THREADS) {
    winner[m] = -1;
    cvt[m] = (unsigned char)1;  // VotingType::Positional (SortTrack::from default)
    s.fw[m] = kNone;
    s.seen_m[m] = 0;
    s.rmax[m] = (-9223372036854775807LL - 1);
    s.cnt_m[m] = 0;
  }
  for (int n = tid; n < N; n += VT_THREADS) { s.excl[n] = 0; s.first_m[n] = 0x7fffffff; }
  __syncthreads();

  // ------------------------------------------------------------------ BestFit on the visual matrix
  if (VISUAL && N > 0) {
    const int K = p.max_obs;
    const float maxd = dec_f32(scene_max[sidx]);
    const float* vis = f.vis + sc.vis_off;
    // column-owned sweep: thread owns columns n = tid + j*VT_THREADS, rows are walked in order
    // s.slack / s.slackx double as per-column best (weight bits, row)
    double* colw = reinterpret_cast<double*>(s.slack);
    int* colm = s.slackx;
    for (int n = tid; n < N; n += VT_THREADS) { colm[n] = -1; colw[n] = 0.0; }
    __syncthreads();
    for (int m0 = 0; m0 < M; m0 += 32) {
      const int mend = min(M, m0 + 32);
      for (int m = m0; m < mend; ++m) {
        BestPair rb; rb.w = 0.0; rb.i = -1;
        for (int n = tid; n < N; n += VT_THREADS) {
          const float* e = vis + ((size_t)m * N + n) * K;
          int votes = 0;
          double w = 0.0;
          for (int k = 0; k < K; ++k) {
            float d = e[k];
            if (!is_nan(d)) { ++votes; w += (double)(maxd - d); }
          }
          if (votes > 0 && votes >= p.min_votes) {
            if (colm[n] < 0 || w > colw[n]) { colw[n] = w; colm[n] = m; }  // strict: earliest row wins ties
            if (rb.i < 0 || w > rb.w) { rb.w = w; rb.i = n; }             // ascending n: earliest column wins
          }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          BestPair t;
          t.w = __shfl_xor_sync(0xffffffffu, rb.w, o);
          t.i = __shfl_xor_sync(0xffffffffu, rb.i, o);
          rb = best_pair(rb, t);
        }
        if (lane == 0) s_rowc[m - m0][wid] = rb;
      }
      __syncthreads();
      if (tid < mend - m0) {
        BestPair rb = s_rowc[tid][0];
        for (int w = 1; w < NWARPS; ++w) rb = best_pair(rb, s_rowc[tid][w]);
        s.fw[m0 + tid] = rb.i;  // provisional: best column, or -1
      }
      __syncthreads();
    }
    // resolve: a query wins its best track iff it is that track's best query (first element naming the track)
    for (int m = tid; m < M; m += VT_THREADS) {
      int n1 = s.fw[m];
      if (n1 >= 0) {
        cvt[m] = (unsigned char)0;  // VotingType::Visual
        if (colm[n1] == m) { winner[m] = n1; s.excl[n1] = 1; }
        else s.fw[m] = kSelf;       // rewritten to self => new track, still excluded from the positional stage
      }
    }
    __syncthreads();
  }

  // ------------------------------------------------------------------ positional stage: SortVoting
  const long long thr = weight_i64(p.positional_kind == 0 ? 1.0f : p.iou_threshold) ;
  // prepass (warp per row): row maxima, row/column "seen" state in stream order
  if (N > 0) {
    for (int m = wid; m < M; m += NWARPS) {
      if (VISUAL && s.fw[m] != kNone) continue;
      long long mx = (-9223372036854775807LL - 1);
      int cnt = 0;
      for (int n = lane; n < N; n += 32) {
        float v = pos[(size_t)m * N + n];
        if (!is_nan(v) && !(VISUAL && s.excl[n])) {
          long long w = weight_i64(v);
          mx = w > mx ? w : mx;
          ++cnt;
          if (m < s.first_m[n]) atomicMin(&s.first_m[n], m);
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        long long t = __shfl_xor_sync(0xffffffffu, mx, o);
        mx = t > mx ? t : mx;
        cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
      }
      if (lane == 0) { s.rmax[m] = mx; s.cnt_m[m] = cnt; s.seen_m[m] = cnt > 0; }
    }
  }
  __syncthreads();
  // rows: seen candidates in ascending order (first-seen order of the stream), then (Sort only) the unseen ones
  const int n_seen_rows = block_scan_flags(s.seen_m, s.row_of_m, M, s_warp, &s_misc[0]);
  for (int m = tid; m < M; m += VT_THREADS)
    if (s.seen_m[m]) s.row_cand[s.row_of_m[m]] = m;
  const int nrows = VISUAL ? n_seen_rows : M;
  // columns: seen tracks ordered by (first row that names them, track index)
  int n_seen_cols = 0;
  {
    // rank by counting; keys are unique
    for (int n = tid; n < N; n += VT_THREADS) {
      int fm = s.first_m[n];
      if (fm == 0x7fffffff) continue;
      int rank = 0;
      for (int q = 0; q < N; ++q) {
        int fq = s.first_m[q];
        if (fq < fm || (fq == fm && q < n)) ++rank;
      }
      s.col_trk[rank] = n;
    }
    // count seen columns
    int c = 0;
    for (int n = tid; n < N; n += VT_THREADS) c += s.first_m[n] != 0x7fffffff;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if (lane == 0) s_warp[wid] = c;
    __syncthreads();
    for (int w = 0; w < NWARPS; ++w) n_seen_cols += s_warp[w];
    __syncthreads();
  }
  const int ntrk = VISUAL ? n_seen_cols : N;   // SortVoting::new(.., tracks_num)
  const int ny = nrows + ntrk;

  if (ntrk > 0 && nrows > 0) {   // `if self.track_num == 0 { return HashMap::default() }`
    // weight accessor
    auto wgt = [&](int r, int y) -> long long {
      if (y < nrows) return y == r ? thr : 0;
      int j = y - nrows;
      if (j >= n_seen_cols || r >= n_seen_rows) return 0;
      float v = pos[(size_t)s.row_cand[r] * N + s.col_trk[j]];
      return is_nan(v) ? 0 : weight_i64(v);
    };
    // labels: lx = row maximum over all ny columns, ly = 0
    for (int r = tid; r < nrows; r += VT_THREADS) {
      long long mx = thr;
      if (ny > 1) {
        int valid = r < n_seen_rows ? s.cnt_m[s.row_cand[r]] : 0;
        if (ny - 1 > valid) mx = mx > 0 ? mx : 0;           // some implicit zero column exists
        if (r < n_seen_rows) { long long rm = s.rmax[s.row_cand[r]]; mx = rm > mx ? rm : mx; }
      }
      s.lx[r] = mx;
      s.xy[r] = -1;
    }
    for (int y = tid; y < ny; y += VT_THREADS) { s.ly[y] = 0; s.yx[y] = -1; }
    __syncthreads();

    int parity = 0;
    for (int root = 0; root < nrows; ++root) {
      // ---- init search tree at `root`
      const long long lxr = s.lx[root];
      MinPair best; best.v = 9223372036854775807LL; best.y = 0x7fffffff;
      for (int y = tid; y < ny; y += VT_THREADS) {
        long long sl = lxr + s.ly[y] - wgt(root, y);
        s.slack[y] = sl; s.slackx[y] = root; s.alt[y] = -1;
        MinPair c; c.v = sl; c.y = y;
        best = min_pair(best, c);
      }
      for (int x = tid; x < nrows; x += VT_THREADS) s.inS[x] = x == root;
      best = warp_min(best);
      if (lane == 0) s_red[parity][wid] = best;
      __syncthreads();
      int y_end = -1, x_end = -1;
      for (;;) {
        MinPair g = s_red[parity][0];
#pragma unroll
        for (int w = 1; w < NWARPS; ++w) g = min_pair(g, s_red[parity][w]);
        parity ^= 1;
        const long long delta = g.v;
        const int ystar = g.y;
        const int xstar = s.slackx[ystar];
        const int x2 = s.yx[ystar];
        // label update of the tree rows; the row's owner also admits x2 (the row matched to ystar) into the tree,
        // after its own label update so that lx[x2] is not touched by this delta
        for (int x = tid; x < nrows; x += VT_THREADS) {
          if (s.inS[x]) { if (delta > 0) s.lx[x] -= delta; }
          else if (x == x2) s.inS[x] = 1;
        }
        if (x2 < 0) {
          // augmenting path found; still apply the label update to the columns
          if (delta > 0)
            for (int y = tid; y < ny; y += VT_THREADS) {
              if (s.alt[y] >= 0) s.ly[y] += delta;
              else s.slack[y] -= delta;
            }
          y_end = ystar; x_end = xstar;
          break;
        }
        const long long lx2 = s.lx[x2];
        MinPair nb; nb.v = 9223372036854775807LL; nb.y = 0x7fffffff;
        for (int y = tid; y < ny; y += VT_THREADS) {
          if (s.alt[y] >= 0) { if (delta > 0) s.ly[y] += delta; continue; }
          long long sl = s.slack[y] - delta;
          if (y == ystar) { s.alt[y] = xstar; s.slack[y] = sl; continue; }
          long long a = lx2 + s.ly[y] - wgt(x2, y);
          if (sl > a) { sl = a; s.slackx[y] = x2; }
          s.slack[y] = sl;
          MinPair c; c.v = sl; c.y = y;
          nb = min_pair(nb, c);
        }
        nb = warp_min(nb);
        if (lane == 0) s_red[parity][wid] = nb;
        __syncthreads();
      }
      __syncthreads();
      if (tid == 0) {
        int y = y_end, x = x_end;
        for (;;) {
          int prec = s.xy[x];
          s.yx[y] = x;
          s.xy[x] = y;
          y = prec;
          if (y < 0) break;
          x = s.alt[y];
        }
      }
      __syncthreads();
    }
    // emit
    for (int r = tid; r < n_seen_rows; r += VT_THREADS) {
      int y = s.xy[r];
      int m = s.row_cand[r];
      if (y >= nrows && (y - nrows) < n_seen_cols) {
        winner[m] = s.col_trk[y - nrows];
        cvt[m] = (unsigned char)1;
      }
    }
  }
  __syncthreads();
  // count new tracks of the scene
  int c = 0;
  for (int m = tid; m < M; m += VT_THREADS) c += winner[m] < 0;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if (lane == 0) s_warp[wid] = c;
  __syncthreads();
  if (tid == 0) {
    int t = 0;
    for (int w = 0; w < NWARPS; ++w) t += s_warp[w];
    f.new_count[sidx] = t;
  }
}

// =====================================================================================================
// Sparse voting: the same algorithms on the sparse views of the cost matrices (valid entries only).
//
// After the 2R gate / thresholds both matrices are ~99 % None, so the voting stage works on per-scene entry lists:
//   BestFit  : sort the scene's valid visual entries by (candidate, track, observation), one thread per (candidate,
//              track) group accumulates votes and the f64 weight in observation order, row / column argmax with
//              lowest-index tie-break (see the dense kernel for why that equals the reference's greedy pass).
//   KM       : CSR (by candidate) and CSC (by track) of the positional entries live in shared memory.  A root whose
//              tightest column is free is matched by a single warp without touching the other columns -- exactly what
//              the first iteration of pathfinding's search would do (delta = 0) -- and only the remaining roots run the
//              block-wide label/slack search, with w(row, col) looked up in the CSC.
struct SparseSmem {
  long long* slack; long long* ly; long long* lx; long long* rmax;
  int* slackx; int* alt; int* yx; int* xy; int* row_cand; int* row_of_m; int* cnt_m; int* col_trk; int* first_m;
  int* col_rank; int* fw; int* row_ptr; int* col_ptr;
  float* csr_v; float* csc_v;
  unsigned short* csr_n; unsigned short* csc_m;
  unsigned char* inS; unsigned char* seen_m; unsigned char* excl;
  // BestFit scratch, overlaid on the KM / CSR region (disjoint in time)
  unsigned long long* vkey; float* vval; unsigned long long* rowW; unsigned long long* colW; int* rown; int* colm;
  int* bstart; int* bcur;   // per-candidate buckets of the valid visual entries (bucket path of BestFit)
};

__host__ __device__ inline int vote_cap(const Params& p) { return p.vote_vis_cap > 0 ? p.vote_vis_cap : kVoteVisCap; }

__host__ __device__ inline size_t sparse_smem_bytes(int M, int N, int viscap) {
  size_t ny = (size_t)M + N;
  size_t km = ny * 8 * 2 + (size_t)M * 8 * 2 + ny * 4 * 3 + (size_t)M * 4 * 4 + (size_t)N * 4 * 3 + (size_t)(M + 1) * 4 +
              (size_t)(N + 1) * 4 + (size_t)kVotePosCap * 12 + 64;
  size_t bf = (size_t)viscap * 12 + (size_t)M * 12 + (size_t)N * 12 + (size_t)(2 * M + 2) * 4 + 64;
  size_t persist = (size_t)M * 4 + (size_t)M * 2 + N + 64;  // fw, inS, seen_m, excl
  return (km > bf ? km : bf) + persist;
}

__device__ inline SparseSmem carve_sparse(unsigned char* base, int M, int N, int viscap) {
  SparseSmem s;
  size_t ny = (size_t)M + N;
  // persistent part first
  int* p4 = reinterpret_cast<int*>(base);
  s.fw = p4; p4 += M;
  unsigned char* p1 = reinterpret_cast<unsigned char*>(p4);
  s.inS = p1; p1 += M;
  s.seen_m = p1; p1 += M;
  s.excl = p1; p1 += N;
  unsigned char* scratch = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(p1) + 15) & ~(uintptr_t)15);
  // KM / CSR / CSC view
  long long* p8 = reinterpret_cast<long long*>(scratch);
  s.slack = p8; p8 += ny;
  s.ly = p8; p8 += ny;
  s.lx = p8; p8 += M;
  s.rmax = p8; p8 += M;
  p4 = reinterpret_cast<int*>(p8);
  s.slackx = p4; p4 += ny;
  s.alt = p4; p4 += ny;
  s.yx = p4; p4 += ny;
  s.xy = p4; p4 += M;
  s.row_cand = p4; p4 += M;
  s.row_of_m = p4; p4 += M;
  s.cnt_m = p4; p4 += M;
  s.col_trk = p4; p4 += N;
  s.first_m = p4; p4 += N;
  s.col_rank = p4; p4 += N;
  s.row_ptr = p4; p4 += M + 1;
  s.col_ptr = p4; p4 += N + 1;
  s.csr_v = reinterpret_cast<float*>(p4); p4 += kVotePosCap;
  s.csc_v = reinterpret_cast<float*>(p4); p4 += kVotePosCap;
  unsigned short* p2 = reinterpret_cast<unsigned short*>(p4);
  s.csr_n = p2; p2 += kVotePosCap;
  s.csc_m = p2; p2 += kVotePosCap;
  // BestFit view of the same scratch
  unsigned long long* q8 = reinterpret_cast<unsigned long long*>(scratch);
  s.vkey = q8; q8 += viscap;
  s.rowW = q8; q8 += M;
  s.colW = q8; q8 += N;
  p4 = reinterpret_cast<int*>(q8);
  s.vval = reinterpret_cast<float*>(p4); p4 += viscap;
  s.rown = p4; p4 += M;
  s.colm = p4; p4 += N;
  s.bstart = p4; p4 += M + 1;
  s.bcur = p4; p4 += M + 1;
  return s;
}

__device__ __forceinline__ unsigned long long enc_f64(double v) {  // order-preserving f64 -> u64
  unsigned long long u = (unsigned long long)__double_as_longlong(v);
  return (u & 0x8000000000000000ull) ? ~u : (u | 0x8000000000000000ull);
}

__device__ int block_exscan_int(int* data, int n, int* s_warp, int* s_carry) {
  // in-place exclusive scan of data[0..n), returns the total
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid == 0) *s_carry = 0;
  __syncthreads();
  for (int base = 0; base < n; base += VT_THREADS) {
    int i = base + tid;
    int v = i < n ? data[i] : 0;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int t = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += t;
    }
    if (lane == 31) s_warp[wid] = x;
    __syncthreads();
    int woff = 0;
    for (int w = 0; w < wid; ++w) woff += s_warp[w];
    int carry = *s_carry;
    if (i < n) data[i] = carry + woff + x - v;
    __syncthreads();
    if (tid == VT_THREADS - 1) *s_carry = carry + woff + x;
    __syncthreads();
  }
  return *s_carry;
}

template <bool VISUAL, bool MASK_ONLY>
__global__ void __launch_bounds__(VT_THREADS) voting_sparse_kernel(Params p, TrackStore ts, Frame f) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ MinPair s_red[2][NWARPS];
  __shared__ int s_warp[NWARPS];
  __shared__ int s_misc[8];
  const int sidx = blockIdx.x;
  if (MASK_ONLY) { if (f.vis_mode[sidx] != 0) return; }  // the scan takes such a scene in full
  else if (f.scene_mode[sidx] != 0) return;  // handled by the dense voting_kernel
  const SceneDesc sc = f.scenes[sidx];
  const int M = sc.m, N = sc.n;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  int* winner = f.winner + sc.det_base;
  unsigned char* cvt = f.c_vt + sc.det_base;
  if (M == 0) {
    if (!MASK_ONLY && tid == 0) f.new_count[sidx] = 0;
    return;
  }
  SparseSmem s = carve_sparse(smem_raw, M, N, vote_cap(p));
  for (int m = tid; m < M; m += VT_THREADS) {
    winner[m] = -1;
    cvt[m] = (unsigned char)1;
    s.fw[m] = kNone;
    s.seen_m[m] = 0;
  }
  for (int n = tid; n < N; n += VT_THREADS) s.excl[n] = 0;
  __syncthreads();

  // ------------------------------------------------------------------ BestFit on the valid visual entries
  // The full pass of a frame whose BestFit pre-pass already ran for this scene (lazy positional stage: f.decided / f.excl
  // are set and the scene's visual list was complete) takes the decisions from there instead of computing them twice.
  const bool have_prepass = VISUAL && !MASK_ONLY && f.decided != nullptr && f.excl != nullptr && f.vis_mode[sidx] == 0;
  if (have_prepass) {
    const unsigned char* dec = f.decided + sc.det_base;
    const unsigned char* ex = f.excl + (size_t)sc.slot * ts.track_cap;
    const int* pw = f.pre_winner + sc.det_base;
    for (int m = tid; m < M; m += VT_THREADS) {
      if (dec[m]) {
        const int n1 = pw[m];
        cvt[m] = (unsigned char)0;
        if (n1 >= 0) { winner[m] = n1; s.fw[m] = n1; }
        else s.fw[m] = kSelf;
      }
    }
    for (int n = tid; n < N; n += VT_THREADS) s.excl[n] = ex[n];
    __syncthreads();
  } else if (VISUAL && N > 0) {
    const int K = p.max_obs;
    const float maxd = dec_f32(f.scene_max[sidx]);
    const int nraw = min(f.vis_cnt[sidx], sc.vis_lcap);
    // The valid entries (value passed the threshold) are grouped per candidate by a counting sort; a candidate's
    // handful of entries is then ordered by logical column by the one thread that owns the candidate, which also
    // walks its (candidate, track) groups: votes and the f64 weight sum_k (max_dist - d_k) in observation order
    // (best.rs:97).  Row maxima need no atomics (a thread owns its row), column maxima are order-preserving
    // atomicMax / atomicMin.  A pathological bucket (> kBucketMax entries of one candidate) takes the whole-list
    // bitonic sort instead.
    constexpr int kBucketMax = 160;   // (the dense tensor-core path lists ~10 near-equal groups for an unmatched candidate)
    for (int m = tid; m <= M; m += VT_THREADS) s.bstart[m] = 0;
    for (int m = tid; m < M; m += VT_THREADS) { s.rowW[m] = 0ull; s.rown[m] = 0x7fffffff; }
    for (int n = tid; n < N; n += VT_THREADS) { s.colW[n] = 0ull; s.colm[n] = 0x7fffffff; }
    if (tid == 0) { s_misc[0] = 0; s_misc[3] = 0; }
    __syncthreads();
    for (int i = tid; i < nraw; i += VT_THREADS) {
      const float v = f.vis_val[sc.vis_lbase + i];
      if (!is_nan(v)) {
        const int m = f.vis_pairs[sc.vis_lbase + i].g - sc.det_base;
        const int c = atomicAdd(&s.bstart[m], 1);
        if (c + 1 > kBucketMax) s_misc[3] = 1;
      }
    }
    __syncthreads();
    const bool buckets = s_misc[3] == 0;
    __syncthreads();
    if (buckets) {
      int* ecol = reinterpret_cast<int*>(s.vkey);   // [L] logical column of the entry (the u64 key array is free here)
      float* eval = s.vval;                         // [L]
      const int L = block_exscan_int(s.bstart, M + 1, s_warp, &s_misc[1]);
      (void)L;
      for (int m = tid; m < M; m += VT_THREADS) s.bcur[m] = s.bstart[m];
      __syncthreads();
      for (int i = tid; i < nraw; i += VT_THREADS) {
        const float v = f.vis_val[sc.vis_lbase + i];
        if (!is_nan(v)) {
          const VisPair vp = f.vis_pairs[sc.vis_lbase + i];
          const int slot = atomicAdd(&s.bcur[vp.g - sc.det_base], 1);
          ecol[slot] = vp.outcol;
          eval[slot] = v;
        }
      }
      __syncthreads();
      for (int pass = 0; pass < 2; ++pass) {
        for (int m = tid; m < M; m += VT_THREADS) {
          const int b0 = s.bstart[m], b1 = s.bstart[m + 1];
          if (b1 == b0) continue;
          if (pass == 0) {   // insertion sort of the bucket by logical column (keys are unique)
            for (int a = b0 + 1; a < b1; ++a) {
              const int ca = ecol[a]; const float va = eval[a];
              int b = a - 1;
              while (b >= b0 && ecol[b] > ca) { ecol[b + 1] = ecol[b]; eval[b + 1] = eval[b]; --b; }
              ecol[b + 1] = ca; eval[b + 1] = va;
            }
          }
          unsigned long long best_w = 0ull;
          int best_n = 0x7fffffff;
          int q = b0;
          while (q < b1) {
            const int n = ecol[q] / K;
            int votes = 0;
            double w = 0.0;
            for (; q < b1 && ecol[q] / K == n; ++q) { ++votes; w += (double)(maxd - eval[q]); }
            if (votes < p.min_votes) continue;
            const unsigned long long we = enc_f64(w);
            if (pass == 0) {
              atomicMax(&s.colW[n], we);
              if (we > best_w) { best_w = we; best_n = n; }   // groups ascend in n: the first maximum is the lowest n
            } else if (we == s.colW[n]) atomicMin(&s.colm[n], m);
          }
          if (pass == 0) { s.rowW[m] = best_w; s.rown[m] = best_n; }
        }
        __syncthreads();
      }
    } else {
    if (tid == 0) s_misc[0] = 0;
    __syncthreads();
    // compact the valid entries into shared memory
    for (int i = tid; i < nraw; i += VT_THREADS) {
      const float v = f.vis_val[sc.vis_lbase + i];
      if (!is_nan(v)) {
        const VisPair vp = f.vis_pairs[sc.vis_lbase + i];
        const int slot = atomicAdd(&s_misc[0], 1);
        s.vkey[slot] = ((unsigned long long)(unsigned int)(vp.g - sc.det_base) << 32) | (unsigned int)vp.outcol;
        s.vval[slot] = v;
      }
    }
    __syncthreads();
    const int L = s_misc[0];
    int Lp = 1;
    while (Lp < L) Lp <<= 1;
    for (int i = L + tid; i < Lp; i += VT_THREADS) { s.vkey[i] = ~0ull; s.vval[i] = 0.0f; }
    __syncthreads();
    // bitonic sort by (candidate, logical column): groups and their observation order become contiguous
    for (int k2 = 2; k2 <= Lp; k2 <<= 1) {
      for (int j = k2 >> 1; j > 0; j >>= 1) {
        for (int i = tid; i < Lp; i += VT_THREADS) {
          const int ixj = i ^ j;
          if (ixj > i) {
            const unsigned long long a = s.vkey[i], b = s.vkey[ixj];
            const bool up = (i & k2) == 0;
            if ((a > b) == up) {
              s.vkey[i] = b; s.vkey[ixj] = a;
              const float t = s.vval[i]; s.vval[i] = s.vval[ixj]; s.vval[ixj] = t;
            }
          }
        }
        __syncthreads();
      }
    }
    // group heads: votes and f64 weight sum_k (max_dist - d_k) as f64, best.rs:97
    for (int pass = 0; pass < 2; ++pass) {
      for (int i = tid; i < L; i += VT_THREADS) {
        const unsigned long long key = s.vkey[i];
        const int m = (int)(key >> 32);
        const int n = (int)((unsigned int)key) / K;
        bool head = true;
        if (i > 0) {
          const unsigned long long pk = s.vkey[i - 1];
          head = !((int)(pk >> 32) == m && (int)((unsigned int)pk) / K == n);
        }
        if (!head) continue;
        int votes = 0;
        double w = 0.0;
        for (int q = i; q < L; ++q) {
          const unsigned long long kq = s.vkey[q];
          if ((int)(kq >> 32) != m || (int)((unsigned int)kq) / K != n) break;
          ++votes;
          w += (double)(maxd - s.vval[q]);
        }
        if (votes < p.min_votes) continue;
        const unsigned long long we = enc_f64(w);
        if (pass == 0) { atomicMax(&s.rowW[m], we); atomicMax(&s.colW[n], we); }
        else {
          if (we == s.rowW[m]) atomicMin(&s.rown[m], n);
          if (we == s.colW[n]) atomicMin(&s.colm[n], m);
        }
      }
      __syncthreads();
    }
    }
    // resolve (dense kernel: "a query wins its best track iff it is that track's best query")
    for (int m = tid; m < M; m += VT_THREADS) {
      const int n1 = s.rown[m];
      if (n1 != 0x7fffffff) {
        cvt[m] = (unsigned char)0;
        if (s.colm[n1] == m) { winner[m] = n1; s.excl[n1] = 1; s.fw[m] = n1; }
        else s.fw[m] = kSelf;
      }
    }
    __syncthreads();
  }
  if (MASK_ONLY) {
    // pre-pass: publish who is still open for the positional stage (the full pass recomputes the same decisions)
    unsigned char* dec = f.decided + sc.det_base;
    unsigned char* ex = f.excl + (size_t)sc.slot * ts.track_cap;
    int* pw = f.pre_winner + sc.det_base;
    for (int m = tid; m < M; m += VT_THREADS) { dec[m] = s.fw[m] != kNone; pw[m] = s.fw[m] >= 0 ? s.fw[m] : -1; }
    for (int n = tid; n < N; n += VT_THREADS) ex[n] = s.excl[n];
    return;
  }

  // ------------------------------------------------------------------ positional stage on the sparse entries
  const long long thr = weight_i64(p.positional_kind == 0 ? 1.0f : p.iou_threshold);
  const int nent = min(f.pos_cnt[sidx], sc.pos_lcap);
  const PosEntry* ents = f.pos_list + sc.pos_lbase;
  auto ent_ok = [&](const PosEntry& e) -> bool {
    return !(VISUAL && (s.fw[e.m] != kNone || s.excl[e.n]));
  };
  for (int m = tid; m < M; m += VT_THREADS) { s.cnt_m[m] = 0; s.rmax[m] = (-9223372036854775807LL - 1); s.row_ptr[m] = 0; }
  for (int n = tid; n < N; n += VT_THREADS) { s.first_m[n] = 0x7fffffff; s.col_ptr[n] = 0; }
  if (tid == 0) { s.row_ptr[M] = 0; s.col_ptr[N] = 0; }
  __syncthreads();
  for (int i = tid; i < nent; i += VT_THREADS) {
    const PosEntry e = ents[i];
    if (!ent_ok(e)) continue;
    atomicAdd(&s.row_ptr[e.m], 1);
    atomicAdd(&s.col_ptr[e.n], 1);
    atomicMax(&s.rmax[e.m], weight_i64(e.v));
    atomicMin(&s.first_m[e.n], (int)e.m);
  }
  __syncthreads();
  for (int m = tid; m < M; m += VT_THREADS) { s.cnt_m[m] = s.row_ptr[m]; s.seen_m[m] = s.row_ptr[m] > 0; }
  __syncthreads();
  block_exscan_int(s.row_ptr, M + 1, s_warp, &s_misc[1]);
  block_exscan_int(s.col_ptr, N + 1, s_warp, &s_misc[1]);
  // scatter into CSR / CSC (slot order inside a row / column is irrelevant); cursors reuse slack / ly as int scratch
  int* rcur = reinterpret_cast<int*>(s.slack);
  int* ccur = reinterpret_cast<int*>(s.ly);
  for (int m = tid; m < M; m += VT_THREADS) rcur[m] = s.row_ptr[m];
  for (int n = tid; n < N; n += VT_THREADS) ccur[n] = s.col_ptr[n];
  __syncthreads();
  for (int i = tid; i < nent; i += VT_THREADS) {
    const PosEntry e = ents[i];
    if (!ent_ok(e)) continue;
    const int a = atomicAdd(&rcur[e.m], 1);
    s.csr_n[a] = e.n; s.csr_v[a] = e.v;
    const int b = atomicAdd(&ccur[e.n], 1);
    s.csc_m[b] = e.m; s.csc_v[b] = e.v;
  }
  __syncthreads();
  // rows: seen candidates ascending, then (Sort only) the unseen ones
  const int n_seen_rows = block_scan_flags(s.seen_m, s.row_of_m, M, s_warp, &s_misc[0]);
  for (int m = tid; m < M; m += VT_THREADS)
    if (s.seen_m[m]) s.row_cand[s.row_of_m[m]] = m;
  const int nrows = VISUAL ? n_seen_rows : M;
  int n_seen_cols = 0;
  {
    // Columns in first-seen order (voting.rs:61-75 with entries visited by candidate, then store order): rank of track
    // n = tracks first touched by an earlier candidate + tracks of the same first candidate with a lower index.  A
    // histogram over the first candidates gives the former; the latter are among the (few) entries of that candidate's
    // CSR row.
    int* hist = s.alt;   // [M + 1]; the alternating-tree array is not in use before the search starts
    for (int m = tid; m <= M; m += VT_THREADS) hist[m] = 0;
    __syncthreads();
    for (int n = tid; n < N; n += VT_THREADS) {
      const int fm = s.first_m[n];
      s.col_rank[n] = -1;
      if (fm != 0x7fffffff) atomicAdd(&hist[fm], 1);
    }
    __syncthreads();
    n_seen_cols = block_exscan_int(hist, M + 1, s_warp, &s_misc[1]);
    for (int n = tid; n < N; n += VT_THREADS) {
      const int fm = s.first_m[n];
      if (fm == 0x7fffffff) continue;
      int rank = hist[fm];
      for (int q = s.row_ptr[fm]; q < s.row_ptr[fm + 1]; ++q) {
        const int n2 = s.csr_n[q];
        if (n2 < n && s.first_m[n2] == fm) ++rank;
      }
      s.col_trk[rank] = n;
      s.col_rank[n] = rank;
    }
    __syncthreads();
  }
  const int ntrk = VISUAL ? n_seen_cols : N;
  const int ny = nrows + ntrk;

  if (ntrk > 0 && nrows > 0) {
    // w(row, col) through the CSC of the column's track
    auto wgt = [&](int r, int y) -> long long {
      if (y < nrows) return y == r ? thr : 0;
      const int j = y - nrows;
      if (j >= n_seen_cols || r >= n_seen_rows) return 0;
      const int n = s.col_trk[j];
      const int m = s.row_cand[r];
      for (int q = s.col_ptr[n]; q < s.col_ptr[n + 1]; ++q)
        if (s.csc_m[q] == m) return weight_i64(s.csc_v[q]);
      return 0;
    };
    for (int r = tid; r < nrows; r += VT_THREADS) {
      long long mx = thr;
      if (ny > 1) {
        const int valid = r < n_seen_rows ? s.cnt_m[s.row_cand[r]] : 0;
        if (ny - 1 > valid) mx = mx > 0 ? mx : 0;
        if (r < n_seen_rows) { const long long rm = s.rmax[s.row_cand[r]]; mx = rm > mx ? rm : mx; }
      }
      s.lx[r] = mx;
      s.xy[r] = -1;
    }
    for (int y = tid; y < ny; y += VT_THREADS) { s.ly[y] = 0; s.yx[y] = -1; }
    __syncthreads();

    int parity = 0;
    int root = 0;
    while (root < nrows) {
      // ---- fast path: roots whose tightest column is free are matched without a block-wide search.  The labels do not
      // change on this path (delta = 0), so the tightest column of EVERY remaining root can be computed at once (one
      // thread per row over its CSR entries); the sequential walk "commit while ok and the column is still free" then
      // stops at the first root that is not ok, whose column was taken before this round, or whose column a lower
      // remaining root also wants -- found with an atomicMin of the row index per column.  Everything below that root is
      // committed in parallel: exactly the state the one-by-one walk reaches (tools/km_root_stats.py: in cfg2 / cfg4
      // scenes every root ends here, so one round replaces a 500-step serial loop of a single warp).
      {
        int* cand = s.alt;        // [ny] scratch between searches: tightest column of row r, or -1
        int* cfirst = s.slackx;   // [ny] lowest remaining row that wants column y
        for (int y = tid; y < ny; y += VT_THREADS) cfirst[y] = 0x7fffffff;
        if (tid == 0) s_misc[2] = nrows;
        __syncthreads();
        for (int r = root + tid; r < nrows; r += VT_THREADS) {
          int besty = -1;
          if (thr > 0) {
            const long long lxr = s.lx[r];
            // candidates for the minimum slack: own diagonal column and the row's valid entries
            MinPair best; best.v = lxr + s.ly[r] - thr; best.y = r;
            if (r < n_seen_rows) {
              const int m = s.row_cand[r];
              for (int q = s.row_ptr[m]; q < s.row_ptr[m + 1]; ++q) {
                const int y = nrows + s.col_rank[s.csr_n[q]];
                MinPair c; c.v = lxr + s.ly[y] - weight_i64(s.csr_v[q]); c.y = y;
                best = min_pair(best, c);
              }
            }
            // every other column has weight 0 and slack >= lx[r] > 0, so a zero here is the global minimum
            if (best.v == 0 && lxr > 0) besty = best.y;
          }
          cand[r] = besty;
          if (besty >= 0) atomicMin(&cfirst[besty], r);
        }
        __syncthreads();
        for (int r = root + tid; r < nrows; r += VT_THREADS) {
          const int y = cand[r];
          if (y < 0 || cfirst[y] != r || s.yx[y] >= 0) atomicMin(&s_misc[2], r);
        }
        __syncthreads();
        const int first_fail = s_misc[2];
        for (int r = root + tid; r < first_fail; r += VT_THREADS) {
          const int y = cand[r];
          s.xy[r] = y; s.yx[y] = r;
        }
      }
      __syncthreads();
      root = s_misc[2];
      if (root >= nrows) break;
      // ---- full label / slack search for `root` (same as the dense kernel, weights from the CSC)
      const long long lxr = s.lx[root];
      MinPair best; best.v = 9223372036854775807LL; best.y = 0x7fffffff;
      for (int y = tid; y < ny; y += VT_THREADS) {
        long long sl = lxr + s.ly[y] - wgt(root, y);
        s.slack[y] = sl; s.slackx[y] = root; s.alt[y] = -1;
        MinPair c; c.v = sl; c.y = y;
        best = min_pair(best, c);
      }
      for (int x = tid; x < nrows; x += VT_THREADS) s.inS[x] = x == root;
      best = warp_min(best);
      if (lane == 0) s_red[parity][wid] = best;
      __syncthreads();
      int y_end = -1, x_end = -1;
      for (;;) {
        MinPair g = s_red[parity][0];
#pragma unroll
        for (int w = 1; w < NWARPS; ++w) g = min_pair(g, s_red[parity][w]);
        parity ^= 1;
        const long long delta = g.v;
        const int ystar = g.y;
        const int xstar = s.slackx[ystar];
        const int x2 = s.yx[ystar];
        for (int x = tid; x < nrows; x += VT_THREADS) {
          if (s.inS[x]) { if (delta > 0) s.lx[x] -= delta; }
          else if (x == x2) s.inS[x] = 1;
        }
        if (x2 < 0) {
          if (delta > 0)
            for (int y = tid; y < ny; y += VT_THREADS) {
              if (s.alt[y] >= 0) s.ly[y] += delta;
              else s.slack[y] -= delta;
            }
          y_end = ystar; x_end = xstar;
          break;
        }
        const long long lx2 = s.lx[x2];
        MinPair nb; nb.v = 9223372036854775807LL; nb.y = 0x7fffffff;
        for (int y = tid; y < ny; y += VT_THREADS) {
          if (s.alt[y] >= 0) { if (delta > 0) s.ly[y] += delta; continue; }
          long long sl = s.slack[y] - delta;
          if (y == ystar) { s.alt[y] = xstar; s.slack[y] = sl; continue; }
          long long a = lx2 + s.ly[y] - wgt(x2, y);
          if (sl > a) { sl = a; s.slackx[y] = x2; }
          s.slack[y] = sl;
          MinPair c; c.v = sl; c.y = y;
          nb = min_pair(nb, c);
        }
        nb = warp_min(nb);
        if (lane == 0) s_red[parity][wid] = nb;
        __syncthreads();
      }
      __syncthreads();
      if (tid == 0) {
        int y = y_end, x = x_end;
        for (;;) {
          int prec = s.xy[x];
          s.yx[y] = x;
          s.xy[x] = y;
          y = prec;
          if (y < 0) break;
          x = s.alt[y];
        }
      }
      __syncthreads();
      ++root;
    }
    for (int r = tid; r < n_seen_rows; r += VT_THREADS) {
      int y = s.xy[r];
      int m = s.row_cand[r];
      if (y >= nrows && (y - nrows) < n_seen_cols) {
        winner[m] = s.col_trk[y - nrows];
        cvt[m] = (unsigned char)1;
      }
    }
  }
  __syncthreads();
  int c = 0;
  for (int m = tid; m < M; m += VT_THREADS) c += winner[m] < 0;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if (lane == 0) s_warp[wid] = c;
  __syncthreads();
  if (tid == 0) {
    int t = 0;
    for (int w = 0; w < NWARPS; ++w) t += s_warp[w];
    f.new_count[sidx] = t;
  }
}

// per-scene mode: 0 = the voting stage consumes the sparse lists, 1 = dense matrices
__device__ __forceinline__ int vis_side_mode(const Params& p, const Frame& f, const SceneDesc& sc, int s, int tc_used) {
  if (sc.m >= 65535 || sc.n >= 65535) return 1;
  if (p.is_visual) {
    if (!tc_used) return 1;
    if (f.vis_cnt[s] > sc.vis_lcap || f.vis_cnt[s] > vote_cap(p)) return 1;
    if (f.dense_bad && f.dense_bad[s]) return 1;   // dense tensor-core path: a precondition failed for this scene
  }
  return 0;
}
__global__ void scene_mode_kernel(Params p, Frame f, int n_scenes, int tc_used) {
  int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n_scenes) return;
  const SceneDesc sc = f.scenes[s];
  int mode = vis_side_mode(p, f, sc, s, tc_used);
  if (f.pos_cnt[s] > sc.pos_lcap || f.pos_cnt[s] > kVotePosCap) mode = 1;
  f.scene_mode[s] = mode;
  if (mode != 0 && f.dense_cnt) atomicAdd(f.dense_cnt, 1);
}
// the visual half alone: decided right after the screen, so the refinement does not wait for the positional stage
__global__ void vis_mode_kernel(Params p, Frame f, int n_scenes, int tc_used) {
  int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n_scenes) return;
  f.vis_mode[s] = vis_side_mode(p, f, f.scenes[s], s, tc_used);
}

void launch_scene_mode(const Params& p, const Frame& f, int n_scenes, bool tc_used, cudaStream_t st) {
  if (n_scenes == 0) return;
  scene_mode_kernel<<<(n_scenes + 127) / 128, 128, 0, st>>>(p, f, n_scenes, tc_used ? 1 : 0);
  note_launch();
}

void launch_vis_mode(const Params& p, const Frame& f, int n_scenes, bool tc_used, cudaStream_t st) {
  if (n_scenes == 0 || !f.vis_mode) return;
  vis_mode_kernel<<<(n_scenes + 127) / 128, 128, 0, st>>>(p, f, n_scenes, tc_used ? 1 : 0);
  note_launch();
}

void launch_scene_max(const Params& p, const Frame& f, int n_scenes, bool init_only, cudaStream_t st) {
  if (n_scenes == 0 || !f.scene_max) return;
  if (init_only) {
    vis_max_init_kernel<<<(n_scenes + 255) / 256, 256, 0, st>>>(f.scene_max, n_scenes);
  } else {
    dim3 grid(32, scene_grid(n_scenes));
    vis_max_kernel<<<grid, 256, 0, st>>>(p, f, f.scene_max, n_scenes);
  }
  note_launch();
}

size_t voting_smem_need(int max_m, int max_n, int viscap) {
  return std::max(vote_smem_bytes(max_m, max_n), sparse_smem_bytes(max_m, max_n, viscap > 0 ? viscap : kVoteVisCap));
}

int launch_voting(const Params& p, const TrackStore& ts, const Frame& f, int n_scenes, int max_m, int max_n,
                  cudaStream_t st) {
  if (n_scenes == 0) return 0;
  const size_t smem_d = vote_smem_bytes(max_m, max_n);
  const size_t smem_s = sparse_smem_bytes(max_m, max_n, vote_cap(p));
  if (smem_d > kVotingSmemLimit || smem_s > kVotingSmemLimit) return -3;
  cudaError_t e;
  if (p.is_visual) {
    if ((e = cudaFuncSetAttribute(voting_sparse_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_s)) != cudaSuccess) return (int)e;
    if ((e = cudaFuncSetAttribute(voting_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_d)) != cudaSuccess) return (int)e;
    voting_sparse_kernel<true, false><<<n_scenes, VT_THREADS, smem_s, st>>>(p, ts, f);
    voting_kernel<true><<<n_scenes, VT_THREADS, smem_d, st>>>(p, f);
    note_launch(2);
  } else {
    if ((e = cudaFuncSetAttribute(voting_sparse_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_s)) != cudaSuccess) return (int)e;
    if ((e = cudaFuncSetAttribute(voting_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_d)) != cudaSuccess) return (int)e;
    voting_sparse_kernel<false, false><<<n_scenes, VT_THREADS, smem_s, st>>>(p, ts, f);
    voting_kernel<false><<<n_scenes, VT_THREADS, smem_d, st>>>(p, f);
    note_launch(2);
  }
  return 0;
}

int launch_vote_masks(const Params& p, const TrackStore& ts, const Frame& f, int n_scenes, int max_m, int max_n,
                      cudaStream_t st) {
  if (n_scenes == 0 || !p.is_visual || !f.decided || !f.excl) return 0;
  const size_t smem_s = sparse_smem_bytes(max_m, max_n, vote_cap(p));
  if (smem_s > kVotingSmemLimit) return -3;
  cudaError_t e = cudaFuncSetAttribute(voting_sparse_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_s);
  if (e != cudaSuccess) return (int)e;
  voting_sparse_kernel<true, true><<<n_scenes, VT_THREADS, smem_s, st>>>(p, ts, f);
  note_launch();
  return 0;
}

}  // namespace sb
