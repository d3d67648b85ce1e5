// kernels_feat_tc.cu -- visual (ReID feature) cost matrix: tensor-core screen (wgmma + TMA + mbarrier) followed by
// an exact f32 refinement of the surviving pairs.
//
// What the reference computes (src/distance.rs:9-47, src/trackers/visual_sort/metric.rs:200-295): for every
// (candidate, track-observation) pair the f32 euclidean / cosine distance, kept only if it passes the metric's
// threshold (euclid d <= thr, cosine cos >= thr).  After thresholding the matrix is sparse: a detection is close to a
// handful of observations of "its" track and far from everything else.
//
// GPU shape:
//   1. screen  : C~[m][c] = sum_d A[m][d] * B[c][d] with BF16 operand copies on the tensor cores (wgmma m64n256k16,
//                fp32 accumulation in registers).  The BF16 rounding error of the dot product is bounded by
//                E = 2^-8 * ||a|| * ||b|| (Cauchy-Schwarz), so a pair can only pass the threshold if its screened value is
//                within E of it.  Everything else is written as None (NaN) straight from the epilogue; survivors are
//                appended to a compact pair list.
//   2. refine  : one warp per surviving pair recomputes the distance in f32 in the reference's exact summation order
//                (8-lane blocks, horizontal reduce_add, sequential block accumulation) and applies is_ok /
//                distance_to_weight.  Every value that reaches the voting stage is therefore bit-identical to the
//                CPU reference -- the tensor cores only decide which pairs are worth computing.
//   If the pair list overflows (a non-selective threshold) the caller falls back to the dense exact SIMT kernel.
//
// Screen kernels: persistent 2-CTA clusters (one CTA per SM), 384 threads = a producer warpgroup (one TMA thread) and two
// consumer warpgroups.  d8 <= 512 (vis_screen_sa_kernel): the cluster's candidate rows stay in shared memory for a whole
// work unit and only the track-observation rows stream; each consumer warpgroup owns whole 128 x 128 output tiles and the
// two take turns on the tensor pipe.  d8 > 512 (vis_screen_kernel): tile 128 (candidates) x 256 (track-observation rows)
// x 64 (features = one 128-byte swizzle atom of bf16), both operands streamed through 4 smem stages of 48 KB; each
// consumer warpgroup accumulates 64 candidate rows x 256 columns in registers and screens them in place.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>

#include "sb_engine.cuh"
#include "sb_tc.cuh"

namespace sb {

constexpr int TC_STAGES = 4;          // 48 KB stages (A tile + whole B tile)
constexpr int TC_STAGE_BYTES = TC_A_BYTES + TC_B_BYTES;  // 48 KB

struct TcHdr { int scene, m0, ncols_left, m, det_base, col0, epoch, vis_lbase, vis_lcap, pad; };
struct TcSmem {
  unsigned char stage[TC_STAGES][TC_STAGE_BYTES];  // 1024-byte aligned operand stages first
  // four slab sets of per-tile metadata, bulk-copied by the producer warp: it runs up to three tiles ahead
  VisColMeta meta[4][TC_BN];
  VisRowMeta rowm[4][TC_BM];
  float colb[4][TC_BN];
  unsigned int colvalid[4][TC_BN / 32];
  TcHdr hdr[4];
  unsigned long long full_bar[TC_STAGES];
  unsigned long long empty_bar[TC_STAGES];
  unsigned long long meta_full[4];
  unsigned long long meta_empty[4];
};
static_assert(sizeof(TcSmem) + 1024 <= 227 * 1024, "screen kernel exceeds the shared memory of an SM");


// ------------------------------------------------------------------------------------------------ screen kernel, d8 > 512
// Clusters of two CTAs work on two candidate tiles (m0, m0 + 128) of the same track-row tile; each CTA loads its own A
// tile and HALF of the B tile, multicast into both CTAs' shared memory, so B crosses L2 -> SM once per pair.
template <bool COSINE>
__global__ void __launch_bounds__(TC_THREADS, 1)
vis_screen_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB, Params p,
                  TrackStore ts, Frame f, const TcTile* tiles, int n_tiles_host, const int* n_tiles_dev,
                  const VisColMeta* colmeta, const VisColGeo* colgeo, const VisRowMeta* rowmeta, const float* colb,
                  const unsigned int* colvalid) {
  // trackers: the tile list is built on the device (frame_setup_kernel) and so is its length
  const int n_tiles = n_tiles_dev ? *n_tiles_dev : n_tiles_host;
  extern __shared__ unsigned char smem_raw_[];
  // offset arithmetic on the __shared__ array (not on an integer) keeps the accesses in the shared address space
  TcSmem& S = *reinterpret_cast<TcSmem*>(smem_raw_ + ((1024u - (smem_u32(smem_raw_) & 1023u)) & 1023u));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int K = p.max_obs;
  const int KB = (p.d8 + TC_BK - 1) / TC_BK;

  unsigned char* const stage_base = &S.stage[0][0];
  const uint32_t crank = cluster_rank();
  const int cta_first = (int)(blockIdx.x >> 1);   // first (cluster) tile of this CTA
  const int cta_step = (int)(gridDim.x >> 1);
  if (threadIdx.x == 0) {
    // empty: one arrival per consumer warpgroup of every CTA that reads the stage's bytes; meta_empty: the 8 consumer warps
    for (int s = 0; s < TC_STAGES; ++s) { mbar_init(&S.full_bar[s], 1); mbar_init(&S.empty_bar[s], 4); }
    for (int b = 0; b < 4; ++b) { mbar_init(&S.meta_full[b], 1); mbar_init(&S.meta_empty[b], 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  cluster_sync_all();   // the peer's barriers are initialised before anything is multicast into them

  if (warp < 4) {
    // ===================================================================== TMA producer (one thread); the warpgroup hands
    // most of its registers to the consumers, whose accumulators alone take 128 per thread
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp == 0 && lane == 0) {
      asm volatile("prefetch.tensormap [%0];" ::"l"((uint64_t)&mapA) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"((uint64_t)&mapB) : "memory");
      int stage = 0;
      uint32_t phase = 0;
      int it = 0;
      TcTile tl_n;
      tl_n.scene = 0; tl_n.m0 = 0; tl_n.c0 = 0; tl_n.pad = 0;
      if (cta_first < n_tiles) tl_n = tiles[cta_first];
      SceneDesc sc_n = f.scenes[tl_n.scene];
      for (int t = cta_first; t < n_tiles; t += cta_step, ++it) {
        const TcTile tl = tl_n;
        const SceneDesc sc = sc_n;
        if (t + cta_step < n_tiles) { tl_n = tiles[t + cta_step]; sc_n = f.scenes[tl_n.scene]; }
        const int m0 = tl.m0 + (int)crank * TC_BM;
        const int rowA = sc.det_base + m0;
        const int rowB = sc.slot * ts.track_cap * K + tl.c0;
        {
          // metadata of this tile: header by plain stores (published by the release of the arrive below), column / row
          // slabs by bulk copies that complete on the same barrier
          const int g = it & 3;
          mbar_wait(&S.meta_empty[g], ((it >> 2) & 1) ^ 1);
          TcHdr h;
          h.scene = tl.scene; h.m0 = m0; h.ncols_left = sc.nb * K - tl.c0; h.m = sc.m; h.det_base = sc.det_base;
          h.col0 = sc.col_off + tl.c0; h.epoch = (int)sc.epoch; h.vis_lbase = sc.vis_lbase; h.vis_lcap = sc.vis_lcap; h.pad = 0;
          S.hdr[g] = h;
          mbar_expect_tx(&S.meta_full[g], (uint32_t)(sizeof(VisColMeta) * TC_BN + sizeof(VisRowMeta) * TC_BM +
                                                    4 * TC_BN + TC_BN / 8));
          bulk_load(S.meta[g], colmeta + h.col0, (uint32_t)(sizeof(VisColMeta) * TC_BN), &S.meta_full[g]);
          bulk_load(S.rowm[g], rowmeta + rowA, (uint32_t)(sizeof(VisRowMeta) * TC_BM), &S.meta_full[g]);
          bulk_load(S.colb[g], colb + h.col0, 4 * TC_BN, &S.meta_full[g]);
          bulk_load(S.colvalid[g], colvalid + (h.col0 >> 5), TC_BN / 8, &S.meta_full[g]);   // col0 is a multiple of 128
        }
        for (int kb = 0; kb < KB; ++kb) {
          mbar_wait(&S.empty_bar[stage], phase ^ 1);   // both CTAs have released the stage
          unsigned char* base = stage_base + stage * TC_STAGE_BYTES;
          mbar_expect_tx(&S.full_bar[stage], TC_STAGE_BYTES);
          tma_load_2d(base, &mapA, kb * TC_BK, rowA, &S.full_bar[stage]);
          // this CTA's half of the B tile (rows rank*128 .. +128), delivered to both CTAs
          tma_load_2d_mc(base + TC_A_BYTES + crank * (TC_B_BYTES / 2), &mapB, kb * TC_BK, rowB + (int)crank * (TC_BN / 2),
                         &S.full_bar[stage], (uint16_t)0x3);
          if (++stage == TC_STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ===================================================================== consumer warpgroups 1 and 2
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    // Warpgroup wg owns candidate rows wg*64 .. +64 of every tile.  Thread layout of the accumulators (wgmma): register i
    // holds row rr[(i >> 1) & 1] and column 8 * (i >> 2) + 2 * (lane & 3) + (i & 1).  All per-tile metadata arrives in
    // shared memory through the producer warp's bulk copies: the epilogue issues no global load on its common path.
    const int wg = (warp >> 2) - 1;
    const int rr[2] = {wg * TC_WG_ROWS + (warp & 3) * 16 + (lane >> 2), wg * TC_WG_ROWS + (warp & 3) * 16 + (lane >> 2) + 8};
    const int q2 = 2 * (lane & 3);
    const bool geo = p.n_constraints > 0;
    int stage = 0;
    uint32_t phase = 0;
    int it = 0;
    for (int t = cta_first; t < n_tiles; t += cta_step, ++it) {
      float acc[128];
      tc_consume_tile<2, TC_STAGES, TC_STAGE_BYTES>(acc, stage_base, S.full_bar, S.empty_bar, KB, wg, stage, phase);
      const int ms = it & 3;   // slab set of this tile (same rule as the producer)
      mbar_wait(&S.meta_full[ms], (it >> 2) & 1);
      const VisColMeta* gmeta = S.meta[ms];
      const TcHdr h = S.hdr[ms];
      const float* gcolb = S.colb[ms];
      // Screen test, E = p.vis_rel_err (screen_rel_err) bounds the BF16 operand rounding (|dot~ - dot| <= E |a||b| <= E (|a|^2 + |b|^2) / 2):
      //   cosine: cos >= thr possible   <=>  dot~ >= (thr - 1e-5 - E) |a| * |b|                                = rowk * colb
      //   euclid: d^2 <= thr^2 possible <=>  dot~ >= 0.5 ((1 - 1e-5 - E)(|a|^2 + |b|^2) - thr^2 (1 + 1e-5))   = rowk + colb
      float rowk[2];
      bool row_ok[2];
      int g[2];
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        const VisRowMeta rm = S.rowm[ms][rr[hr]];
        const int m = h.m0 + rr[hr];
        row_ok[hr] = m < h.m && rm.ok;
        g[hr] = h.det_base + m;
        rowk[hr] = rm.rowk;
      }
      // bit i of keep[i >> 5]: the pair of accumulator register i survives the screen
      unsigned int keep[4] = {0u, 0u, 0u, 0u};
#pragma unroll
      for (int j = 0; j < TC_BN / 8; ++j) {
        const int c0 = 8 * j + q2;
        const float2 cb = *reinterpret_cast<const float2*>(gcolb + c0);
        const unsigned int vw = S.colvalid[ms][c0 >> 5] >> (c0 & 31);   // columns without a usable observation never survive
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int hr = e >> 1, cl = e & 1;
          const float b = COSINE ? rowk[hr] * (cl ? cb.y : cb.x) : rowk[hr] + (cl ? cb.y : cb.x);
          // a NaN anywhere keeps the pair: the exact pass decides; columns past the scene's last track row hold foreign
          // metadata
          const bool k = !(acc[4 * j + e] < b) && ((vw >> cl) & 1u) && c0 + cl < h.ncols_left && row_ok[hr];
          if (k) keep[j >> 3] |= 1u << (((4 * j) & 31) + e);
        }
      }
      if (geo) {
        float cx[2], cy[2], cr[2];
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          cx[hr] = 0.0f; cy[hr] = 0.0f; cr[hr] = 0.0f;
          if (row_ok[hr]) { cx[hr] = f.c_box[(size_t)g[hr] * 6]; cy[hr] = f.c_box[(size_t)g[hr] * 6 + 1]; cr[hr] = f.c_radius[g[hr]]; }
        }
#pragma unroll
        for (int w = 0; w < 4; ++w) {
          unsigned int kk = keep[w];
          while (kk) {
            const int b = __ffs(kk) - 1;
            kk &= kk - 1;
            const int i = w * 32 + b, hr = (i >> 1) & 1;
            const int col = 8 * (i >> 2) + q2 + (i & 1);
            const VisColGeo cg = colgeo[h.col0 + col];   // rare path: straight from global memory
            if (!compat_ok(p, (unsigned int)h.epoch, cg.tep, cx[hr], cy[hr], cr[hr], cg.tx, cg.ty, cg.tr)) keep[w] &= ~(1u << b);
          }
        }
      }
      // survivors -> pair list, ONE warp-aggregated append per tile (a thread's pairs row by row); everything else is None
      int cnt = 0;
#pragma unroll
      for (int w = 0; w < 4; ++w) cnt += __popc(keep[w]);
      if (__any_sync(0xffffffffu, cnt != 0)) {
        int incl = cnt;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          int tt = __shfl_up_sync(0xffffffffu, incl, o);
          if (lane >= o) incl += tt;
        }
        const int total = __shfl_sync(0xffffffffu, incl, 31);
        int base = 0;
        if (lane == 31) base = atomicAdd(&f.vis_cnt[h.scene], total);
        base = __shfl_sync(0xffffffffu, base, 31);
        int pos = base + incl - cnt;
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
#pragma unroll
          for (int w = 0; w < 4; ++w) {
            unsigned int kk = keep[w] & (hr ? 0xccccccccu : 0x33333333u);
            while (kk) {
              const int b = __ffs(kk) - 1;
              kk &= kk - 1;
              if (pos < h.vis_lcap) {
                const int i = w * 32 + b;
                const VisColMeta cm = gmeta[8 * (i >> 2) + q2 + (i & 1)];
                VisPair vp;
                vp.g = g[hr]; vp.row = cm.row; vp.scene = h.scene; vp.outcol = cm.outcol;
                f.vis_pairs[h.vis_lbase + pos] = vp;
              }
              ++pos;
            }
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&S.meta_empty[ms]);   // the slabs of this tile may be overwritten
    }
  }
  __syncthreads();
  cluster_sync_all();   // no CTA leaves while its peer may still multicast into / arrive on its smem
}

// ------------------------------------------------------------------------------------------------ screen kernel, d8 <= 512
// A-stationary organisation.  A work unit is (scene, pair of 128-row candidate tiles, range of track-observation rows)
// and one 2-CTA cluster runs it: each CTA keeps its 128 candidate rows x d8 resident in shared memory (loaded once per
// unit, each 64-feature block on its own barrier so the first column tile starts on the first block) and streams the
// unit's B rows through a FIFO ring of 128-row x 64-feature stages, half of every stage loaded by each CTA and multicast
// to both.  Only B crosses L2 -> SM per output tile: 64 KB per CTA per 128 x 128 x 512 tile.
//
// Ping-pong consumers: the column tiles of the cluster's units form one sequence; consumer warpgroup 0 takes the even
// positions, warpgroup 1 the odd ones, and each holds a whole 128 x 128 tile (two m64n128 MMAs per k16 step, 128 fp32
// accumulators).  A pair of named barriers hands the tensor pipe from one warpgroup's mainloop to the other's, so one
// warpgroup screens its tile while the other's MMAs run.
constexpr int SA_BN = 128;                          // track-observation rows per column tile (one warpgroup's tile)
constexpr int SA_KMAX = 8;                          // 64-feature blocks of A kept resident: d8 <= 512
constexpr int SA_A_BLOCK = TC_BM * TC_BK * 2;       // 16 KB
constexpr int SA_B_STAGE = SA_BN * TC_BK * 2;       // 16 KB
constexpr int SA_STAGES = 5;
constexpr int SA_SLABS = 4;                         // column-tile metadata slabs in flight
struct SaHdr { int scene, m0, ncols, m, det_base, col0, epoch, vis_lbase, vis_lcap, unit, last, pad; };
struct SaSmem {
  unsigned char a[SA_KMAX][SA_A_BLOCK];             // 1024-byte aligned operand buffers first
  unsigned char b[SA_STAGES][SA_B_STAGE];
  VisColMeta meta[SA_SLABS][SA_BN];
  float colb[SA_SLABS][SA_BN];
  float colsb[SA_SLABS][SA_BN];                     // e4m3 Euclidean screen only: the columns' scales
  unsigned int colvalid[SA_SLABS][SA_BN / 32];
  SaHdr hdr[SA_SLABS];
  unsigned long long a_full[SA_KMAX];
  unsigned long long a_empty;
  unsigned long long full_bar[SA_STAGES];
  unsigned long long empty_bar[SA_STAGES];
  unsigned long long meta_full[SA_SLABS];
  unsigned long long meta_empty[SA_SLABS];
};
static_assert(sizeof(SaSmem) + 1024 <= 227 * 1024, "A-stationary screen kernel exceeds the shared memory of an SM");
constexpr int kScreenStationaryMaxD8 = SA_KMAX * TC_BK;

// units: TcTile (scene, m0, c0) with m0 a multiple of 256 and c0 a multiple of ucols; the unit covers the scene's rows
// c0 .. min(c0 + ucols, nb * K)
//
// FP8: the operands are the e4m3 copies (f.c_fp8, ts.feat_fp8) and every MMA is m64n128k32.e4m3.  A 128-byte swizzle row
// then holds 128 features instead of 64: the same 16 KB blocks and stages carry twice the features, so A takes half the
// blocks and the k-loop half the trips.  The row and column constants carry the rows' scales (vis_rowmeta_kernel,
// vis_meta_kernel): the cosine test stays rowk * colb, the Euclidean one becomes acc * rowi >= fma(colsb, rowk, colb).
template <bool COSINE, bool FP8>
__global__ void __launch_bounds__(TC_THREADS, 1)
vis_screen_sa_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB, Params p,
                     TrackStore ts, Frame f, const TcTile* units, int n_units_host, const int* n_units_dev, int ucols,
                     const VisColMeta* colmeta, const VisColGeo* colgeo, const VisRowMeta* rowmeta, const float* colb,
                     const float* colsb, const unsigned int* colvalid) {
  constexpr bool kScaled = FP8 && !COSINE;   // the Euclidean e4m3 test needs the columns' scales
  constexpr int BKF = FP8 ? 2 * TC_BK : TC_BK;   // features per 128-byte swizzle row
  const int n_units = n_units_dev ? *n_units_dev : n_units_host;
  extern __shared__ unsigned char smem_raw_[];
  SaSmem& S = *reinterpret_cast<SaSmem*>(smem_raw_ + ((1024u - (smem_u32(smem_raw_) & 1023u)) & 1023u));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int K = p.max_obs;
  const int KB = (p.d8 + BKF - 1) / BKF;
  const uint32_t crank = cluster_rank();
  if (threadIdx.x == 0) {
    // full: the local producer's expect_tx; empty: the consuming warpgroup of each CTA; a_empty: both local consumer
    // warpgroups (or the producer for a warpgroup without a tile in the unit); meta_empty: the 4 warps of the consumer
    for (int kb = 0; kb < SA_KMAX; ++kb) mbar_init(&S.a_full[kb], 1);
    mbar_init(&S.a_empty, 2);
    for (int s = 0; s < SA_STAGES; ++s) { mbar_init(&S.full_bar[s], 1); mbar_init(&S.empty_bar[s], 2); }
    for (int b = 0; b < SA_SLABS; ++b) { mbar_init(&S.meta_full[b], 1); mbar_init(&S.meta_empty[b], 4); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  cluster_sync_all();   // the peer's barriers are initialised before anything is multicast into them

  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp == 0 && lane == 0) {
      asm volatile("prefetch.tensormap [%0];" ::"l"((uint64_t)&mapA) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"((uint64_t)&mapB) : "memory");
      int seq = 0, gk = 0, unit = 0;
      for (int u = (int)(blockIdx.x >> 1); u < n_units; u += (int)(gridDim.x >> 1), ++unit) {
        const TcTile tl = units[u];
        const SceneDesc sc = f.scenes[tl.scene];
        const int m0 = tl.m0 + (int)crank * TC_BM;
        const int rowA = sc.det_base + m0;
        const int cols = min(ucols, sc.nb * K - tl.c0);
        const int nct = (cols + SA_BN - 1) / SA_BN;
        const int rowB = sc.slot * ts.track_cap * K + tl.c0;
        // A stays until both warpgroups have completed the MMAs of the previous unit
        if (unit > 0) mbar_wait(&S.a_empty, (unit - 1) & 1);
        if (nct == 1) mbar_arrive(&S.a_empty);   // on behalf of the warpgroup without a tile in this unit
        for (int ct = 0; ct < nct; ++ct, ++seq) {
          const int g = seq % SA_SLABS;
          mbar_wait(&S.meta_empty[g], ((seq / SA_SLABS) & 1) ^ 1);
          SaHdr h;
          h.scene = tl.scene; h.m0 = m0; h.ncols = min(SA_BN, cols - ct * SA_BN); h.m = sc.m; h.det_base = sc.det_base;
          h.col0 = sc.col_off + tl.c0 + ct * SA_BN; h.epoch = (int)sc.epoch; h.vis_lbase = sc.vis_lbase;
          h.vis_lcap = sc.vis_lcap; h.unit = unit; h.last = ct + 2 >= nct; h.pad = 0;
          S.hdr[g] = h;   // published by the release of the arrive below
          mbar_expect_tx(&S.meta_full[g], (uint32_t)(sizeof(VisColMeta) * SA_BN + (kScaled ? 8 : 4) * SA_BN + SA_BN / 8));
          bulk_load(S.meta[g], colmeta + h.col0, (uint32_t)(sizeof(VisColMeta) * SA_BN), &S.meta_full[g]);
          bulk_load(S.colb[g], colb + h.col0, 4 * SA_BN, &S.meta_full[g]);
          if (kScaled) bulk_load(S.colsb[g], colsb + h.col0, 4 * SA_BN, &S.meta_full[g]);
          bulk_load(S.colvalid[g], colvalid + (h.col0 >> 5), SA_BN / 8, &S.meta_full[g]);   // col0 is a multiple of 128
          for (int kb = 0; kb < KB; ++kb, ++gk) {
            if (ct == 0) {
              mbar_expect_tx(&S.a_full[kb], SA_A_BLOCK);
              tma_load_2d(S.a[kb], &mapA, kb * BKF, rowA, &S.a_full[kb]);
            }
            const int s = gk % SA_STAGES;
            mbar_wait(&S.empty_bar[s], ((gk / SA_STAGES) & 1) ^ 1);   // both CTAs have released the stage
            mbar_expect_tx(&S.full_bar[s], SA_B_STAGE);
            // this CTA's half of the stage (rows rank*64 .. +64), delivered to both CTAs
            tma_load_2d_mc(S.b[s] + crank * (SA_B_STAGE / 2), &mapB, kb * BKF, rowB + ct * SA_BN + (int)crank * (SA_BN / 2),
                           &S.full_bar[s], (uint16_t)0x3);
          }
        }
      }
      // two end markers: one for each consumer warpgroup
      for (int e = 0; e < 2; ++e, ++seq) {
        const int g = seq % SA_SLABS;
        mbar_wait(&S.meta_empty[g], ((seq / SA_SLABS) & 1) ^ 1);
        S.hdr[g].scene = -1 - e;
        mbar_arrive(&S.meta_full[g]);
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    // Warpgroup wg screens the column tiles at positions wg, wg + 2, ... of the cluster's sequence.  Accumulator register
    // i (0..127) holds row 64 * (i >> 6) + rr[(i >> 1) & 1] and column 8 * ((i & 63) >> 2) + q2 + (i & 1).
    const int wg = (warp >> 2) - 1;
    const int rr[2] = {(warp & 3) * 16 + (lane >> 2), (warp & 3) * 16 + (lane >> 2) + 8};
    const int q2 = 2 * (lane & 3);
    const bool geo = p.n_constraints > 0;
    const bool elected = (threadIdx.x & 127) == 0;
    for (int pos = wg;; pos += 2) {
      const int ms = pos % SA_SLABS;
      mbar_wait(&S.meta_full[ms], (pos / SA_SLABS) & 1);
      const SaHdr h = S.hdr[ms];
      // named barriers 1 + (pos & 1): the warpgroup at position pos waits for the mainloop of position pos - 1
      if (pos > 0) wg2_bar_sync(1 + (pos & 1));
      if (h.scene < 0) {
        if (h.scene == -1) wg2_bar_arrive(1 + ((pos + 1) & 1));   // lets the other warpgroup reach its end marker
        break;
      }
      // row constants of the 4 rows of this thread (rows past the tile's candidates read padding and are masked)
      float rowk[2][2], rowi[2][2];
      bool row_ok[2][2];
#pragma unroll
      for (int hh = 0; hh < 2; ++hh)
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          const int m = h.m0 + 64 * hh + rr[hr];
          const VisRowMeta rm = rowmeta[h.det_base + m];
          rowk[hh][hr] = rm.rowk;
          rowi[hh][hr] = rm.rowi;
          row_ok[hh][hr] = m < h.m && rm.ok;
        }

      float acc[128];
      {
        const int g0 = pos * KB;
        int stage = g0 % SA_STAGES;
        uint32_t phase = (g0 / SA_STAGES) & 1;
        int prev = -1;
        auto release = [&](int s) {
          if (elected)
            for (uint32_t r = 0; r < 2; ++r) mbar_arrive_cluster(cluster_addr(&S.empty_bar[s], r));
        };
        for (int kb = 0; kb < KB; ++kb) {
          mbar_wait(&S.a_full[kb], (uint32_t)h.unit & 1u);
          mbar_wait(&S.full_bar[stage], phase);
          const uint32_t a0 = smem_u32(S.a[kb]);
          const uint32_t b0 = smem_u32(S.b[stage]);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < 4; ++k) {   // 32 bytes of the 128-byte swizzle row per MMA: k16 of BF16, k32 of e4m3
            const uint32_t acc_on = (kb | k) != 0 ? 1u : 0u;
            if (FP8) {
              wgmma_e4m3_m64n128(acc, wgmma_desc(a0 + k * 32), wgmma_desc(b0 + k * 32), acc_on);
              wgmma_e4m3_m64n128(acc + 64, wgmma_desc(a0 + 64 * 128 + k * 32), wgmma_desc(b0 + k * 32), acc_on);
            } else {
              wgmma_bf16_m64n128(acc, wgmma_desc(a0 + k * 32), wgmma_desc(b0 + k * 32), acc_on);
              wgmma_bf16_m64n128(acc + 64, wgmma_desc(a0 + 64 * 128 + k * 32), wgmma_desc(b0 + k * 32), acc_on);
            }
          }
          wgmma_commit();
          wgmma_wait<1>();   // the previous stage's MMAs have completed
          if (prev >= 0) release(prev);
          prev = stage;
          if (++stage == SA_STAGES) { stage = 0; phase ^= 1; }
        }
        wg2_bar_arrive(1 + ((pos + 1) & 1));   // the other warpgroup's mainloop may start
        wgmma_wait<0>();
        wgmma_fence_acc(acc);
        release(prev);
        if (h.last && elected) mbar_arrive(&S.a_empty);   // this warpgroup's last MMAs on the unit's A have completed
      }

      // Screen test (see vis_screen_kernel).  Column and row conditions are folded into masks built once per tile, so
      // the inner loop is the test alone; a NaN accumulator keeps the pair.
      const VisColMeta* gmeta = S.meta[ms];
      const float* gcolb = S.colb[ms];
      unsigned int colm[2] = {0u, 0u};   // bit i & 31 of colm[i >> 5] (i = register index within a 64-row half)
#pragma unroll
      for (int j = 0; j < SA_BN / 8; ++j) {
        const int c0 = 8 * j + q2;
        unsigned int m2 = (S.colvalid[ms][c0 >> 5] >> (c0 & 31)) & 3u;
        m2 &= (c0 < h.ncols ? 1u : 0u) | (c0 + 1 < h.ncols ? 2u : 0u);
        colm[j >> 3] |= (m2 | (m2 << 2)) << ((4 * j) & 31);
      }
      unsigned int keep[4];
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const unsigned int rowm = (row_ok[hh][0] ? 0x33333333u : 0u) | (row_ok[hh][1] ? 0xccccccccu : 0u);
        keep[2 * hh] = 0u;
        keep[2 * hh + 1] = 0u;
#pragma unroll
        for (int j = 0; j < SA_BN / 8; ++j) {
          const float2 cb = *reinterpret_cast<const float2*>(gcolb + 8 * j + q2);
          float2 cs = make_float2(1.0f, 1.0f);
          if (kScaled) cs = *reinterpret_cast<const float2*>(&S.colsb[ms][8 * j + q2]);
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float rk = rowk[hh][e >> 1], c = (e & 1) ? cb.y : cb.x;
            if (kScaled) {
              // acc = 2^(ka + kb) dot~: acc 2^-ka >= 2^kb (rowk + colb), both sides exact scalings of the BF16 test's
              const float b = __fmaf_rn((e & 1) ? cs.y : cs.x, rk, c);
              if (!(acc[64 * hh + 4 * j + e] * rowi[hh][e >> 1] < b)) keep[2 * hh + (j >> 3)] |= 1u << ((4 * j + e) & 31);
            } else {
              const float b = COSINE ? rk * c : rk + c;
              if (!(acc[64 * hh + 4 * j + e] < b)) keep[2 * hh + (j >> 3)] |= 1u << ((4 * j + e) & 31);
            }
          }
        }
        keep[2 * hh] &= colm[0] & rowm;
        keep[2 * hh + 1] &= colm[1] & rowm;
      }
      if (geo) {
        float cx[2][2], cy[2][2], cr[2][2];
#pragma unroll
        for (int hh = 0; hh < 2; ++hh)
#pragma unroll
          for (int hr = 0; hr < 2; ++hr) {
            cx[hh][hr] = 0.0f; cy[hh][hr] = 0.0f; cr[hh][hr] = 0.0f;
            if (row_ok[hh][hr]) {
              const size_t g = (size_t)h.det_base + h.m0 + 64 * hh + rr[hr];
              cx[hh][hr] = f.c_box[g * 6]; cy[hh][hr] = f.c_box[g * 6 + 1]; cr[hh][hr] = f.c_radius[g];
            }
          }
#pragma unroll
        for (int w = 0; w < 4; ++w) {
          unsigned int kk = keep[w];
          while (kk) {
            const int b = __ffs(kk) - 1;
            kk &= kk - 1;
            const int i = (w & 1) * 32 + b, hh = w >> 1;
            const bool r8 = (i >> 1) & 1;   // selects, not an index: the row arrays stay in registers
            const int col = 8 * (i >> 2) + q2 + (i & 1);
            const VisColGeo cg = colgeo[h.col0 + col];   // rare path: straight from global memory
            if (!compat_ok(p, (unsigned int)h.epoch, cg.tep, r8 ? cx[hh][1] : cx[hh][0], r8 ? cy[hh][1] : cy[hh][0],
                           r8 ? cr[hh][1] : cr[hh][0], cg.tx, cg.ty, cg.tr))
              keep[w] &= ~(1u << b);
          }
        }
      }
      // survivors -> pair list, ONE warp-aggregated append per tile (a thread's pairs row by row)
      int cnt = 0;
#pragma unroll
      for (int w = 0; w < 4; ++w) cnt += __popc(keep[w]);
      if (__any_sync(0xffffffffu, cnt != 0)) {
        int incl = cnt;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          int tt = __shfl_up_sync(0xffffffffu, incl, o);
          if (lane >= o) incl += tt;
        }
        const int total = __shfl_sync(0xffffffffu, incl, 31);
        int base = 0;
        if (lane == 31) base = atomicAdd(&f.vis_cnt[h.scene], total);
        base = __shfl_sync(0xffffffffu, base, 31);
        int at = base + incl - cnt;
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
#pragma unroll
          for (int hr = 0; hr < 2; ++hr) {
            const int g = h.det_base + h.m0 + 64 * hh + rr[hr];
#pragma unroll
            for (int w = 0; w < 2; ++w) {
              unsigned int kk = keep[2 * hh + w] & (hr ? 0xccccccccu : 0x33333333u);
              while (kk) {
                const int b = __ffs(kk) - 1;
                kk &= kk - 1;
                if (at < h.vis_lcap) {
                  const int i = w * 32 + b;
                  const VisColMeta cm = gmeta[8 * (i >> 2) + q2 + (i & 1)];
                  VisPair vp;
                  vp.g = g; vp.row = cm.row; vp.scene = h.scene; vp.outcol = cm.outcol;
                  f.vis_pairs[h.vis_lbase + at] = vp;
                }
                ++at;
              }
            }
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&S.meta_empty[ms]);   // the slabs of this tile may be overwritten
    }
  }
  __syncthreads();
  cluster_sync_all();   // no CTA leaves while its peer may still multicast into / arrive on its smem
}

// ------------------------------------------------------------------------------------------------ refine kernel
// One warp per surviving pair: f32 distance in the reference's summation order (src/distance.rs:9-47).

// A warp takes RF_CLAIM pairs at a time.  Phase 1 (cooperative, coalesced): for every pair the lanes compute the 8-element
// block sums s_blk = reduce_add8(...) of up to 64 blocks and park them in shared memory.  Phase 2: lane p owns pair p and
// adds its block sums strictly in block order, acc = (..((0 + s_0) + s_1) + ..), which is the reference's order; the
// serial chains run side by side instead of one 64-step shuffle chain per pair.
constexpr int RF_WARPS = 4;
constexpr int RF_SEG = 64;             // blocks per segment
constexpr int RF_PITCH = RF_SEG + 1;   // +1: lane p reads row p, rows must start in different banks
// 16 survivors per claim rather than 32: half the parked block sums, so eight CTAs fit an SM instead of six
constexpr int RF_CLAIM = 16;

// a-side of a block sum: the candidate's 8 features of block `blk` (zero padded past D on the TAIL path), widened to f32
// when the request's column is a 2-byte type (one 16-byte load per block)
template <bool TAIL>
__device__ __forceinline__ void refine_load_a(const float* __restrict__ a, int blk, int D, float* av) {
  if (!TAIL) {
    const float4 a0 = *reinterpret_cast<const float4*>(a + blk * 8);
    const float4 a1 = *reinterpret_cast<const float4*>(a + blk * 8 + 4);
    av[0] = a0.x; av[1] = a0.y; av[2] = a0.z; av[3] = a0.w; av[4] = a1.x; av[5] = a1.y; av[6] = a1.z; av[7] = a1.w;
  } else {
#pragma unroll
    for (int l = 0; l < 8; ++l) av[l] = blk * 8 + l < D ? a[blk * 8 + l] : 0.0f;   // the input row has D, not d8, floats
  }
}
template <bool TAIL, class T>
__device__ __forceinline__ void refine_load_a(const T* __restrict__ a, int blk, int D, float* av) {
  if (!TAIL) {
    feat_widen8(*reinterpret_cast<const uint4*>(a + blk * 8), a, av);
  } else {
#pragma unroll
    for (int l = 0; l < 8; ++l) av[l] = blk * 8 + l < D ? feat_elem(a, blk * 8 + l) : 0.0f;
  }
}
template <bool COSINE>
__device__ __forceinline__ float refine_block_sum(const float* av, const float* __restrict__ b, int blk) {
  const float4 b0 = *reinterpret_cast<const float4*>(b + blk * 8);
  const float4 b1 = *reinterpret_cast<const float4*>(b + blk * 8 + 4);
  const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
  float t[8];
#pragma unroll
  for (int l = 0; l < 8; ++l) {
    if (COSINE) t[l] = av[l] * bb[l];
    else { const float df = av[l] - bb[l]; t[l] = df * df; }
  }
  return reduce_add8(t);
}

// T: element type of the request's feature column
template <bool COSINE, bool TAIL, class T>
__global__ void __launch_bounds__(RF_WARPS * 32, 8) vis_refine_kernel(Params p, TrackStore ts, Frame f, int* nan_flag,
                                                                      int n_scenes) {
  __shared__ float s_bs[RF_WARPS][RF_CLAIM][RF_PITCH];
  __shared__ int s_cnt[2];
  for (int scene = blockIdx.y; scene < n_scenes; scene += gridDim.y) {
    if (f.vis_mode[scene] != 0) {   // survivor list overflowed: this scene is computed densely
      if (f.screen_cnt && blockIdx.x == 0 && threadIdx.x == 0) atomicAdd(f.screen_cnt + 2, 1);
      continue;
    }
    const SceneDesc sc = f.scenes[scene];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (f.screen_cnt) {
      if (threadIdx.x < 2) s_cnt[threadIdx.x] = 0;
      __syncthreads();
    }
    int n_ref = 0, n_cut = 0;   // survivors this lane refined, and how many of them the exact test cut
    const int n_pairs = min(f.vis_cnt[scene], sc.vis_lcap);
    const int nblk = p.d8 / 8;
    const int D = p.feature_dim;
    float (*bs)[RF_PITCH] = s_bs[w];
    float vmax = nanf("");
    // warps claim RF_CLAIM survivors at a time from the scene's counter: however many survive, the scene's warps finish together
    for (;;) {
      int i0 = 0;
      if (lane == 0) i0 = atomicAdd(f.refine_next + scene, RF_CLAIM);
      i0 = __shfl_sync(0xffffffffu, i0, 0);
      if (i0 >= n_pairs) break;
      const int npair = min(RF_CLAIM, n_pairs - i0);
      VisPair mine;
      mine.g = 0; mine.row = 0; mine.scene = 0; mine.outcol = 0;
      if (lane < npair) mine = f.vis_pairs[sc.vis_lbase + i0 + lane];
      float acc = 0.0f;
      for (int seg0 = 0; seg0 < nblk; seg0 += RF_SEG) {
        const int segn = min(RF_SEG, nblk - seg0);
        // A candidate's survivors sit next to each other in the list (the observations of its track are adjacent columns
        // of one screen tile; the dense path emits whole groups): its row is loaded once and reused while the candidate
        // stays the same -- a third of the L2 -> SM traffic of this kernel.
        int g_prev = -1;
        float av[RF_SEG / 32][8];
#pragma unroll 4
        for (int pp = 0; pp < npair; ++pp) {
          const int g = __shfl_sync(0xffffffffu, mine.g, pp);
          const int row = __shfl_sync(0xffffffffu, mine.row, pp);
          const float* b = ts.feat + (size_t)row * p.d8;
          if (g != g_prev) {   // warp-uniform
            const T* a = static_cast<const T*>(f.in_feat) + (size_t)g * D;
#pragma unroll
            for (int h = 0; h < RF_SEG / 32; ++h)
              if (h * 32 + lane < segn) refine_load_a<TAIL>(a, seg0 + h * 32 + lane, D, av[h]);
            g_prev = g;
          }
#pragma unroll
          for (int h = 0; h < RF_SEG / 32; ++h) {
            const int j = h * 32 + lane;
            if (j < segn) bs[pp][j] = refine_block_sum<COSINE>(av[h], b, seg0 + j);
          }
        }
        __syncwarp();
        if (lane < npair)
          for (int j = 0; j < segn; ++j) acc = acc + bs[lane][j];
        __syncwarp();
      }
      if (lane < npair) {
        float v = nanf("");
        if (COSINE) {
          const float d = acc / sqrtf(f.c_norm2[mine.g] * ts.fnorm2[mine.row]);
          if (d >= p.visual_threshold) v = 1.0f - d;       // is_ok + distance_to_weight
        } else {
          const float d = sqrtf(acc);
          if (d <= p.visual_threshold) v = d;
        }
        f.vis_val[sc.vis_lbase + i0 + lane] = v;
        n_ref += 1;
        n_cut += is_nan(v) ? 1 : 0;
        if (!is_nan(v) && !(v <= vmax)) vmax = v;   // best.rs "max_dist": maximum over the entries that exist
        if (nan_flag && is_nan(v)) nan_flag[scene] = 1;   // dense path: an entry the threshold cuts voids its precondition
      }
    }
    // one atomic per warp
    unsigned int u = 0u;
    if (!is_nan(vmax)) {
      u = __float_as_uint(vmax);
      u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) u = max(u, __shfl_xor_sync(0xffffffffu, u, o));
    if (lane == 0 && u != 0u) atomicMax(f.scene_max + scene, u);
    if (f.screen_cnt) {   // the screen's selectivity: one shared atomic per warp, one global atomic per CTA
      n_ref = __reduce_add_sync(0xffffffffu, n_ref);
      n_cut = __reduce_add_sync(0xffffffffu, n_cut);
      if (lane == 0 && n_ref) { atomicAdd(&s_cnt[0], n_ref); atomicAdd(&s_cnt[1], n_cut); }
      __syncthreads();
      if (threadIdx.x == 0 && s_cnt[0]) { atomicAdd(f.screen_cnt, s_cnt[0]); if (s_cnt[1]) atomicAdd(f.screen_cnt + 1, s_cnt[1]); }
      __syncthreads();   // thread 0 has read s_cnt before the next scene zeroes it
    }
  }
}

// dense view of the sparse scenes' visual entries (operators / debugging): None everywhere, then the refined survivors
__global__ void vis_fill_none_kernel(Params p, Frame f, int n_scenes) {
  for (int scene = blockIdx.y; scene < n_scenes; scene += gridDim.y) {
    if (f.scene_mode[scene] != 0) continue;
    const SceneDesc sc = f.scenes[scene];
    const long long cnt = (long long)sc.m * sc.n * p.max_obs;
    float* out = f.vis + sc.vis_off;
    const float qnan = nanf("");
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < cnt; i += (long long)gridDim.x * blockDim.x) out[i] = qnan;
  }
}
__global__ void vis_scatter_kernel(Params p, Frame f, int n_scenes) {
  for (int scene = blockIdx.y; scene < n_scenes; scene += gridDim.y) {
    if (f.scene_mode[scene] != 0) continue;
    const SceneDesc sc = f.scenes[scene];
    const int n_pairs = min(f.vis_cnt[scene], sc.vis_lcap);
    float* out = f.vis + sc.vis_off;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_pairs; i += gridDim.x * blockDim.x) {
      const VisPair vp = f.vis_pairs[sc.vis_lbase + i];
      out[(size_t)(vp.g - sc.det_base) * (sc.n * p.max_obs) + vp.outcol] = f.vis_val[sc.vis_lbase + i];
    }
  }
}
void launch_vis_densify(const Params& p, const Frame& f, int n_scenes, cudaStream_t st) {
  if (n_scenes == 0) return;
  dim3 grid(64, scene_grid(n_scenes));
  vis_fill_none_kernel<<<grid, 256, 0, st>>>(p, f, n_scenes);
  vis_scatter_kernel<<<grid, 256, 0, st>>>(p, f, n_scenes);
  note_launch(2);
}

// ------------------------------------------------------------------------------------------------ bf16 operand copies
__global__ void to_bf16_kernel(const float* src, int src_pitch, int d, int d8, long long rows, __nv_bfloat16* dst) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * d8) return;
  long long r = i / d8;
  int c = (int)(i - r * d8);
  float x = c < d ? src[r * src_pitch + c] : 0.0f;
  dst[i] = __float2bfloat16_rn(x);
}

void launch_to_bf16(const float* src, int src_pitch, int d, int d8, long long rows, void* dst, cudaStream_t st) {
  if (rows == 0) return;
  long long n = rows * d8;
  to_bf16_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(src, src_pitch, d, d8, rows, (__nv_bfloat16*)dst);
  note_launch();
}

// e4m3 operand copies: one warp per row (d8 <= 512)
__global__ void to_fp8_kernel(const float* src, int src_pitch, int d, int d8, long long rows, unsigned char* dst, float* scale) {
  const long long r = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (r >= rows) return;
  const float s = fp8_row_from(src + r * src_pitch, d, d8, dst + r * fp8_pitch(d8));
  if ((threadIdx.x & 31) == 0) scale[r] = s;
}

void launch_to_fp8(const float* src, int src_pitch, int d, int d8, long long rows, unsigned char* dst, float* scale,
                   cudaStream_t st) {
  if (rows == 0) return;
  to_fp8_kernel<<<(unsigned)((rows * 32 + 255) / 256), 256, 0, st>>>(src, src_pitch, d, d8, rows, dst, scale);
  note_launch();
}

// ------------------------------------------------------------------------------------------------ host launcher
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qr) == cudaSuccess && p) fn = (EncodeTiledFn)p;
  }
  return fn;
}

int make_map(CUtensorMap* m, const void* base, long long rows, int d8, int box_rows, bool fp8) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return -1;
  // a box row is one 128-byte swizzle row: 64 BF16 or 128 e4m3 features; past d8 the box is zero-filled
  cuuint64_t dims[2] = {(cuuint64_t)d8, (cuuint64_t)rows};
  cuuint64_t strides[1] = {fp8 ? (cuuint64_t)fp8_pitch(d8) : (cuuint64_t)d8 * 2};
  cuuint32_t box[2] = {(cuuint32_t)(fp8 ? 2 * TC_BK : TC_BK), (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(m, fp8 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, (void*)base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : -2;
}

// the frame's screen runs on the e4m3 copies
static bool screen_fp8(const Params& p, const TcArgs& tc) { return tc.fp8 && !tc.dense && p.d8 <= kFp8MaxD8; }

// per-frame metadata: one thread per physical feature row (scene, arena block b, physical slot p) and per candidate.
// A block without an owner (free list) is an invalid column; otherwise the row belongs to track n = blk_owner[b].
// fp8: the constants of the e4m3 screen -- colb scaled by the row's 2^k (NaN, which keeps every pair, for a row outside
// fp8_norm_ok), and the scale itself in colsb.
__global__ void vis_meta_kernel(Params p, TrackStore ts, Frame f, int n_scenes, int max_rows, VisColMeta* colmeta,
                                VisColGeo* colgeo, float* colb, float* colsb, unsigned int* colvalid, bool fp8) {
  for (int s = blockIdx.y; s < n_scenes; s += gridDim.y) {
    const SceneDesc sc = f.scenes[s];
    const int K = p.max_obs;
    const int prow = blockIdx.x * blockDim.x + threadIdx.x;
    const bool in = prow < sc.nb * K && prow < max_rows;
    VisColMeta cm;
    cm.colb = 0.0f; cm.colc = 0.0f; cm.outcol = -1; cm.row = -1;
    float csb = 1.0f;
    if (in) {
      const int b = prow / K, ph = prow - b * K;
      const size_t sbase = (size_t)sc.slot * ts.track_cap;
      const int n = ts.blk_owner ? ts.blk_owner[sbase + b] : b;
      const size_t ti = sbase + (n >= 0 ? n : 0);
      const size_t frow = (sbase + b) * K + ph;   // feature row of this column
      unsigned int tep = 0u;
      if (n >= 0) {
        const int on = ts.obs_n[ti];
        // logical <-> physical observation bookkeeping of this track
        int k_of = -1, live_mask = 0;
        for (int k = 0; k < K; ++k) {
          if (k < on && ts.obs_hasf[ti * K + k]) {
            int pp = ts.obs_phys[ti * K + k];
            live_mask |= 1 << pp;
            if (pp == ph) k_of = k;
          }
        }
        tep = ts.epoch[ti];
        if (k_of >= 0) {
          const unsigned int delta = sc.epoch > tep ? sc.epoch - tep : tep - sc.epoch;
          cm.outcol = n * K + k_of;
          const bool valid = (ts.feat_cnt[ti] >= p.min_track_length) && ((unsigned int)p.max_idle_epochs >= delta);
          const float nb = ts.fnorm2[frow];
          const float E = fp8 ? p.vis_rel_err8 : p.vis_rel_err;
          cm.colb = p.visual_kind == 1 ? sqrtf(nb) : 0.5f * nb * (1.0f - 1e-5f - E);
          if (fp8) {
            if (fp8_norm_ok(nb)) { csb = ts.fscale[frow]; cm.colb *= csb; }
            else cm.colb = nanf("");
          }
          cm.row = valid ? (int)frow : -1;
        } else {
          // dead physical slot -> owns the dead_rank-th logical column without a feature (written as None)
          int dead_rank = 0;
          for (int pp = 0; pp < ph; ++pp) dead_rank += ((live_mask >> pp) & 1) ? 0 : 1;
          int seen = 0;
          for (int k = 0; k < K; ++k) {
            bool lv = k < on && ts.obs_hasf[ti * K + k];
            if (!lv) { if (seen == dead_rank) { cm.outcol = n * K + k; break; } ++seen; }
          }
        }
      }
      colmeta[sc.col_off + prow] = cm;
      colb[sc.col_off + prow] = cm.colb;
      if (fp8 && p.visual_kind != 1) colsb[sc.col_off + prow] = csb;
      if (p.n_constraints > 0) {
        VisColGeo cg;
        cg.tx = 0.0f; cg.ty = 0.0f; cg.tr = 0.0f; cg.tep = tep;
        if (n >= 0) { const float* tb = ts.pred + ti * 6; cg.tx = tb[0]; cg.ty = tb[1]; cg.tr = ts.radius[ti]; }
        colgeo[sc.col_off + prow] = cg;
      }
    }
    // col_off is a multiple of 128, so the 32 columns of a warp are exactly one word of the validity mask
    const unsigned int vb = __ballot_sync(0xffffffffu, cm.row >= 0);
    if ((threadIdx.x & 31) == 0 && vb != 0) colvalid[(sc.col_off + prow) >> 5] = vb;
    else if ((threadIdx.x & 31) == 0 && in) colvalid[(sc.col_off + prow) >> 5] = 0u;
  }
}

// fp8: cosine rowk carries the row's 2^k, Euclidean rowi = 2^-k; NaN rowk (every pair kept) outside fp8_norm_ok
__global__ void vis_rowmeta_kernel(Params p, Frame f, VisRowMeta* rowmeta, bool fp8) {
  int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= f.total) return;
  g += f.det0;
  const float na = f.c_norm2[g];
  VisRowMeta rm;
  rm.ok = (f.c_flags[g] & 2) ? 1 : 0;
  rm.rowi = 1.0f;
  rm.pad = 0;
  const float thr = p.visual_threshold;
  const float E = fp8 ? p.vis_rel_err8 : p.vis_rel_err;
  if (p.visual_kind == 1) rm.rowk = (thr - 1e-5f - E) * sqrtf(na);
  else rm.rowk = 0.5f * (na * (1.0f - 1e-5f - E) - thr * thr * (1.0f + 1e-5f));
  if (fp8) {
    const float s = f.c_scale[g];
    if (!fp8_norm_ok(na)) rm.rowk = nanf("");
    else if (p.visual_kind == 1) rm.rowk *= s;
    else rm.rowi = 1.0f / s;
  }
  rowmeta[g] = rm;
}

// exact refinement of the scene pair lists (f.vis_pairs / vis_cnt / refine_next / vis_val; scenes with vis_mode != 0 skipped)
int launch_vis_refine(const Params& p, const TrackStore& ts, const Frame& f, int n_scenes, int* nan_flag, cudaStream_t st) {
  if (n_scenes == 0) return 0;
  dim3 grid(16, scene_grid(n_scenes));   // 64 warps x RF_CLAIM survivors per scene in flight; more survivors are claimed in further rounds
  // the vector path needs 16-byte aligned input rows (a caller-owned device pointer on the device-io path); rows of d8
  // elements are 16-byte multiples for every element type
  const bool tail = p.feature_dim != p.d8 || (reinterpret_cast<uintptr_t>(f.in_feat) & 15) != 0;
  feat_dispatch(f.feat_type, [&](auto t) {
    using T = decltype(t);
    if (p.visual_kind == 1) {
      if (tail) vis_refine_kernel<true, true, T><<<grid, RF_WARPS * 32, 0, st>>>(p, ts, f, nan_flag, n_scenes);
      else vis_refine_kernel<true, false, T><<<grid, RF_WARPS * 32, 0, st>>>(p, ts, f, nan_flag, n_scenes);
    } else {
      if (tail) vis_refine_kernel<false, true, T><<<grid, RF_WARPS * 32, 0, st>>>(p, ts, f, nan_flag, n_scenes);
      else vis_refine_kernel<false, false, T><<<grid, RF_WARPS * 32, 0, st>>>(p, ts, f, nan_flag, n_scenes);
    }
  });
  note_launch();
  return 0;
}

void launch_vis_colmeta(const Params& p, const TrackStore& ts, const Frame& f, int n_scenes, int max_n, const TcArgs& tc,
                        cudaStream_t st) {
  const int max_rows = tc.max_rows > 0 ? tc.max_rows : max_n * p.max_obs;
  if (tc.n_tiles == 0 || max_rows <= 0) return;
  dim3 grid((max_rows + 255) / 256, scene_grid(n_scenes));
  vis_meta_kernel<<<grid, 256, 0, st>>>(p, ts, f, n_scenes, max_rows, tc.colmeta, tc.colgeo, tc.colb, tc.colsb, tc.colvalid,
                                        screen_fp8(p, tc));
  note_launch();
}

int vis_screen_ucols(int d8, int num_sms, int n_scenes, const int* m, const int* nb, int K) {
  if (d8 > kScreenStationaryMaxD8) return TC_BN;
  long long pairs = 0, pair_tiles = 0;
  int max_ct = 1;
  for (int s = 0; s < n_scenes; ++s) {
    const int ct = (nb[s] * K + SA_BN - 1) / SA_BN, rp = (m[s] + 2 * TC_BM - 1) / (2 * TC_BM);
    pairs += rp;
    pair_tiles += (long long)rp * ct;
    max_ct = std::max(max_ct, ct);
  }
  // whole scenes when the candidate-tile pairs alone give every cluster two units; else split the columns until they do,
  // but not below two column tiles, one for each consumer warpgroup
  const long long units = 2ll * std::max(1, num_sms / 2);
  if (pairs >= units) return max_ct * SA_BN;
  const long long per = (pair_tiles + units - 1) / units;
  return (int)std::max<long long>(2, std::min<long long>(per, max_ct)) * SA_BN;
}

int launch_vis_cost_tc(const Params& p, const TrackStore& ts, const Frame& f, int n_scenes, int max_n, const TcArgs& tc,
                       int phase, cudaStream_t st) {
  if (tc.n_tiles == 0) return 0;
  if (phase == 1) {
    // dense path: an exact value the threshold cuts (a NaN or infinite distance) voids the scene's dense result too
    int rc = launch_vis_refine(p, ts, f, n_scenes, tc.dense ? tc.dense_bad : nullptr, st);
    if (tc.ev_refine1) cudaEventRecord(tc.ev_refine1, st);
    return rc;
  }
  // d8 <= 512: the A-stationary kernel over work units of tc.cstep columns; wider features do not fit A in shared
  // memory, they take the streaming kernel over 256-column tiles
  const bool stationary = p.d8 <= kScreenStationaryMaxD8;
  // e4m3 operands (TcArgs::fp8): the A-stationary kernel only; a missing copy is an error, not a quiet BF16 run
  const bool fp8 = screen_fp8(p, tc);
  if (fp8 && (!f.c_fp8 || !f.c_scale || !ts.feat_fp8 || !ts.fscale || (p.visual_kind != 1 && !tc.colsb))) return -3;
  CUtensorMap mA, mB;
  if (make_map(&mA, fp8 ? (const void*)f.c_fp8 : f.c_bf16, tc.a_rows, p.d8, TC_BM, fp8) ||
      make_map(&mB, fp8 ? (const void*)ts.feat_fp8 : ts.feat_bf16, tc.b_rows, p.d8, stationary ? SA_BN / 2 : TC_BN / 2, fp8))
    return -1;
  const size_t smem = (stationary ? sizeof(SaSmem) : sizeof(TcSmem)) + 1024;
  const bool cosine = p.visual_kind == 1;
  cudaError_t e = cudaSuccess;
  const void* fn;
  if (!stationary) fn = cosine ? (const void*)vis_screen_kernel<true> : (const void*)vis_screen_kernel<false>;
  else if (fp8) fn = cosine ? (const void*)vis_screen_sa_kernel<true, true> : (const void*)vis_screen_sa_kernel<false, true>;
  else fn = cosine ? (const void*)vis_screen_sa_kernel<true, false> : (const void*)vis_screen_sa_kernel<false, false>;
  e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return (int)e;
  if (!tc.colmeta_done) launch_vis_colmeta(p, ts, f, n_scenes, max_n, tc, st);
  vis_rowmeta_kernel<<<(f.total + 255) / 256, 256, 0, st>>>(p, f, tc.rowmeta, fp8);
  note_launch();
  if (tc.ev_screen0) cudaEventRecord(tc.ev_screen0, st);
  {
    const int ncta = 2 * std::min(tc.n_tiles, tc.num_sms / 2);
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(ncta);
    cfg.blockDim = dim3(TC_THREADS);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 2; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    const TcTile* d_tiles = tc.d_tiles;
    int n_tiles = tc.n_tiles;
    const int* d_n_tiles = tc.d_n_tiles;
    const VisColMeta* cmeta = tc.colmeta;
    const VisColGeo* cgeo = tc.colgeo;
    const VisRowMeta* rmeta = tc.rowmeta;
    const float* cb = tc.colb;
    const float* csb = tc.colsb;
    const unsigned int* cv = tc.colvalid;
    int ucols = tc.cstep;
    void* args[] = {(void*)&mA, (void*)&mB, (void*)&p, (void*)&ts, (void*)&f, (void*)&d_tiles, (void*)&n_tiles,
                    (void*)&d_n_tiles, (void*)&cmeta, (void*)&cgeo, (void*)&rmeta, (void*)&cb, (void*)&cv};
    void* args_sa[] = {(void*)&mA, (void*)&mB, (void*)&p, (void*)&ts, (void*)&f, (void*)&d_tiles, (void*)&n_tiles,
                       (void*)&d_n_tiles, (void*)&ucols, (void*)&cmeta, (void*)&cgeo, (void*)&rmeta, (void*)&cb, (void*)&csb,
                       (void*)&cv};
    e = cudaLaunchKernelExC(&cfg, fn, stationary ? args_sa : args);
    if (e != cudaSuccess) return (int)e;
    note_launch();
  }
  if (tc.ev_screen1) cudaEventRecord(tc.ev_screen1, st);
  return 0;
}

}  // namespace sb
