// kernels_feat_dense.cu -- visual (ReID feature) cost for thresholds that cut nothing: the dense tensor-core path.
//
// The reference's default visual metric is Euclidean(f32::MAX) (src/trackers/visual_sort/metric/builder.rs:26-42) and its
// published VisualSORT bench uses Euclidean(10.0) on unit vectors (benches/simple_visual_sort_tracker.rs:111): every
// (candidate, track observation) distance is an entry of the metric.  The screen + refine path of kernels_feat_tc.cu lives on
// sparsity and has none to exploit here.  What the voting stage needs from the dense matrix is much less than the matrix:
// BestFitVoting (src/track/voting/best.rs:52-128, consumed by VisualVoting, src/trackers/visual_sort/voting.rs:45-100) gives
// every (candidate q, track t) group the weight W(q,t) = sum_k (max_dist - d(q,t,k)), a candidate's decision is its row
// maximum and it wins that track iff it is also the column maximum (kernels_assign.cu).  So:
//
//   1. vis_wsum_kernel  : C~ = A B^T on the tensor cores (wgmma BF16, the same TMA / mbarrier pipeline as the screen).  The
//                         epilogue turns every accumulator into an approximate distance d~ with a rigorous error bound
//                         (BF16 operand rounding, screen_rel_err), sums the observations of a track -- the column tiles are
//                         cut at track boundaries -- and stores {S~(q,t), bound} once per (candidate, track): 8 B per
//                         3 * 512 MACs.  Elements that can be the scene's maximal distance (needed exactly: it is best.rs's
//                         max_dist) are appended to a short list, found with a lower bound sampled beforehand.
//   2. refine (max)     : the exact f32 distances of those few elements, reference summation order -> exact max_dist.
//   3. vis_dense_select : weight intervals [W_lo, W_hi] from S~, the bound and max_dist; every group whose interval reaches
//                         its row's or its column's best lower bound can be a BestFit maximum and is emitted -- all its
//                         observations -- to the scene's pair list.  Everything else provably cannot win anything.
//   4. refine + voting  : unchanged (kernels_feat_tc.cu, kernels_assign.cu): exact f32 values in the reference's summation
//                         order, exact f64 weights, the oracle's tie order.  The tensor cores only decide which groups are
//                         worth computing exactly, so assignments stay bit-identical to the CPU reference.
//
// Preconditions checked on the device per scene (else dense_bad -> the exact SIMT kernels take the scene): the exact max_dist
// passes the threshold (then every entry does), every feature norm is in the range of dense_norm_ok, the lists did not
// overflow.
// The final refinement also sends a scene to the exact kernels when one of its exact values is cut by the threshold.
// Spatio-temporal constraints switch the path off on the host (they make the matrix sparse in a way only the per-pair gate
// knows).
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>

#include "sb_engine.cuh"
#include "sb_tc.cuh"

namespace sb {

// error of x~ = |a|^2 + |b|^2 - 2 dot~ against the reference's f32 squared distance, relative to (|a|^2 + |b|^2):
// 2 E |a||b| <= E (|a|^2 + |b|^2) for the BF16 dot product (E = p.vis_rel_err, screen_rel_err), plus 2e-4 for the f32
// roundings of the norms, of x~ itself and of the reference's own 512-term summation.  Cosine: |cos~ - cos| <= E + 2e-4
// absolute.
__device__ __forceinline__ float dense_err(const Params& p) { return p.vis_rel_err + 2e-4f; }

// The bounds above hold for finite operands whose squared norms stay below FLT_MAX / 4 (then neither |a|^2 + |b|^2 nor
// 2 dot~ overflows) and, under cosine, are not zero.  A scene with any other feature (a NaN or infinite component, a zero
// vector under cosine, an overflowing norm) goes to the exact kernels: its approximate distances bound nothing, and a
// NaN among them would poison the order-preserving row and column maxima of the selection.
__device__ __forceinline__ bool dense_norm_ok(const Params& p, float n2) {
  return n2 <= 0.25f * 3.402823466e38f && (p.visual_kind != 1 || n2 > 0.0f);
}

constexpr int DS_STAGES = 4;
constexpr int DS_STAGE_BYTES = TC_A_BYTES + TC_B_BYTES;   // A tile (128 x 64 bf16) + B tile (256 x 64 bf16, half from each CTA)
constexpr int DS_CH = 16;                                 // accumulator columns per epilogue chunk
constexpr int DS_PITCH = DS_CH + 1;                       // +1: the row owners read column cc of 32 rows from 32 banks

struct DsHdr {
  int scene, m0, m, det_base;
  int rowB;          // feature row of the tile's column 0
  int vis_lbase, vis_lcap, mpad;
  long long ws_base; // ws element of (first block of the tile, candidate 0)
  float l0, scmax;
  int blk0;          // global index (frame-wide) of the tile's first block
  int nblk;          // blocks of the scene inside this tile (the last tile of a scene is partial)
};
struct DsSmem {
  unsigned char stage[DS_STAGES][DS_STAGE_BYTES];   // 1024-byte aligned operand stages first
  float colc[4][TC_BN];
  float cmax[4][TC_BN];
  float ktf[4][TC_BN];   // valid observations of the column's block when the block can vote (>= min_votes), else 0
  VisRowMeta rowm[4][TC_BM];
  unsigned int vmask[4][TC_BN / 32];
  unsigned int bmask[4][TC_BN / 32];
  float dist[2][TC_WG_ROWS][DS_PITCH];   // per consumer warpgroup: one chunk of approximate distances, row-major
  DsHdr hdr[4];
  unsigned long long full_bar[DS_STAGES];
  unsigned long long empty_bar[DS_STAGES];
  unsigned long long meta_full[4];
  unsigned long long meta_empty[4];
};
static_assert(sizeof(DsSmem) + 1024 <= 227 * 1024, "weight-sum kernel exceeds the shared memory of an SM");

constexpr int kDenseKClasses = 5;   // observation counts the fused row bounds distinguish (templated kernels: K <= 5)
constexpr float kHalfRel = 4.9e-4f; // 2^-11 (+): relative rounding error of a sum stored as fp16

__device__ __forceinline__ unsigned int enc_ord(float v) {   // order-preserving f32 -> u32 (0 is below every value)
  const unsigned int u = __float_as_uint(v);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float dec_ord(unsigned int u) {
  return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

struct DenseDev {   // device pointers of the path (TcArgs subset, passed by value)
  __half2* ws;           // {sum of the block's distances (rn), per-observation error bound (ru)} per (block, candidate)
  unsigned int* rowb;    // [total][kDenseKClasses] best lower bound of -(S + k del) per candidate and observation count
  unsigned int* colb;    // [blocks of the frame] the same per block (column of the weight matrix)
  const float* slab_ktf;
  const float* slab_colc; const float* slab_cmax;
  const unsigned int* slab_vmask; const unsigned int* slab_bmask;
  const float* scene_l0; const float* scene_cmax;
  VisPair* maxc; int* maxc_cnt;
  const VisRowMeta* rowmeta;
};

// ------------------------------------------------------------------------------------------------ weight-sum kernel
// Clusters of two CTAs: each CTA takes 128 candidate rows of the cluster's 256 and loads half of the shared B tile,
// multicast into both CTAs' shared memory.  Two consumer warpgroups per CTA, 64 rows x 256 columns of accumulators each.
// approximate MUFU operations (2 ulp), one instruction each: only upper bounds and the approximate distances use them
__device__ __forceinline__ float rsqrt_approx(float x) { float r; asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
__device__ __forceinline__ float rcp_approx(float x) { float r; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }

// Rare path of the weight-sum epilogue (about one element in a thousand): the element may be the scene's maximal distance.
__device__ __noinline__ void dense_append_candidate(VisPair* maxc, int* maxc_cnt, int scene, int lbase, int lcap, int g, int row) {
  const int slot = atomicAdd(&maxc_cnt[scene], 1);
  if (slot < lcap) {
    VisPair vp;
    vp.g = g; vp.row = row; vp.scene = scene; vp.outcol = -1;
    maxc[lbase + slot] = vp;
  }
}

// KT > 0: the number of observations per track is a compile-time constant, so the positions where a block of the
// accumulator ends (every KT-th column: tiles start at block boundaries) are too and the epilogue is straight-line code.
// KT == 0: any K, block ends come from the bmask slab (uniform branches).
template <bool COSINE, int KT>
__global__ void __launch_bounds__(TC_THREADS, 1)
vis_wsum_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB, Params p, TrackStore ts,
                Frame f, const TcTile* tiles, const int* n_tiles_dev, DenseDev dd) {
  extern __shared__ unsigned char smem_raw_[];
  DsSmem& S = *reinterpret_cast<DsSmem*>(smem_raw_ + ((1024u - (smem_u32(smem_raw_) & 1023u)) & 1023u));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int K = p.max_obs;
  const int KB = (p.d8 + TC_BK - 1) / TC_BK;
  const int n_tiles = *n_tiles_dev;
  const uint32_t crank = cluster_rank();
  const int cta_first = (int)(blockIdx.x >> 1);
  const int cta_step = (int)(gridDim.x >> 1);
  unsigned char* const stage_base = &S.stage[0][0];
  if (threadIdx.x == 0) {
    for (int s = 0; s < DS_STAGES; ++s) { mbar_init(&S.full_bar[s], 1); mbar_init(&S.empty_bar[s], 4); }
    for (int b = 0; b < 4; ++b) { mbar_init(&S.meta_full[b], 1); mbar_init(&S.meta_empty[b], 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  cluster_sync_all();

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
      for (int t = cta_first; t < n_tiles; t += cta_step, ++it) {
        const TcTile tl = tiles[t];
        const SceneDesc sc = f.scenes[tl.scene];
        const int m0 = tl.m0 + (int)crank * TC_BM;
        const int rowA = sc.det_base + m0;
        const int rowB = sc.slot * ts.track_cap * K + tl.c0;
        {
          const int g = it & 3;
          mbar_wait(&S.meta_empty[g], ((it >> 2) & 1) ^ 1);
          DsHdr h;
          h.scene = tl.scene; h.m0 = m0; h.m = sc.m; h.det_base = sc.det_base; h.rowB = rowB;
          h.vis_lbase = sc.vis_lbase; h.vis_lcap = sc.vis_lcap;
          h.mpad = (sc.m + 127) / 128 * 128;
          h.ws_base = sc.ws_off + (long long)(tl.c0 / K) * h.mpad;
          h.l0 = dd.scene_l0[tl.scene]; h.scmax = dd.scene_cmax[tl.scene];
          h.blk0 = sc.blk_off + tl.c0 / K;
          h.nblk = min(TC_BN / K, sc.nb - tl.c0 / K);
          S.hdr[g] = h;
          const size_t slab = (size_t)sc.slab_off + tl.pad;
          mbar_expect_tx(&S.meta_full[g], (uint32_t)(4 * TC_BN * 3 + sizeof(VisRowMeta) * TC_BM + (TC_BN / 8) * 2));
          bulk_load(S.ktf[g], dd.slab_ktf + slab * TC_BN, 4 * TC_BN, &S.meta_full[g]);
          bulk_load(S.colc[g], dd.slab_colc + slab * TC_BN, 4 * TC_BN, &S.meta_full[g]);
          bulk_load(S.cmax[g], dd.slab_cmax + slab * TC_BN, 4 * TC_BN, &S.meta_full[g]);
          bulk_load(S.rowm[g], dd.rowmeta + rowA, (uint32_t)(sizeof(VisRowMeta) * TC_BM), &S.meta_full[g]);
          bulk_load(S.vmask[g], dd.slab_vmask + slab * (TC_BN / 32), TC_BN / 8, &S.meta_full[g]);
          bulk_load(S.bmask[g], dd.slab_bmask + slab * (TC_BN / 32), TC_BN / 8, &S.meta_full[g]);
        }
        for (int kb = 0; kb < KB; ++kb) {
          mbar_wait(&S.empty_bar[stage], phase ^ 1);   // both CTAs have released the stage
          unsigned char* base = stage_base + stage * DS_STAGE_BYTES;
          mbar_expect_tx(&S.full_bar[stage], DS_STAGE_BYTES);
          tma_load_2d(base, &mapA, kb * TC_BK, rowA, &S.full_bar[stage]);
          tma_load_2d_mc(base + TC_A_BYTES + crank * (TC_B_BYTES / 2), &mapB, kb * TC_BK, rowB + (int)crank * (TC_BN / 2),
                         &S.full_bar[stage], (uint16_t)0x3);
          if (++stage == DS_STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ===================================================================== consumer warpgroups 1 and 2
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    // Per 16-column chunk: every thread turns its accumulators (wgmma layout: register i is row er[(i >> 1) & 1], column
    // 8 * (i >> 2) + 2 * (lane & 3) + (i & 1)) into approximate distances in place and parks them in S.dist; then the
    // warpgroup's first two warps, one thread per row, add them up block by block in column order.
    const int wg = (warp >> 2) - 1;
    const int wtid = threadIdx.x & 127;
    const bool owner = wtid < TC_WG_ROWS;   // warp-uniform
    const int er[2] = {(warp & 3) * 16 + (lane >> 2), (warp & 3) * 16 + (lane >> 2) + 8};   // rows inside the warpgroup
    const int q2 = 2 * (lane & 3);
    const float finf = __int_as_float(0x7f800000);
    float (*dist)[DS_PITCH] = S.dist[wg];
    int stage = 0;
    uint32_t phase = 0;
    int it = 0;
    for (int t = cta_first; t < n_tiles; t += cta_step, ++it) {
      float acc[128];
      tc_consume_tile<2, DS_STAGES, DS_STAGE_BYTES>(acc, stage_base, S.full_bar, S.empty_bar, KB, wg, stage, phase);
      const int ms = it & 3;
      mbar_wait(&S.meta_full[ms], (it >> 2) & 1);
      const DsHdr h = S.hdr[ms];
      const float* gcolc = S.colc[ms];
      const float* gcmax = S.cmax[ms];
      const float* gktf = S.ktf[ms];
      // element view: the two rows of this thread's accumulators
      float erowc[2], eTd[2];
      int eg[2];
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        const int r = wg * TC_WG_ROWS + er[hr];
        const VisRowMeta rm = S.rowm[ms][r];
        const int m = h.m0 + r;
        erowc[hr] = rm.rowk;   // |a|^2 (euclidean) or 1 / |a| (cosine)
        eg[hr] = h.det_base + m;
        // an element can be the scene's maximal distance only above the sampled lower bound minus the error bound
        float T = COSINE ? h.l0 - dense_err(p) : h.l0 - dense_err(p) * (erowc[hr] + h.scmax);
        if (!(m < h.m && rm.ok)) T = finf;
        eTd[hr] = COSINE ? T : (T > 0.0f ? T * rsqrt_approx(T) * (1.0f - 1e-6f) : -1.0f);   // sqrt(T), a hair low
      }
      // row view (owners): the row this thread sums
      const int rrow = wg * TC_WG_ROWS + (wtid & (TC_WG_ROWS - 1));
      const VisRowMeta rm = S.rowm[ms][rrow];
      const int m = h.m0 + rrow;
      const bool row_ok = m < h.m && rm.ok;
      const int g = h.det_base + m;
      const float rowc = rm.rowk;
      __half2* wsp = dd.ws + h.ws_base + m;
      float s_acc = 0.0f, dmin = finf;
      // fused "pass A" of the selection (templated kernels): best lower bound of the maxd-independent part of the weight,
      // -(S + k del), per observation count for this row, per block over the rows (warp maximum + one atomic)
      constexpr bool FUSED = KT > 0;
      float lrow[kDenseKClasses];
#pragma unroll
      for (int kc = 0; kc < kDenseKClasses; ++kc) lrow[kc] = -finf;
      int bidx = h.blk0;
      // one flush per block: {sum of the block's distances, per-observation error bound}
      auto flush = [&](int col) {
        const float cmx = gcmax[col];
        float del;
        if (COSINE) del = dense_err(p);
        else {
          const float rc = rowc + cmx;
          const float e = dense_err(p) * rc;
          // |d - d~| <= |d^2 - d~^2| / (d + d~) <= e / d~ always, <= 0.536 e / d~ once d~^2 >= 4 e (then d >= 0.866 d~),
          // and <= sqrt(e) always.  Approximate reciprocal / rsqrt (2 ulp) under a 1.0001 safety factor; 1e-6 (rc + 1) >=
          // 1e-6 sqrt(rc) covers the rsqrt approximation of d~ itself.
          const float dm = dmin * (1.0f - 1e-6f);
          const float q = e * rcp_approx(dm);
          del = fminf(dm * dm >= 4.0f * e ? 0.536f * q : q, e * rsqrt_approx(e));
          del = __fmaf_rn(del, 1.0001f, 1e-6f * (rc + 1.0f));
        }
        if (row_ok) *wsp = __halves2half2(__float2half_rn(s_acc), __float2half_ru(del));
        wsp += h.mpad;
        if (FUSED) {
          const float kf = gktf[col];   // block-uniform; 0: the block takes no part in the voting
          float base = -finf;
          if (row_ok && kf > 0.0f) base = -(s_acc * (1.0f + 2e-6f) + kf * del);
#pragma unroll
          for (int kc = 0; kc < (KT > 0 ? KT : 1); ++kc) lrow[kc] = fmaxf(lrow[kc], kf == (float)(kc + 1) ? base : -finf);
          const unsigned int u = __reduce_max_sync(0xffffffffu, enc_ord(base));
          if (lane == 0 && kf > 0.0f && u > 0x007fffffu) atomicMax(&dd.colb[bidx], u);   // 0x007fffff == enc(-inf)
        }
        ++bidx;
        s_acc = 0.0f; dmin = finf;
      };
      // distances of one chunk in place (accumulator groups j = 2 ch, 2 ch + 1); an element that can be the scene's maximal
      // distance (approximate distance above the bound Td, valid column) is appended to the candidate list on the spot;
      // then the chunk goes to S.dist
      auto distances = [&](int ch, unsigned int vm) {
#pragma unroll
        for (int jj = 0; jj < 2; ++jj) {
          const int j = 2 * ch + jj;
          const int cc = 8 * jj + q2;   // column inside the chunk
          const float2 c2 = *reinterpret_cast<const float2*>(gcolc + 8 * j + q2);
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int hr = e >> 1, cl = e & 1;
            const float a = acc[4 * j + e];
            const float cv = cl ? c2.y : c2.x;
            float dval;
            if (COSINE) dval = __fsub_rn(1.0f, __fmul_rn(__fmul_rn(a, erowc[hr]), cv));
            else {
              float x = __fmaf_rn(-2.0f, a, __fadd_rn(erowc[hr], cv));
              x = fmaxf(x, 1e-30f);
              dval = __fmul_rn(x, rsqrt_approx(x));
            }
            // about one element in a thousand
            if (dval >= eTd[hr] && ((vm >> (cc + cl)) & 1u))
              dense_append_candidate(dd.maxc, dd.maxc_cnt, h.scene, h.vis_lbase, h.vis_lcap, eg[hr], h.rowB + 8 * j + q2 + cl);
            dist[er[hr]][cc + cl] = dval;
          }
        }
      };
      if (KT > 0) {
        constexpr int KC = KT > 0 ? KT : 1;
        constexpr int CSTEP = (TC_BN / KC) * KC;   // columns of the tile that belong to whole blocks
#pragma unroll
        for (int ch = 0; ch < TC_BN / DS_CH; ++ch) {
          const unsigned int vm = (S.vmask[ms][ch >> 1] >> ((ch & 1) * DS_CH)) & 0xffffu;
          distances(ch, vm);
          wg_bar(1 + wg);
          if (owner) {
#pragma unroll
            for (int cc = 0; cc < DS_CH; ++cc) {
              const int col = ch * DS_CH + cc;
              if (col < CSTEP) {   // compile time
                const bool valid = (vm >> cc) & 1u;
                const float dval = dist[wtid][cc];
                s_acc = __fadd_rn(s_acc, valid ? dval : 0.0f);
                dmin = fminf(dmin, valid ? dval : finf);
                // compile-time position: last physical slot of a block (the per-scene arrays are padded to whole tiles, so a
                // block position past the scene's arena is stored too: kt = 0 there, nobody reads it)
                if (col % KC == KC - 1) flush(col);
              }
            }
          }
          wg_bar(1 + wg);   // S.dist may be overwritten
        }
      } else {
#pragma unroll
        for (int ch = 0; ch < TC_BN / DS_CH; ++ch) {   // unrolled: the accumulators are indexed at compile time
          const unsigned int vm = (S.vmask[ms][ch >> 1] >> ((ch & 1) * DS_CH)) & 0xffffu;
          const unsigned int bm = (S.bmask[ms][ch >> 1] >> ((ch & 1) * DS_CH)) & 0xffffu;
          if ((vm | bm) == 0u) continue;   // uniform over the warpgroup, like every test on vm / bm below: column properties
          distances(ch, vm);
          wg_bar(1 + wg);
          if (owner) {
#pragma unroll
            for (int cc = 0; cc < DS_CH; ++cc) {
              const bool valid = (vm >> cc) & 1u;
              const float dval = dist[wtid][cc];
              s_acc = __fadd_rn(s_acc, valid ? dval : 0.0f);
              dmin = fminf(dmin, valid ? dval : finf);
              if (bm & (1u << cc)) flush(ch * DS_CH + cc);
            }
          }
          wg_bar(1 + wg);
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&S.meta_empty[ms]);
      if (FUSED && owner && row_ok) {
#pragma unroll
        for (int kc = 0; kc < (KT > 0 ? KT : 1); ++kc)
          if (lrow[kc] > -finf) atomicMax(&dd.rowb[(size_t)g * kDenseKClasses + kc], enc_ord(lrow[kc]));
      }
    }
  }
  __syncthreads();
  cluster_sync_all();   // no CTA leaves while its peer may still multicast into / arrive on its smem
}

// ------------------------------------------------------------------------------------------------ per-frame metadata
// One thread per arena block (scene, b): the block's K physical feature rows -> rowinfo (logical column, feature row or -1),
// the tile-major slabs the weight-sum kernel bulk-copies (column constant, block maximum, validity / block-end masks) and
// the block record of the selection kernel (owner, valid observations).  Same validity rule as vis_meta_kernel.
__global__ void vis_dense_meta_kernel(Params p, TrackStore ts, Frame f, int max_blocks, int cstep, DenseTrackMeta* tmeta,
                                      int2* rowinfo, float* slab_colc, float* slab_cmax, float* slab_ktf,
                                      unsigned int* slab_vmask, unsigned int* slab_bmask, float* scene_cmax,
                                      int* dense_bad) {
  const int s = blockIdx.y;
  const SceneDesc sc = f.scenes[s];
  const int K = p.max_obs;
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  float cmax = 0.0f;
  if (b < sc.nb && b < max_blocks) {
    const size_t sbase = (size_t)sc.slot * ts.track_cap;
    const int n = ts.blk_owner ? ts.blk_owner[sbase + b] : b;
    DenseTrackMeta tm;
    tm.n = n; tm.kt = 0; tm.cmax = 0.0f; tm.pad = 0;
    int outcol[kMaxObs], frow_of[kMaxObs];
    float colc[kMaxObs];
    for (int ph = 0; ph < K; ++ph) { outcol[ph] = -1; frow_of[ph] = -1; colc[ph] = 0.0f; }
    if (n >= 0) {
      const size_t ti = sbase + n;
      const int on = ts.obs_n[ti];
      const unsigned int tep = ts.epoch[ti];
      const unsigned int delta = sc.epoch > tep ? sc.epoch - tep : tep - sc.epoch;
      const bool valid = (ts.feat_cnt[ti] >= p.min_track_length) && ((unsigned int)p.max_idle_epochs >= delta);
      for (int k = 0; k < K; ++k) {
        if (k < on && ts.obs_hasf[ti * K + k]) {
          const int ph = ts.obs_phys[ti * K + k];
          const size_t frow = (sbase + b) * K + ph;
          outcol[ph] = n * K + k;
          if (valid) {
            frow_of[ph] = (int)frow;
            const float nb2 = ts.fnorm2[frow];
            if (!dense_norm_ok(p, nb2)) dense_bad[s] = 1;
            colc[ph] = p.visual_kind == 1 ? rsqrtf(nb2) : nb2;
            cmax = fmaxf(cmax, nb2);
            tm.kt += 1;
          }
        }
      }
      tm.cmax = cmax;
    }
    tmeta[sc.blk_off + b] = tm;
    const int need_votes = p.min_votes > 1 ? p.min_votes : 1;
    const float ktf = (tm.n >= 0 && tm.kt >= need_votes) ? (float)tm.kt : 0.0f;
    for (int ph = 0; ph < K; ++ph) {
      const int prow = b * K + ph;
      rowinfo[(size_t)sc.blk_off * K + prow] = make_int2(outcol[ph], frow_of[ph]);
      const int j = prow / cstep, cc = prow - j * cstep;
      const size_t slab = (size_t)sc.slab_off + j;
      slab_colc[slab * TC_BN + cc] = colc[ph];
      slab_cmax[slab * TC_BN + cc] = cmax;
      slab_ktf[slab * TC_BN + cc] = ktf;
      if (frow_of[ph] >= 0) atomicOr(&slab_vmask[slab * (TC_BN / 32) + (cc >> 5)], 1u << (cc & 31));
      if (ph == K - 1) atomicOr(&slab_bmask[slab * (TC_BN / 32) + (cc >> 5)], 1u << (cc & 31));
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) cmax = fmaxf(cmax, __shfl_xor_sync(0xffffffffu, cmax, o));
  if ((threadIdx.x & 31) == 0 && cmax > 0.0f) atomicMax(reinterpret_cast<int*>(scene_cmax) + s, __float_as_int(cmax));
}

// K > kMaxObs: one warp per arena block, lane k reading logical observation k and lane ph writing physical row ph, the
// two joined through the warp's shared-memory row (rowinfo and colc of every physical slot).  Same records as above.
constexpr int DMW_WARPS = 4;
__global__ void __launch_bounds__(DMW_WARPS * 32)
vis_dense_meta_wide_kernel(Params p, TrackStore ts, Frame f, int max_blocks, int cstep, DenseTrackMeta* tmeta, int2* rowinfo,
                           float* slab_colc, float* slab_cmax, float* slab_ktf, unsigned int* slab_vmask,
                           unsigned int* slab_bmask, float* scene_cmax, int* dense_bad) {
  __shared__ int2 s_ri[DMW_WARPS][32];
  __shared__ float s_colc[DMW_WARPS][32];
  const int s = blockIdx.y;
  const SceneDesc sc = f.scenes[s];
  const int K = p.max_obs;
  const int wi = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.x * DMW_WARPS + wi;
  if (!(b < sc.nb && b < max_blocks)) return;   // warp-uniform
  const unsigned int all = 0xffffffffu;
  const size_t sbase = (size_t)sc.slot * ts.track_cap;
  const int n = ts.blk_owner ? ts.blk_owner[sbase + b] : b;
  s_ri[wi][lane] = make_int2(-1, -1);
  s_colc[wi][lane] = 0.0f;
  __syncwarp();
  bool use = false;   // lane's logical observation holds a feature of a valid track
  float nb2 = 0.0f;
  if (n >= 0) {
    const size_t ti = sbase + n;
    const int on = ts.obs_n[ti];
    const unsigned int tep = ts.epoch[ti];
    const unsigned int delta = sc.epoch > tep ? sc.epoch - tep : tep - sc.epoch;
    const bool valid = (ts.feat_cnt[ti] >= p.min_track_length) && ((unsigned int)p.max_idle_epochs >= delta);
    const int k = lane;
    if (k < K && k < on && ts.obs_hasf[ti * K + k]) {
      const int ph = ts.obs_phys[ti * K + k];
      const size_t frow = (sbase + b) * K + ph;
      int fr = -1;
      if (valid) {
        fr = (int)frow;
        nb2 = ts.fnorm2[frow];
        if (!dense_norm_ok(p, nb2)) dense_bad[s] = 1;
        s_colc[wi][ph] = p.visual_kind == 1 ? rsqrtf(nb2) : nb2;
        use = true;
      }
      s_ri[wi][ph] = make_int2(n * K + k, fr);
    }
  }
  float cmax = use ? nb2 : 0.0f;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) cmax = fmaxf(cmax, __shfl_xor_sync(all, cmax, o));
  const int kt = __popc(__ballot_sync(all, use));
  __syncwarp();
  if (lane == 0) {
    DenseTrackMeta tm;
    tm.n = n; tm.kt = n >= 0 ? kt : 0; tm.cmax = n >= 0 ? cmax : 0.0f; tm.pad = 0;
    tmeta[sc.blk_off + b] = tm;
    if (cmax > 0.0f) atomicMax(reinterpret_cast<int*>(scene_cmax) + s, __float_as_int(cmax));
  }
  const int need_votes = p.min_votes > 1 ? p.min_votes : 1;
  const float ktf = (n >= 0 && kt >= need_votes) ? (float)kt : 0.0f;
  const int ph = lane;
  if (ph < K) {
    const int2 ri = s_ri[wi][ph];
    const int prow = b * K + ph;
    rowinfo[(size_t)sc.blk_off * K + prow] = ri;
    const int j = prow / cstep, cc = prow - j * cstep;
    const size_t slab = (size_t)sc.slab_off + j;
    slab_colc[slab * TC_BN + cc] = s_colc[wi][ph];
    slab_cmax[slab * TC_BN + cc] = cmax;
    slab_ktf[slab * TC_BN + cc] = ktf;
    if (ri.y >= 0) atomicOr(&slab_vmask[slab * (TC_BN / 32) + (cc >> 5)], 1u << (cc & 31));
    if (ph == K - 1) atomicOr(&slab_bmask[slab * (TC_BN / 32) + (cc >> 5)], 1u << (cc & 31));
  }
}

__global__ void vis_dense_rowmeta_kernel(Params p, Frame f, VisRowMeta* rowmeta) {
  int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= f.total) return;
  g += f.det0;
  const float na = f.c_norm2[g];
  VisRowMeta rm;
  rm.ok = (f.c_flags[g] & 2) ? 1 : 0;
  rm.rowk = p.visual_kind == 1 ? rsqrtf(na) : na;
  rm.rowi = 1.0f; rm.pad = 0;
  rowmeta[g] = rm;
}

// Sampled lower bound of the scene's maximal distance (in the weight-sum kernel's domain: squared distance, or 1 - cos):
// up to 64 candidates x 64 valid feature rows, plain f32 dot products.  Any real element bounds the maximum from below, so
// whatever the sample is, the candidates the weight-sum kernel keeps (x~ >= l0 - bound) contain the true maximum.
// T: element type of the request's feature column (widened on load).
constexpr int DSAMP = 32;
template <class T>
__global__ void __launch_bounds__(256) vis_dense_sample_kernel(Params p, TrackStore ts, Frame f, const int2* rowinfo, float* scene_l0,
                                                                int* dense_bad) {
  __shared__ int s_q[DSAMP], s_r[DSAMP];
  __shared__ int s_nq, s_nr;
  __shared__ float s_w[8];
  const int s = blockIdx.x;
  const SceneDesc sc = f.scenes[s];
  const int K = p.max_obs;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid == 0) { s_nq = 0; s_nr = 0; }
  __syncthreads();
  const int rows = sc.nb * K;
  for (int i = tid; i < sc.m; i += 256) {   // the candidate side of the dense_norm_ok rule
    const int g = sc.det_base + i;
    if ((f.c_flags[g] & 2) && !dense_norm_ok(p, f.c_norm2[g])) dense_bad[s] = 1;
  }
  if (tid < DSAMP) {
    if (sc.m > 0) {
      const int m = (int)(((long long)tid * sc.m) / DSAMP);
      const bool dup = tid > 0 && (int)(((long long)(tid - 1) * sc.m) / DSAMP) == m;
      if (!dup && (f.c_flags[sc.det_base + m] & 2)) s_q[atomicAdd(&s_nq, 1)] = sc.det_base + m;
    }
  } else if (tid < 2 * DSAMP) {
    const int i = tid - DSAMP;
    if (rows > 0) {
      // evenly spaced starting points; a free block or an unused slot moves on to the next valid row (at most 2 K steps)
      int pr = (int)(((long long)i * rows) / DSAMP);
      int fr = -1;
      for (int step = 0; step < 2 * K && pr < rows; ++step, ++pr) {
        fr = rowinfo[(size_t)sc.blk_off * K + pr].y;
        if (fr >= 0) break;
      }
      if (fr >= 0) s_r[atomicAdd(&s_nr, 1)] = fr;   // duplicates are harmless: any real element is a lower bound
    }
  }
  __syncthreads();
  const int nq = s_nq, nr = s_nr;
  float best = 0.0f;
  const int D = p.feature_dim;
  // one warp per sampled pair: the lanes stride over the features (coalesced), shuffle tree at the end
  for (int pi = wid; pi < nq * nr; pi += 8) {
    const int g = s_q[pi / nr], fr = s_r[pi % nr];
    const T* a = static_cast<const T*>(f.in_feat) + (size_t)g * D;
    const float* b = ts.feat + (size_t)fr * p.d8;
    float dot = 0.0f;
    for (int d = lane; d < D; d += 32) dot = __fmaf_rn(feat_elem(a, d), b[d], dot);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
    const float na = f.c_norm2[g], nb2 = ts.fnorm2[fr];
    float v;
    if (p.visual_kind == 1) v = 1.0f - dot * rsqrtf(na) * rsqrtf(nb2) - 1e-4f;
    else v = (na + nb2 - 2.0f * dot) - 1e-4f * (na + nb2);
    best = fmaxf(best, v);
  }
  if (lane == 0) s_w[wid] = best;
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < 8; ++w) best = fmaxf(best, s_w[w]);
    scene_l0[s] = best;
  }
}

// ------------------------------------------------------------------------------------------------ selection kernel
// One CTA per scene.  Pass A: best lower bound of every row (candidate) and column (block) of the weight matrix; pass B:
// every group whose upper bound reaches one of the two is emitted to the scene's pair list with all its valid observations.
constexpr int SEL_T = 512;
// WIDE (K > kMaxObs): an emitted group reads its block's rowinfo twice (count, then list) instead of keeping it per thread.
template <bool WIDE>
__global__ void __launch_bounds__(SEL_T) vis_dense_select_kernel(Params p, Frame f, const __half2* ws, const DenseTrackMeta* tmeta,
                                                                 const int2* rowinfo, const int* maxc_cnt, const int* max_nan,
                                                                 int* dense_bad, int* dbg_counts, const unsigned int* rowb,
                                                                 const unsigned int* colb, int fused) {
  extern __shared__ unsigned char sel_smem[];
  const int s = blockIdx.x;
  const SceneDesc sc = f.scenes[s];
  const int tid = threadIdx.x, lane = tid & 31;
  const int K = p.max_obs;
  const int nb = sc.nb, M = sc.m;
  if (M == 0 || nb == 0) return;
  // preconditions of the dense result
  const unsigned int um = f.scene_max[s];
  const float maxd = __uint_as_float((um & 0x80000000u) ? (um & 0x7fffffffu) : ~um);
  // reasons: 1 an entry the threshold cuts (set by the max refinement and the final refinement) or a feature norm outside
  // dense_norm_ok (set by the metadata and sample kernels), 2 max-candidate list overflow, 4 no maximum found
  const int reason = (max_nan[s] != 0 ? 1 : 0) | (maxc_cnt[s] > sc.vis_lcap ? 2 : 0) | (!(maxd >= 0.0f) ? 4 : 0);
  if (tid == 0) {   // diagnostics of the frame (SB200_TRACE): fallback reasons, list lengths
    if (reason & 1) atomicAdd(&dbg_counts[0], 1);
    if (reason & 2) atomicAdd(&dbg_counts[1], 1);
    if (reason & 4) atomicAdd(&dbg_counts[2], 1);
    atomicAdd(&dbg_counts[3], maxc_cnt[s]);
  }
  if (reason) { if (tid == 0) dense_bad[s] = reason; return; }
  unsigned int* lcol = reinterpret_cast<unsigned int*>(sel_smem);          // [nb] order-preserving f32 encoding
  short* kt = reinterpret_cast<short*>(lcol + nb);                          // [nb] valid observations (0: block takes no part)
  const int need_votes = p.min_votes > 1 ? p.min_votes : 1;
  for (int b = tid; b < nb; b += SEL_T) {
    const DenseTrackMeta tm = tmeta[sc.blk_off + b];
    const int kb = (tm.n >= 0 && tm.kt >= need_votes) ? tm.kt : 0;
    kt[b] = (short)kb;
    unsigned int u = 0x00800000u;   // encoding of -3.4e38-ish: below every real bound, decodes to a finite value
    if (fused && kb > 0) {
      // the weight-sum kernel left max over the rows of -(S + k del); W_lo = k maxd (1 - 2e-6) - 1e-7 + that
      const unsigned int cb = colb[sc.blk_off + b];
      if (cb != 0u) u = enc_ord(((float)kb * maxd * (1.0f - 2e-6f) - 1e-7f) + dec_ord(cb));
    }
    lcol[b] = u;
  }
  __syncthreads();
  const int mpad = (M + 127) / 128 * 128;
  const __half2* w0 = ws + sc.ws_off;
  const float fneg = -3.0e38f;
  // W = k maxd - S, slack = k del + 2e-6 (k maxd + S) + 1e-7 (f32 roundings of both sides):
  //   W_lo = k maxd (1 - 2e-6) - 1e-7 - (1 + 2e-6) S - k del,   W_hi = k maxd (1 + 2e-6) + 1e-7 - (1 - 2e-6) S + k del
  for (int pass = fused ? 1 : 0; pass < 2; ++pass) {
    for (int m0 = 0; m0 < mpad; m0 += SEL_T) {
      const int m = m0 + tid;
      const bool row_ok = m < M && (f.c_flags[sc.det_base + m] & 2);
      float lrow = fneg;
      if (pass == 1 && row_ok) {
        if (!fused) lrow = f.vis_val[sc.vis_lbase + m];   // pass A parked the row bounds in the (still unused) value list
        else {
          const unsigned int* rb = rowb + (size_t)(sc.det_base + m) * kDenseKClasses;
#pragma unroll
          for (int kc = 0; kc < kDenseKClasses; ++kc) {
            const unsigned int u = rb[kc];
            if (u != 0u) lrow = fmaxf(lrow, ((float)(kc + 1) * maxd * (1.0f - 2e-6f) - 1e-7f) + dec_ord(u));
          }
        }
      }
      const __half2* wrow = w0 + m;
      constexpr int UB = 8;   // blocks per round: the loads of a round are issued together (memory-level parallelism)
      for (int b0 = 0; b0 < nb; b0 += UB) {
        int kk[UB];
        float2 ee[UB];
#pragma unroll
        for (int u = 0; u < UB; ++u) {
          kk[u] = b0 + u < nb ? (int)kt[b0 + u] : 0;
          ee[u] = make_float2(0.0f, 0.0f);
          if (row_ok && kk[u] != 0) {
            const unsigned int raw = __ldcs(reinterpret_cast<const unsigned int*>(wrow + (size_t)(b0 + u) * mpad));
            const float2 v = __half22float2(*reinterpret_cast<const __half2*>(&raw));
            // the sum was rounded to fp16 (relative 2^-11): widen the bound by that much
            ee[u] = make_float2(v.x, v.y + (v.x * kHalfRel) / (float)kk[u]);
          }
        }
#pragma unroll
        for (int u = 0; u < UB; ++u) {
          const int k = kk[u], b = b0 + u;
          if (k == 0) continue;   // block-uniform
          const float fk = (float)k, a = fk * maxd;
          const float2 e = ee[u];
          if (pass == 0) {
            float wlo = fneg;
            if (row_ok) wlo = (a * (1.0f - 2e-6f) - 1e-7f) - (e.x * (1.0f + 2e-6f) + fk * e.y);
            lrow = fmaxf(lrow, wlo);
            unsigned int uu = __float_as_uint(wlo);
            uu = (uu & 0x80000000u) ? ~uu : (uu | 0x80000000u);
            uu = __reduce_max_sync(0xffffffffu, uu);   // one instruction: the warp's best lower bound for this column
            if (lane == 0 && uu > lcol[b]) atomicMax(&lcol[b], uu);   // (pass A only runs for the any-K kernel)
          } else if (row_ok) {
            float whi = (a * (1.0f + 2e-6f) + 1e-7f) - (e.x * (1.0f - 2e-6f) - fk * e.y);
            if (!(e.x < 6.0e4f)) whi = 3.0e38f;   // the fp16 sum overflowed (huge unnormalised features): never rule the group out
            const unsigned int uu = lcol[b];
            const float lc = __uint_as_float((uu & 0x80000000u) ? (uu & 0x7fffffffu) : ~uu);
            if (whi >= lrow || whi >= lc) {
              // the group may hold a row or column maximum: all its valid observations go to the exact pass
              const int g = sc.det_base + m;
              int cnt = 0;
              int2 ri[WIDE ? 1 : kMaxObs];
              for (int ph = 0; ph < K; ++ph) {
                const int r = WIDE ? 0 : ph;
                ri[r] = rowinfo[(size_t)sc.blk_off * K + (size_t)b * K + ph];
                cnt += ri[r].y >= 0;
              }
              int pos = atomicAdd(&f.vis_cnt[s], cnt);
              for (int ph = 0; ph < K; ++ph) {
                const int r = WIDE ? 0 : ph;
                if (WIDE) ri[r] = rowinfo[(size_t)sc.blk_off * K + (size_t)b * K + ph];
                if (ri[r].y < 0) continue;
                if (pos < sc.vis_lcap) {
                  VisPair vp;
                  vp.g = g; vp.row = ri[r].y; vp.scene = s; vp.outcol = ri[r].x;
                  f.vis_pairs[sc.vis_lbase + pos] = vp;
                }
                ++pos;
              }
            }
          }
        }
      }
      if (pass == 0 && m < M) f.vis_val[sc.vis_lbase + m] = lrow;
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------ host launcher
// the max-candidate refinement reuses the refine kernel of kernels_feat_tc.cu on a view of the frame
int launch_vis_refine(const Params& p, const TrackStore& ts, const Frame& f, int n_scenes, int* nan_flag, cudaStream_t st);

int launch_vis_dense(const Params& p, const TrackStore& ts, const Frame& f, int n_scenes, int max_m, const TcArgs& tc,
                     cudaStream_t st) {
  if (n_scenes == 0) return 0;
  cudaMemsetAsync(tc.maxc_cnt, 0, (size_t)n_scenes * 4 * 4, st);   // maxc_cnt | maxc_next | dense_bad | zeros (contiguous)
  cudaMemsetAsync(tc.dbg_counts, 0, 8 * 4, st);
  if (tc.n_tiles == 0 || max_m == 0) return 0;
  CUtensorMap mA, mB;
  if (make_map(&mA, f.c_bf16, tc.a_rows, p.d8, TC_BM) || make_map(&mB, ts.feat_bf16, tc.b_rows, p.d8, TC_BN / 2)) return -1;
  const bool cosine = p.visual_kind == 1;
  // metadata: zeroed masks / maxima, then one thread per arena block
  cudaMemsetAsync(tc.slab_vmask, 0, (size_t)tc.n_slabs_ub * (TC_BN / 32) * 4, st);
  cudaMemsetAsync(tc.slab_bmask, 0, (size_t)tc.n_slabs_ub * (TC_BN / 32) * 4, st);
  cudaMemsetAsync(tc.scene_cmax, 0, (size_t)n_scenes * 4, st);
  // block positions past a scene's arena (the last column tile is padded to whole blocks) must read "no voting observations"
  cudaMemsetAsync(tc.slab_ktf, 0, (size_t)tc.n_slabs_ub * TC_BN * 4, st);
  // SB200_DENSE_GENERIC (tests): the any-K epilogue also for K <= kDenseKClasses
  const bool fused = p.max_obs <= kDenseKClasses && getenv("SB200_DENSE_GENERIC") == nullptr;
  if (fused) {
    cudaMemsetAsync(tc.d_rowb, 0, (size_t)f.total * kDenseKClasses * 4, st);
    cudaMemsetAsync(tc.d_colb, 0, (size_t)tc.blk_ub * 4, st);
  }
  const bool wide = p.max_obs > kMaxObs;
  if (tc.max_blocks > 0 && wide) {
    dim3 grid((tc.max_blocks + DMW_WARPS - 1) / DMW_WARPS, n_scenes);
    vis_dense_meta_wide_kernel<<<grid, DMW_WARPS * 32, 0, st>>>(p, ts, f, tc.max_blocks, tc.cstep, tc.tmeta, tc.rowinfo,
                                                              tc.slab_colc, tc.slab_cmax, tc.slab_ktf, tc.slab_vmask,
                                                              tc.slab_bmask, tc.scene_cmax, tc.dense_bad);
    note_launch();
  } else if (tc.max_blocks > 0) {
    dim3 grid((tc.max_blocks + 127) / 128, n_scenes);
    vis_dense_meta_kernel<<<grid, 128, 0, st>>>(p, ts, f, tc.max_blocks, tc.cstep, tc.tmeta, tc.rowinfo, tc.slab_colc, tc.slab_cmax,
                                                tc.slab_ktf, tc.slab_vmask, tc.slab_bmask, tc.scene_cmax,
                                                tc.dense_bad);
    note_launch();
  }
  vis_dense_rowmeta_kernel<<<(f.total + 255) / 256, 256, 0, st>>>(p, f, tc.rowmeta);
  feat_dispatch(f.feat_type, [&](auto t) {
    vis_dense_sample_kernel<decltype(t)><<<n_scenes, 256, 0, st>>>(p, ts, f, tc.rowinfo, tc.scene_l0, tc.dense_bad);
  });
  note_launch(2);
  if (tc.ev_screen0) cudaEventRecord(tc.ev_screen0, st);
  {
    const size_t smem = sizeof(DsSmem) + 1024;
    const void* fn = nullptr;
#define SB_WSUM(KT) (cosine ? (const void*)vis_wsum_kernel<true, KT> : (const void*)vis_wsum_kernel<false, KT>)
    switch (fused ? p.max_obs : 0) {   // the reference's default is 5 observations per track, its published bench uses 3
      case 1: fn = SB_WSUM(1); break;
      case 2: fn = SB_WSUM(2); break;
      case 3: fn = SB_WSUM(3); break;
      case 4: fn = SB_WSUM(4); break;
      case 5: fn = SB_WSUM(5); break;
      default: fn = SB_WSUM(0); break;
    }
#undef SB_WSUM
    cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
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
    DenseDev dd;
    dd.ws = reinterpret_cast<__half2*>(tc.ws); dd.rowb = tc.d_rowb; dd.colb = tc.d_colb; dd.slab_ktf = tc.slab_ktf;
    dd.slab_colc = tc.slab_colc; dd.slab_cmax = tc.slab_cmax; dd.slab_vmask = tc.slab_vmask;
    dd.slab_bmask = tc.slab_bmask; dd.scene_l0 = tc.scene_l0; dd.scene_cmax = tc.scene_cmax; dd.maxc = tc.maxc;
    dd.maxc_cnt = tc.maxc_cnt; dd.rowmeta = tc.rowmeta;
    const TcTile* d_tiles = tc.d_tiles;
    const int* d_n_tiles = tc.d_n_tiles;
    void* args[] = {(void*)&mA, (void*)&mB, (void*)&p, (void*)&ts, (void*)&f, (void*)&d_tiles, (void*)&d_n_tiles, (void*)&dd};
    e = cudaLaunchKernelExC(&cfg, fn, args);
    if (e != cudaSuccess) return (int)e;
    note_launch();
  }
  if (tc.ev_screen1) cudaEventRecord(tc.ev_screen1, st);
  // exact maximal distance: the refine kernel on the candidate list (writes scene_max; flags a value the threshold cuts)
  {
    Frame fm = f;
    fm.vis_pairs = tc.maxc; fm.vis_val = tc.maxc_val; fm.vis_cnt = tc.maxc_cnt; fm.refine_next = tc.maxc_next;
    fm.vis_mode = tc.zeros;
    int rc = launch_vis_refine(p, ts, fm, n_scenes, tc.dense_bad, st);
    if (rc != 0) return rc;
  }
  {
    const size_t smem = (size_t)std::max(1, tc.max_blocks) * 6 + 64;
    const auto kernel = wide ? vis_dense_select_kernel<true> : vis_dense_select_kernel<false>;
    if (smem > 48 * 1024) cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    kernel<<<n_scenes, SEL_T, smem, st>>>(p, f, reinterpret_cast<const __half2*>(tc.ws), tc.tmeta, tc.rowinfo, tc.maxc_cnt,
                                          tc.dense_bad, tc.dense_bad, tc.dbg_counts, tc.d_rowb, tc.d_colb, fused ? 1 : 0);
    note_launch();
  }
  return 0;
}

}  // namespace sb
