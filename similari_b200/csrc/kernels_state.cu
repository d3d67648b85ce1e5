// kernels_state.cu -- applying the voting decisions to the device-resident track store.
//
// Replaces the per-candidate tail of the reference's predict functions
//   (src/trackers/sort/simple_api.rs:165-192, sort/batch_api.rs:98-139, visual_sort/simple_api.rs:188-227):
//   new track   -> TrackStore::add_track of the candidate built by SortMetric::optimize / VisualMetric::optimize
//   merge       -> TrackStore::merge_external -> Track::merge (src/track.rs:522-588) -> optimize(is_merge = true):
//                  Kalman predict + update with the candidate box (src/trackers/kalman_prediction.rs:13-32),
//                  history push, feature-set pruning (src/trackers/visual_sort/metric.rs:129-154,297-374)
// and the lifecycle sweep TrackerAPI::auto_waste (src/trackers/tracker_api.rs:70-88).
#include <cuda_bf16.h>

#include <algorithm>
#include <type_traits>

#include "sb_engine.cuh"

namespace sb {

constexpr int AT = 512;

__device__ __forceinline__ void write_box(float* dst, const Box& b) {
  dst[0] = b.xc; dst[1] = b.yc; dst[2] = b.angle; dst[3] = b.aspect; dst[4] = b.height; dst[5] = b.conf;
}
// the store's own box rows (24-byte rows of a 256-byte aligned allocation): three 8-byte stores
__device__ __forceinline__ void write_box_row(float* dst, const Box& b) {
  float2* d2 = reinterpret_cast<float2*>(dst);
  d2[0] = make_float2(b.xc, b.yc); d2[1] = make_float2(b.angle, b.aspect); d2[2] = make_float2(b.height, b.conf);
}

// Phase 1 of apply (one CTA per scene): rank of every new-track candidate among the scene's new candidates (candidate
// order), the scene's counters, and the inverse map of the frame: for every store row j of the scene, the detection that
// updates it (app_row, -1: no detection).  Phase 2 runs by store row, so that consecutive lanes write consecutive rows.
__global__ void __launch_bounds__(AT) apply_rank_kernel(Params p, TrackStore ts, Frame f, int n_scenes, int* n_tracks) {
  __shared__ int s_warp[AT / 32];
  __shared__ int s_carry;
  __shared__ int s_newbefore;
  const int sidx = blockIdx.x;
  const SceneDesc sc = f.scenes[sidx];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  // ids of non-batch trackers are consumed by new tracks only, in request order => prefix over earlier scenes; the
  // feature-history pool hands out blocks by the same frame-wide rank, for every kind
  const bool need_before = !p.is_batch || ts.hblk != nullptr;
  if (need_before) {
    int c = 0;
    for (int s2 = tid; s2 < f.scene0 + sidx; s2 += AT) c += f.new_count_all[s2];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if (lane == 0) s_warp[wid] = c;
    __syncthreads();
    if (tid == 0) {
      int t = 0;
      for (int w = 0; w < AT / 32; ++w) t += s_warp[w];
      s_newbefore = t;
    }
  }
  // the stored rows nobody matches stay -1; rows [n, n + added) are all taken by the new tracks below
  int* row_det = f.app_row + (size_t)sidx * ts.track_cap;
  for (int j = tid; j < sc.n; j += AT) row_det[j] = -1;
  if (tid == 0) { s_carry = 0; if (!need_before) s_newbefore = 0; }
  __syncthreads();
  const int* winner = f.winner + sc.det_base;
  for (int base = 0; base < sc.m; base += AT) {
    const int m = base + tid;
    const bool active = m < sc.m;
    const int win = active ? winner[m] : 0;
    const int isnew = (active && win < 0) ? 1 : 0;
    int x = isnew;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int t = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += t;
    }
    if (lane == 31) s_warp[wid] = x;
    __syncthreads();
    int woff = 0;
    for (int w = 0; w < wid; ++w) woff += s_warp[w];
    const int carry = s_carry;
    const int rank = carry + woff + x - isnew;
    __syncthreads();
    if (tid == AT - 1) s_carry = carry + woff + x;
    __syncthreads();
    if (active) {
      const int g = sc.det_base + m;
      if (!isnew) row_det[win] = g;
      else if (sc.n + rank < ts.track_cap) row_det[sc.n + rank] = g;
      else {   // store overflow: the frame fails; nothing of this detection may be stored later
        atomicOr(&f.status[sidx], 1);
        if (f.feat_dst) f.feat_dst[g] = -1;
        if (f.hist_dst) f.hist_dst[g] = -1;
      }
    }
  }
  __syncthreads();
  if (tid == 0) {
    // feature arena of this scene (visual trackers): new tracks take blocks from the free list first, then fresh ones
    const int nfree0 = ts.fblk ? ts.n_free[sc.slot] : 0;
    const int top0 = ts.fblk ? ts.arena_top[sc.slot] : 0;
    const int added = min(sc.n + s_carry, ts.track_cap) - sc.n;
    f.app_meta[sidx] = make_int4(s_newbefore, nfree0, top0, sc.n + added);
    n_tracks[sc.slot] = sc.n + added;
    if (ts.fblk) {
      ts.n_free[sc.slot] = nfree0 - min(nfree0, added);
      ts.arena_top[sc.slot] = top0 + max(0, added - nfree0);
    }
  }
}

// K <= kMaxObs: the observation list of a visual merge, unrolled to kMaxObs entries with only static indices, so that every
// list stays in registers.  optimize_observations (visual_sort/metric.rs:297-374): retain the observations with a feature,
// stable insertion sort by descending quality (the swaps make the same comparisons as the sequential shifts, NaN included),
// drop the last when K are kept, push the new observation into the lowest free physical slot and swap it to the front.
// Returns the physical slot of the new observation.
struct ObsList {   // a track's stored list as loaded, entries k < K (those at and beyond n were never written)
  int n;
  unsigned long long hasf, phys;   // byte k: entry k (packed: the whole list fits the registers of the apply)
  float q[kMaxObs];
};
// loaded without waiting for the count, so that the loads go out with the track's other loads
__device__ __forceinline__ ObsList load_obs_list(const TrackStore& ts, size_t idx, int K) {
  ObsList l;
  l.n = ts.obs_n[idx];
  l.hasf = l.phys = 0;
#pragma unroll
  for (int k = 0; k < kMaxObs; ++k) {
    if (k < K) {
      l.hasf |= (unsigned long long)ts.obs_hasf[idx * K + k] << (8 * k);
      l.phys |= (unsigned long long)ts.obs_phys[idx * K + k] << (8 * k);
    }
    l.q[k] = k < K ? ts.obs_q[idx * K + k] : 0.0f;
  }
  return l;
}
__device__ __forceinline__ int merge_obs_list(const TrackStore& ts, size_t idx, int K, const ObsList& l, float quality,
                                              bool keep) {
  unsigned char phys[kMaxObs], hasf[kMaxObs];
  float q[kMaxObs];
  int cnt = 0;
#pragma unroll
  for (int k = 0; k < kMaxObs; ++k) {
    const bool have = k < K && k < l.n;
    const unsigned char lh = have ? (unsigned char)(l.hasf >> (8 * k)) : (unsigned char)0;
    const unsigned char lp = (unsigned char)(l.phys >> (8 * k));
    const float lq = l.q[k];
    phys[k] = 0; q[k] = 0.0f; hasf[k] = 0;
#pragma unroll
    for (int c = 0; c <= k; ++c)
      if (lh && c == cnt) { phys[c] = lp; q[c] = lq; }
    cnt += lh ? 1 : 0;
  }
#pragma unroll
  for (int a = 1; a < kMaxObs; ++a) {
    bool shift = a < cnt;
#pragma unroll
    for (int b = a - 1; b >= 0; --b) {
      shift = shift && q[b] < q[b + 1];
      if (shift) {
        const unsigned char tp = phys[b]; phys[b] = phys[b + 1]; phys[b + 1] = tp;
        const float tq = q[b]; q[b] = q[b + 1]; q[b + 1] = tq;
      }
    }
  }
  if (cnt >= K && cnt > 0) --cnt;
  unsigned int used = 0;
#pragma unroll
  for (int k = 0; k < kMaxObs; ++k)
    if (k < cnt) { used |= 1u << phys[k]; hasf[k] = 1; }
  const int freep = __ffs((int)~used) - 1;   // cnt < K <= kMaxObs: a slot is free
  // push new, swap(0, last)
#pragma unroll
  for (int c = 0; c < kMaxObs; ++c)
    if (c == cnt) { phys[c] = (unsigned char)freep; q[c] = quality; hasf[c] = keep ? 1 : 0; }
  ++cnt;
  unsigned char pl = 0, hl = 0;
  float ql = 0.0f;
#pragma unroll
  for (int c = 0; c < kMaxObs; ++c)
    if (c == cnt - 1) { pl = phys[c]; ql = q[c]; hl = hasf[c]; }
#pragma unroll
  for (int c = 1; c < kMaxObs; ++c)
    if (c == cnt - 1) { phys[c] = phys[0]; q[c] = q[0]; hasf[c] = hasf[0]; }
  phys[0] = pl; q[0] = ql; hasf[0] = hl;
  int fc = 0;
#pragma unroll
  for (int k = 0; k < kMaxObs; ++k)
    if (k < cnt) {
      ts.obs_phys[idx * K + k] = phys[k]; ts.obs_q[idx * K + k] = q[k]; ts.obs_hasf[idx * K + k] = hasf[k];
      fc += hasf[k];
    }
  ts.obs_n[idx] = (unsigned char)cnt;
  ts.feat_cnt[idx] = (unsigned char)fc;
  return freep;
}

// Phase 2 of apply, by store row: grid (row tiles, scenes), thread j of a scene creates or merges store row j from the
// detection app_row names, and leaves at once when it names none.  Consecutive lanes hold consecutive rows, so the narrow
// columns are written in whole sectors; the detection side is a gather inside the scene's candidate range.  The 128-byte
// Kalman rows and the 64-byte vertex rows go through a per-warp tile of shared memory, so that each load or store instruction
// moves whole rows (float4 chunk c of the warp's row r at r * 8 + (c ^ (r & 7)): no bank conflicts either way).
// WIDE (K > kMaxObs): a merge leaves the track's observation list, its feature count and the detection's feature row to
// apply_obs_wide_kernel, which runs next, one warp per row, instead of holding K-sized lists per thread.
constexpr int APT = 128;   // threads of the row-indexed apply: ~10 CTAs for a scene of ~1,200 rows

template <bool WIDE>
__global__ void __launch_bounds__(APT, 4) apply_kernel(Params p, TrackStore ts, Frame f, int n_scenes,
                                                    unsigned long long id_base) {
  __shared__ float4 s_tile[APT / 32][32 * 8];
  __shared__ double2 s_vtile[APT / 32][32 * 4];
  const int K = p.max_obs;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  float4* tile = s_tile[wid];
  double2* vtile = s_vtile[wid];
  if (f.id_counter) id_base = *f.id_counter;   // stream-ordered predict: the counter lives on the device
  for (int sidx = blockIdx.y; sidx < n_scenes; sidx += gridDim.y) {
    const SceneDesc& sc = f.scenes[sidx];
    const int4 meta = f.app_meta[sidx];
    const int s_newbefore = meta.x, nfree0 = meta.y, top0 = meta.z, rows = meta.w;
    const size_t sbase = (size_t)sc.slot * ts.track_cap;
    const int* row_det = f.app_row + (size_t)sidx * ts.track_cap;
    for (int w0 = blockIdx.x * APT + wid * 32; w0 < rows; w0 += gridDim.x * APT) {   // warp-uniform
      const int j = w0 + lane;
      const int g = j < rows ? row_det[j] : -1;
      const bool valid = g >= 0, isnew = j >= sc.n;
      const unsigned int vmask = __ballot_sync(0xffffffffu, valid);
      if (vmask == 0) continue;
      const unsigned int mmask = __ballot_sync(0xffffffffu, valid && !isnew);
      const size_t idx = sbase + j;
      float4* k4 = reinterpret_cast<float4*>(ts.kst) + (sbase + w0) * (kStateStride / 4);
      // the Kalman rows of the warp's merges, whole rows per load
#pragma unroll
      for (int it = 0; it < 8; ++it) {
        const int r = it * 4 + (lane >> 3), c = lane & 7;
        if ((mmask >> r) & 1u) tile[r * 8 + (c ^ (r & 7))] = k4[r * 8 + c];
      }
      __syncwarp();
      if (valid) {
        const float* cbp = f.c_box + (size_t)g * 6;
        const Box cb{cbp[0], cbp[1], cbp[2], cbp[3], cbp[4], cbp[5]};
        const long long custom = f.in_custom ? f.in_custom[g] : (-9223372036854775807LL - 1);
        const unsigned char flags = p.is_visual ? f.c_flags[g] : 0;
        const float quality = (p.is_visual && f.in_quality) ? f.in_quality[g] : 1.0f;
        const int rank = j - sc.n;
        unsigned long long tid64;
        if (p.is_batch) tid64 = id_base + (unsigned long long)g + 1ull;  // one id per candidate (batch_api.rs:102-106)
        else tid64 = id_base + (unsigned long long)(s_newbefore + rank) + 1ull;
        // every load of the row first (one round trip to memory), then the arithmetic, then the stores
        unsigned int len0 = 0; unsigned long long id0 = 0; int blk_b = 0, hb = 0;
        ObsList ol;
        if (!isnew) {
          len0 = ts.length[idx];
          id0 = ts.id[idx];
          if (!WIDE && p.is_visual) {
            ol = load_obs_list(ts, idx, K);
            if (ts.fblk) blk_b = ts.fblk[idx];
          }
          if (ts.hblk) hb = ts.hblk[idx];
        } else {
          if (ts.fblk) blk_b = rank < nfree0 ? ts.blk_free[sbase + (nfree0 - 1 - rank)] : top0 + (rank - nfree0);
          if (ts.hblk) {
            // a new track takes the history-pool block of its frame-wide rank: the free list first, then fresh blocks
            const int r = s_newbefore + rank, hn0 = ts.hpool[0];
            hb = r < hn0 ? ts.hfree[hn0 - 1 - r] : ts.hpool[1] + (r - hn0);
          }
        }
        float st[kStateFloats], st2[kStateFloats];
        Box pred;
        // this lane's new Kalman row (zero-padded to 128 bytes) and vertex row into the warp's tiles, as soon as they are
        // known: the state is dead before the observation list is merged
        auto stage = [&](const Box& pr) {
#pragma unroll
          for (int c = 0; c < 8; ++c) {
            float e[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) e[i] = 4 * c + i < kStateFloats ? st[4 * c + i] : 0.0f;
            tile[lane * 8 + (c ^ (lane & 7))] = make_float4(e[0], e[1], e[2], e[3]);
          }
          if (p.positional_kind == 1) {   // double2 chunk c of row r at r * 4 + (c ^ ((r >> 1) & 3))
            double vx[8];
            box_vertices(pr.xc, pr.yc, pr.angle, pr.aspect, pr.height, vx);
#pragma unroll
            for (int c = 0; c < 4; ++c) vtile[lane * 4 + (c ^ ((lane >> 1) & 3))] = make_double2(vx[2 * c], vx[2 * c + 1]);
          }
        };
        int fdst = -1;
        unsigned long long o_id = 0; unsigned int o_len = 0; signed char o_vt = -1;   // SortTrack columns of this detection
        if (isnew) {
          const float* rb = f.in_boxes + (size_t)g * 6;
          const Box raw{rb[0], rb[1], rb[2], rb[3], rb[4], rb[5]};
          kalman_initiate(p.pos_weight, p.vel_weight, raw, st);
          kalman_predict(p.pos_weight, p.vel_weight, st, st2);
          kalman_update(p.pos_weight, st2, raw, st);
          pred = state_box(st, raw.conf);
          stage(pred);
          ts.id[idx] = tid64;
          ts.length[idx] = 1;
          ts.vt[idx] = -1;
          o_id = tid64; o_len = 1; o_vt = -1;
          write_box_row(ts.obs + idx * 6, raw);
          if (p.is_visual) {
            ts.obs_n[idx] = 1;
            ts.obs_phys[idx * K] = 0;
            ts.obs_hasf[idx * K] = flags & 1;
            ts.obs_q[idx * K] = quality;
            ts.feat_cnt[idx] = flags & 1;
            size_t blk = idx;
            if (ts.fblk) {
              ts.fblk[idx] = blk_b;
              ts.blk_owner[sbase + blk_b] = j;
              blk = sbase + blk_b;
            }
            if (flags & 1) fdst = (int)(blk * K);
          }
        } else {
#pragma unroll
          for (int c = 0; c < 8; ++c) {
            const float4 v = tile[lane * 8 + (c ^ (lane & 7))];
            const float e[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
              if (4 * c + i < kStateFloats) st2[4 * c + i] = e[i];
          }
          o_id = id0;
          kalman_predict(p.pos_weight, p.vel_weight, st2, st);
          kalman_update(p.pos_weight, st, cb, st2);
#pragma unroll
          for (int i = 0; i < kStateFloats; ++i) st[i] = st2[i];
          pred = state_box(st, cb.conf);
          stage(pred);
          o_len = len0 + 1;
          ts.length[idx] = o_len;
          write_box_row(ts.obs + idx * 6, cb);
          if (p.is_visual) {
            o_vt = (signed char)f.c_vt[g];
            ts.vt[idx] = o_vt;
            if (!WIDE) {   // WIDE: apply_obs_wide_kernel
              // is_merge && !feature_can_be_used(collect thresholds) => feature dropped (visual_sort/metric.rs:327-337)
              bool keep = (flags & 1) != 0;
              if (keep) {
                bool ok = quality >= p.min_quality_collect;
                if (p.use_own_area && f.in_own) ok = ok && (f.in_own[g] >= p.min_own_collect);
                ok = ok && (box_area(cb.aspect, cb.height) >= p.min_area);
                keep = ok;
              }
              const size_t blk = ts.fblk ? sbase + blk_b : idx;   // feat_block
              const int freep = merge_obs_list(ts, idx, K, ol, quality, keep);
              if (keep) fdst = (int)(blk * K + freep);
            }
          }
        }
        ts.epoch[idx] = sc.epoch;
        ts.custom[idx] = custom;
        write_box_row(ts.pred + idx * 6, pred);
        ts.radius[idx] = box_radius(pred.aspect, pred.height);
        if (f.feat_dst && !(WIDE && !isnew)) f.feat_dst[g] = fdst;
        if (ts.hblk) {
          // feature history: every observation pushes its feature, or None, before the collect gate
          // (VisualMetric::optimize, visual_sort/metric.rs:319-324).  The sweep at the end of the frame advances hpool by
          // the count of new tracks.
          if (isnew) ts.hblk[idx] = hb;
          const size_t hrow = (size_t)hb * ts.fhist_len + (o_len - 1u) % (unsigned int)ts.fhist_len;
          ts.hpresent[hrow] = flags & 1;
          f.hist_dst[g] = (flags & 1) ? (int)hrow : -1;
        }
        const float* rb2 = f.in_boxes + (size_t)g * 6;
        const Box obs = isnew ? Box{rb2[0], rb2[1], rb2[2], rb2[3], rb2[4], rb2[5]} : cb;
        if (ts.hist_len > 1) {   // update_history: observation number o_len - 1 goes to ring slot (o_len - 1) % hist_len
          const size_t hslot = (idx * ts.hist_len + (size_t)((o_len - 1u) % (unsigned int)ts.hist_len)) * 6;
          write_box_row(ts.hist_pred + hslot, pred);
          write_box_row(ts.hist_obs + hslot, obs);
        }
        // SortTrack (src/trackers/sort.rs:286-311)
        if (f.o_ids) f.o_ids[g] = o_id;
        if (f.o_epochs) f.o_epochs[g] = sc.epoch;
        if (f.o_lengths) f.o_lengths[g] = o_len;
        if (f.o_vt) f.o_vt[g] = p.is_visual ? (o_vt < 0 ? (unsigned char)1 : (unsigned char)o_vt) : (unsigned char)1;
        if (f.o_pred) write_box(f.o_pred + (size_t)g * 6, pred);
        if (f.o_obs) write_box(f.o_obs + (size_t)g * 6, obs);
      }
      // the new Kalman and vertex rows, whole rows per store
      __syncwarp();
#pragma unroll
      for (int it = 0; it < 8; ++it) {
        const int r = it * 4 + (lane >> 3), c = lane & 7;
        if ((vmask >> r) & 1u) k4[r * 8 + c] = tile[r * 8 + (c ^ (r & 7))];
      }
      if (p.positional_kind == 1) {
        double2* v2 = reinterpret_cast<double2*>(ts.vert) + (sbase + w0) * 4;
#pragma unroll
        for (int it = 0; it < 4; ++it) {
          const int r = it * 8 + (lane >> 2), c = lane & 3;
          if ((vmask >> r) & 1u) v2[r * 4 + c] = vtile[r * 4 + (c ^ ((r >> 1) & 3))];
        }
      }
      __syncwarp();   // the next round refills the tiles
    }
  }
}

// The observation list of a visual merge for K > kMaxObs (K <= 32): one warp per stored row, lane k holding logical
// observation k (physical slot, quality, feature flag).  Same steps as merge_obs_list, in the same order:
// optimize_observations keeps the observations with a feature, insertion-sorts them by descending quality (one
// insertion per step; the ballot finds where the shifting stops, exactly as the sequential loop does, NaN qualities
// included), drops the last when K are kept, then pushes the new observation into the lowest free physical slot and swaps
// it to the front.  A 32-bit mask holds every physical slot, which bounds K at 32.  Rows below the scene's n are merges.
__global__ void __launch_bounds__(256) apply_obs_wide_kernel(Params p, TrackStore ts, Frame f, int n_scenes) {
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  const int K = p.max_obs;
  const unsigned int all = 0xffffffffu;
  for (int sidx = blockIdx.y; sidx < n_scenes; sidx += gridDim.y) {
    const int slot = f.scenes[sidx].slot, n = f.scenes[sidx].n;
    const int* row_det = f.app_row + (size_t)sidx * ts.track_cap;
    for (int j = blockIdx.x * wpb + (int)(threadIdx.x >> 5); j < n; j += gridDim.x * wpb) {
      const int g = row_det[j];
      if (g < 0) continue;
      const size_t idx = (size_t)slot * ts.track_cap + j;
      const unsigned char flags = f.c_flags[g];
      const float quality = f.in_quality ? f.in_quality[g] : 1.0f;
      bool keep = (flags & 1) != 0;   // the collect gate of apply_kernel
      if (keep) {
        const float* cbp = f.c_box + (size_t)g * 6;
        bool ok = quality >= p.min_quality_collect;
        if (p.use_own_area && f.in_own) ok = ok && (f.in_own[g] >= p.min_own_collect);
        ok = ok && (box_area(cbp[3], cbp[4]) >= p.min_area);
        keep = ok;
      }
      const int on = ts.obs_n[idx];
      const bool have = lane < on && lane < K;   // slots at and beyond obs_n were never written
      const bool retain = have && ts.obs_hasf[idx * K + lane];
      const int ph0 = retain ? ts.obs_phys[idx * K + lane] : 0;
      const float q0 = retain ? ts.obs_q[idx * K + lane] : 0.0f;
      // retain featured, in logical order: lane j takes the j-th retained observation
      const unsigned int rmask = __ballot_sync(all, retain);
      int cnt = __popc(rmask);
      int src = 0;   // lowest bit s with popc(rmask & bits 0..s) == lane + 1 (binary search; 31 when lane >= cnt)
      for (int b = 16; b > 0; b >>= 1)
        if (__popc(rmask & ((2u << (src + b - 1)) - 1u)) < lane + 1) src += b;
      int ph = __shfl_sync(all, ph0, src);
      float q = __shfl_sync(all, q0, src);
      for (int a = 1; a < cnt; ++a) {   // stable insertion sort, descending quality
        const float qa = __shfl_sync(all, q, a);
        const int pa = __shfl_sync(all, ph, a);
        // the sequential loop shifts while q[b] < qa, from b = a - 1 down: it stops below the highest b < a without that
        const unsigned int stop = __ballot_sync(all, lane < a && !(q < qa));
        const int pos = stop ? 32 - __clz((int)stop) : 0;
        const float qu = __shfl_up_sync(all, q, 1);
        const int pu = __shfl_up_sync(all, ph, 1);
        if (lane > pos && lane <= a) { q = qu; ph = pu; }
        if (lane == pos) { q = qa; ph = pa; }
      }
      if (cnt >= K && cnt > 0) --cnt;
      const unsigned int used = __reduce_or_sync(all, lane < cnt ? 1u << ph : 0u);
      const int freep = __ffs((int)~used) - 1;   // cnt < K <= 32: a slot is free
      // push new, swap(0, last)
      unsigned char hasf = lane < cnt ? 1 : 0;
      if (lane == cnt) { ph = freep; q = quality; hasf = keep ? 1 : 0; }
      ++cnt;
      const int from = lane == 0 ? cnt - 1 : (lane == cnt - 1 ? 0 : lane);
      ph = __shfl_sync(all, ph, from);
      q = __shfl_sync(all, q, from);
      hasf = (unsigned char)__shfl_sync(all, (int)hasf, from);
      if (lane < cnt) {
        ts.obs_phys[idx * K + lane] = (unsigned char)ph; ts.obs_q[idx * K + lane] = q; ts.obs_hasf[idx * K + lane] = hasf;
      }
      const int fc = __popc(__ballot_sync(all, lane < cnt && hasf));
      if (lane == 0) {
        ts.obs_n[idx] = (unsigned char)cnt;
        ts.feat_cnt[idx] = (unsigned char)fc;
        if (f.feat_dst) f.feat_dst[g] = keep ? (int)(feat_block(ts, slot, idx) * K + freep) : -1;
      }
    }
  }
}

// copies the features that VisualMetric::optimize keeps into the track's free physical slot (warp per detection), and
// every present feature -- kept or dropped by the collect gate -- into the track's history ring when history is on.
// This kernel runs beside the end-of-frame sweep (side stream).  It writes history rows only of the blocks of tracks
// updated in this frame (epoch == the scene's new epoch); the sweep moves only the block indices of tracks with
// epoch + max_idle < that epoch, and no block changes hands in between (blocks are freed on the host, after a drain, and
// reused only by frames enqueued after it).  The two sets are disjoint.
// T: element type of the request's feature column; a 2-byte row is widened to f32 where it is loaded, and the arena row,
// its BF16 and e4m3 copies and the history row are written from the widened values.  With d8 <= 512 (the only rows with
// an e4m3 copy) the vector paths hold the whole row in registers after their first round: the e4m3 copy comes from there.
template <class T>
__global__ void feat_store_kernel(Params p, TrackStore ts, Frame f) {
  int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  int lane = threadIdx.x & 31;
  if (w >= f.total) return;
  if (lane == 0 && f.bf16_log) f.bf16_log[w] = f.feat_dst[f.det0 + w];
  w += f.det0;
  const int dst = f.feat_dst[w];
  const int hdst = f.hist_dst ? f.hist_dst[w] : -1;
  if (dst < 0 && hdst < 0) return;
  const T* src = static_cast<const T*>(f.in_feat) + (size_t)w * p.feature_dim;
  float* d = ts.feat + (size_t)max(dst, 0) * p.d8;
  __nv_bfloat16* db = reinterpret_cast<__nv_bfloat16*>(ts.feat_bf16) + (size_t)max(dst, 0) * p.d8;
  const bool wb = dst >= 0 && !f.skip_bf16;
  float* hd = hdst >= 0 ? ts.hrows + (size_t)hdst * p.d8 : nullptr;
  unsigned char* d8p = dst >= 0 && ts.feat_fp8 ? ts.feat_fp8 + (size_t)dst * fp8_pitch(p.d8) : nullptr;
  if constexpr (!std::is_same<T, float>::value) {
    if (p.feature_dim == p.d8 && (reinterpret_cast<uintptr_t>(f.in_feat) & 15) == 0) {
      // rows are 16-byte multiples: one 16-byte load is 8 elements, four in flight per lane
      const uint4* s8 = reinterpret_cast<const uint4*>(src);
      float4* d4 = reinterpret_cast<float4*>(d);
      float4* h4 = reinterpret_cast<float4*>(hd);
      uint4* b8 = reinterpret_cast<uint4*>(db);
      const int n8 = p.d8 >> 3;
      uint4 r[4];
      for (int i0 = 0; i0 < n8; i0 += 128) {
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int i = i0 + u * 32 + lane;
          if (i < n8) r[u] = __ldcs(s8 + i);   // the input row is dead after this kernel
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int i = i0 + u * 32 + lane;
          if (i < n8) {
            float x[8];
            feat_widen8(r[u], src, x);
            const float4 lo = make_float4(x[0], x[1], x[2], x[3]), hi = make_float4(x[4], x[5], x[6], x[7]);
            if (dst >= 0) {
              d4[2 * i] = lo;
              d4[2 * i + 1] = hi;
            }
            if (wb) {
              __nv_bfloat162 bb[4];
#pragma unroll
              for (int l = 0; l < 4; ++l) bb[l] = __floats2bfloat162_rn(x[2 * l], x[2 * l + 1]);
              b8[i] = *reinterpret_cast<const uint4*>(bb);   // B operand of the tensor-core screen
            }
            if (h4) { __stcs(h4 + 2 * i, lo); __stcs(h4 + 2 * i + 1, hi); }
          }
        }
      }
      if (d8p) {   // n8 <= 64: blocks lane and lane + 32 of the row are r[0] and r[1]
        float x[2][8];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (h * 32 + lane < n8) feat_widen8(r[h], src, x[h]);
          else
#pragma unroll
            for (int l = 0; l < 8; ++l) x[h][l] = 0.0f;
        }
        const float s = fp8_row_store(x, p.d8, d8p);
        if (lane == 0) ts.fscale[dst] = s;
      }
    } else {
      for (int i = lane; i < p.d8; i += 32) {
        float x = i < p.feature_dim ? feat_elem(src, i) : 0.0f;   // Feature::from_vec zero-pads to the 8-lane multiple
        if (dst >= 0) d[i] = x;
        if (wb) db[i] = __float2bfloat16_rn(x);
        if (hd) hd[i] = x;
      }
      if (d8p) {   // from the f32 row this warp has just written
        __syncwarp();
        const float s = fp8_row_from(d, p.d8, p.d8, d8p);
        if (lane == 0) ts.fscale[dst] = s;
      }
    }
  } else if (p.feature_dim == p.d8 && (reinterpret_cast<uintptr_t>(f.in_feat) & 15) == 0) {
    // rows are 32-byte multiples: 16-byte vectors, four in flight per lane
    const float4* s4 = reinterpret_cast<const float4*>(src);
    float4* d4 = reinterpret_cast<float4*>(d);
    float4* h4 = reinterpret_cast<float4*>(hd);
    uint2* b4 = reinterpret_cast<uint2*>(db);
    const int n4 = p.d8 >> 2;
    float4 v[4];
    for (int i0 = 0; i0 < n4; i0 += 128) {
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int i = i0 + u * 32 + lane;
        if (i < n4) v[u] = __ldcs(s4 + i);   // the input row is dead after this kernel
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int i = i0 + u * 32 + lane;
        if (i < n4) {
          if (dst >= 0) d4[i] = v[u];
          if (wb) {
            const __nv_bfloat162 lo = __floats2bfloat162_rn(v[u].x, v[u].y), hi = __floats2bfloat162_rn(v[u].z, v[u].w);
            uint2 pk;
            pk.x = *reinterpret_cast<const unsigned int*>(&lo);
            pk.y = *reinterpret_cast<const unsigned int*>(&hi);
            b4[i] = pk;   // B operand of the tensor-core screen
          }
          if (h4) __stcs(h4 + i, v[u]);   // read back only when the track is collected: streaming store
        }
      }
    }
    if (d8p) {   // n4 <= 128: element 4 i of the row is v[i / 32] of lane i % 32
      float amax = 0.0f;   // the maximum of fp8_row_store (NaN does not enter it)
#pragma unroll
      for (int u = 0; u < 4; ++u)
        if (u * 32 + lane < n4)
          amax = fmaxf(amax, fmaxf(fmaxf(fabsf(v[u].x), fabsf(v[u].y)), fmaxf(fabsf(v[u].z), fabsf(v[u].w))));
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
      const float s = fp8_row_scale(amax);
      unsigned int* o4 = reinterpret_cast<unsigned int*>(d8p);
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int i = u * 32 + lane;
        if (i < n4) o4[i] = fp8_pack4(v[u].x, v[u].y, v[u].z, v[u].w, s);
      }
      if (lane == 0) ts.fscale[dst] = s;
    }
  } else {
    for (int i = lane; i < p.d8; i += 32) {
      float x = i < p.feature_dim ? src[i] : 0.0f;   // Feature::from_vec zero-pads to the 8-lane multiple
      if (dst >= 0) d[i] = x;
      if (wb) db[i] = __float2bfloat16_rn(x);
      if (hd) hd[i] = x;
    }
    if (d8p) {   // from the f32 row this warp has just written
      __syncwarp();
      const float s = fp8_row_from(d, p.d8, p.d8, d8p);
      if (lane == 0) ts.fscale[dst] = s;
    }
  }
  if (lane == 0 && dst >= 0) ts.fnorm2[dst] = f.c_norm2[w];
}

__global__ void bf16_regen_kernel(TrackStore ts, int d8, int K, const int* __restrict__ rows, long long n, int n_slots) {
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  auto convert = [&](long long r) {
    const float4* s4 = reinterpret_cast<const float4*>(ts.feat + (size_t)r * d8);
    uint2* b4 = reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(ts.feat_bf16) + (size_t)r * d8);
    for (int k = lane; k < (d8 >> 2); k += 32) {
      const float4 v = s4[k];
      const __nv_bfloat162 lo = __floats2bfloat162_rn(v.x, v.y), hi = __floats2bfloat162_rn(v.z, v.w);
      b4[k] = make_uint2(*reinterpret_cast<const unsigned int*>(&lo), *reinterpret_cast<const unsigned int*>(&hi));
    }
  };
  const long long w0 = (long long)blockIdx.x * wpb + (threadIdx.x >> 5), ws = (long long)gridDim.x * wpb;
  if (rows) {
    for (long long i = w0; i < n; i += ws)
      if (rows[i] >= 0) convert(rows[i]);
    return;
  }
  for (int s = blockIdx.y; s < n_slots; s += gridDim.y) {
    const long long r0 = (long long)s * ts.track_cap * K, nr = (long long)ts.arena_top[s] * K;
    for (long long i = w0; i < nr; i += ws) convert(r0 + i);
  }
}

void launch_bf16_regen(const TrackStore& ts, int d8, int K, const int* rows, long long n, int n_slots, cudaStream_t st) {
  if (rows ? n <= 0 : n_slots <= 0) return;
  const long long warps = rows ? n : (long long)ts.track_cap * K;   // per slot: an upper bound of its arena rows
  const dim3 grid((unsigned)std::min<long long>((warps + 7) / 8, 2048), rows ? 1u : scene_grid(n_slots));
  bf16_regen_kernel<<<grid, 256, 0, st>>>(ts, d8, K, rows, n, n_slots);
  note_launch();
}

// feature histories of wasted records, one warp per (record, entry)
__global__ void hist_gather_kernel(TrackStore ts, int d8, const int* __restrict__ blk, const unsigned int* __restrict__ lengths,
                                   int n, int hist_cap, float* __restrict__ out_rows, unsigned char* __restrict__ out_present) {
  const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= (long long)n * hist_cap) return;
  const int i = (int)(w / hist_cap), c = (int)(w - (long long)i * hist_cap);
  const unsigned int len = lengths[i], H = (unsigned int)ts.fhist_len;
  const int cnt = (int)min(min(len, H), (unsigned int)hist_cap);
  // every output row is written: the entry's feature, or zeros (no feature, or past the record's count)
  unsigned char present = 0;
  size_t row = 0;
  if (c < cnt) {
    const unsigned int j = len - (unsigned int)cnt + (unsigned int)c;   // observation number, oldest kept first
    row = (size_t)blk[i] * H + j % H;
    present = ts.hpresent[row];
  }
  if (lane == 0) out_present[w] = present;
  const float4* s4 = reinterpret_cast<const float4*>(ts.hrows + row * d8);
  float4* d4 = reinterpret_cast<float4*>(out_rows + (size_t)w * d8);
  for (int k = lane; k < (d8 >> 2); k += 32) d4[k] = present ? s4[k] : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
}

void launch_hist_gather(const TrackStore& ts, int d8, const int* blk, const unsigned int* lengths, int n, int hist_cap,
                        float* out_rows, unsigned char* out_present, cudaStream_t st) {
  const long long threads = (long long)n * hist_cap * 32;
  if (threads == 0) return;
  hist_gather_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(ts, d8, blk, lengths, n, hist_cap, out_rows,
                                                                        out_present);
  note_launch();
}

void launch_apply(const Params& p, const TrackStore& ts, const Frame& f, int n_scenes, int max_rows,
                  unsigned long long id_base, int* d_n_tracks, cudaStream_t st) {
  if (n_scenes == 0) return;
  apply_rank_kernel<<<n_scenes, AT, 0, st>>>(p, ts, f, n_scenes, d_n_tracks);
  note_launch();
  if (f.total > 0) {
    // max_rows bounds every scene's rows (stored tracks + detections); the kernels stride past it all the same
    const int rows = std::max(1, std::min(max_rows, ts.track_cap));
    const dim3 grid((unsigned)((rows + APT - 1) / APT), scene_grid(n_scenes));
    if (p.max_obs > kMaxObs) {
      apply_kernel<true><<<grid, APT, 0, st>>>(p, ts, f, n_scenes, id_base);
      apply_obs_wide_kernel<<<dim3((unsigned)((rows + 7) / 8), scene_grid(n_scenes)), 256, 0, st>>>(p, ts, f, n_scenes);
      note_launch(2);
    } else {
      apply_kernel<false><<<grid, APT, 0, st>>>(p, ts, f, n_scenes, id_base);
      note_launch();
    }
  }
}

bool launch_feat_store(const Params& p, const TrackStore& ts, const Frame& f, cudaStream_t st) {
  if (!(p.is_visual && f.in_feat && f.total > 0)) return false;
  long long threads = (long long)f.total * 32;
  feat_dispatch(f.feat_type, [&](auto t) {
    feat_store_kernel<decltype(t)><<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(p, ts, f);
  });
  note_launch();
  return true;
}

// --------------------------------------------------------------------------------------------------------
// auto_waste: EpochDb::baked (src/trackers/epoch_db.rs:51-66): last_updated + max_idle < current_epoch => Wasted.
// One CTA per scene; a stable compaction keeps the store order.
//
// Two callers: the reference's collection points (auto-waste tick, wasted(), skip_epochs: all scene slots, epochs from the
// host's epoch db) and the end-of-frame sweep (the scenes of the request, `scenes` != null, epoch = the scene's new epoch).
// Only the small per-track arrays move (about 300 B per track).  Feature rows never do: an expired track's block of the
// scene's feature arena goes to the free list and is handed to the next new track.
constexpr int WT = 512;    // threads of the sweep kernel: two CTAs per SM, so 256 scenes are one wave
constexpr int WR = 8;      // elements in flight per thread and round of compact_rows

// Moves row j to row s_dst[j] (<= j; -1: dropped) for j in [first, n).  The flattened (row, column) elements are taken in
// ascending rounds of AT * WR: a round reads all its elements, synchronises, then writes them.  Destinations never lie
// above sources, so a round can only overwrite elements it has already read or that an earlier round has moved away.
template <typename T>
__device__ __forceinline__ void compact_rows(T* arr, size_t base, int width, const int* s_dst, int first, int n) {
  T* a = arr + base * width;
  const int total = n * width;
  for (int e0 = first * width; e0 < total; e0 += WT * WR) {
    T v[WR];
    int de[WR];
#pragma unroll
    for (int r = 0; r < WR; ++r) {
      const int e = e0 + r * WT + (int)threadIdx.x;
      de[r] = -1;
      if (e < total) {
        const int j = e / width, c = e - j * width;
        const int d = s_dst[j];
        if (d >= 0 && d != j) { v[r] = a[e]; de[r] = d * width + c; }
      }
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < WR; ++r)
      if (de[r] >= 0) a[de[r]] = v[r];
    __syncthreads();
  }
}

// WIDE (K > kMaxObs): the observation columns move as K-wide rows through compact_rows instead of per-thread lists.
template <bool WIDE>
__global__ void __launch_bounds__(WT) waste_kernel(Params p, TrackStore ts, const unsigned int* cur_epoch,
                                                   const unsigned long long* scene_ids, int* n_tracks, WastedBuf wb,
                                                   const SceneDesc* scenes, int* frame_out, unsigned long long* id_counter,
                                                   long long id_add, const int* new_count, int n_scenes) {
  extern __shared__ int s_dst[];   // [n] destination row of every track (-1: expired)
  __shared__ int s_warp[WT / 32];
  __shared__ int s_wbase, s_wcount, s_first;
  if (id_counter && blockIdx.x == 0 && threadIdx.x == 0) {
    // ids consumed by this frame: one per detection (batch trackers) or one per new track (sort/simple_api.rs:99-102,170).
    // Every apply_kernel CTA has read the old value: that kernel completed before this one started.
    unsigned long long add = 0;
    if (id_add >= 0) add = (unsigned long long)id_add;
    else for (int s2 = 0; s2 < n_scenes; ++s2) add += (unsigned long long)new_count[s2];
    *id_counter += add;
  }
  if (ts.hblk && scenes && blockIdx.x == 0 && threadIdx.x == 0) {
    // feature-history pool: the new tracks of this frame took its first free blocks, then fresh ones (apply_kernel, which
    // completed before this kernel started, read the old values)
    int add = 0;
    for (int s2 = 0; s2 < n_scenes; ++s2) add += new_count[s2];
    const int nf = ts.hpool[0];
    ts.hpool[0] = nf - min(nf, add);
    ts.hpool[1] += max(0, add - nf);
  }
  const int slot = scenes ? scenes[blockIdx.x].slot : (int)blockIdx.x;
  const int n = n_tracks[slot];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const size_t base = (size_t)slot * ts.track_cap;
  const unsigned int cur = scenes ? scenes[blockIdx.x].epoch : cur_epoch[slot];
  const unsigned long long scene_id = scenes ? scenes[blockIdx.x].scene_id : scene_ids[slot];
  const int K = p.max_obs;
  const bool arena = ts.fblk != nullptr;
  if (n == 0) {
    if (frame_out && tid == 0) {
      frame_out[blockIdx.x * 3] = 0; frame_out[blockIdx.x * 3 + 1] = arena ? ts.arena_top[slot] : 0; frame_out[blockIdx.x * 3 + 2] = 0;
    }
    return;
  }
  // pass 1: destination of every track = index minus the expired tracks before it
  if (tid == 0) s_first = n;
  int seen = 0;   // expired tracks in the chunks before (uniform)
  for (int j0 = 0; j0 < n; j0 += WT) {
    const int j = j0 + tid;
    // cur - ep > max_idle: the reference's ep + max_idle < cur in usize, which ep + max_idle in u32 can wrap past
    const unsigned int ep = j < n ? ts.epoch[base + j] : cur;
    const int w = (cur > ep && cur - ep > (unsigned int)p.max_idle_epochs) ? 1 : 0;
    int x = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int t = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += t;
    }
    if (lane == 31) s_warp[wid] = x;
    __syncthreads();
    int woff = 0, wtot = 0;
    for (int q = 0; q < WT / 32; ++q) { if (q < wid) woff += s_warp[q]; wtot += s_warp[q]; }
    const int before = seen + woff + x - w;
    if (j < n) {
      s_dst[j] = w ? -1 - before : j - before;   // expired: -(rank among the expired) - 1
      if (w) atomicMin(&s_first, j);
    }
    seen += wtot;
    __syncthreads();
  }
  if (tid == 0) {
    s_wcount = seen;
    s_wbase = seen > 0 ? atomicAdd(wb.count, seen) : 0;
  }
  __syncthreads();
  const int wcount = s_wcount;
  if (frame_out && tid == 0) {
    frame_out[blockIdx.x * 3] = n - wcount;
    frame_out[blockIdx.x * 3 + 1] = arena ? ts.arena_top[slot] : 0;
    frame_out[blockIdx.x * 3 + 2] = wcount;
  }
  if (wcount == 0) return;
  const int first = s_first;
  const int nfree0 = arena ? ts.n_free[slot] : 0;
  // pass 2: records of the expired tracks -> wasted buffer, their feature blocks -> free list (store order)
  for (int j = first + tid; j < n; j += WT) {
    const int d = s_dst[j];
    if (d >= 0) continue;
    const int wrank = -1 - d;
    const int o = s_wbase + wrank;
    if (o < wb.cap) {
      wb.id[o] = ts.id[base + j]; wb.scene[o] = scene_id; wb.epoch[o] = ts.epoch[base + j];
      wb.length[o] = ts.length[base + j];
      for (int c = 0; c < 6; ++c) { wb.pred[(size_t)o * 6 + c] = ts.pred[(base + j) * 6 + c]; wb.obs[(size_t)o * 6 + c] = ts.obs[(base + j) * 6 + c]; }
      if (ts.hist_len > 1) {
        const int hw = ts.hist_len * 6;
        // observation j lives in ring slot j % hist_len: a track shorter than the ring has written slots [0, length) only
        const int hv = (int)min((unsigned int)ts.hist_len, ts.length[base + j]) * 6;
        for (int c = 0; c < hv; ++c) {
          wb.hist_pred[(size_t)o * hw + c] = ts.hist_pred[(base + j) * hw + c];
          wb.hist_obs[(size_t)o * hw + c] = ts.hist_obs[(base + j) * hw + c];
        }
      }
      if (ts.hblk) wb.hblk[o] = ts.hblk[base + j];   // the feature history stays in the pool: only its block moves
    }
    if (arena) {
      const int b = ts.fblk[base + j];
      ts.blk_free[base + nfree0 + wrank] = b;
      ts.blk_owner[base + b] = -1;
    }
  }
  __syncthreads();
  // pass 3: stable compaction of the per-track arrays.  The narrow columns of a track travel together (one thread per
  // track, one read / write round per WT tracks); the wide rows go through compact_rows.
  for (int j0 = first; j0 < n; j0 += WT) {
    const int j = j0 + tid;
    int d = -1;
    unsigned long long v_id = 0; unsigned int v_ep = 0, v_len = 0; long long v_cu = 0; signed char v_vt = 0; float v_r = 0.0f;
    unsigned char v_on = 0, v_fc = 0, v_ph[kMaxObs], v_hf[kMaxObs]; float v_q[kMaxObs]; int v_fb = 0, v_hb = 0;
    if (j < n) {
      d = s_dst[j];
      if (d >= 0 && d != j) {
        const size_t t = base + j;
        v_id = ts.id[t]; v_ep = ts.epoch[t]; v_len = ts.length[t]; v_cu = ts.custom[t]; v_vt = ts.vt[t]; v_r = ts.radius[t];
        if (p.is_visual) {
          v_on = ts.obs_n[t]; v_fc = ts.feat_cnt[t];
          if (arena) v_fb = ts.fblk[t];
          if (ts.hblk) v_hb = ts.hblk[t];
          for (int k = 0; k < (WIDE ? 0 : K); ++k) {   // slots at and beyond obs_n were never written
            const bool have = k < (int)v_on;
            v_ph[k] = have ? ts.obs_phys[t * K + k] : (unsigned char)0; v_hf[k] = have ? ts.obs_hasf[t * K + k] : (unsigned char)0;
            v_q[k] = have ? ts.obs_q[t * K + k] : 0.0f;
          }
        }
      } else d = -1;
    }
    __syncthreads();
    if (d >= 0) {
      const size_t t = base + d;
      ts.id[t] = v_id; ts.epoch[t] = v_ep; ts.length[t] = v_len; ts.custom[t] = v_cu; ts.vt[t] = v_vt; ts.radius[t] = v_r;
      if (p.is_visual) {
        ts.obs_n[t] = v_on; ts.feat_cnt[t] = v_fc;
        if (arena) ts.fblk[t] = v_fb;
        if (ts.hblk) ts.hblk[t] = v_hb;
        for (int k = 0; k < (WIDE ? 0 : K); ++k) { ts.obs_phys[t * K + k] = v_ph[k]; ts.obs_hasf[t * K + k] = v_hf[k]; ts.obs_q[t * K + k] = v_q[k]; }
      }
    }
    __syncthreads();
  }
  compact_rows(ts.pred, base, 6, s_dst, first, n);
  compact_rows(ts.obs, base, 6, s_dst, first, n);
  compact_rows(ts.kst, base, ts.kst_stride, s_dst, first, n);
  if (p.positional_kind == 1) compact_rows(ts.vert, base, 8, s_dst, first, n);
  if (WIDE && p.is_visual) {
    compact_rows(ts.obs_phys, base, K, s_dst, first, n);
    compact_rows(ts.obs_hasf, base, K, s_dst, first, n);
    compact_rows(ts.obs_q, base, K, s_dst, first, n);
  }
  if (ts.hist_len > 1) {
    compact_rows(ts.hist_pred, base, ts.hist_len * 6, s_dst, first, n);
    compact_rows(ts.hist_obs, base, ts.hist_len * 6, s_dst, first, n);
  }
  const int kept = n - wcount;
  if (arena) {   // owners follow the compaction
    for (int j = first + tid; j < kept; j += WT) ts.blk_owner[base + ts.fblk[base + j]] = j;
    if (tid == 0) ts.n_free[slot] = nfree0 + wcount;
  }
  if (tid == 0) n_tracks[slot] = kept;
}

static void launch_waste_kernel(const Params& p, const TrackStore& ts, int n_ctas, const unsigned int* d_cur_epoch,
                                const unsigned long long* d_scene_ids, int* d_n_tracks, const WastedBuf& wb,
                                const SceneDesc* scenes, int* frame_out, unsigned long long* id_counter, long long id_add,
                                const int* new_count, cudaStream_t st) {
  const size_t smem = (size_t)std::max(1, ts.track_cap) * sizeof(int);   // s_dst for the largest possible scene
  const auto kernel = p.max_obs > kMaxObs ? waste_kernel<true> : waste_kernel<false>;
  if (smem > 48 * 1024) cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  kernel<<<n_ctas, WT, smem, st>>>(p, ts, d_cur_epoch, d_scene_ids, d_n_tracks, wb, scenes, frame_out, id_counter, id_add,
                                   new_count, n_ctas);
  note_launch();
}

void launch_waste(const Params& p, const TrackStore& ts, int n_slots, const unsigned int* d_cur_epoch,
                  const unsigned long long* d_scene_ids, int* d_n_tracks, const WastedBuf& wb, int max_n,
                  cudaStream_t st) {
  (void)max_n;
  if (n_slots == 0) return;
  launch_waste_kernel(p, ts, n_slots, d_cur_epoch, d_scene_ids, d_n_tracks, wb, nullptr, nullptr, nullptr, 0, nullptr, st);
}

void launch_frame_sweep(const Params& p, const TrackStore& ts, const Frame& f, int n_scenes, int* d_n_tracks,
                        const WastedBuf& wb, cudaStream_t st) {
  if (n_scenes == 0) return;
  launch_waste_kernel(p, ts, n_scenes, nullptr, nullptr, d_n_tracks, wb, f.scenes, f.frame_out, f.id_counter, f.id_add,
                      f.new_count, st);
}

// --------------------------------------------------------------------------------------------------------
// stateless Kalman operators (parity tests / callers that keep their own state)
__global__ void kalman_ops_kernel(int op, float pw, float vw, const float* in30, const float* boxes, int n, float* out30) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float a[kStateFloats], b[kStateFloats];
  Box bx{};
  if (boxes) { const float* q = boxes + (size_t)i * 6; bx = Box{q[0], q[1], q[2], q[3], q[4], q[5]}; }
  if (op == 0) kalman_initiate(pw, vw, bx, b);
  else {
    for (int k = 0; k < kStateFloats; ++k) a[k] = in30[(size_t)i * kStateFloats + k];
    if (op == 1) kalman_predict(pw, vw, a, b);
    else kalman_update(pw, a, bx, b);
  }
  for (int k = 0; k < kStateFloats; ++k) out30[(size_t)i * kStateFloats + k] = b[k];
}

void launch_kalman_ops(int op, float pw, float vw, const float* in30, const float* boxes, int n, float* out30,
                       cudaStream_t st) {
  if (n == 0) return;
  kalman_ops_kernel<<<(n + 127) / 128, 128, 0, st>>>(op, pw, vw, in30, boxes, n, out30);
  note_launch();
}

// Universal2DBoxKalmanFilter::distance over n (state, box) pairs
__global__ void kalman_distance_kernel(float pw, const float* __restrict__ in30, const float* __restrict__ boxes, int n,
                                       float* __restrict__ out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float a[kStateFloats];
  for (int k = 0; k < kStateFloats; ++k) a[k] = in30[(size_t)i * kStateFloats + k];
  const float* q = boxes + (size_t)i * 6;
  out[i] = kalman_distance(pw, a, Box{q[0], q[1], q[2], q[3], q[4], q[5]});
}

void launch_kalman_distance(float pw, const float* in30, const float* boxes, int n, float* out, cudaStream_t st) {
  if (n == 0) return;
  kalman_distance_kernel<<<(n + 127) / 128, 128, 0, st>>>(pw, in30, boxes, n, out);
  note_launch();
}

// Point2DKalmanFilter over n packed 12-float states, one thread per state.  op: 0 initiate (points -> out12),
// 1 predict (in12 -> out12), 2 update (in12, points -> out12), 3 distance (in12, points -> out_f32).
__global__ void point_kalman_kernel(int op, float pw, float vw, const float* __restrict__ in12,
                                    const float* __restrict__ points, int n, float* __restrict__ out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float a[kPointStateFloats], b[kPointStateFloats];
  float x = 0.0f, y = 0.0f;
  if (points) { x = points[(size_t)i * 2]; y = points[(size_t)i * 2 + 1]; }
  if (op != 0) {
    const float4* s4 = reinterpret_cast<const float4*>(in12 + (size_t)i * kPointStateFloats);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const float4 v = s4[k];
      a[4 * k] = v.x; a[4 * k + 1] = v.y; a[4 * k + 2] = v.z; a[4 * k + 3] = v.w;
    }
  }
  if (op == 3) { out[i] = point_kalman_distance(pw, a, x, y); return; }
  if (op == 0) point_kalman_initiate(pw, vw, x, y, b);
  else if (op == 1) point_kalman_predict(pw, vw, a, b);
  else point_kalman_update(pw, a, x, y, b);
  float4* o4 = reinterpret_cast<float4*>(out + (size_t)i * kPointStateFloats);
#pragma unroll
  for (int k = 0; k < 3; ++k) o4[k] = make_float4(b[4 * k], b[4 * k + 1], b[4 * k + 2], b[4 * k + 3]);
}

void launch_point_kalman(int op, float pw, float vw, const float* in12, const float* points, int n, float* out,
                         cudaStream_t st) {
  if (n == 0) return;
  point_kalman_kernel<<<(n + 255) / 256, 256, 0, st>>>(op, pw, vw, in12, points, n, out);
  note_launch();
}

// ------------------------------------------------------------------------------------------------------------
// Small per-frame tables (scene descriptors, tile list) are read straight from mapped pinned host memory.
__global__ void pull_kernel(unsigned int* __restrict__ dst, const unsigned int* __restrict__ src, size_t n4, size_t n1) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n4) reinterpret_cast<uint4*>(dst)[i] = reinterpret_cast<const uint4*>(src)[i];
  if (i < n1) dst[n4 * 4 + i] = src[n4 * 4 + i];
}

void launch_pull(void* dst, const void* src, size_t bytes, cudaStream_t st) {
  if (bytes == 0) return;
  const size_t words = bytes / 4, n4 = words / 4, n1 = words - n4 * 4;
  const size_t threads = n4 > n1 ? n4 : n1;
  pull_kernel<<<(unsigned int)((threads + 255) / 256), 256, 0, st>>>(reinterpret_cast<unsigned int*>(dst),
                                                                    reinterpret_cast<const unsigned int*>(src), n4, n1);
  note_launch();
}

// ------------------------------------------------------------------------------------------------------------
// frame_setup_kernel: the per-frame tables, built where the track counts live.  The host writes what it knows about the
// request (SceneReq, mapped pinned memory: read over PCIe by this kernel, no copy-engine transfer) and upper bounds for
// every buffer; the number of tracks each scene holds WHEN THIS FRAME RUNS (n_tracks, arena_top: left there by the previous
// frame's apply / sweep kernels) is joined in here: matrix offsets, column offsets, the tile list of the tensor-core
// kernel and the frame scalars.  One CTA: the tables are a few KB and three prefix sums.
constexpr int FS_T = 1024;

__global__ void __launch_bounds__(FS_T) frame_setup_kernel(Params p, TrackStore ts, Frame f, const SceneReq* req, int n_scenes,
                                                           const int* n_tracks, int mstep, int cstep, int dense_i,
                                                           TcTile* tiles, FrameDyn* dyn, int* zero, int n_zero) {
  constexpr int NQ = 6;   // scanned quantities: pos, vis, columns, tiles, weight sums, blocks
  __shared__ long long s_w[NQ][FS_T / 32];
  __shared__ long long s_carry[NQ];
  __shared__ unsigned long long s_red[3][FS_T / 32];
  __shared__ int s_maxn, s_maxrows;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  for (int i = tid; i < n_zero; i += FS_T) zero[i] = 0;
  // per-scene maximum of the valid visual distances starts at -1.0 (order-preserving u32 code of kernels_assign.cu: ~bits)
  if (f.scene_max) for (int i = tid; i < n_scenes; i += FS_T) f.scene_max[i] = ~__float_as_uint(-1.0f);
  if (tid < NQ) s_carry[tid] = 0;
  if (tid == 0) { s_maxn = 0; s_maxrows = 0; }
  const bool dense = dense_i != 0;
  __syncthreads();
  const int K = p.max_obs;
  unsigned long long u_mn = 0, u_rows = 0, live = 0;
  for (int base = 0; base < n_scenes; base += FS_T) {
    const int s = base + tid;
    SceneReq r;
    r.slot = 0; r.m = 0; r.det_base = 0; r.epoch = 0; r.scene_id = 0; r.pos_lbase = r.pos_lcap = r.vis_lbase = r.vis_lcap = 0;
    int n = 0, nb = 0, rows = 0;
    long long v[NQ] = {0, 0, 0, 0, 0, 0};
    int ctiles = 0;
    if (s < n_scenes) {
      r = req[s];
      n = n_tracks[r.slot];
      nb = (p.is_visual && ts.arena_top) ? ts.arena_top[r.slot] : 0;
      rows = nb * K;
      v[0] = (long long)r.m * n;
      v[1] = p.is_visual ? (long long)r.m * n * K : 0;
      ctiles = (rows + cstep - 1) / cstep;          // column tiles of the scene
      // screen: 128-padded columns (16-byte aligned bulk copies of 256-column slabs); dense: one 256-entry slab per tile
      v[2] = dense ? (long long)ctiles * 256 : ((long long)rows + 127) / 128 * 128;
      v[3] = mstep > 0 ? (long long)((r.m + mstep - 1) / mstep) * ctiles : 0;
      // dense kernel: the weight-sum matrix and the per-block arrays are padded to whole column tiles, so its epilogue
      // stores one record per block position of every tile without asking whether the block exists
      const int nbpad = dense ? ctiles * (cstep / (K > 0 ? K : 1)) : nb;
      v[4] = dense ? (long long)nbpad * ((r.m + 127) / 128 * 128) : 0;
      v[5] = nbpad;
      u_mn += (unsigned long long)v[0];
      u_rows += (unsigned long long)r.m * (unsigned long long)rows;
      live += (unsigned long long)n;
      atomicMax(&s_maxn, n);
      atomicMax(&s_maxrows, rows);
    }
    long long x[NQ];
#pragma unroll
    for (int q = 0; q < NQ; ++q) {
      x[q] = v[q];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const long long t = __shfl_up_sync(0xffffffffu, x[q], o);
        if (lane >= o) x[q] += t;
      }
      if (lane == 31) s_w[q][wid] = x[q];
    }
    __syncthreads();
    long long ex[NQ];
#pragma unroll
    for (int q = 0; q < NQ; ++q) {
      long long woff = 0;
      for (int w = 0; w < wid; ++w) woff += s_w[q][w];
      ex[q] = s_carry[q] + woff + x[q] - v[q];
    }
    __syncthreads();
    if (tid == FS_T - 1) {
#pragma unroll
      for (int q = 0; q < NQ; ++q) s_carry[q] = ex[q] + v[q];
    }
    if (s < n_scenes) {
      SceneDesc d;
      d.slot = r.slot; d.m = r.m; d.n = n; d.det_base = r.det_base;
      d.pos_off = ex[0]; d.vis_off = ex[1];
      d.epoch = r.epoch; d.col_off = (int)ex[2]; d.scene_id = r.scene_id;
      d.pos_lbase = r.pos_lbase; d.pos_lcap = r.pos_lcap; d.vis_lbase = r.vis_lbase; d.vis_lcap = r.vis_lcap;
      d.nb = nb; d.pad0 = 0;
      d.ws_off = ex[4]; d.blk_off = (int)ex[5]; d.slab_off = dense ? (int)(ex[2] / 256) : 0;
      f.scenes[s] = d;
      if (mstep > 0 && tiles) {
        int k = (int)ex[3];
        for (int m0 = 0; m0 < r.m; m0 += mstep)
          for (int j = 0; j < ctiles; ++j) { TcTile t; t.scene = s; t.m0 = m0; t.c0 = j * cstep; t.pad = j; tiles[k++] = t; }
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    u_mn += __shfl_xor_sync(0xffffffffu, u_mn, o);
    u_rows += __shfl_xor_sync(0xffffffffu, u_rows, o);
    live += __shfl_xor_sync(0xffffffffu, live, o);
  }
  if (lane == 0) { s_red[0][wid] = u_mn; s_red[1][wid] = u_rows; s_red[2][wid] = live; }
  __syncthreads();
  if (tid == 0) {
    unsigned long long a = 0, b = 0, c = 0;
    for (int w = 0; w < FS_T / 32; ++w) { a += s_red[0][w]; b += s_red[1][w]; c += s_red[2][w]; }
    FrameDyn d;
    d.n_tiles = (int)s_carry[3]; d.total_cols = (int)s_carry[2]; d.max_rows = s_maxrows; d.max_n = s_maxn;
    d.pos_total = s_carry[0]; d.vis_total = s_carry[1];
    d.units_mn = a; d.units_rows = b; d.live_total = (long long)c;
    d.ws_total = s_carry[4]; d.blk_total = (int)s_carry[5]; d.dense_scenes = 0;
    *dyn = d;
  }
}

void launch_frame_setup(const Params& p, const TrackStore& ts, const Frame& f, const SceneReq* req, int n_scenes,
                        const int* d_n_tracks, int mstep, int cstep, bool dense, TcTile* tiles, FrameDyn* dyn, int* zero,
                        int n_zero, cudaStream_t st) {
  frame_setup_kernel<<<1, FS_T, 0, st>>>(p, ts, f, req, n_scenes, d_n_tracks, mstep, cstep > 0 ? cstep : 256, dense ? 1 : 0, tiles,
                                         dyn, zero, n_zero);
  note_launch();
}

}  // namespace sb
