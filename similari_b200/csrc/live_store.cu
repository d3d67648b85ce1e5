// live_store.cu -- the live tracks of a visual tracker read where the tracker keeps them (DESIGN.md §3d.10):
// sb200_scene_observations, the read-back of Track::obs, and sb200_fstore_search_tracks, which searches a feature track
// store with the present observations of live tracks.  For a search the host reads back only an index and a present count
// per pair (and, on a quality store, the present rows' qualities); the request rows of the store call are written from
// the tracker's f32 arena by ls_stage_kernel on the store's stream.  Neither call changes the tracker or the store.
#include <cuda_runtime.h>

#include <algorithm>
#include <climits>
#include <cstring>
#include <utility>
#include <vector>

#include "../../include/similari_b200.h"
#include "sb_engine.cuh"
#include "sb_host.cuh"
#include "sb_wstore.cuh"

using sb::fail;

namespace sb {

// One warp per (track i, logical observation j) of a scene whose live tracks start at store index `base`: the track's id
// and n_obs (j == 0), the observation's present byte and quality, and its feature row trimmed to D; zeros where the
// observation has no feature and past n_obs.
__global__ void ls_gather_kernel(LiveTracks lt, long long base, int n, int D, unsigned long long* __restrict__ ids,
                                 int* __restrict__ n_obs, unsigned char* __restrict__ hasf, float* __restrict__ q,
                                 float* __restrict__ feats) {
  const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31, K = lt.K;
  if (w >= (long long)n * K) return;
  const int i = (int)(w / K), j = (int)(w % K);
  const size_t idx = (size_t)(base + i);
  const int on = lt.obs_n[idx];
  const bool live = j < on, has = live && lt.obs_hasf[idx * K + j] != 0;
  if (lane == 0) {
    if (j == 0) {
      ids[i] = lt.id[idx];
      n_obs[i] = on;
    }
    hasf[w] = has ? 1 : 0;
    q[w] = live ? lt.obs_q[idx * K + j] : 0.0f;
  }
  const float* src = lt.feat + ((size_t)(base + lt.fblk[idx]) * K + (has ? lt.obs_phys[idx * K + j] : 0)) * lt.d8;
  float* dst = feats + (size_t)w * D;
  for (int k = lane; k < D; k += 32) dst[k] = has ? src[k] : 0.0f;
}

// One pair of sb200_fstore_search_tracks as the lookup reads it: track `want` among the n_tracks live tracks from `base`
struct LsPair {
  long long base;   // -1: no such scene
  unsigned long long want;
  int n_tracks, pad;
};

// One warp per pair i: the position of its track among the scene's live tracks (-1: not live) and the number of its
// present observations (look[i]), and their logical positions as a mask (bit j: obs_hasf[idx][j], j < obs_n[idx]).
__global__ void ls_lookup_kernel(LiveTracks lt, const LsPair* __restrict__ pairs, int n, int2* __restrict__ look,
                                 unsigned int* __restrict__ mask) {
  const long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (i >= n) return;
  const LsPair p = pairs[i];
  int at = -1;
  for (int k = 0; p.base >= 0 && k < p.n_tracks; k += 32) {
    const int j = k + lane;
    const unsigned int hit = __ballot_sync(0xffffffffu, j < p.n_tracks && lt.id[p.base + j] == p.want);
    if (hit) {
      at = k + __ffs(hit) - 1;
      break;
    }
  }
  unsigned int m = 0;
  if (at >= 0) {
    const size_t idx = (size_t)(p.base + at);
    m = __ballot_sync(0xffffffffu, lane < lt.obs_n[idx] && lt.obs_hasf[idx * lt.K + lane] != 0);
  }
  if (lane == 0) {
    look[i] = make_int2(at, __popc(m));
    mask[i] = m;
  }
}

// One warp per queried pair q = pairs[qpair[q]]: the qualities of its present observations, in logical order, at
// out[poff[q] ..) (a quality store's row qualities).
__global__ void ls_quality_kernel(LiveTracks lt, const LsPair* __restrict__ pairs, const int2* __restrict__ look,
                                  const unsigned int* __restrict__ mask, const int* __restrict__ qpair,
                                  const int* __restrict__ poff, int Q, float* __restrict__ out) {
  const long long q = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (q >= Q) return;
  const int i = qpair[q];
  const unsigned int m = mask[i];
  if (m >> lane & 1u) {
    const size_t idx = (size_t)(pairs[i].base + look[i].x);
    out[poff[q] + __popc(m & ((1u << lane) - 1u))] = lt.obs_q[idx * lt.K + lane];
  }
}

// One warp per request row r of the store call: query q = row_q[r] is pair qpair[q], and the row is its present
// observation number row_table[r] - poff[q] (in logical order), found by rank-select in the pair's mask.  The arena row
// is copied with 16-byte accesses; the lanes from D on are written as zero (the store's padding).
__global__ void ls_stage_kernel(LiveTracks lt, const LsPair* __restrict__ pairs, const int2* __restrict__ look,
                                const unsigned int* __restrict__ mask, const int* __restrict__ qpair,
                                const int* __restrict__ poff, const int* __restrict__ row_table,
                                const int* __restrict__ row_q, int R, int D, float* __restrict__ rows) {
  const long long r = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= R) return;
  const int q = row_q[r], i = qpair[q];
  unsigned int m = mask[i];
  for (int k = row_table[r] - poff[q]; k > 0; --k) m &= m - 1;
  const int j = __ffs(m) - 1;
  const long long base = pairs[i].base;
  const size_t idx = (size_t)(base + look[i].x);
  const size_t row = (size_t)(base + lt.fblk[idx]) * lt.K + lt.obs_phys[idx * lt.K + j];
  const float4* s4 = reinterpret_cast<const float4*>(lt.feat + row * lt.d8);
  float4* d4 = reinterpret_cast<float4*>(rows + (size_t)r * lt.d8);
  for (int k = lane; k < (lt.d8 >> 2); k += 32) {
    float4 v = s4[k];
    const int e = 4 * k;
    if (e + 0 >= D) v.x = 0.0f;
    if (e + 1 >= D) v.y = 0.0f;
    if (e + 2 >= D) v.z = 0.0f;
    if (e + 3 >= D) v.w = 0.0f;
    d4[k] = v;
  }
}

static unsigned blocks_of_warps(long long warps) { return (unsigned)((warps * 32 + 255) / 256); }

// what ls_stage_kernel reads besides the store call's own tables
struct LiveCtx {
  LiveTracks lt;
  const LsPair* pairs;
  const int2* look;
  const unsigned int* mask;
  const int* qpair;
  const int* poff;
  int* d_table;
  const std::vector<int>* table;
};

static int stage_live_rows(void* ctx, float* rows, const int* qoff, const int* row_q, int R, cudaStream_t st) {
  (void)qoff;
  const LiveCtx& c = *static_cast<const LiveCtx*>(ctx);
  CU(cudaMemcpyAsync(c.d_table, c.table->data(), (size_t)R * 4, cudaMemcpyHostToDevice, st));
  ls_stage_kernel<<<blocks_of_warps(R), 256, 0, st>>>(c.lt, c.pairs, c.look, c.mask, c.qpair, c.poff, c.d_table, row_q,
                                                       R, c.lt.feature_dim, rows);
  sb::note_launch();
  CU(cudaGetLastError());
  return 0;
}

static size_t align16(size_t v) { return (v + 15) & ~size_t(15); }

}  // namespace sb

extern "C" {

int64_t sb200_scene_observations(sb200_tracker* t, uint64_t scene_id, int64_t cap, uint64_t* ids, int32_t* n_obs,
                                 uint8_t* has_feature, float* quality, float* features) {
  if (!t) return fail(SB200_ERR_INVALID, "tracker is NULL");
  if (cap < 0) return fail(SB200_ERR_INVALID, "cap < 0");
  if (!sb::tracker_feature_info(t).visual) return fail(SB200_ERR_INVALID, "the tracker is not a visual tracker");
  sb::LiveTracks lt{};
  std::vector<sb::LiveScene> sc;
  if (int rc = sb::tracker_live(t, 1, &scene_id, &lt, &sc)) return rc;
  const int n = (int)std::min<int64_t>(cap, sc[0].n_tracks);
  if (n <= 0) return 0;
  // one staging buffer, one copy down: ids [n], n_obs [n], has_feature [n][K], quality [n][K], features [n][K][D]
  const size_t K = (size_t)lt.K, D = (size_t)lt.feature_dim;
  const size_t o_obs = sb::align16((size_t)n * 8), o_hf = sb::align16(o_obs + (size_t)n * 4);
  const size_t o_q = sb::align16(o_hf + n * K), o_f = sb::align16(o_q + n * K * 4), total = o_f + n * K * D * 4;
  sb::DBuf buf;
  if (int rc = buf.ensure(total)) return rc;
  char* d = buf.as<char>();
  sb::ls_gather_kernel<<<sb::blocks_of_warps((long long)n * lt.K), 256, 0, lt.st>>>(
      lt, sc[0].base, n, (int)D, reinterpret_cast<unsigned long long*>(d), reinterpret_cast<int*>(d + o_obs),
      reinterpret_cast<unsigned char*>(d + o_hf), reinterpret_cast<float*>(d + o_q), reinterpret_cast<float*>(d + o_f));
  sb::note_launch();
  CU(cudaGetLastError());
  std::vector<char> h(total);
  CU(cudaMemcpyAsync(h.data(), d, total, cudaMemcpyDeviceToHost, lt.st));
  CU(cudaStreamSynchronize(lt.st));
  if (ids) memcpy(ids, h.data(), (size_t)n * 8);
  if (n_obs) memcpy(n_obs, h.data() + o_obs, (size_t)n * 4);
  if (has_feature) memcpy(has_feature, h.data() + o_hf, n * K);
  if (quality) memcpy(quality, h.data() + o_q, n * K * 4);
  if (features) memcpy(features, h.data() + o_f, n * K * D * 4);
  return n;
}

int sb200_fstore_search_tracks(sb200_fstore* s, sb200_tracker* t, int32_t n, const uint64_t* scene_ids,
                               const uint64_t* track_ids, uint64_t id_offset, const sb200_fstore_attrs* attrs,
                               uint8_t* found, int32_t* feature_counts, uint8_t* queried, int32_t* counts,
                               uint64_t* winners, double* weights) {
  if (!s || !t) return fail(SB200_ERR_INVALID, "store / tracker is NULL");
  if (n < 0) return fail(SB200_ERR_INVALID, "n < 0");
  if (n > 0 && (!scene_ids || !track_ids)) return fail(SB200_ERR_INVALID, "scene_ids / track_ids is NULL");
  const sb::TrackerFeatureInfo ti = sb::tracker_feature_info(t);
  if (!ti.visual) return fail(SB200_ERR_INVALID, "the tracker is not a visual tracker");
  int sdev = 0, sdim = 0, topn = 0;
  sb::fstore_info(s, &sdev, &sdim, &topn);
  if (sdev != ti.device)
    return fail(SB200_ERR_INVALID, "the tracker is on device %d and the store on device %d", ti.device, sdev);
  if (ti.dim_fixed && ti.feature_dim != sdim)
    return fail(SB200_ERR_INVALID, "feature_dim differs: %d in the tracker, %d in the store", ti.feature_dim, sdim);
  const bool gated = sb::fstore_gate(s) != SB200_FSTORE_GATE_NONE, keep = sb::fstore_retention(s) != 0;
  if (gated && !attrs)
    return fail(SB200_ERR_INVALID, "the store is gated: attrs needs a source and a window per pair");
  if (!gated && attrs) return fail(SB200_ERR_INVALID, "attrs must be NULL on an ungated store");
  if (gated)
    if (int rc = sb::fstore_check_attrs(s, n, attrs)) return rc;
  {
    std::vector<std::pair<uint64_t, uint64_t>> pairs((size_t)n);   // (scene, id), sorted: a repeated pair is adjacent
    for (int i = 0; i < n; ++i) pairs[(size_t)i] = {scene_ids[i], track_ids[i]};
    std::sort(pairs.begin(), pairs.end());
    for (int i = 1; i < n; ++i)
      if (pairs[(size_t)i] == pairs[(size_t)i - 1])
        return fail(SB200_ERR_INVALID, "track %llu of scene %llu appears twice in the call",
                    (unsigned long long)pairs[(size_t)i].second, (unsigned long long)pairs[(size_t)i].first);
  }
  sb::LiveTracks lt{};
  std::vector<sb::LiveScene> sc;
  if (int rc = sb::tracker_live(t, n, scene_ids, &lt, &sc)) return rc;
  // lookup: n x 8 bytes come back, the rows stay where they are
  std::vector<sb::LsPair> hp((size_t)n);
  for (int i = 0; i < n; ++i) hp[(size_t)i] = {sc[(size_t)i].base, track_ids[i], sc[(size_t)i].n_tracks, 0};
  std::vector<int2> look((size_t)n);
  const size_t o_look = sb::align16((size_t)n * sizeof(sb::LsPair)), o_mask = sb::align16(o_look + (size_t)n * 8);
  const size_t o_qpair = sb::align16(o_mask + (size_t)n * 4), o_poff = sb::align16(o_qpair + (size_t)n * 4);
  const size_t o_end = sb::align16(o_poff + ((size_t)n + 1) * 4);
  sb::DBuf scratch, rowbuf;
  char* d = nullptr;
  if (n > 0) {
    if (int rc = scratch.ensure(o_end)) return rc;
    d = scratch.as<char>();
    CU(cudaMemcpyAsync(d, hp.data(), (size_t)n * sizeof(sb::LsPair), cudaMemcpyHostToDevice, lt.st));
    sb::ls_lookup_kernel<<<sb::blocks_of_warps(n), 256, 0, lt.st>>>(
        lt, reinterpret_cast<const sb::LsPair*>(d), n, reinterpret_cast<int2*>(d + o_look),
        reinterpret_cast<unsigned int*>(d + o_mask));
    sb::note_launch();
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(look.data(), d + o_look, (size_t)n * 8, cudaMemcpyDeviceToHost, lt.st));
    CU(cudaStreamSynchronize(lt.st));
  }
  // the queried pairs: track id + id_offset, their present rows (in logical order) as the CSR of one search call
  std::vector<int> qpair;
  std::vector<uint64_t> qid, qsrc;
  std::vector<int64_t> qt0, qt1;
  std::vector<int32_t> offs(1, 0);
  long long rows = 0;
  for (int i = 0; i < n; ++i) {
    if (look[(size_t)i].y == 0) continue;
    rows += look[(size_t)i].y;
    if (rows > INT_MAX) return fail(SB200_ERR_CAPACITY, "the call holds more than 2^31 - 1 observations");
    qpair.push_back(i);
    qid.push_back(track_ids[i] + id_offset);
    offs.push_back((int32_t)rows);
    if (gated) {
      qsrc.push_back(attrs->source[i]);
      qt0.push_back(attrs->t_start[i]);
      qt1.push_back(attrs->t_end[i]);
    }
  }
  const int Q = (int)qpair.size();
  std::vector<float> rq;
  if (Q > 0) {
    if (int rc = rowbuf.ensure((size_t)rows * 4)) return rc;   // the row table, and first the qualities
    CU(cudaMemcpyAsync(d + o_qpair, qpair.data(), (size_t)Q * 4, cudaMemcpyHostToDevice, lt.st));
    CU(cudaMemcpyAsync(d + o_poff, offs.data(), ((size_t)Q + 1) * 4, cudaMemcpyHostToDevice, lt.st));
    if (keep) {
      rq.resize((size_t)rows);
      sb::ls_quality_kernel<<<sb::blocks_of_warps(Q), 256, 0, lt.st>>>(
          lt, reinterpret_cast<const sb::LsPair*>(d), reinterpret_cast<const int2*>(d + o_look),
          reinterpret_cast<const unsigned int*>(d + o_mask), reinterpret_cast<const int*>(d + o_qpair),
          reinterpret_cast<const int*>(d + o_poff), Q, rowbuf.as<float>());
      sb::note_launch();
      CU(cudaGetLastError());
      CU(cudaMemcpyAsync(rq.data(), rowbuf.p, (size_t)rows * 4, cudaMemcpyDeviceToHost, lt.st));
    }
    CU(cudaStreamSynchronize(lt.st));   // the tracker's stream is idle before the store's reads the arena
  }
  std::vector<int32_t> qc((size_t)Q);
  std::vector<uint64_t> qw((size_t)Q * topn);
  std::vector<double> qwt((size_t)Q * topn);
  std::vector<int> table;
  const sb200_fstore_attrs qa{qsrc.data(), qt0.data(), qt1.data()};
  sb::LiveCtx ctx{lt,
                  reinterpret_cast<const sb::LsPair*>(d),
                  reinterpret_cast<const int2*>(d + o_look),
                  reinterpret_cast<const unsigned int*>(d + o_mask),
                  reinterpret_cast<const int*>(d + o_qpair),
                  reinterpret_cast<const int*>(d + o_poff),
                  rowbuf.as<int>(),
                  &table};
  // returns once the store's stream has finished, so no kernel reads the arena after this point
  if (int rc = sb::fstore_search_rows(s, Q, qid.data(), offs.data(), keep ? rq.data() : nullptr, gated ? &qa : nullptr,
                                      {sb::stage_live_rows, &ctx}, &table, qc.data(), qw.data(), qwt.data()))
    return rc;
  for (int i = 0, q = 0; i < n; ++i) {
    const bool on = q < Q && qpair[(size_t)q] == i;
    if (found) found[i] = look[(size_t)i].x >= 0 ? 1 : 0;
    if (feature_counts) feature_counts[i] = look[(size_t)i].y;
    if (queried) queried[i] = on ? 1 : 0;
    if (counts) counts[i] = on ? qc[(size_t)q] : 0;
    for (int e = 0; e < topn; ++e) {
      if (winners) winners[(size_t)i * topn + e] = on ? qw[(size_t)q * topn + e] : 0;
      if (weights) weights[(size_t)i * topn + e] = on ? qwt[(size_t)q * topn + e] : 0.0;
    }
    if (on) ++q;
  }
  return 0;
}

}  // extern "C"
