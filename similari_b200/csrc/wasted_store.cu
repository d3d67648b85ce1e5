// wasted_store.cu -- sb200_fstore_associate_wasted: the wasted records of a visual tracker associated with a feature
// track store, their feature histories read on the device where the tracker keeps them (DESIGN.md §3d.4).
// The host reads back only the records (as sb200_wasted_history does) and one present count per record; the request rows
// of the store call are written from the tracker's history pool by ws_stage_kernel, on the store's stream, and the
// records leave the wasted buffer only once the store's work is complete.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <vector>

#include "../../include/similari_b200.h"
#include "sb_engine.cuh"
#include "sb_host.cuh"
#include "sb_wstore.cuh"

using sb::fail;

namespace sb {

// One warp per record: the present bytes of its kept history (its newest min(length, H) observations, H <= 64) as a
// chronological mask (bit c: entry c, oldest first) and their count.
__global__ void ws_count_kernel(const int* __restrict__ hblk, const unsigned int* __restrict__ length,
                                const unsigned char* __restrict__ hpresent, int H, int n,
                                unsigned long long* __restrict__ mask, int* __restrict__ count) {
  const long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (i >= n) return;
  const unsigned int len = length[i], nk = min(len, (unsigned int)H);
  const size_t b = (size_t)hblk[i] * H;
  bool p[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const unsigned int c = (unsigned int)(h * 32 + lane);
    p[h] = c < nk && hpresent[b + (len - nk + c) % (unsigned int)H] != 0;
  }
  const unsigned int lo = __ballot_sync(0xffffffffu, p[0]), hi = __ballot_sync(0xffffffffu, p[1]);
  if (lane == 0) {
    mask[i] = (unsigned long long)hi << 32 | lo;
    count[i] = __popc(lo) + __popc(hi);
  }
}

// One warp per request row r of the store call: query q = row_q[r] is record qrec[q], whose kept rows are its newest
// qoff[q + 1] - qoff[q] present entries.  The row's entry is found by rank-select in the record's mask, then copied
// from the pool with 16-byte accesses; the lanes from D on are written as zero (the store's padding).
__global__ void ws_stage_kernel(const float* __restrict__ hrows, const int* __restrict__ hblk,
                                const unsigned int* __restrict__ length, int H, int d8, int D,
                                const unsigned long long* __restrict__ mask, const int* __restrict__ count,
                                const int* __restrict__ qrec, const int* __restrict__ qoff,
                                const int* __restrict__ row_q, int R, float* __restrict__ rows) {
  const long long r = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= R) return;
  const int q = row_q[r], i = qrec[q];
  const int rank = count[i] - (qoff[q + 1] - qoff[q]) + ((int)r - qoff[q]);   // among the present entries, oldest first
  unsigned long long m = mask[i];
  for (int k = 0; k < rank; ++k) m &= m - 1;
  const unsigned int c = (unsigned int)(__ffsll((long long)m) - 1);
  const unsigned int len = length[i], nk = min(len, (unsigned int)H);
  const size_t row = (size_t)hblk[i] * H + (len - nk + c) % (unsigned int)H;
  const float4* s4 = reinterpret_cast<const float4*>(hrows + row * d8);
  float4* d4 = reinterpret_cast<float4*>(rows + (size_t)r * d8);
  for (int k = lane; k < (d8 >> 2); k += 32) {
    float4 v = s4[k];
    const int e = 4 * k;
    if (e + 0 >= D) v.x = 0.0f;
    if (e + 1 >= D) v.y = 0.0f;
    if (e + 2 >= D) v.z = 0.0f;
    if (e + 3 >= D) v.w = 0.0f;
    d4[k] = v;
  }
}

// what ws_stage_kernel reads besides the store call's own tables
struct StageCtx {
  sb::WastedFeatures f;
  int D;
  const unsigned long long* mask;
  const int* count;
  int* d_qrec;
  const std::vector<int>* qrec;
};

int stage_rows(void* ctx, float* rows, const int* qoff, const int* row_q, int R, cudaStream_t st) {
  const StageCtx& c = *static_cast<const StageCtx*>(ctx);
  CU(cudaMemcpyAsync(c.d_qrec, c.qrec->data(), c.qrec->size() * 4, cudaMemcpyHostToDevice, st));
  const long long threads = (long long)R * 32;
  ws_stage_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(c.f.hrows, c.f.hblk, c.f.length, c.f.H, c.f.d8, c.D,
                                                                      c.mask, c.count, c.d_qrec, qoff, row_q, R, rows);
  sb::note_launch();
  CU(cudaGetLastError());
  return 0;
}

}  // namespace sb

extern "C" {

int64_t sb200_fstore_associate_wasted(sb200_fstore* s, sb200_tracker* t, int64_t cap, uint64_t id_offset, uint64_t* ids,
                                      uint64_t* scene_ids, uint32_t* epochs, uint32_t* lengths, float* predicted_boxes,
                                      float* observed_boxes, int32_t history_cap, float* predicted_history,
                                      float* observed_history, int32_t* history_counts, int32_t* feature_counts,
                                      uint8_t* queried, int32_t* counts, uint64_t* winners, double* weights,
                                      uint64_t* track_ids, uint8_t* merged) {
  if (!s || !t) return fail(SB200_ERR_INVALID, "store / tracker is NULL");
  if (cap < 0 || history_cap < 0) return fail(SB200_ERR_INVALID, "cap < 0 or history_cap < 0");
  if (sb::fstore_gate(s))
    return fail(SB200_ERR_INVALID, "associate_wasted needs an ungated store: a wasted record has no exact window (the "
                                   "tracker keeps no birth epoch)");
  if (sb::fstore_retention(s))
    return fail(SB200_ERR_INVALID, "associate_wasted needs a store that keeps its newest observations: the tracker's "
                                   "feature history keeps no quality");
  const sb::TrackerFeatureInfo ti = sb::tracker_feature_info(t);
  if (!ti.visual) return fail(SB200_ERR_INVALID, "the tracker is not a visual tracker");
  if (!ti.history) return fail(SB200_ERR_INVALID, "the tracker's feature history is off (sb200_set_feature_history)");
  int sdev = 0, sdim = 0, topn = 0;
  sb::fstore_info(s, &sdev, &sdim, &topn);
  if (sdev != ti.device)
    return fail(SB200_ERR_INVALID, "the tracker is on device %d and the store on device %d", ti.device, sdev);
  if (ti.dim_fixed && ti.feature_dim != sdim)
    return fail(SB200_ERR_INVALID, "feature_dim differs: %d in the tracker, %d in the store", ti.feature_dim, sdim);
  // the collection point, and the records read back; they stay in the wasted buffer until the store is done
  std::vector<uint64_t> rid;
  sb::WastedFeatures wf{};
  const int64_t n = sb::tracker_collect_wasted(t, cap, {ids, scene_ids, epochs, lengths, predicted_boxes, observed_boxes,
                                                        history_cap, predicted_history, observed_history, history_counts},
                                               &rid, &wf);
  if (n <= 0) return n;
  // present entries of every record: n x 4 bytes come back, the rows stay where they are
  sb::DBuf scratch;
  if (int rc = scratch.ensure((size_t)n * 16)) return rc;
  unsigned long long* d_mask = scratch.as<unsigned long long>();
  int* d_count = reinterpret_cast<int*>(d_mask + n);
  int* d_qrec = d_count + n;
  sb::ws_count_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, wf.st>>>(wf.hblk, wf.length, wf.hpresent, wf.H, (int)n,
                                                                        d_mask, d_count);
  sb::note_launch();
  CU(cudaGetLastError());
  std::vector<int> pc((size_t)n);
  CU(cudaMemcpyAsync(pc.data(), d_count, 4 * (size_t)n, cudaMemcpyDeviceToHost, wf.st));
  CU(cudaStreamSynchronize(wf.st));
  // the queried records: ids + id_offset, their present rows as the CSR of one associate call
  std::vector<int> qrec;
  std::vector<uint64_t> qid;
  std::vector<int32_t> offs(1, 0);
  for (int64_t i = 0; i < n; ++i) {
    if (pc[(size_t)i] == 0) continue;
    qrec.push_back((int)i);
    qid.push_back(rid[(size_t)i] + id_offset);
    offs.push_back(offs.back() + pc[(size_t)i]);
  }
  const int Q = (int)qrec.size();
  std::vector<int32_t> qc(Q);
  std::vector<uint64_t> qw((size_t)Q * topn), qt(Q);
  std::vector<double> qwt((size_t)Q * topn);
  std::vector<uint8_t> qm(Q);
  if (Q > 0) {
    sb::StageCtx ctx{wf, sdim, d_mask, d_count, d_qrec, &qrec};
    // returns once the store's stream has finished, so no kernel reads the records' blocks after this point
    if (int rc = sb::fstore_associate_rows(s, Q, qid.data(), offs.data(), {sb::stage_rows, &ctx}, qc.data(), qw.data(),
                                           qwt.data(), qt.data(), qm.data()))
      return rc;
  }
  for (int64_t i = 0, q = 0; i < n; ++i) {
    const bool on = q < Q && qrec[(size_t)q] == (int)i;
    if (feature_counts) feature_counts[i] = pc[(size_t)i];
    if (queried) queried[i] = on ? 1 : 0;
    if (counts) counts[i] = on ? qc[(size_t)q] : 0;
    if (track_ids) track_ids[i] = on ? qt[(size_t)q] : 0;
    if (merged) merged[i] = on ? qm[(size_t)q] : 0;
    for (int e = 0; e < topn; ++e) {
      if (winners) winners[(size_t)i * topn + e] = on ? qw[(size_t)q * topn + e] : 0;
      if (weights) weights[(size_t)i * topn + e] = on ? qwt[(size_t)q * topn + e] : 0.0;
    }
    if (on) ++q;
  }
  if (int rc = sb::tracker_drop_wasted(t, n)) return rc;   // the records' history blocks go back to the pool
  return n;
}

}  // extern "C"
