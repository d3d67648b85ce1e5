// sb_wstore.cuh -- the internal interfaces behind sb200_fstore_associate_wasted (wasted_store.cu): what that call needs of
// a visual tracker (engine.cu) and of a feature track store (fstore.cu).  Host code; each handle stays opaque outside
// its own file.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <vector>

#include "../../include/similari_b200.h"

namespace sb {

// ---- tracker side (engine.cu)
struct TrackerFeatureInfo {
  int device;
  bool visual, history;   // a visual tracker; its feature history is on (sb200_set_feature_history)
  int feature_dim;
  bool dim_fixed;         // a request has carried features (the dimension can no longer change)
};
TrackerFeatureInfo tracker_feature_info(sb200_tracker* t);

// The record outputs of sb200_wasted_history; every pointer may be NULL.
struct WastedOut {
  uint64_t* ids;
  uint64_t* scene_ids;
  uint32_t* epochs;
  uint32_t* lengths;
  float* predicted_boxes;
  float* observed_boxes;
  int32_t history_cap;
  float* predicted_history;
  float* observed_history;
  int32_t* history_counts;
};

// Where the feature histories of collected records lie (tracker with the feature history on): record i of the wasted
// buffer has history block hblk[i] and length[i] observations; observation number j of block b is row b * H + j % H of
// hrows ([.][d8] f32, zero-padded from feature_dim) and hpresent.  Valid until tracker_drop_wasted.  `st` is the
// tracker's work stream, idle when tracker_collect_wasted returns.
struct WastedFeatures {
  const int* hblk;
  const unsigned int* length;
  const float* hrows;
  const unsigned char* hpresent;
  int H, d8;
  cudaStream_t st;
};

// A collection point (drain, then the auto-waste step) and the read-back of the first min(cap, wasted count) records as
// sb200_wasted_history reads them, their ids also into ids[] (host, room for them sized here).  The records stay in
// the buffer.  Returns their number or a negative status.
int64_t tracker_collect_wasted(sb200_tracker* t, int64_t cap, const WastedOut& out, std::vector<uint64_t>* ids,
                               WastedFeatures* feat);
// The end of a collection: takes the first n records out of the wasted buffer and returns their history blocks to the
// pool.  The caller has finished every read of those blocks.
int tracker_drop_wasted(sb200_tracker* t, int64_t n);

// ---- store side (fstore.cu)
void fstore_info(sb200_fstore* s, int* device, int* feature_dim, int* topn);
// the store's gate rule (SB200_FSTORE_GATE_*); a gated store refuses associate_wasted
int fstore_gate(sb200_fstore* s);
// the store's retention rule (SB200_FSTORE_KEEP_*); a quality store refuses associate_wasted
int fstore_retention(sb200_fstore* s);

// Writes the request rows of a store call on the store's stream `st`: rows[R][d8] f32 (zero-padded from feature_dim),
// request row r holding observation r - qoff[q] of the rows query q = row_q[r] keeps (its newest max_observations,
// oldest first).  qoff / row_q / rows are device pointers of the call.  Returns 0 or a negative status.
struct FsRowSource {
  int (*fill)(void* ctx, float* rows, const int* qoff, const int* row_q, int R, cudaStream_t st);
  void* ctx;
};

// sb200_fstore_associate of Q queries, query q with offs[q + 1] - offs[q] >= 1 rows, written on the device by `src`.
// Checks (ids, pair bound), outputs and store changes as there; every rejection comes before the store changes.
int fstore_associate_rows(sb200_fstore* s, int Q, const uint64_t* qids, const int32_t* offs, const FsRowSource& src,
                          int32_t* counts, uint64_t* winners, double* weights, uint64_t* track_ids, uint8_t* merged);

}  // namespace sb
