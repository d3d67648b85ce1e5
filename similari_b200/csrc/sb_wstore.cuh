// sb_wstore.cuh -- the internal interfaces behind sb200_fstore_associate_wasted (wasted_store.cu) and the live-track calls
// (live_store.cu): what those calls need of a visual tracker (engine.cu) and of a feature track store (fstore.cu).  Host
// code; each handle stays opaque outside its own file.
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

// Where a visual tracker keeps Track::obs of its live tracks (sb200_scene_observations, sb200_fstore_search_tracks,
// live_store.cu): the TrackStore columns.  The live tracks of a scene are the store indices [base, base + n_tracks) of
// its slot (base = slot * track_cap); logical observation j < obs_n[idx] of track idx has the present byte
// obs_hasf[idx * K + j], the quality obs_q[idx * K + j] and the f32 row (base + fblk[idx]) * K + obs_phys[idx * K + j]
// of feat ([.][d8], zero-padded from feature_dim).  `st` is the tracker's work stream, idle when tracker_live returns.
struct LiveTracks {
  const unsigned long long* id;
  const int* fblk;
  const unsigned char* obs_phys;
  const unsigned char* obs_hasf;
  const unsigned char* obs_n;
  const float* obs_q;
  const float* feat;
  int track_cap, K, d8, feature_dim;
  cudaStream_t st;
};
struct LiveScene {
  long long base;   // -1: the tracker holds no such scene
  int n_tracks;
};
// A query point of a visual tracker (a drain; no auto-waste step, nothing changes): the columns, and the slot of each of
// the n scene ids.  Valid until the next call that enqueues a frame or changes the tracker.
int tracker_live(sb200_tracker* t, int n, const uint64_t* scene_ids, LiveTracks* lt, std::vector<LiveScene>* scenes);

// ---- store side (fstore.cu)
void fstore_info(sb200_fstore* s, int* device, int* feature_dim, int* topn);
// the store's gate rule (SB200_FSTORE_GATE_*); a gated store refuses associate_wasted
int fstore_gate(sb200_fstore* s);
// the store's retention rule (SB200_FSTORE_KEEP_*); a quality store refuses associate_wasted
int fstore_retention(sb200_fstore* s);

// Writes the request rows of a store call on the store's stream `st`: rows[R][d8] f32 (zero-padded from feature_dim),
// request row r holding observation r - qoff[q] of the rows query q = row_q[r] keeps (associate: its newest
// max_observations, oldest first; fstore_search_rows: the rows its row table names).  qoff / row_q / rows are device
// pointers of the call.  Returns 0 or a negative status.
struct FsRowSource {
  int (*fill)(void* ctx, float* rows, const int* qoff, const int* row_q, int R, cudaStream_t st);
  void* ctx;
};

// sb200_fstore_associate of Q queries, query q with offs[q + 1] - offs[q] >= 1 rows, written on the device by `src`.
// Checks (ids, pair bound), outputs and store changes as there; every rejection comes before the store changes.
int fstore_associate_rows(sb200_fstore* s, int Q, const uint64_t* qids, const int32_t* offs, const FsRowSource& src,
                          int32_t* counts, uint64_t* winners, double* weights, uint64_t* track_ids, uint8_t* merged);

// The checks of sb200_fstore_search_attr's triples for n queries (a gated store; columns present; t_start <= t_end).
int fstore_check_attrs(sb200_fstore* s, int n, const sb200_fstore_attrs* attrs);

// sb200_fstore_search of Q queries, query q with offs[q + 1] - offs[q] >= 1 rows written on the device by `src`; on a
// quality store sb200_fstore_search_quality with quality[offs[Q]] the rows' qualities (a NaN is refused here), on a gated
// store the _attr form with `attrs` (checked by the caller).  The store's query rule picks the request rows: request row
// r is row (*row_table)[r] of the call, set before src.fill runs.  Checks (ids, pair bound) and outputs as there.
int fstore_search_rows(sb200_fstore* s, int Q, const uint64_t* qids, const int32_t* offs, const float* quality,
                       const sb200_fstore_attrs* attrs, const FsRowSource& src, std::vector<int>* row_table,
                       int32_t* counts, uint64_t* winners, double* weights);

}  // namespace sb
