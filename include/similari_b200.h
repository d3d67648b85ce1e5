/*
 * similari_b200.h -- C ABI of the H100-native association engine (libsimilari_b200.so).
 *
 * Drop-in boundary for Similari's per-frame cost-matrix + assignment hot path.  The reference has no C ABI
 * (it is a Rust crate with PyO3 classes); these entry points are what a Rust `extern "C"` block inside
 * Sort / BatchSort / VisualSort / BatchVisualSort (or the ctypes/PyO3 layer) binds in place of
 *     TrackStore::foreign_track_distances  (src/track/store.rs:429-460)
 *   + Voting::winners                       (src/trackers/sort/voting.rs:30-100, src/trackers/visual_sort/voting.rs:45-100)
 *   + TrackStore::merge_external / add_track (src/track/store.rs:625-691)
 * INTEGRATION.md shows the Rust-side and Python-side bindings.  All paths cited below are relative to the
 * reference tree (insight-platform/Similari, crate similari-trackers-rs v0.26.12).
 *
 * Conventions
 *   - plain pointers and sizes only; the caller allocates every output; the library never frees caller memory;
 *   - a box is 6 floats (xc, yc, angle, aspect, height, confidence) = Universal2DBox (src/utils/bbox.rs:79-87);
 *     angle == NaN encodes Option::None;
 *   - custom_object_id == INT64_MIN encodes Option::None; feature quality NULL means 1.0 (unwrap_or(1.0),
 *     src/trackers/visual_sort/simple_api.rs:141-151);
 *   - every function returns 0 on success, a negative sb200_status otherwise (the reference panics instead);
 *     sb200_last_error() returns the message of the calling thread's last failure;
 *   - a tracker handle is single-threaded (`&mut self` in the reference); handles are independent;
 *   - there is NO CPU fallback: without a CUDA device every compute entry point fails with SB200_ERR_CUDA.
 */
#ifndef SIMILARI_B200_H
#define SIMILARI_B200_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define SB200_VERSION 3

typedef enum {
  SB200_OK = 0,
  SB200_ERR_INVALID = -1,   /* bad argument (the reference's assert!/panic paths) */
  SB200_ERR_CUDA = -2,      /* CUDA runtime error or no device */
  SB200_ERR_CAPACITY = -3,  /* problem exceeds a documented device limit */
  SB200_ERR_INTERNAL = -4
} sb200_status;

/* TrackerKind: which reference tracker's semantics the handle follows (id numbering, voting cascade).
 *   SORT             src/trackers/sort/simple_api.rs:21-29
 *   BATCH_SORT       src/trackers/sort/batch_api.rs:46-53
 *   VISUAL_SORT      src/trackers/visual_sort/simple_api.rs
 *   BATCH_VISUAL_SORT src/trackers/visual_sort/batch_api.rs */
#define SB200_KIND_SORT 0
#define SB200_KIND_BATCH_SORT 1
#define SB200_KIND_VISUAL_SORT 2
#define SB200_KIND_BATCH_VISUAL_SORT 3
/* PositionalMetricType, src/trackers/sort.rs:364-369 */
#define SB200_POS_MAHA 0
#define SB200_POS_IOU 1
/* VisualSortMetricType, src/trackers/visual_sort/metric.rs:20-24 */
#define SB200_VIS_EUCLIDEAN 0
#define SB200_VIS_COSINE 1
/* VotingType, src/trackers/sort.rs:357-362 */
#define SB200_VOTING_VISUAL 0
#define SB200_VOTING_POSITIONAL 1
#define SB200_MAX_CONSTRAINTS 8
#define SB200_NONE_ID INT64_MIN

/* Constructor arguments of the four trackers folded into one struct:
 *   Sort::new / BatchSort::new              src/trackers/sort/simple_api.rs:41-50, batch_api.rs:157-167
 *   VisualSortOptions + VisualMetricBuilder src/trackers/visual_sort/options.rs:10-205, metric/builder.rs:9-42 */
typedef struct {
  int32_t kind;
  int32_t positional_kind;        /* method / positional_metric */
  float iou_threshold;            /* PositionalMetricType::IoU(t) */
  float min_confidence;           /* min_confidence / positional_min_confidence */
  int32_t max_idle_epochs;
  int32_t history_length;         /* bbox_history / kept_history_length: boxes of history per track (device cap 64; 0 = that cap) */
  float kalman_position_weight;
  float kalman_velocity_weight;
  int32_t n_constraints;          /* SpatioTemporalConstraints: (epoch_delta, max_distance) pairs */
  int32_t constraint_epochs[SB200_MAX_CONSTRAINTS];
  float constraint_max_dist[SB200_MAX_CONSTRAINTS];
  int32_t visual_kind;
  float visual_threshold;
  int32_t feature_dim;            /* D; 0 for Sort / BatchSort */
  int32_t visual_max_observations; /* observations kept per track, 1..32 (reference default 5, its examples 25); above
                                    * 32 the tracker is refused with SB200_ERR_CAPACITY before anything is created */
  int32_t visual_min_votes;
  int32_t visual_minimal_track_length;
  float visual_minimal_area;
  float visual_minimal_quality_use;
  float visual_minimal_quality_collect;
  float visual_minimal_own_area_percentage_use;
  float visual_minimal_own_area_percentage_collect;
  int32_t max_scenes_hint;            /* capacity hints (0 = grow on demand) */
  int32_t max_tracks_per_scene_hint;
  int32_t max_dets_per_scene_hint;
  int32_t device;                     /* CUDA device ordinal */
} sb200_options;

/* Fills `o` with the reference's defaults (PySort::new defaults, src/trackers/sort/simple_api.rs:461-470;
 * VisualMetricBuilder::default, src/trackers/visual_sort/metric/builder.rs:26-42). */
void sb200_options_default(sb200_options* o);

typedef struct sb200_tracker sb200_tracker;

/* Per-detection result columns = SortTrack (src/trackers/sort.rs:286-311) as struct-of-arrays.  Any pointer
 * may be NULL (that column is then neither computed into host memory nor copied back). */
typedef struct {
  uint64_t* ids;            /* SortTrack.id */
  uint32_t* epochs;         /* SortTrack.epoch */
  uint32_t* lengths;        /* SortTrack.length */
  uint8_t* voting_types;    /* SortTrack.voting_type (SB200_VOTING_*) */
  float* predicted_boxes;   /* [total][6] SortTrack.predicted_bbox */
  float* observed_boxes;    /* [total][6] SortTrack.observed_bbox */
} sb200_predict_out;

const char* sb200_last_error(void);
int sb200_device_count(void);

/* ---- tracker lifecycle (Sort::new ... ) ---- */
int sb200_tracker_create(const sb200_options* opts, sb200_tracker** out);
void sb200_tracker_destroy(sb200_tracker* t);
/* Orders the tracker's work with `cuda_stream` (a cudaStream_t; NULL is the legacy default stream): every predict call first waits
 * for what that stream holds when the call is made (so device-resident inputs may be produced on it just before the call)
 * and the stream waits for the call's frame (so its outputs can be consumed on it, and the caller can bracket the work
 * with its own CUDA events).  The kernels themselves run on the tracker's own streams. */
int sb200_tracker_set_stream(sb200_tracker* t, void* cuda_stream);
/* per_call != 0 (the default): the caller's stream waits for the frame of every predict call.  0: it does not -- successive
 * frames then overlap where they can (the next frame's candidate preparation runs under the current frame's cost kernels);
 * a stream that consumes device-resident outputs -- or overwrites device-resident inputs of a frame that may still be
 * running -- waits explicitly with sb200_stream_join (or the host calls sb200_sync).  Counterpart of taking the results off PredictionBatchResult's channel when they are needed
 * (src/trackers/batch.rs:24-38) instead of blocking in predict. */
int sb200_set_stream_join(sb200_tracker* t, int32_t per_call);
/* Makes `cuda_stream` wait (on the device) for every frame enqueued so far. */
int sb200_stream_join(sb200_tracker* t, void* cuda_stream);

/* VisualSortObservation::feature is an Option (src/trackers/visual_sort.rs:42-55): a tracker may see frames without any
 * feature before it learns the feature length.  Until a request has carried feature rows the dimension given at creation
 * is provisional and can be changed here; afterwards a different value is SB200_ERR_INVALID. */
int sb200_set_feature_dim(sb200_tracker* t, int32_t feature_dim);

/* Element type of the `features` column of the predict entry points and sb200_prefetch_inputs.  The column stays
 * [total][feature_dim] row-major; with F16 (IEEE binary16) or BF16 the `const float* features` parameter carries a pointer
 * to 2-byte elements.  Widening either type to f32 is exact: a frame fed half-precision rows returns exactly what the same
 * frame fed the widened f32 rows returns (results, stored features, wasted feature histories, state blobs). */
#define SB200_FEATURE_F32 0
#define SB200_FEATURE_F16 1
#define SB200_FEATURE_BF16 2
/* Sets the element type of the features column for every later sb200_predict_batch / _async / _device and
 * sb200_prefetch_inputs call on the tracker.  It may change between calls: each frame keeps the type it was enqueued
 * with, and a prefetch made under one type is not used by a predict call under another (the columns are copied again).
 * The type is an input format, not tracker state: it is not saved in the state blob, and a new or loaded tracker reads
 * F32.  SB200_ERR_INVALID for a NULL handle, a non-visual tracker or an unknown type. */
int sb200_set_feature_type(sb200_tracker* t, int32_t type);

/* ---- the hot path ----
 * One call == Sort::predict_with_scene (n_scenes = 1, src/trackers/sort/simple_api.rs:110-196) or
 * BatchSort::predict / BatchVisualSort::predict over a PredictionBatchRequest (src/trackers/sort/batch_api.rs:222-290,
 * src/trackers/visual_sort/batch_api.rs:213-317, src/trackers/batch.rs:12-38) flattened as:
 *   scene_ids[n_scenes], det_offsets[n_scenes+1] (CSR over detections),
 *   boxes[total][6], features[total][D] or NULL (f32, or the type set by sb200_set_feature_type), has_feature[total]
 *   or NULL (all present),
 *   quality[total] or NULL, custom_ids[total] or NULL, own_area[total] or NULL
 *   (own-area shares of exclusively_owned_areas, computed by the caller; src/utils/clipping/bbox_own_areas.rs).
 * All pointers are HOST pointers; inputs are copied to the device and the requested result columns copied back
 * before the call returns (results in input order, like the reference's Vec<SortTrack>). */
int sb200_predict_batch(sb200_tracker* t, int32_t n_scenes, const uint64_t* scene_ids, const int32_t* det_offsets,
                        const float* boxes, const float* features, const uint8_t* has_feature, const float* quality,
                        const int64_t* custom_ids, const float* own_area, const sb200_predict_out* out);
/* Optional input prefetch for pipelined callers (BatchSort::predict is asynchronous in the reference too,
 * src/trackers/sort/batch_api.rs:222-290): starts the host-to-device copy of a FUTURE request's columns on a copy
 * stream and returns immediately.  A later sb200_predict_batch() called with the same `boxes` / `features` pointers
 * and the same detection count uses the prefetched copy instead of copying again, so the copy of frame i+1 overlaps
 * the kernels of frame i.  The host buffers must stay unchanged until that predict call returns. */
int sb200_prefetch_inputs(sb200_tracker* t, int32_t total, const float* boxes, const float* features,
                          const uint8_t* has_feature, const float* quality, const int64_t* custom_ids,
                          const float* own_area);
/* The asynchronous form of the same call -- what BatchSort::predict is in the reference, where the request is queued
 * and the per-scene results arrive later on PredictionBatchResult's channel (src/trackers/sort/batch_api.rs:222-290,
 * src/trackers/batch.rs:24-38).  The frame is enqueued on the tracker's stream and the call returns; up to three frames
 * are in flight (a fourth call waits for the oldest).  The host buffers (inputs, and the `out` columns, which should be
 * pinned: sb200_host_alloc) must stay valid and are only defined after sb200_sync() -- or after a later call has
 * reported sb200_frames_in_flight() low enough.  An error inside an asynchronous frame is returned by the next
 * predict / sync / query call on the tracker. */
int sb200_predict_batch_async(sb200_tracker* t, int32_t n_scenes, const uint64_t* scene_ids, const int32_t* det_offsets,
                              const float* boxes, const float* features, const uint8_t* has_feature, const float* quality,
                              const int64_t* custom_ids, const float* own_area, const sb200_predict_out* out);
/* Waits for every frame in flight (PredictionBatchResult::get until batch_size results arrived) and hands their
 * bookkeeping to the host side of the tracker; returns the first error an asynchronous frame raised, if any. */
int sb200_sync(sb200_tracker* t);
/* Frames enqueued and not yet completed (PredictionBatchResult::ready is `== 0`); never blocks. */
int sb200_frames_in_flight(sb200_tracker* t);

/* Host-side cost of the predict entry points since the tracker was created: out3 = {calls, wall milliseconds spent inside
 * them, milliseconds of that spent blocked on the device (ring of frames in flight full, wait == true, reallocation)}.
 * (total - blocked) / calls is what one frame costs the calling thread; the stream-ordered design needs it below the
 * frame's device time (no reference counterpart: the reference's predict is synchronous). */
int sb200_host_counters(sb200_tracker* t, double* out3);
/* Same call with boxes / features / has_feature / quality / custom_ids / own_area and every non-NULL `out` column
 * being DEVICE pointers (inputs already resident in HBM).  scene_ids and det_offsets stay host pointers (they are
 * consumed before the call returns).  Stream-ordered like sb200_predict_batch_async: nothing in the call waits for
 * the device -- the per-frame tables that depend on the previous frame's outcome (tracks per scene, matrix offsets, the
 * tile list of the tensor-core kernel, the id counter) are built by a kernel -- so consecutive frames queue back to back
 * and a caller can order its own work after the results with an event on the tracker's stream. */
int sb200_predict_batch_device(sb200_tracker* t, int32_t n_scenes, const uint64_t* scene_ids,
                               const int32_t* det_offsets, const float* boxes, const float* features,
                               const uint8_t* has_feature, const float* quality, const int64_t* custom_ids,
                               const float* own_area, const sb200_predict_out* out);

/* ---- TrackerAPI (src/trackers/tracker_api.rs:27-117) ---- */
int sb200_skip_epochs(sb200_tracker* t, uint64_t scene_id, int32_t n);
int64_t sb200_current_epoch(sb200_tracker* t, uint64_t scene_id);
int64_t sb200_active_tracks(sb200_tracker* t);                 /* sum(active_shard_stats()) */
/* stored tracks per scene (0 for unknown scenes) as the reference's store would count them: the N of the next frame's
 * N x M cost matrix, expired tracks that the reference has not collected yet included */
int sb200_scene_track_counts(sb200_tracker* t, int32_t n_scenes, const uint64_t* scene_ids, int32_t* out);
/* what the device actually holds and scans per scene: `live` = tracks that can still match (expired tracks leave the
 * device store at the end of the frame in which they expire and wait, hidden, for the reference's collection point:
 * auto-waste tick, wasted(), skip_epochs), `blocks` = feature blocks of the scene's arena (rows scanned by the visual
 * cost kernel = blocks * visual_max_observations).  Either output may be NULL. */
int sb200_scene_live_counts(sb200_tracker* t, int32_t n_scenes, const uint64_t* scene_ids, int32_t* live, int32_t* blocks);
int sb200_set_auto_waste(sb200_tracker* t, int32_t periodicity);
int sb200_clear_wasted(sb200_tracker* t);
/* wasted(): drains up to `cap` wasted tracks; returns the count (>= 0) or a negative status. */
int64_t sb200_wasted(sb200_tracker* t, int64_t cap, uint64_t* ids, uint64_t* scene_ids, uint32_t* epochs,
                     uint32_t* lengths, float* predicted_boxes, float* observed_boxes);
/* wasted() with the box history of WastedSortTrack (src/trackers/sort.rs:316-341: predicted_boxes / observed_boxes, the last
 * history_length boxes of the track, oldest first, kept by SortAttributes::update_history, sort.rs:157-171).
 * predicted_history / observed_history: [cap][history_cap][6], history_counts[cap] = boxes filled for each track. */
int64_t sb200_wasted_history(sb200_tracker* t, int64_t cap, uint64_t* ids, uint64_t* scene_ids, uint32_t* epochs,
                             uint32_t* lengths, float* predicted_boxes, float* observed_boxes, int32_t history_cap,
                             float* predicted_history, float* observed_history, int32_t* history_counts);
/* Feature history of the visual trackers (WastedVisualSortTrack::observed_features, src/trackers/visual_sort.rs:117-119,
 * 210-213): the input feature of each of a track's last history_length observations (capped at 64 like the box history),
 * kept on the device while the track lives and until its wasted record is collected.  Off by default; on == 1 switches
 * it on.  SB200_ERR_INVALID for a non-visual tracker or once a predict has been enqueued. */
int sb200_set_feature_history(sb200_tracker* t, int32_t on);
/* Size of the feature-history pool (waits for the frames in flight): out3 = {blocks allocated, blocks ever handed out,
 * free blocks}.  A block holds history_length * (4 * d8 + 1) bytes.  SB200_ERR_INVALID when the history is off. */
int sb200_feature_history_pool(sb200_tracker* t, int64_t* out3);
/* sb200_wasted_history (same records, same order, same "newest history_cap entries" rule) plus each entry's feature:
 * features[cap][history_cap][d8] f32 (d8 = feature_dim rounded up to 8, zero-padded as Feature::from_vec does) and
 * feature_present[cap][history_cap] (0: the observation had no feature; also 0 past history_counts[i]).  Every row of
 * the first returned-count records is written: rows whose present byte is 0 are all zero.  SB200_ERR_INVALID when the
 * feature history is off or an output is NULL. */
int64_t sb200_wasted_visual(sb200_tracker* t, int64_t cap, uint64_t* ids, uint64_t* scene_ids, uint32_t* epochs,
                            uint32_t* lengths, float* predicted_boxes, float* observed_boxes, int32_t history_cap,
                            float* predicted_history, float* observed_history, int32_t* history_counts, float* features,
                            uint8_t* feature_present);
/* idle_tracks_with_scene() (src/trackers/sort/simple_api.rs:198-215) */
int64_t sb200_idle_tracks(sb200_tracker* t, uint64_t scene_id, int64_t cap, uint64_t* ids, uint32_t* epochs,
                          uint32_t* lengths, float* predicted_boxes, float* observed_boxes);
/* Debug / parity: dense dump of one scene's store in store order.  states: [n][30] = mean[10] + 5 x (Pxx,Pxv,Pvx,Pvv). */
int64_t sb200_scene_tracks(sb200_tracker* t, uint64_t scene_id, int64_t cap, uint64_t* ids, float* boxes,
                           float* states30, int32_t* feature_counts);
/* Debug / parity: last frame's positional cost matrix of a scene ([m][n] f32, NaN == None), n = the scene's live tracks
 * in store order.  Visual trackers on the tensor-core path evaluate the positional metric lazily -- only for candidates
 * the visual BestFit pass left undecided against tracks it did not claim, the pairs VisualVoting::winners
 * (src/trackers/visual_sort/voting.rs:45-100) can still consult -- so the other entries read None; with the environment
 * variable SB200_FULL_COSTS=1 every pair is evaluated as the reference does. */
int64_t sb200_last_costs(sb200_tracker* t, uint64_t scene_id, int64_t cap, float* out, int32_t* m, int32_t* n);
/* Cumulative work of all completed frames (waits for the frames in flight): counters4 = { sum over frames and scenes of
 * M x N (pair-associations, N = tracks the device store held when the frame ran), sum of M x (feature rows scanned by the
 * visual cost kernel), frames, scenes the exact SIMT fallback kernels had to take }, ms8 = { summed per-stage device times: prep, positional cost, visual cost, voting, apply;
 * summed times of the dominant visual-cost kernel and of the refinement; frames in which those two ran }.  Either may
 * be NULL.  bench.py reads it before and after its timed region. */
int sb200_work_counters(sb200_tracker* t, uint64_t* counters4, double* ms8);
/* Screen precision counters, cumulative over the frames absorbed so far: frames screened on e4m3 operands, frames screened
   on BF16 operands, survivors of those screens refined, survivors the exact test cut.  Waits for the frames in flight. */
int sb200_screen_counters(sb200_tracker* t, uint64_t* counters4);
/* Kernels this library has launched since it was loaded (every launch site counts itself). */
uint64_t sb200_launch_count(void);
/* Per-stage device times (ms) of the last completed predict call: prep, positional cost, visual cost, voting, apply. */
int sb200_last_stage_ms(sb200_tracker* t, float* out5);
/* Device times (ms) of the dominant visual-cost kernels of the last predict call: [0] tensor-core screen kernel,
 * [1] scene-mode + exact refinement kernels; 0 when the tensor-core path was not used. */
int sb200_last_kernel_ms(sb200_tracker* t, float* out2);

/* ---- state blob: save / restore a tracker, move scenes between trackers and GPUs (no reference counterpart: the
 * reference's state lives in host memory).  One versioned binary format; DESIGN.md section 3b describes it.
 * `dst` / `src` may be host memory or device memory on any device, at any address: a device blob that is not 16-byte
 * aligned, or not on the tracker's device, goes through a device copy.  Every entry first waits for the frames in flight
 * (an error of an asynchronous frame is returned there).  Size query: with dst == NULL or cap too small, save and export
 * write nothing, set *bytes to the size they need and return SB200_ERR_CAPACITY.  A rejected call changes nothing.
 * Stream order of a device blob: save, export and import are ordered after what the stream named with
 * sb200_tracker_set_stream holds when the call is made (a blob the caller is still receiving on that stream is read
 * after the receive; pending reads of the destination come before it is written) and return after the blob work is
 * done.  load has no tracker stream yet, and a tracker without a named stream has none to wait for: there a device blob
 * must be complete when the call is made (e.g. cudaStreamSynchronize on the stream of the receive).
 * A blob is checked before anything is copied: header, section bounds, alignment and sizes, and every index it carries
 * (arena blocks, free lists, block owners, observation slots, history blocks) against the counts it declares.
 * sb200_set_feature_history is refused on a loaded tracker and after an import, as after a predict.
 *
 * Whole tracker: options, every scene slot in slot order, the wasted buffer (revealed and hidden records, with box and
 * feature histories), the id counter, the auto-waste counter and periodicity, the feature dimension state, adapt_dense.
 * A loaded tracker fed the same requests returns the same results, bit for bit.  load builds its tracker from the
 * blob's options on `device` (the capacity hints are the blob's); it rejects a scene blob. */
int sb200_tracker_save(sb200_tracker* t, void* dst, size_t cap, size_t* bytes);
int sb200_tracker_load(const void* src, size_t bytes, int32_t device, sb200_tracker** out);
/* Scenes: the live tracks and the epoch of each listed scene (SB200_ERR_INVALID for an unknown id).  remove != 0 takes
 * them out of the source: the slot starts over (no tracks, epoch 0) and the scene's hidden wasted records stay with the
 * source until its next collection point.  import checks the format, that every option but the capacity hints and
 * `device` matches (the constraints up to n_constraints), the feature-history flag, and that no imported scene already
 * holds tracks or epochs here; the id counter becomes max(its own, the source's at export), so a new id never repeats an
 * imported one.  The ids the destination's own scenes already hold come from its own counter and may equal imported ids
 * of other scenes.  import rejects a whole-tracker blob. */
int sb200_scenes_export(sb200_tracker* t, int32_t n_scenes, const uint64_t* scene_ids, int32_t remove,
                        void* dst, size_t cap, size_t* bytes);
int sb200_scenes_import(sb200_tracker* t, const void* src, size_t bytes);
/* The tracker's options as they stand (feature_dim after sb200_set_feature_dim; a loaded tracker's from its blob) and,
 * if `feature_dim_fixed` is not NULL, whether a request has carried feature rows (sb200_set_feature_dim then refuses a
 * change).  No device call. */
int sb200_tracker_options(sb200_tracker* t, sb200_options* out, int32_t* feature_dim_fixed);

/* ---- stateless operators (host pointers) used by parity tests and by callers that keep their own state ----
 * Positional cost matrix = SortMetric::metric over all pairs (src/trackers/sort/metric.rs:38-77):
 * out[m][n] = IoU*conf (>= thr) or (100 - d^2)/conf, NaN == None.  track_states30 only for Mahalanobis. */
int sb200_sort_cost_matrix(int32_t positional_kind, float iou_threshold, float min_confidence, float pos_weight,
                           float vel_weight, const float* cand_boxes, int32_t m, const float* track_boxes,
                           const float* track_states30, int32_t n, float* out_mn, int32_t device);
/* Visual cost matrix = euclidean / cosine (src/distance.rs:9-47) + is_ok/distance_to_weight
 * (src/trackers/visual_sort/metric.rs:52-64); out[m][n], NaN == None. */
int sb200_visual_cost_matrix(int32_t visual_kind, float threshold, const float* cand_features, int32_t m,
                             const float* track_features, int32_t n, int32_t d, float* out_mn, int32_t device);
/* SortVoting::winners on a dense cost matrix (NaN == None): winner[m] = track index or -1 (new track). */
int sb200_sort_voting(float threshold, const float* cost_mn, int32_t m, int32_t n, int32_t* winner, int32_t device);
/* VisualVoting::winners on dense matrices: pos[m][n], vis[m][n][k] (NaN == None), k = observations per track in 1..32. */
int sb200_visual_voting(float positional_threshold, int32_t min_votes, const float* pos_mn, const float* vis_mnk,
                        int32_t m, int32_t n, int32_t k, int32_t* winner, uint8_t* voting_type, int32_t device);
/* Kalman filter steps on packed states (src/utils/kalman/kalman_2d_box.rs:58-148), n states at once. */
int sb200_kalman_initiate(float pos_weight, float vel_weight, const float* boxes, int32_t n, float* states30, int32_t device);
int sb200_kalman_predict(float pos_weight, float vel_weight, const float* in30, int32_t n, float* out30, int32_t device);
int sb200_kalman_update(float pos_weight, float vel_weight, const float* in30, const float* boxes, int32_t n,
                        float* out30, int32_t device);
/* Universal2DBoxKalmanFilter::distance (kalman_2d_box.rs:150-170): out[i] = squared Mahalanobis distance of boxes[i]
 * from states30[i] (vel_weight is accepted for symmetry and unused: the distance reads the position weight only). */
int sb200_kalman_distance(float pos_weight, float vel_weight, const float* states30, const float* boxes, int32_t n,
                          float* out, int32_t device);
/* Point2DKalmanFilter (src/utils/kalman/kalman_2d_point.rs:51-137) on n packed 12-float states: mean (x, y, vx, vy),
 * then for i in {x, y} the covariance block P[i][i], P[i][i+2], P[i+2][i], P[i+2][i+2].  points2 = (x, y) pairs. */
int sb200_point_kalman_initiate(float pos_weight, float vel_weight, const float* points2, int32_t n, float* states12,
                                int32_t device);
int sb200_point_kalman_predict(float pos_weight, float vel_weight, const float* in12, int32_t n, float* out12,
                               int32_t device);
int sb200_point_kalman_update(float pos_weight, float vel_weight, const float* in12, const float* points2, int32_t n,
                              float* out12, int32_t device);
int sb200_point_kalman_distance(float pos_weight, float vel_weight, const float* states12, const float* points2,
                                int32_t n, float* out, int32_t device);
/* Universal2DBox::get_vertices (src/utils/bbox.rs:169-171,287-330): out8[n][4][2] f64, angle NaN == 0. */
int sb200_box_vertices(const float* boxes, int32_t n, double* out8, int32_t device);
/* sutherland_hodgman_clip_py / intersection_area_py (src/utils/clipping/clipping_py.rs:29-46) of n (subject, clipping)
 * box pairs: out_vertices[n][16][2] f64 = the clipped ring without its closing repeat (slots past the count are 0),
 * out_counts[n] = its vertex count, out_areas[n] = its unsigned area.  SB200_ERR_CAPACITY, with no output written, when a
 * pair's clip would need more than 16 vertices (the reference's Vec has no bound). */
int sb200_clip_polygons(const float* subjects, const float* clippings, int32_t n, double* out_vertices,
                        int32_t* out_counts, double* out_areas, int32_t device);
/* out_mn[i][j] = intersection_area_py(a[i], b[j]) (f64; no too_far and no IoU gate).  SB200_ERR_CAPACITY, with no output
 * written, as for sb200_clip_polygons. */
int sb200_intersection_areas(const float* a, int32_t m, const float* b, int32_t n, double* out_mn, int32_t device);
/* exclusively_owned_areas + exclusively_owned_areas_normalized_shares (src/utils/clipping/bbox_own_areas.rs:8-46) for the
 * boxes of ONE scene: out[i] = share of box i that no other box covers, in [0, 1].  The visual trackers call the same
 * kernel themselves when an own-area threshold is set and the request carries no `own_area` column
 * (src/trackers/visual_sort/simple_api.rs:110-127).  A box that more than 32 others overlap takes a second,
 * CTA-per-box pass; SB200_ERR_CAPACITY only beyond 2800 overlapping boxes on one box. */
int sb200_own_area_shares(const float* boxes, int32_t n, float* out, int32_t device);

/* nms (src/utils/nms.rs:32-72): scores NULL or NaN entries == None; out_idx = kept input indices in rank order;
 * returns kept count or negative status.  The one-set case of sb200_nms_batch; at most 1,638,400 boxes
 * (SB200_ERR_CAPACITY above: the suppressed-box bitmap, ceil(n / 64) * 8 bytes, must fit in 200 KB of shared memory). */
int64_t sb200_nms(const float* boxes, const float* scores, int32_t n, float nms_threshold, float score_threshold,
                  int32_t has_score_threshold, int32_t* out_idx, int32_t device);
/* nms (src/utils/nms.rs:32-72) applied independently to each of n_sets sets; set s = rows [offsets[s], offsets[s+1]).
 * keep_idx[offsets[s] .. offsets[s] + keep_counts[s]) = kept row indices RELATIVE to the set, in rank order; the rest of
 * the set's range = -1.  keep_mask (optional) [total] = 1 for kept rows, input order.  scores NULL or NaN == None.
 * Returns the total kept count or a negative status. Host pointers; offsets[n_sets + 1] host.
 * Checks, before anything is launched or written: n_sets >= 0, offsets[0] == 0, offsets non-decreasing, keep_counts
 * non-NULL when n_sets > 0 and boxes / keep_idx non-NULL when the total is above 0 (else SB200_ERR_INVALID); a CUDA
 * device (SB200_ERR_CUDA); every set within sb200_nms's limit (SB200_ERR_CAPACITY, naming the set).  Empty sets and
 * n_sets == 0 are valid.  All sets run in one fixed sequence of kernel launches, whatever their number. */
int64_t sb200_nms_batch(int32_t n_sets, const int32_t* offsets, const float* boxes, const float* scores,
                        float nms_threshold, float score_threshold, int32_t has_score_threshold,
                        int32_t* keep_idx, int32_t* keep_counts, uint8_t* keep_mask, int32_t device);
/* The same with boxes / scores / keep_idx / keep_counts / keep_mask as DEVICE pointers, enqueued on cuda_stream (NULL:
 * the legacy default stream); offsets stays a host pointer and may be reused as soon as the call returns.  Returns after
 * the enqueue (0 or a negative status); no host synchronisation, except that a call waits when eight earlier calls on
 * the device still have the copy of their (pinned) set tables queued.  The workspace is allocated and freed
 * stream-ordered on cuda_stream. */
int sb200_nms_batch_device(int32_t n_sets, const int32_t* offsets, const float* boxes, const float* scores,
                           float nms_threshold, float score_threshold, int32_t has_score_threshold,
                           int32_t* keep_idx, int32_t* keep_counts, uint8_t* keep_mask, int32_t device, void* cuda_stream);

/* ---- multi-GPU: the one exchange step of the scene-sharded path (csrc/comm.cu) ----
 * Scenes are independent and track state is sticky per GPU (rank = scene shard), so N GPUs run N independent trackers; the
 * only data that crosses GPUs is the request on its way from an ingest rank to the owners of its scenes and the assigned
 * track records on their way back -- the counterpart of the reference's voting-shard fan-out and result channel
 * (src/trackers/sort/batch_api.rs:197-207,222-290).  One process per GPU.  NCCL (send/recv over NVLink) is loaded at run
 * time; rank 0 creates the 128-byte unique id and the caller ships it to the other ranks on its own control channel.
 * All data pointers are DEVICE pointers; calls are asynchronous on `cuda_stream`, so the scatter of frame i+1 can overlap
 * the kernels of frame i on another stream.  det_range[world + 1]: rank r owns detections [det_range[r], det_range[r+1])
 * of the root's request (its scenes' detections are contiguous).  Non-root ranks pass NULL for the `all_*` arguments. */
typedef struct sb200_comm sb200_comm;
int sb200_comm_unique_id(void* out128);
int sb200_comm_create(int32_t rank, int32_t world, const void* id128, int32_t device, sb200_comm** out);
void sb200_comm_destroy(sb200_comm* c);
/* root -> owners: boxes [6 f32], features [feature_dim f32], has_feature, quality, custom ids; a column is skipped on every
 * rank when its `my_*` pointer is NULL (all ranks must agree). */
int sb200_shard_scatter(sb200_comm* c, int32_t root, const int32_t* det_range, int32_t feature_dim, const float* all_boxes,
                        const float* all_features, const uint8_t* all_has_feature, const float* all_quality,
                        const int64_t* all_custom_ids, float* my_boxes, float* my_features, uint8_t* my_has_feature,
                        float* my_quality, int64_t* my_custom_ids, void* cuda_stream);
/* owners -> root: the SortTrack columns (`mine`: this rank's results as written by sb200_predict_batch_device; `all`: the
 * root's buffers for the whole request; a column is skipped when `mine` has it NULL). */
int sb200_shard_gather(sb200_comm* c, int32_t root, const int32_t* det_range, const sb200_predict_out* mine,
                       const sb200_predict_out* all, void* cuda_stream);

/* ---- feature track store: TrackStore (src/track/store.rs) for feature-only tracks, with TopNVoting on top ----
 * The tracks of benches/feature_tracker.rs: one feature class, baked is always Ready, every observation carries a
 * feature.  Without a gate (the default) there are no track attributes and compatible is always true; a gated store
 * (sb200_fstore_set_gate, below) keeps the attributes of examples/track_merging.rs.  Each track keeps its newest max_observations (K) observations in
 * their original order (the bench's optimize: reverse / truncate(K) / reverse).  The store lives on the device.
 *
 * Order rules (the reference's shard / HashMap order is replaced by these, which the oracle defines):
 *   - store order is insertion order; removal (sb200_fstore_fetch with remove) is a stable compaction;
 *   - the entries of a search are enumerated as (query, stored track in store order, query observation, track
 *     observation), both observation lists oldest first (cartesian_product(query, track), src/track.rs:618-645); each
 *     group's f64 weight is summed in that order;
 *   - TopN results are sorted by weight, descending; equal weights go to the lower store position.
 * Bounds: topn <= 64, max_observations <= 64, feature_dim <= 8192.  One search / associate call computes a distance
 * matrix of (query observations taking part) x (stored tracks x max_observations) entries, 4 B each; a call that needs
 * more than 2^30 of them returns SB200_ERR_CAPACITY before anything runs.
 * Every rejected call changes nothing.  Host pointers; the caller allocates the outputs.  A handle is single-threaded. */
#define SB200_FSTORE_MAX_TOPN 64
#define SB200_FSTORE_MAX_OBS 64
#define SB200_FSTORE_MAX_DIM 8192
typedef struct {
  int32_t metric;           /* SB200_VIS_EUCLIDEAN: euclidean (src/distance.rs:9-19); SB200_VIS_COSINE: 1 - cosine
                               (src/distance.rs:26-47, as VisualSortMetricType::distance_to_weight maps it) */
  float distance_filter;    /* postprocess_distances keeps d < distance_filter (strict) */
  int32_t max_observations; /* K, 1..64 */
  int32_t feature_dim;      /* D, 1..8192; rows are zero-padded to a multiple of 8 as Feature::from_vec pads */
  int32_t topn;             /* TopNVoting::new(topn, max_distance, min_votes), src/track/voting/topn.rs:37-44 */
  float max_distance;
  int32_t min_votes;
  int32_t device;
} sb200_fstore_options;
typedef struct sb200_fstore sb200_fstore;
/* TrackStoreBuilder::build + TopNVoting::new.  SB200_ERR_INVALID for an unknown metric or a bound outside the caps above. */
int sb200_fstore_create(const sb200_fstore_options* opts, sb200_fstore** out);
void sb200_fstore_destroy(sb200_fstore* s);
/* TrackStore::add (src/track/store.rs:530-568) for each (ids[i], features[i][D]) in order: an unknown id creates a
 * track, at the end of the store, with that one observation; a known id appends the observation and keeps the newest K. */
int sb200_fstore_add(sb200_fstore* s, int32_t n, const uint64_t* ids, const float* features);
/* foreign_track_distances (src/track/store.rs:429-460, Track::distances src/track.rs:604-652) + TopNVoting::winners
 * (src/track/voting/topn.rs:74-138).  Queries in CSR form: query q has id query_ids[q] and the observations
 * features[obs_offsets[q] .. obs_offsets[q+1])[D], oldest first; like a track built by TrackBuilder
 * (src/track/builder.rs:168-179) only its newest K take part.  Stored tracks with the query's id are skipped
 * (src/track/store.rs:206).  max_dist is taken over every entry of the call that passed distance_filter (all queries,
 * also entries above max_distance and entries of groups short of min_votes, topn.rs:78-95).  Outputs: counts[q] results,
 * winners[q][topn] their track ids and weights[q][topn] their f64 weights (entries past counts[q] are 0).
 * SB200_ERR_INVALID for a query without observations or an id twice in the call. */
int sb200_fstore_search(sb200_fstore* s, int32_t n_queries, const uint64_t* query_ids, const int32_t* obs_offsets,
                        const float* features, int32_t* counts, uint64_t* winners, double* weights);
/* One iteration of benches/feature_tracker.rs: search, then, in query order, each query with a result is merged into
 * its first winner (merge_external -> Track::merge, src/track/store.rs:265-277, 625-691: the query's observations are
 * appended and the newest K kept), and every other query becomes a new track under its own id at the end of the store
 * (add_track, src/track/store.rs:510-519).  Queries never see each other within a call.  Outputs as for search, plus
 * track_ids[q] = the id the query ended up in and merged[q] = 1 when it was merged.  SB200_ERR_INVALID, before anything
 * changes, as for search and for a query id that is already stored (where the reference returns DuplicateTrackId after
 * merging the queries before it). */
int sb200_fstore_associate(sb200_fstore* s, int32_t n_queries, const uint64_t* query_ids, const int32_t* obs_offsets,
                           const float* features, int32_t* counts, uint64_t* winners, double* weights,
                           uint64_t* track_ids, uint8_t* merged);
/* fetch_tracks (src/track/store.rs:388-401) when remove != 0, else a read-only lookup: counts[i] = observations of track
 * ids[i] (0: not stored), features[i][K][D] = its observations oldest first (rows past counts[i] are 0).  Returns how
 * many of the ids were found, or a negative status. */
int64_t sb200_fstore_fetch(sb200_fstore* s, int32_t n, const uint64_t* ids, int32_t remove, int32_t* counts,
                           float* features);
/* sum(shard_stats()) (src/track/store.rs:378-384): stored tracks. */
int64_t sb200_fstore_size(sb200_fstore* s);
/* Ids of the stored tracks in store order; writes min(cap, size) and returns the size. */
int64_t sb200_fstore_ids(sb200_fstore* s, int64_t cap, uint64_t* ids);
/* Device times (ms) of the last search / associate / add / search_owned / merge_owned call: distances, TopN, apply (0 for
 * a stage that did not run).  search_owned counts its on-device row staging as distances and sums its chunks.  Under
 * BestFit voting (sb200_fstore_set_voting) the TopN stage includes the claim passes. */
int sb200_fstore_last_stage_ms(sb200_fstore* s, float* out3);

/* Element type (SB200_FEATURE_F32 | _F16 | _BF16) of the `features` argument of every later sb200_fstore_add / _search /
 * _associate call and of their _device forms.  The column stays [rows][feature_dim] row-major; with F16 or BF16 the
 * `const float* features` parameter carries a pointer to 2-byte elements.  Widening either type to f32 is exact, so
 * every output and every stored row is bit for bit what the same call returns for the widened f32 request.  The stored
 * rows are in the store's storage type (sb200_fstore_set_storage_type), which does not depend on this one: every
 * combination works, and sb200_fstore_fetch keeps returning f32.  A new store reads F32; a loaded store reads the type its
 * blob was saved under.  SB200_ERR_INVALID for an unknown type.  No counterpart in the reference (its features are f32). */
int sb200_fstore_set_feature_type(sb200_fstore* s, int32_t type);
/* The options the store was created (or loaded) with, `device` included, and the element type now set.  Either output may
 * be NULL.  What a caller that loads a blob needs to size the outputs of the other calls.  No counterpart in the
 * reference. */
int sb200_fstore_get_options(sb200_fstore* s, sb200_fstore_options* out, int32_t* feature_type);
/* Storage type of the stored rows: SB200_FEATURE_F32 (the default), _F16 or _BF16.  A 2-byte store halves the device
 * memory of the rows, their growth peak and the blob.  A row is stored by rounding its widened f32 value to the storage
 * type once (__float2half_rn / __float2bfloat16_rn: to nearest, ties to even, overflow to +-inf, subnormals kept; a NaN
 * stays some NaN, its payload unspecified).  Queries are never rounded: search and associate compare the request's f32
 * rows with the stored rows widened to f32, the owned calls widened stored rows with widened stored rows, and
 * sb200_fstore_fetch returns the stored values widened to f32.  So a 2-byte store fed a column of its own type returns,
 * bit for bit, what an f32 store fed the same column returns; in general its results are those of an f32 store that
 * holds the rounded rows.  Allowed while the store holds no tracks (also after sb200_fstore_fetch with remove emptied
 * it); reallocates nothing.  SB200_ERR_INVALID, changing nothing, for an unknown type or a store that holds tracks.  A
 * loaded store has the type its blob was saved under.  No counterpart in the reference (its features are f32). */
int sb200_fstore_set_storage_type(sb200_fstore* s, int32_t type);
int sb200_fstore_get_storage_type(sb200_fstore* s, int32_t* out);

/* sb200_fstore_add / _search / _associate with `d_features` a DEVICE pointer on the store's device, in the element type
 * set by sb200_fstore_set_feature_type: the column an embedding network has just written.  ids, query_ids, obs_offsets
 * and every output stay HOST pointers, and every rejection is still decided on the host before anything is launched or
 * changed; a `d_features` that is not device memory on the store's device is SB200_ERR_INVALID.  The request rows are
 * read from the caller's column by a kernel: the features cross PCIe in neither direction.
 * Stream order: the call's work waits, by an event, for what `cuda_stream` (a cudaStream_t; NULL: the legacy default
 * stream) holds when the call is made, so a column that stream is still writing is complete before it is read.  The
 * call returns after its results are on the host, so nothing enqueued after it can race the column.  There are no
 * asynchronous forms: associate needs its results on the host to extend the id -> position map before the next call.
 * Results are those of the host-pointer call on the same values.  They stand for the same reference functions as the
 * host-pointer forms (TrackStore::add, foreign_track_distances + TopNVoting::winners, the loop of
 * benches/feature_tracker.rs); device residency has no counterpart in the reference. */
int sb200_fstore_add_device(sb200_fstore* s, int32_t n, const uint64_t* ids, const void* d_features, void* cuda_stream);
int sb200_fstore_search_device(sb200_fstore* s, int32_t n_queries, const uint64_t* query_ids,
                               const int32_t* obs_offsets, const void* d_features, int32_t* counts, uint64_t* winners,
                               double* weights, void* cuda_stream);
int sb200_fstore_associate_device(sb200_fstore* s, int32_t n_queries, const uint64_t* query_ids,
                                  const int32_t* obs_offsets, const void* d_features, int32_t* counts,
                                  uint64_t* winners, double* weights, uint64_t* track_ids, uint8_t* merged,
                                  void* cuda_stream);

/* TrackStore::owned_track_distances (src/track/store.rs:471-486) + TopNVoting::winners: the queries are STORED tracks,
 * each with its stored observations, oldest first, as its observation list.  Outputs as for sb200_fstore_search.  The
 * store is not changed and the feature type does not matter (the rows are the stored rows, widened to f32 from the
 * storage type).
 *   each == 0: one owned_track_distances(ids) call.  As the reference fetches every queried track first, no query is
 *     scored against another queried track: the candidates are the store minus the queried set.  max_dist is taken over
 *     every kept entry of the call.  The 2^30-pair bound of sb200_fstore_search applies to the whole call.
 *   each == 1: what owned_track_distances([id]) + winners gives when called once per id, in order, on the unchanged
 *     store: each query excludes only itself and has its own max_dist.  The library splits the call into chunks within
 *     the pair bound, so a whole store can be searched against itself in one call (deduplication of a gallery); only a
 *     single query whose rows x (stored tracks x max_observations) exceed 2^30 is SB200_ERR_CAPACITY.
 * An id that is not stored gets count 0 (fetch_tracks skips it).  SB200_ERR_INVALID for an id twice in the call or
 * `each` outside {0, 1}.  Every stored track keeps its store position (the reference's fetch_tracks + add_track moves it
 * within a HashMap, which has no order); ties go to the lower store position, as for search. */
int sb200_fstore_search_owned(sb200_fstore* s, int32_t n, const uint64_t* ids, int32_t each, int32_t* counts,
                              uint64_t* winners, double* weights);
/* TrackStore::merge_owned(dest, src, None, remove_src, false) (src/track/store.rs:584-611) for each pair (dest_ids[i],
 * src_ids[i]) in order, each pair seeing the state the earlier ones left: dest's observations are extended by src's
 * current ones and the newest K kept (Track::merge, src/track.rs:522-588, with the bench's optimize).  Chains (A<-B then
 * C<-A: C receives A's rows after A absorbed B) and stars (many sources into one destination) are allowed.  remove_src
 * takes every source out of the store, a stable compaction as sb200_fstore_fetch with remove.  After the call the store
 * (its blob, byte for byte) is that of the sequential emulation fetch([src]), add([dest] * n, rows), then fetch([src],
 * remove) when remove_src.  SB200_ERR_INVALID, before anything changes, for dest == src (the reference's TrackNotFound:
 * it fetched src first), a dest or src that is not stored, and, with remove_src, a pair that names a track an earlier
 * pair removed; the reference would apply the pairs in front and then return the error, the same deviation as
 * sb200_fstore_associate's.  `classes` is the reference's None: every feature class the source holds, walked in
 * ascending class id (the reference walks a HashMap; this order is the store's own, as the store order and the TopN tie
 * order are).  A newest store keeps no merge history; a quality store (sb200_fstore_set_retention) merges with
 * merge_history = true and its rule, each class step appending the source's history before it truncates that class's
 * list, so a source holding m classes appends its history m times and class step j truncates at
 * c(h_dest + j * h_src).  On a gated store the windows' hull is taken once per pair.
 * sb200_fstore_last_stage_ms reports the row moves as the apply stage. */
int sb200_fstore_merge_owned(sb200_fstore* s, int32_t n, const uint64_t* dest_ids, const uint64_t* src_ids,
                             int32_t remove_src);

/* Feature classes (the reference's `feature_class` of TrackStore::add, foreign_track_distances, owned_track_distances
 * and Track::get_feature_classes, src/track/store.rs, src/track.rs).  A store declares its n classes (1..16, distinct
 * ids, each with its own feature_dim in 1..8192) once, while it holds no tracks; a new store has one class, id 0, of the
 * options' feature_dim.  max_observations, the storage type, the gate and the retention rule are store-wide.  Capacity
 * is shared: every class holds cap * max_observations rows of its own dim, also for tracks without rows in it, so a
 * class costs its rows' device memory whether few or all tracks hold it.  SB200_ERR_INVALID for a bad n, a repeated
 * id, a dim out of range or a store that holds tracks. */
#define SB200_FSTORE_MAX_CLASSES 16
int sb200_fstore_set_classes(sb200_fstore* s, int32_t n, const uint64_t* class_ids, const int32_t* feature_dims);
/* The declared classes in declared order: the first min(cap, n) ids and dims; returns n. */
int32_t sb200_fstore_get_classes(sb200_fstore* s, int32_t cap, uint64_t* class_ids, int32_t* feature_dims);
/* Selects the class of every later call that takes or returns rows: add, search and associate in every form, fetch,
 * fetch_quality, search_owned, associate_wasted and associate_store.  Handle state, like sb200_fstore_set_feature_type:
 * a new or loaded store selects its first declared class.  The row length of those calls' feature columns is the
 * selected class's dim, and sb200_fstore_get_options reports it as feature_dim.  Per call on class c:
 *   - add: an unknown id creates a track whose other classes are empty; a known id appends to class c under the
 *     store's rule (a quality store: at the track's c(h); the history does not change).
 *   - search / associate: a stored track without class-c rows gives no entries (the reference's
 *     ObservationForClassNotFound): it does not vote and does not raise max_dist.  A merged query extends its winner's
 *     class c alone (a quality store extends the history once); a query that becomes a new track holds class c alone.
 *   - search_owned: a queried track without class-c rows gets count 0.
 *   - fetch / fetch_quality: class c's rows; counts[i] can be 0 for a stored track, and the return value still counts
 *     the stored ids.  With remove the whole track leaves, every class with it: read the other classes' rows first.
 *   - associate_wasted: refused unless class c's dim is the tracker's feature dim.
 *   - associate_store: the queries are src's class-c rows; a queried track without them has no results and is added
 *     whole.  A merged query then moves every class it holds into its winner, in ascending class id, each class step
 *     on a quality store appending the query's history as merge_owned's does; a new track keeps every class.  Both
 *     stores must declare the same class ids with the same dims.
 * merge_owned moves every class (see there); find_baked, the attributes, merge histories, ids and size do not depend on
 * the class.  SB200_ERR_INVALID for an id the store does not declare. */
int sb200_fstore_use_class(sb200_fstore* s, uint64_t class_id);
/* counts[i][k] (n rows of get_classes' n entries, declared order): the rows of track ids[i] in class k, 0 in every
 * class for an id that is not stored; the reference's get_feature_classes with their lengths.  One gather kernel.
 * Returns the number of ids found. */
int64_t sb200_fstore_class_counts(sb200_fstore* s, int32_t n, const uint64_t* ids, int32_t* counts);

/* The TrackStore side of examples/track_merging.rs for the visual trackers: a collection of tracker `t`'s wasted records
 * whose feature histories go into store `s` without leaving the device.
 * Records: collects up to `cap` wasted records exactly as sb200_wasted_history(t, cap, ..., history_cap, ...) does (the
 * same collection point with its auto-waste step, the same records in the same order, the same outputs); any of those
 * output pointers may be NULL.  history_cap bounds only the box histories.
 * Query of record i: the present features of its whole kept history (its newest min(length, history_length)
 * observations), oldest first; feature_counts[i] is their number and queried[i] is 1 when it is > 0.  The queried
 * records are associated with the store as ONE sb200_fstore_associate call would associate them, with query id
 * ids[i] + id_offset (mod 2^64) and those rows as the f32 request (so max_dist is taken over every kept entry of the
 * call; the store keeps the newest max_observations rows of each query).  The store outputs are indexed by record:
 * counts[n], winners[n][topn], weights[n][topn], track_ids[n], merged[n], each meaning what it means for
 * sb200_fstore_associate; a record that is not queried gets 0 in every one of them.  Every output may be NULL.
 * Exactness: outputs, the store (its blob) and the tracker (its blob) afterwards are, bit for bit, those of
 * sb200_wasted_visual(t, cap, ..., history_cap) followed by sb200_fstore_associate on the present rows of the queried
 * records, for every storage type, feature type and feature column type.
 * Refusals, SB200_ERR_INVALID unless noted, sb200_last_error naming the cause.  Before anything happens: a NULL handle,
 * cap < 0 or history_cap < 0, a tracker that is not visual or whose feature history is off, tracker and store on
 * different devices, a feature_dim that differs (checked once the tracker's dimension is fixed: a tracker that has never
 * seen a feature holds no present rows).  After the auto-waste step, before any record leaves the wasted buffer and
 * before the store changes: a query id that is already stored; a call whose distance matrix needs more than 2^30
 * observation pairs (SB200_ERR_CAPACITY: the call is not split, as that would change max_dist; lower `cap`).  After a
 * refusal the records are all still in the wasted buffer and the store is unchanged; the auto-waste step, which any
 * collection point runs, is the only effect.
 * The call is synchronous and both handles are single-threaded.  The records' history blocks go back to the tracker's
 * pool only after the store's work on them is complete, so a frame enqueued after the call may reuse them.  An empty
 * buffer, or records without a present feature, launch no store kernel and leave the store unchanged.  Returns the
 * records collected (>= 0) or a negative status.  No counterpart in the reference's Python API. */
int64_t sb200_fstore_associate_wasted(sb200_fstore* s, sb200_tracker* t, int64_t cap, uint64_t id_offset, uint64_t* ids,
                                      uint64_t* scene_ids, uint32_t* epochs, uint32_t* lengths, float* predicted_boxes,
                                      float* observed_boxes, int32_t history_cap, float* predicted_history,
                                      float* observed_history, int32_t* history_counts, int32_t* feature_counts,
                                      uint8_t* queried, int32_t* counts, uint64_t* winners, double* weights,
                                      uint64_t* track_ids, uint8_t* merged);

/* ---- track attributes: a time window and a source per track, and the reference's `compatible` as a gate ----
 * The CamTrackingAttributes of examples/track_merging.rs:218-245: each track of a GATED store carries a source (camera)
 * id and a window [t_start, t_end] (i64, in the caller's unit; t_start <= t_end).  The rule:
 *   SB200_FSTORE_GATE_NONE (0, the default): no attributes; every call behaves as it always has.
 *   SB200_FSTORE_GATE_SAME_SOURCE (1): compatible(a, b) = (a.t_start >= b.t_end || a.t_end <= b.t_start) &&
 *     a.source == b.source, the example's `compatible` exactly: the windows are disjoint, touching windows count as
 *     disjoint.  Two tracks seen at the same time by the same camera are different objects.
 *   SB200_FSTORE_GATE_ANY_SOURCE (2): the windows are disjoint, whatever the sources (cross-camera galleries).
 * merge (CamTrackingAttributes::merge) gives the destination the hull of the two windows; it keeps its source.
 * Semantics on a gated store:
 *   search: an incompatible (query, stored track) pair gives no entries: it does not vote and does not raise max_dist,
 *     the error path of Track::distances (src/track.rs:604-652).  So weights may differ from an ungated search's, as in
 *     the reference.
 *   add: an unknown id creates a track with the row's triple; a known id takes the hull of the windows; a source that
 *     differs from the track's (or from an earlier row's of the same new id) is SB200_ERR_INVALID (WrongCamID).
 *   associate: queries in order; a query is merged into its first winner only if it is compatible with that track's
 *     window as extended by the queries merged into it earlier in the same call; otherwise it becomes a new track with
 *     its own triple.  A merged destination takes the hull.  The reference's merge_external instead returns
 *     IncompatibleAttributes at that point, after merging the queries in front of it (Track::merge,
 *     src/track.rs:522-530): a documented deviation.  It keeps two coexisting queries that win one track apart.
 *   search_owned: each query is gated against every candidate it is scored with, by their stored attributes.
 *   merge_owned: each pair is checked, in order, against the windows the earlier pairs left; an incompatible pair
 *     refuses the whole call (SB200_ERR_INVALID) before anything changes.  A destination takes the hull.
 *   fetch with remove: the attributes leave with their tracks.
 * Refusals, SB200_ERR_INVALID with sb200_last_error naming the cause, decided before anything changes: the plain add /
 * search / associate (and their _device forms) on a gated store; an _attr call on an ungated store; t_start > t_end;
 * sb200_fstore_associate_wasted on a gated store (the tracker keeps no birth epoch, so a wasted record has no exact
 * window).  The host keeps no copy of the attributes: a call reads back those of the tracks it touches only. */
#define SB200_FSTORE_GATE_NONE 0
#define SB200_FSTORE_GATE_SAME_SOURCE 1
#define SB200_FSTORE_GATE_ANY_SOURCE 2
/* Sets the rule.  Allowed while the store holds no tracks (also after sb200_fstore_fetch with remove emptied it), as
 * sb200_fstore_set_storage_type.  SB200_ERR_INVALID, changing nothing, for an unknown rule or a store that holds tracks.
 * A loaded store has its blob's rule. */
int sb200_fstore_set_gate(sb200_fstore* s, int32_t rule);
int sb200_fstore_get_gate(sb200_fstore* s, int32_t* out);
/* One triple per row (add) or per query (search / associate): host arrays. */
typedef struct {
  const uint64_t* source;
  const int64_t* t_start;
  const int64_t* t_end;
} sb200_fstore_attrs;
/* sb200_fstore_add / _search / _associate of a gated store.  Exactly one of `features` (host) and `d_features` (device,
 * with `cuda_stream` as for the _device forms) is non-NULL; either is in the type set by sb200_fstore_set_feature_type.
 * Outputs as for the calls without attributes. */
int sb200_fstore_add_attr(sb200_fstore* s, int32_t n, const uint64_t* ids, const sb200_fstore_attrs* attrs,
                          const float* features, const void* d_features, void* cuda_stream);
int sb200_fstore_search_attr(sb200_fstore* s, int32_t n_queries, const uint64_t* query_ids, const int32_t* obs_offsets,
                             const sb200_fstore_attrs* attrs, const float* features, const void* d_features,
                             int32_t* counts, uint64_t* winners, double* weights, void* cuda_stream);
int sb200_fstore_associate_attr(sb200_fstore* s, int32_t n_queries, const uint64_t* query_ids,
                                const int32_t* obs_offsets, const sb200_fstore_attrs* attrs, const float* features,
                                const void* d_features, int32_t* counts, uint64_t* winners, double* weights,
                                uint64_t* track_ids, uint8_t* merged, void* cuda_stream);
/* The triples of the tracks `ids` of a gated store (0 in every column for an id that is not stored).  Returns how many of
 * the ids were found, or a negative status. */
int64_t sb200_fstore_fetch_attr(sb200_fstore* s, int32_t n, const uint64_t* ids, uint64_t* source, int64_t* t_start,
                                int64_t* t_end);

/* ---- voting: TopNVoting or BestFitVoting on top of the store's distances ----
 * The reference's TrackStore leaves the voting to its caller (foreign_track_distances -> any Voting::winners).  The
 * store has the two built-in rules of src/track/voting:
 *   SB200_FSTORE_VOTING_TOPN (0, the default): TopNVoting (topn.rs:74-138), each query ranked on its own, as every call
 *     above describes.  Several queries of one associate call whose first winner is the same track are all merged
 *     into it.
 *   SB200_FSTORE_VOTING_BEST_FIT (1): BestFitVoting (best.rs:52-128), the rule of the reference's VisualVoting.  Groups,
 *     votes, min_votes, max_distance, max_dist and the f64 weights are TopN's.  Every group of the call that reaches
 *     min_votes is an element; elements are ordered by weight descending, then query (call order) ascending, then store
 *     position ascending (the reference sorts stably over HashMap order, which leaves ties open; this order is the
 *     store's own).  An element wins its track iff no earlier element names that track: the heaviest group naming a
 *     track takes it, the lowest query on ties.  All groups claim, also those past a query's topn cut.
 *     - search, search_owned (each == 0) and the search part of every associate: counts[q] and the weights are TopN's
 *       (q's elements in order, at most topn); the winner of an element that does not win its track is the query's own
 *       id (best.rs:112-120).
 *     - associate in every form, associate_store and associate_wasted: a query is merged into its first element's track
 *       iff that element wins it; otherwise it becomes a new track under its own id, as the reference's callers read a
 *       winner equal to the query (examples/middleware_sort_tracker.rs:76-81).  So no two queries of one call merge into
 *       one track, and merged[q] can be 0 with counts[q] > 0.  On a gated store every destination is exclusive and every
 *       scored pair compatible, so the gate keeps each of them.
 *     - search_owned with each == 1: one voting call per query, where BestFit gives TopN's results.
 *   The claims cost two more passes over the call's distance matrix, which sb200_fstore_last_stage_ms counts in the
 *   voting stage.  Quality stores, feature classes, storage, feature and column types and gates work unchanged.
 * The rule is handle state, like the feature type: it decides how a call reads the store, not what the store holds, so
 * it may be changed at any time and is not saved in the blob (every blob is what it was); a new or loaded store votes
 * TopN.  sb200_fstore_associate_store votes with dst's rule.  No per-call argument. */
#define SB200_FSTORE_VOTING_TOPN 0
#define SB200_FSTORE_VOTING_BEST_FIT 1
/* SB200_ERR_INVALID, changing nothing, for an unknown rule. */
int sb200_fstore_set_voting(sb200_fstore* s, int32_t rule);
int sb200_fstore_get_voting(sb200_fstore* s, int32_t* out);

/* ---- retention by quality: each track keeps its best observations, and its capacity grows with its merges ----
 * The store semantics of examples/track_merging.rs (its `optimize`, :279-297, with the defaults of :257-265) in place of
 * the newest K of benches/feature_tracker.rs:
 *   SB200_FSTORE_KEEP_NEWEST (0, the default): every track keeps its newest K observations; every call behaves as it
 *     always has, and the store saves as version 1 or 2.
 *   SB200_FSTORE_KEEP_BEST_QUALITY (1): every observation carries an f32 quality (the example's observation attribute,
 *     e.g. VisualSortObservation.feature_quality) and every track a merge history (Track::get_merge_history): [id] when
 *     the track is created (add of an unknown id, a query that becomes a new track), to which every merge appends the
 *     source's whole history (Track::merge with merge_history = true, src/track.rs:522-588): associate merging a query
 *     into its winner, and each merge_owned pair.  A source left in the store keeps its history.  A track of history
 *     length h holds at most
 *       c(h) = min(K, (u64)((float)initial_capacity * powf(merge_extension, (float)h)))
 *     observations, f32 arithmetic and a truncating cast as Rust's `as u64`; the host tabulates c(h) with the C
 *     library's powf (which Rust's f32::powf calls on Linux) up to the first h with c(h) == K, and the device never
 *     evaluates powf.  After a row is appended (add) or a merge concatenates dest ++ src, the track's list is stably
 *     sorted by quality, descending (equal qualities keep their order: dest's rows first, then src's; -0.0 == +0.0), and
 *     truncated to c(h) at the destination's new h.  Merges of one call are applied in order, each at its own c(h): a
 *     row dropped by an earlier merge does not come back.  A query of search / associate is a fresh track (h = 1): its
 *     best c(1) rows in quality order (ties to the earlier row) take part, and entries are enumerated in that order, so
 *     the f64 weights follow it.  Stored tracks are searched in their order, best first.
 * Calls on a quality store: sb200_fstore_add_quality, _search_quality and _associate_quality (the plain, _device and
 * _attr forms are refused; the _quality forms are refused on a newest store); search_owned and merge_owned as always,
 * with the rule above for merge_owned; sb200_fstore_fetch returns each track's rows in its order, best first, and
 * sb200_fstore_fetch_quality their qualities too.  A gated quality store decides every associate destination as a gated
 * store does, then applies the quality merge.  sb200_fstore_associate_wasted on a quality store is refused, changing
 * nothing (the tracker's feature history keeps no quality).
 * Refusals, SB200_ERR_INVALID with sb200_last_error naming the cause, decided on the host before anything changes: a NaN
 * quality (the reference panics on it, partial_cmp().unwrap()); in sb200_fstore_set_retention an unknown rule, a store
 * that holds tracks, initial_capacity < 1, a merge_extension that is not finite or is below 1, and parameters whose
 * capacity has not reached K by h = 65536 unless merge_extension == 1 (a constant capacity) -- values the reference
 * would accept. */
#define SB200_FSTORE_KEEP_NEWEST 0
#define SB200_FSTORE_KEEP_BEST_QUALITY 1
/* Sets the rule and its parameters (the example's defaults are 4 and 1.5; ignored for SB200_FSTORE_KEEP_NEWEST).
 * Allowed while the store holds no tracks, as sb200_fstore_set_gate.  A loaded store has its blob's. */
int sb200_fstore_set_retention(sb200_fstore* s, int32_t rule, int32_t initial_capacity, float merge_extension);
/* Any output may be NULL. */
int sb200_fstore_get_retention(sb200_fstore* s, int32_t* rule, int32_t* initial_capacity, float* merge_extension);
/* sb200_fstore_add / _search / _associate of a quality store.  quality: host memory, one value per row of the feature
 * column (n for add, obs_offsets[n_queries] for search / associate).  attrs: a gated store's triples, NULL on an ungated
 * store.  Exactly one of `features` (host) and `d_features` (device, with `cuda_stream` as for the _device forms) is
 * non-NULL; either is in the type set by sb200_fstore_set_feature_type.  Outputs as for the calls without quality. */
int sb200_fstore_add_quality(sb200_fstore* s, int32_t n, const uint64_t* ids, const float* quality,
                             const sb200_fstore_attrs* attrs, const float* features, const void* d_features,
                             void* cuda_stream);
int sb200_fstore_search_quality(sb200_fstore* s, int32_t n_queries, const uint64_t* query_ids,
                                const int32_t* obs_offsets, const float* quality, const sb200_fstore_attrs* attrs,
                                const float* features, const void* d_features, int32_t* counts, uint64_t* winners,
                                double* weights, void* cuda_stream);
int sb200_fstore_associate_quality(sb200_fstore* s, int32_t n_queries, const uint64_t* query_ids,
                                   const int32_t* obs_offsets, const float* quality, const sb200_fstore_attrs* attrs,
                                   const float* features, const void* d_features, int32_t* counts, uint64_t* winners,
                                   double* weights, uint64_t* track_ids, uint8_t* merged, void* cuda_stream);
/* sb200_fstore_fetch of a quality store, plus quality[n][K]: the quality of each returned row (0 past counts[i]). */
int64_t sb200_fstore_fetch_quality(sb200_fstore* s, int32_t n, const uint64_t* ids, int32_t remove, int32_t* counts,
                                   float* features, float* quality);
/* The merge histories of the tracks `ids` of a quality store in CSR form: lengths[i] (0: not stored), and the histories
 * concatenated, in order, into out (at most `cap` entries written; out may be NULL when cap == 0).  Returns their total
 * length, or a negative status. */
int64_t sb200_fstore_merge_history(sb200_fstore* s, int32_t n, const uint64_t* ids, int32_t* lengths, int64_t cap,
                                   uint64_t* out);

/* ---- store to store: the main loop of the reference's examples/track_merging.rs (:371-481) ----
 * A collecting store gathers each tracklet's observations; the tracks that are baked move into a merge store (the
 * gallery), each merged into its winner or added whole.  Both calls run on the device: no stored row, window or quality
 * crosses PCIe. */
/* TrackStore::find_usable (src/track/store.rs:348-374) with the example's `baked` (:240-247) on a gated store: the ids of
 * the tracks with now > t_end + baked_period, compared exactly for every int64 value (the reference compares in u128),
 * in store order.  The first min(cap, total) are written to ids (NULL allowed when cap == 0); returns the total, or a
 * negative status.  One kernel selects on the device; only the count and the selected positions are read back.
 * Deviation: the reference keeps baked_period per track (the example resets it with BakedPeriodUpdate(0) when it
 * promotes a track); here it is an argument of the call, so the store keeps no extra state and its blob is unchanged.
 * There are no Wasted or Err statuses.  SB200_ERR_INVALID, changing nothing: an ungated store (it keeps no windows),
 * cap < 0, ids == NULL with cap > 0. */
int64_t sb200_fstore_find_baked(sb200_fstore* s, int64_t now, int64_t baked_period, int64_t cap, uint64_t* ids);
/* fetch_tracks(ids) of `src`, then one sb200_fstore_associate of `dst` with those tracks as its queries, in the order of
 * ids, each merged into its winner with merge_external(winner, &track, .., true) or added with add_track
 * (examples/track_merging.rs:371-481, Track::merge src/track.rs:522-588).  A query's id is its src id, its rows its kept
 * rows in its own order (a newest store: oldest first; a quality store: best first, with their qualities), widened
 * exactly from src's storage type and rounded to dst's at apply time as any f32 request.  A gated query carries its
 * src source and window, and the gate decides the merges as in sb200_fstore_associate_attr.  On quality stores a query
 * brings its history length h_q and its history: a merge sets h += h_q, merges the two quality lists stably (dst rows
 * first on ties), truncates at c(h) and appends the query's history to the destination's; a new track keeps src's list,
 * h_q and history whole.  Outputs as sb200_fstore_associate.  remove = 1 then takes the queried tracks out of src (a
 * stable compaction, as sb200_fstore_fetch with remove); remove = 0 leaves src unchanged.  The call is synchronous: it
 * reads src's columns on dst's stream once src's stream is idle, and compacts src after dst's work is complete.  On
 * newest stores both stores end exactly as after src.fetch(ids, remove) (+ sb200_fstore_fetch_attr on a gated store)
 * then dst.associate of the fetched rows.  dst and src must be distinct handles on one device with equal feature_dim,
 * max_observations, gate rule, retention rule and retention parameters; storage types, metric, topn and thresholds may
 * differ (they belong to dst's voting).  SB200_ERR_INVALID, before either store changes: a NULL handle, dst == src,
 * a mismatch above, n < 0, remove not 0 or 1, an id given twice, an id not stored in src, an id already stored in dst
 * (the reference's DuplicateTrackId).  SB200_ERR_CAPACITY: more than 2^30 observation pairs (the call is not split,
 * which would change max_dist).  n == 0 changes nothing.  sb200_fstore_last_stage_ms(dst) reports the call's stages. */
int sb200_fstore_associate_store(sb200_fstore* dst, sb200_fstore* src, int32_t n, const uint64_t* ids, int32_t remove,
                                 int32_t* counts, uint64_t* winners, double* weights, uint64_t* track_ids,
                                 uint8_t* merged);

/* ---- the store blob ----
 * The whole store as one relocatable block of bytes: this header, then four sections at 256-byte aligned offsets, gaps
 * zeroed, in this order: ids[live] (u64), cnt[live] (i32 observations held), start[live] (i32 ring slot of the oldest
 * observation), feat[live][max_observations][d8] (rows as stored, in the storage type: 4 or 2 bytes per element;
 * observation j of a track sits in ring slot (start + j) % max_observations).  Ring slots a track has never filled are
 * written as zeros, so two stores that hold the same tracks in the same ring state give byte-equal blobs.  The magic
 * differs from the tracker blob's: each loader refuses the other's blob.  A blob may sit in host memory or in device
 * memory on any device, at any address: a device blob that is not 16-byte aligned, or not on the store's device, goes
 * through a device copy.
 * storage_type was a reserved 0 before 2-byte stores existed, which is SB200_FEATURE_F32: older blobs load unchanged, and
 * an f32 store's blob is what it was.  A library from before 2-byte stores refuses a non-empty 2-byte store's blob by
 * its feat section size (half of what an f32 store needs), so it cannot misread one; an empty 2-byte store's blob has
 * a 0-byte feat section, and such a library loads it as an empty f32 store. */
#define SB200_FSTORE_BLOB_MAGIC 0x53464253u /* "SBFS" */
#define SB200_FSTORE_BLOB_VERSION 1u
#define SB200_FSTORE_BLOB_ALIGN 256u
#define SB200_FSTORE_BLOB_SECTIONS 4
typedef struct {
  uint32_t magic;
  uint32_t version;
  uint64_t total_bytes;
  int32_t metric; /* the fields of sb200_fstore_options, `device` excepted */
  float distance_filter;
  int32_t max_observations;
  int32_t feature_dim;
  int32_t topn;
  float max_distance;
  int32_t min_votes;
  int32_t d8;           /* feature_dim rounded up to a multiple of 8: the stored row length */
  int32_t feature_type; /* the element type set when the blob was written */
  int32_t storage_type; /* the element type of the stored rows and of the feat section */
  int64_t live;         /* stored tracks */
  uint64_t sec_off[SB200_FSTORE_BLOB_SECTIONS];
  uint64_t sec_bytes[SB200_FSTORE_BLOB_SECTIONS];
} sb200_fstore_blob_header;
/* The blob of a gated store: version 2, this header (the version-1 fields through `live`, then the rule), then seven
 * sections laid out as version 1's: ids, cnt, start, feat, then source[live] (u64), t_start[live] and t_end[live] (i64).
 * An ungated store writes version 1, byte for byte as before, and a version-1 blob loads as an ungated store.  A library
 * from before gated stores refuses a version-2 blob by its version check. */
#define SB200_FSTORE_BLOB_VERSION_GATED 2u
#define SB200_FSTORE_BLOB_SECTIONS_V2 7
typedef struct {
  uint32_t magic;
  uint32_t version; /* SB200_FSTORE_BLOB_VERSION_GATED */
  uint64_t total_bytes;
  int32_t metric;
  float distance_filter;
  int32_t max_observations;
  int32_t feature_dim;
  int32_t topn;
  float max_distance;
  int32_t min_votes;
  int32_t d8;
  int32_t feature_type;
  int32_t storage_type;
  int64_t live;
  int32_t gate;      /* SB200_FSTORE_GATE_SAME_SOURCE or _ANY_SOURCE */
  int32_t reserved;  /* 0 */
  uint64_t sec_off[SB200_FSTORE_BLOB_SECTIONS_V2];
  uint64_t sec_bytes[SB200_FSTORE_BLOB_SECTIONS_V2];
} sb200_fstore_blob_header_v2;
/* The blob of a quality store: version 3, this header (the version-2 fields, the retention rule and its parameters),
 * then ten sections laid out as version 1's: ids, cnt, start, feat, source, t_start, t_end (0 bytes each on an ungated
 * store), quality[live][max_observations] (f32, slot by slot as feat, 0 in a slot that holds no observation),
 * history_length[live] (i32, >= 1) and history[sum of history_length] (u64, the histories concatenated in store order,
 * each starting with its track's id).  A newest store writes version 1 or 2 as before.  Load also refuses an unknown
 * rule or bad parameters, a history length of 0, a history whose first id is not its track's id, a history section
 * whose size is not the sum of the lengths, and every state the rule cannot produce: a ring start other than 0, a count
 * above c(history length), and (by kernel) a NaN quality in a filled slot or a list out of quality order.  Empty slots
 * of feat and quality are written as zeros, so two stores holding the same lists and histories give byte-equal blobs. */
#define SB200_FSTORE_BLOB_VERSION_QUALITY 3u
#define SB200_FSTORE_BLOB_SECTIONS_V3 10
typedef struct {
  uint32_t magic;
  uint32_t version; /* SB200_FSTORE_BLOB_VERSION_QUALITY */
  uint64_t total_bytes;
  int32_t metric;
  float distance_filter;
  int32_t max_observations;
  int32_t feature_dim;
  int32_t topn;
  float max_distance;
  int32_t min_votes;
  int32_t d8;
  int32_t feature_type;
  int32_t storage_type;
  int64_t live;
  int32_t gate;             /* SB200_FSTORE_GATE_* (NONE allowed) */
  int32_t retention;        /* SB200_FSTORE_KEEP_BEST_QUALITY */
  int32_t initial_capacity;
  float merge_extension;
  uint64_t sec_off[SB200_FSTORE_BLOB_SECTIONS_V3];
  uint64_t sec_bytes[SB200_FSTORE_BLOB_SECTIONS_V3];
} sb200_fstore_blob_header_v3;
/* The blob of a store of several feature classes, or of one class whose id is not 0: version 4, this header (the
 * version-3 fields, with gate and retention NONE allowed, then n_classes; feature_dim and d8 are the first declared
 * class's), then 8 + 4 * n_classes sections laid out as version 1's:
 *   shared: ids, source, t_start, t_end (0 bytes each on an ungated store), history_length, history (0 bytes each on a
 *   newest store);
 *   the class table: class_ids[n_classes] (u64), class_dims[n_classes] (i32), in declared order;
 *   per class, in declared order: cnt[live], start[live], feat[live][max_observations][d8 of the class] and
 *   quality[live][max_observations] (0 bytes on a newest store).
 * A store of the single class 0 (every store that never declared other classes) writes version 1, 2 or 3 byte for byte
 * as before, and those blobs load as one class of id 0.  Load also refuses a version-4 blob with n_classes outside
 * 1..16, a class id twice or a dim outside 1..8192, and, by kernel, a cnt outside [0, max_observations], a start
 * outside [0, max_observations) or a track without a row in any class; a quality store's checks of version 3 hold per
 * class. */
#define SB200_FSTORE_BLOB_VERSION_CLASSES 4u
#define SB200_FSTORE_BLOB_SECTIONS_V4 (8 + 4 * SB200_FSTORE_MAX_CLASSES)
typedef struct {
  uint32_t magic;
  uint32_t version; /* SB200_FSTORE_BLOB_VERSION_CLASSES */
  uint64_t total_bytes;
  int32_t metric;
  float distance_filter;
  int32_t max_observations;
  int32_t feature_dim;
  int32_t topn;
  float max_distance;
  int32_t min_votes;
  int32_t d8;
  int32_t feature_type;
  int32_t storage_type;
  int64_t live;
  int32_t gate;             /* SB200_FSTORE_GATE_* */
  int32_t retention;        /* SB200_FSTORE_KEEP_* */
  int32_t initial_capacity;
  float merge_extension;
  int32_t n_classes;
  int32_t reserved;         /* 0 */
  uint64_t sec_off[SB200_FSTORE_BLOB_SECTIONS_V4];
  uint64_t sec_bytes[SB200_FSTORE_BLOB_SECTIONS_V4];
} sb200_fstore_blob_header_v4;
/* Writes the blob to `buf` (`cap` bytes; host memory, or device memory on any device) and its size to *bytes.
 * buf == NULL: reports the size and writes nothing.  SB200_ERR_CAPACITY when cap is too small: nothing is written and
 * *bytes is still set.  Rows are copied, not re-derived; the store is not changed.  Timers and the stream are not part
 * of the state.  No counterpart in the reference (its store is not serialisable). */
int sb200_fstore_save(sb200_fstore* s, void* buf, uint64_t cap, uint64_t* bytes);
/* A new store on `device` from a blob (host or device memory).  Exact continuation: fed the same calls, the loaded
 * store returns what the saved one returns (counts, winner ids, f64 weights, track_ids, merged, fetched rows, id order,
 * size).  A damaged blob is refused with SB200_ERR_INVALID before a store exists, sb200_last_error naming the field:
 * magic, version, truncation, section bounds / order / 256-byte alignment / sizes, options outside the caps of
 * sb200_fstore_create, d8 != round_up(feature_dim, 8), an unknown feature_type or storage_type (checked before the
 * section sizes, which depend on it), an id twice, and (by one kernel over the blob, before any row is
 * copied) a cnt outside [1, max_observations] or a start outside [0, max_observations); in a version-2 blob also an
 * unknown gate rule and (by kernel) a stored window with t_start > t_end.  A flipped feature value is not
 * detected: the blob carries no checksum.  A failed load leaves no handle and no device memory behind.  No counterpart
 * in the reference. */
int sb200_fstore_load(const void* buf, uint64_t bytes, int32_t device, sb200_fstore** out);

/* Pinned host memory for callers that want the predict H2D/D2H copies to run at full PCIe speed. */
void* sb200_host_alloc(size_t bytes);
void sb200_host_free(void* p);

#ifdef __cplusplus
}
#endif
#endif
