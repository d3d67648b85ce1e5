/*
 * similari_oracle.h -- CPU ORACLE for Similari's cost-matrix + assignment hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  This is a CPU restatement of the reference's algorithm
 * (insight-platform/Similari, crate similari-trackers-rs v0.26.12) used as the parity
 * checker for the CUDA engine and as the timed CPU baseline ("port") of bench.py.
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
 * legs may load it.  The product (libsimilari_b200.so) never links or calls it.
 *
 * Parity status: the reference is Rust and cannot be compiled in this image (no
 * cargo/rustc), so the oracle is pinned against every known-answer test the reference
 * holds for this path (tests/test_oracle_golden.py lists them with file:line).
 * Unpinned by any reference test (documented in DESIGN.md):
 *   - pathfinding::kuhn_munkres tie-break order (restated from the published algorithm),
 *   - wide::f32x8::reduce_add lane order (irrelevant at 1e-5),
 *   - nms (the reference's only nms test is commented out).
 *
 * All arrays are flat, row-major.  A box is 6 floats: xc, yc, angle, aspect, height,
 * confidence; angle == NaN encodes Option::None.  custom_object_id == INT64_MIN encodes None.
 */
#ifndef SIMILARI_ORACLE_H
#define SIMILARI_ORACLE_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define ORC_POS_MAHA 0
#define ORC_POS_IOU 1
#define ORC_VIS_EUCLIDEAN 0
#define ORC_VIS_COSINE 1
#define ORC_KIND_SORT 0
#define ORC_KIND_BATCH_SORT 1
#define ORC_KIND_VISUAL_SORT 2
#define ORC_KIND_BATCH_VISUAL_SORT 3
#define ORC_VOTING_VISUAL 0
#define ORC_VOTING_POSITIONAL 1
#define ORC_MAX_CONSTRAINTS 8

/* mirrors include/similari_b200.h :: sb200_options field-for-field (kept as a separate
 * declaration so the oracle never includes product headers). */
typedef struct {
  int32_t kind;
  int32_t positional_kind;
  float iou_threshold;
  float min_confidence;
  int32_t max_idle_epochs;
  int32_t history_length;
  float kalman_position_weight;
  float kalman_velocity_weight;
  int32_t n_constraints;
  int32_t constraint_epochs[ORC_MAX_CONSTRAINTS];
  float constraint_max_dist[ORC_MAX_CONSTRAINTS];
  int32_t visual_kind;
  float visual_threshold;
  int32_t feature_dim;
  int32_t visual_max_observations;
  int32_t visual_min_votes;
  int32_t visual_minimal_track_length;
  float visual_minimal_area;
  float visual_minimal_quality_use;
  float visual_minimal_quality_collect;
  float visual_minimal_own_area_percentage_use;
  float visual_minimal_own_area_percentage_collect;
  int32_t max_scenes_hint;
  int32_t max_tracks_per_scene_hint;
  int32_t max_dets_per_scene_hint;
  int32_t device;
} orc_options;

/* ---- geometry: src/utils/bbox.rs, src/utils/clipping.rs ---- */
float orc_radius(const float* box);
int orc_too_far(const float* l, const float* r);
float orc_dist_in_2r(const float* l, const float* r);
void orc_vertices(const float* box, double* out8);
/* returns number of vertices (<= 16) written to out (x,y pairs) */
int orc_sutherland_hodgman_clip(const double* subject, int ns, const double* clip, int nc, double* out);
double orc_polygon_area(const double* poly, int n);
double orc_intersection(const float* l, const float* r);
/* returns 1 and *out when Some, 0 when None */
int orc_iou(const float* l, const float* r, float* out);

/* ---- Kalman: src/utils/kalman/kalman_2d_box.rs ; state = mean[10] + cov[100] (row-major) ---- */
void orc_kalman_initiate(float pw, float vw, const float* box, float* state110);
void orc_kalman_predict(float pw, float vw, const float* in110, float* out110);
void orc_kalman_update(float pw, float vw, const float* in110, const float* box, float* out110);
float orc_kalman_distance(float pw, float vw, const float* state110, const float* box);
float orc_kalman_calculate_cost(float distance, int inverted);
void orc_kalman_state_box(const float* state110, float* box6);

/* ---- feature distances: src/distance.rs (inputs are raw length-d vectors; zero-padded to x8 inside) ---- */
float orc_euclidean(const float* a, const float* b, int d);
float orc_cosine(const float* a, const float* b, int d);

/* ---- cost matrices (dense restatement of the N x M pair loop; NaN == None) ---- */
/* SortMetric::metric, src/trackers/sort/metric.rs:38-77; tracks: boxes6 (+ states110 for maha) */
void orc_sort_cost_matrix(int positional_kind, float iou_threshold, float min_confidence, float pw, float vw,
                          const float* cand_boxes, int m, const float* track_boxes, const float* track_states110,
                          int n, float* out_mn, int threads);
/* visual distances, M x N (one observation per track), NaN == None (threshold applied, weight mapped) */
void orc_visual_cost_matrix(int visual_kind, float threshold, const float* cand_feats, int m,
                            const float* track_feats, int n, int d, float* out_mn, int threads);

/* ---- voting ---- */
/* pathfinding::kuhn_munkres restated; w is rows x cols (rows <= cols); out_row_to_col[rows]; returns total */
int64_t orc_kuhn_munkres(const int64_t* w, int rows, int cols, int32_t* out_row_to_col);
/* COO entries: from/to ids, attr (NaN None), feat (NaN None). Outputs: n winners written as (from,to[,type]) */
int orc_sort_voting(float threshold, int candidates_num, int tracks_num, int n_ent, const uint64_t* from,
                    const uint64_t* to, const float* attr, uint64_t* out_from, uint64_t* out_to);
int orc_bestfit_voting(float max_distance, int min_votes, int n_ent, const uint64_t* from, const uint64_t* to,
                       const float* feat, uint64_t* out_query, uint64_t* out_winner, double* out_weight);
int orc_visual_voting(float positional_threshold, float max_allowed_feature_distance, int min_votes, int n_ent,
                      const uint64_t* from, const uint64_t* to, const float* attr, const float* feat,
                      uint64_t* out_from, uint64_t* out_to, int32_t* out_type);

/* ---- test hooks for the two restatements of the feature distances (scalar lanes / AVX2 vectors), blocks of 8 floats ---- */
float orc_euclidean_scalar(const float* a, const float* b, int blocks);
float orc_cosine_scalar(const float* a, const float* b, int blocks);
float orc_euclidean_blocks(const float* a, const float* b, int blocks);
float orc_cosine_blocks(const float* a, const float* b, int blocks);
int orc_simd_active(void);

/* ---- exclusively owned area shares: src/utils/clipping/bbox_own_areas.rs:8-46 (one scene's boxes) ---- */
int orc_own_area_shares(const float* boxes, int n, float* out);

/* ---- NMS: src/utils/nms.rs:32-72; scores NaN == None; returns kept count, out_idx = input indices in rank order ---- */
int orc_nms(const float* boxes, const float* scores, int n, float nms_threshold, float score_threshold,
            int has_score_threshold, int32_t* out_idx);

/* ---- full trackers (Sort / BatchSort / VisualSort / BatchVisualSort semantics) ---- */
typedef struct orc_tracker orc_tracker;
orc_tracker* orc_tracker_create(const orc_options* o);
void orc_tracker_destroy(orc_tracker* t);
void orc_tracker_set_threads(orc_tracker* t, int threads);
/* same flat request layout as sb200_predict_batch; any out pointer may be NULL */
int orc_tracker_predict_batch(orc_tracker* t, int n_scenes, const uint64_t* scene_ids, const int32_t* det_offsets,
                              const float* boxes, const float* features, const uint8_t* has_feature,
                              const float* quality, const int64_t* custom_ids, const float* own_area,
                              uint64_t* out_ids, uint32_t* out_epochs, uint32_t* out_lengths,
                              uint8_t* out_voting_types, float* out_predicted, float* out_observed);
void orc_tracker_skip_epochs(orc_tracker* t, uint64_t scene_id, int n);
int64_t orc_tracker_current_epoch(orc_tracker* t, uint64_t scene_id);
int orc_tracker_active_tracks(orc_tracker* t);
/* drains wasted store; returns count; arrays sized by cap */
int orc_tracker_wasted(orc_tracker* t, int cap, uint64_t* ids, uint64_t* scene_ids, uint32_t* epochs,
                       uint32_t* lengths, float* predicted, float* observed);
int orc_tracker_idle_tracks(orc_tracker* t, uint64_t scene_id, int cap, uint64_t* ids, uint32_t* epochs,
                            uint32_t* lengths, float* predicted, float* observed);
void orc_tracker_clear_wasted(orc_tracker* t);
/* debugging / parity: dump dense per-scene store (track order == store order) */
int orc_tracker_scene_tracks(orc_tracker* t, uint64_t scene_id, int cap, uint64_t* ids, float* boxes6,
                             float* states110, int32_t* feat_counts);
/* each track's logical observation list Track::obs (store order): n_obs[cap]; per observation [cap][K]: has_feat,
 * quality, the feature zero-padded to d8 (zeros when absent) and its squared norm in the order cosine accumulates it
 * (distance.rs:36-44); entries past n_obs are zero.  Returns the number of tracks written. */
int orc_tracker_scene_observations(orc_tracker* t, uint64_t scene_id, int cap, int K, int d8, int32_t* n_obs,
                                   uint8_t* has_feat, float* quality, float* feats, float* norm2);
/* last frame's per-scene dense cost matrices (positional M x N, NaN none) for parity tests */
int orc_tracker_last_costs(orc_tracker* t, uint64_t scene_id, int cap, float* out, int32_t* m, int32_t* n);

#ifdef __cplusplus
}
#endif
#endif
