// engine.cu -- host side of libsimilari_b200.so: the C ABI of include/similari_b200.h, device memory management
// and the per-frame launch sequence (prep -> positional cost -> visual cost -> voting -> apply).
// There is no CPU execution path in this library: every compute entry point needs a CUDA device.
#include <cuda_runtime.h>

#include <algorithm>
#include <array>
#include <chrono>
#include <cmath>
#include <cstddef>
#include <cstdlib>
#include <cstdio>
#include <cstring>
#include <map>
#include <string>
#include <type_traits>
#include <unordered_map>
#include <utility>
#include <vector>

#include "../../include/similari_b200.h"
#include "sb_blob.cuh"
#include "sb_engine.cuh"
#include "sb_host.cuh"
#include "sb_wstore.cuh"

#include <atomic>

namespace sb {
static std::atomic<unsigned long long> g_launches{0};
void note_launch(int n) { g_launches.fetch_add((unsigned long long)n, std::memory_order_relaxed); }
unsigned long long launch_count() { return g_launches.load(std::memory_order_relaxed); }
}  // namespace sb

using sb::DBuf;
using sb::HBuf;
using sb::fail;

namespace {

// A column of the tracker's device state (sb200_tracker::store_table, slot_table, wasted_table, pool_table): the buffer
// that owns it, the TrackStore / WastedBuf pointer the kernels read it through, and its row width.  `rows` says what a
// row counts, and so how many rows a state-blob section of the column holds: live tracks, arena blocks or free-list
// entries of each listed scene; the records of the wasted buffer; the history blocks handed out or the pool's free stack;
// or, in a scene blob, the history rows of the live tracks.
enum ColRows { kRowTrack, kRowBlock, kRowFree, kRowWasted, kRowHistTop, kRowHistFree, kRowTrackHist };
enum ColBlob { kBlobNo, kBlobAll, kBlobTrackerOnly };
// index-valued columns that a load checks against the blob's counts (kTagHblk: a history block, below the pool's top)
enum ColTag { kTagNone, kTagFblk, kTagHblk, kTagObsN, kTagObsPhys, kTagOwner, kTagFree };
struct Col {
  DBuf* buf;
  void (*point)(sb200_tracker&, void*);   // sets the column's pointer in the TrackStore / WastedBuf (null: there is none)
  size_t w;                                // bytes per row
  bool zero = false;   // growth zero-fills the column: rows moved whole although only partly written (history rings)
  int rows = kRowTrack;
  int blob = kBlobAll;   // which state blobs carry the column
  int tag = kTagNone;
};

int make_params(const sb200_options& o, sb::Params* out) {
  sb::Params p;
  memset(&p, 0, sizeof(p));
  if (o.kind < 0 || o.kind > 3) return fail(SB200_ERR_INVALID, "unknown tracker kind %d", o.kind);
  if (o.positional_kind != SB200_POS_MAHA && o.positional_kind != SB200_POS_IOU)
    return fail(SB200_ERR_INVALID, "unknown positional metric %d", o.positional_kind);
  p.kind = o.kind;
  p.positional_kind = o.positional_kind;
  p.visual_kind = o.visual_kind;
  p.iou_threshold = o.iou_threshold;
  p.min_confidence = o.min_confidence;
  p.pos_weight = o.kalman_position_weight;
  p.vel_weight = o.kalman_velocity_weight;
  p.max_idle_epochs = o.max_idle_epochs;
  if (o.max_idle_epochs < 0) return fail(SB200_ERR_INVALID, "max_idle_epochs must be >= 0");
  if (o.n_constraints < 0 || o.n_constraints > SB200_MAX_CONSTRAINTS)
    return fail(SB200_ERR_INVALID, "at most %d spatio-temporal constraints", SB200_MAX_CONSTRAINTS);
  // SpatioTemporalConstraints::add_constraints: stable sort by epoch, dedup keeping the first
  std::vector<std::pair<int, float>> c;
  for (int i = 0; i < o.n_constraints; ++i) {
    if (!(o.constraint_max_dist[i] > 0.0f))
      return fail(SB200_ERR_INVALID, "The distance is expected to be a positive float");
    // the reference's epochs are usize; compat_ok compares them as unsigned
    if (o.constraint_epochs[i] < 0) return fail(SB200_ERR_INVALID, "constraint epochs must be >= 0");
    c.emplace_back(o.constraint_epochs[i], o.constraint_max_dist[i]);
  }
  std::stable_sort(c.begin(), c.end(), [](const std::pair<int, float>& a, const std::pair<int, float>& b) { return a.first < b.first; });
  c.erase(std::unique(c.begin(), c.end(), [](const std::pair<int, float>& a, const std::pair<int, float>& b) { return a.first == b.first; }), c.end());
  p.n_constraints = (int)c.size();
  for (size_t i = 0; i < c.size(); ++i) { p.constraint_epochs[i] = c[i].first; p.constraint_max_dist[i] = c[i].second; }
  p.is_visual = o.kind == SB200_KIND_VISUAL_SORT || o.kind == SB200_KIND_BATCH_VISUAL_SORT;
  p.is_batch = o.kind == SB200_KIND_BATCH_SORT || o.kind == SB200_KIND_BATCH_VISUAL_SORT;
  if (p.is_visual) {
    if (o.visual_kind != SB200_VIS_EUCLIDEAN && o.visual_kind != SB200_VIS_COSINE)
      return fail(SB200_ERR_INVALID, "unknown visual metric %d", o.visual_kind);
    if (o.feature_dim <= 0) return fail(SB200_ERR_INVALID, "feature_dim must be > 0 for visual trackers");
    if (o.visual_max_observations < 1 || o.visual_max_observations > sb::kMaxObsWide)
      return fail(SB200_ERR_CAPACITY, "visual_max_observations must be in [1, %d]", sb::kMaxObsWide);
    p.visual_threshold = o.visual_threshold;
    p.feature_dim = o.feature_dim;
    p.d8 = (o.feature_dim + 7) / 8 * 8;
    p.vis_rel_err = sb::screen_rel_err(o.feature_dim);
    p.vis_rel_err8 = sb::screen_rel_err_fp8(o.feature_dim);
    p.vis_dense_f32 = sb::dense_f32_err(o.feature_dim);
    p.vis_sample_margin = sb::dense_sample_margin(o.feature_dim);
    p.max_obs = o.visual_max_observations;
    p.min_votes = o.visual_min_votes;
    p.min_track_length = o.visual_minimal_track_length;
    p.min_area = o.visual_minimal_area;
    p.min_quality_use = o.visual_minimal_quality_use;
    p.min_quality_collect = o.visual_minimal_quality_collect;
    p.min_own_use = o.visual_minimal_own_area_percentage_use;
    p.min_own_collect = o.visual_minimal_own_area_percentage_collect;
    p.use_own_area = (o.visual_minimal_own_area_percentage_collect + o.visual_minimal_own_area_percentage_use) > 0.0f;
  } else {
    p.max_obs = 1;
    p.d8 = 8;
  }
  *out = p;
  return 0;
}

}  // namespace

struct sb200_tracker {
  sb200_options opts{};
  sb::Params P{};
  int device = 0;
  // `stream` is the tracker's own work stream.  A caller's stream (sb200_tracker_set_stream) is joined by events: the work
  // of a call is ordered after what the caller's stream held when the call was made, and that stream waits for the call's
  // frame -- the stream-order contract, without the library's kernels sitting in the caller's stream (so the library is free
  // to start the next frame's candidate preparation under the current frame, see prep_stream).
  cudaStream_t stream = nullptr;
  cudaStream_t user_stream = nullptr;   // valid when has_user_stream (0 is the legacy default stream)
  bool has_user_stream = false;
  bool join_per_call = true;   // the caller's stream waits for every call's frame (else: sb200_stream_join)
  cudaEvent_t ev_join_req = nullptr;
  cudaEvent_t ev_user_in = nullptr, ev_user_out = nullptr;
  // candidate preparation (prep + norms / BF16 rows: needs the request only) one frame ahead, on its own stream, into one
  // of two sets of candidate-side buffers
  cudaStream_t prep_stream = nullptr;
  cudaEvent_t ev_prep_done = nullptr, ev_set_free[2]{}, ev_inputs = nullptr;
  cudaEvent_t ev_cost_done = nullptr;   // the cost kernels of the newest frame have been issued up to here (work stream)
  bool cost_done_valid = false;
  bool set_busy[2]{};
  unsigned long long frame_seq = 0;
  float kernel_ms[2]{};    // screen, refine(+mode) of the last absorbed frame
  bool tc_timed = false;
  cudaStream_t copy_stream = nullptr;
  // ---- frames in flight.  predict() is stream-ordered: it enqueues a frame and returns; what only the device knows when
  // the call is made (tracks per scene, ids consumed, expired tracks) is joined in by frame_setup_kernel and read back
  // into the host mirrors when the frame is absorbed -- lazily, by a later call, or by sb200_sync().
  static constexpr int kDepth = 3;
  // What a frame leaves for the host in Pending::h_out: frame_out[n][3] {live tracks, arena blocks, newly expired} and
  // status[n] per scene, then, at back_offset(n), this record.
  struct FrameBack {
    sb::FrameDyn dyn;
    int dense_scenes;   // scenes the exact SIMT kernels had to take (Frame::dense_cnt)
    int hpool[2];       // the history pool's {free, handed out} blocks after the sweep (feature history on only)
    int screen[3];      // screen survivors refined, how many the exact test cut, scenes whose list overflowed
  };
  static_assert(offsetof(FrameBack, dense_scenes) == sizeof(sb::FrameDyn) && sizeof(FrameBack) == sizeof(sb::FrameDyn) + 24,
                "FrameBack: FrameDyn followed by the counters, without padding");
  static size_t back_offset(int n_scenes) { return ((size_t)n_scenes * 16 + 15) / 16 * 16; }
  struct Pending {
    bool active = false;
    int n_scenes = 0, total = 0;
    std::vector<int> slots, m;
    long long live_ub = 0;     // upper bound of the records this frame's sweep appends to the wasted buffer
    HBuf h_req;                // SceneReq[n_scenes], written by the host, read by frame_setup_kernel over PCIe
    HBuf h_out;                // frame_out[n][3] | status[n] | FrameBack, copied back at the end of the frame
    FrameBack* back() const { return reinterpret_cast<FrameBack*>(h_out.as<char>() + back_offset(n_scenes)); }
    cudaEvent_t done = nullptr;
    cudaEvent_t ev[6]{}, ev_k[3]{}, ev_pos[2]{};
    bool tc_timed = false, pos_forked = false;
    int mode = 0;              // visual cost path of the frame: 0 none / exact SIMT, 1 screen + refine, 2 dense tensor-core
    bool fp8 = false;          // mode 1 on the e4m3 screen
  } pend[kDepth];
  int pend_head = 0, pend_count = 0;
  std::vector<int> pending_add;   // per slot: detections of the frames in flight (each can add at most that many tracks)
  long long inflight_live_ub = 0;
  int async_rc = 0;
  std::string async_err;
  // cumulative work counters over the absorbed frames (bench.py reads them around its timed region)
  unsigned long long acc_units_mn = 0, acc_units_rows = 0, acc_frames = 0;
  double host_ms_total = 0.0, host_ms_blocked = 0.0;   // wall time inside predict(), and the part of it spent waiting for the device
  unsigned long long host_calls = 0;
  double acc_stage_ms[5]{}, acc_kernel_ms[2]{};
  unsigned long long acc_tc_frames = 0;
  // Screen precision.  The e4m3 screen (twice the tensor rate of BF16) is the default where d8 <= 512; its slack is ~30x
  // the BF16 one, too wide when the threshold sits in the bulk of the distance distribution.  After a frame on it where
  // most survivors failed the exact test, or a survivor list overflowed, the next kFp8Hold screened frames take the BF16
  // screen, then e4m3 is tried again.
  static constexpr int kFp8Hold = 64;
  int fp8_hold = 0;
  // cumulative over the absorbed screened frames: frames on e4m3, frames on BF16, survivors refined, survivors cut
  unsigned long long acc_screen[4] = {0, 0, 0, 0};
  // high-priority side stream: the frame tables and the screen's column metadata beside the candidate preparation, the
  // end-of-frame sweep beside the feature store
  cudaStream_t side_stream = nullptr;
  cudaEvent_t ev_fork[2]{}, ev_join = nullptr;
  float stage_ms[5]{};
  // scene table
  std::unordered_map<uint64_t, int> slot_of;
  std::vector<uint64_t> scene_of_slot;
  std::vector<uint32_t> epoch;      // host epoch db
  std::vector<int> n_tracks;        // host mirror: live tracks per slot (expired tracks leave the device store every frame)
  std::vector<int> n_hidden;        // expired tracks per slot swept early and not yet collected in the reference's sense
  std::vector<int> arena_top;       // host mirror: feature blocks handed out per slot (rows the screen scans = top * K)
  std::vector<uint64_t> last_req_scenes;   // scene ids of the previous request and their slots (steady-state fast path)
  std::vector<int> last_req_slots;
  int64_t revealed = 0;             // wasted-buffer records [0, revealed) are collected; [revealed, wasted_count) hidden
  int scene_cap = 0, track_cap = 0;
  DBuf b_idc;                       // device id counter (ids consumed so far)
  int auto_waste_counter = 100, auto_waste_periodicity = 100;
  int64_t wasted_count = 0;
  // device track store
  sb::TrackStore ts{};
  DBuf b_id, b_epoch, b_length, b_custom, b_vt, b_pred, b_obs, b_radius, b_kst, b_vert, b_hpred, b_hobs, b_feat, b_feat_bf16, b_fnorm2, b_obs_phys,
      b_feat_fp8, b_fscale, b_obs_hasf, b_obs_q, b_obs_n, b_feat_cnt, b_fblk, b_blk_owner, b_blk_free;
  DBuf b_ntracks, b_cur_epoch, b_scene_ids, b_nfree, b_atop;
  // wasted
  sb::WastedBuf wb{};
  DBuf w_count, w_id, w_scene, w_epoch, w_length, w_pred, w_obs, w_hpred, w_hobs;
  int hist_len = 1;   // boxes of history kept per track (1: only the last ones, the SortTrack columns)
  // feature history of the visual trackers (sb200_set_feature_history): hist_len features per track in a pool of history
  // blocks (TrackStore::hblk ...), owned by the live track, then by its wasted record until the record is collected
  bool fhist_on = false;
  DBuf b_hblk, b_hrows, b_hpresent, b_hfree, b_hpool, w_hblk, f_histdst;
  long long hpool_cap = 0;    // blocks the pool can hold
  long long hpool_top = 0;    // blocks ever handed out, as of the last absorbed frame (exact when nothing is in flight)
  long long hpool_free = 0;   // free blocks, as of the last absorbed frame or the last collection (exact likewise)
  long long hpool_pend = 0;   // detections of the frames in flight (each can take at most one block)
  // frame buffers
  // The input columns of a request.  Each has a staging buffer in both sets (Staging::col), a Frame field the kernels
  // read it through and a row width; only visual trackers read the feature-side ones, and has_feature only with features.
  enum InColumn { kBoxes, kFeat, kHasf, kQuality, kCustom, kOwn, kInCols };
  using InPtrs = std::array<const void*, kInCols>;
  InPtrs in_ptrs(const void* boxes, const void* feat, const void* hasf, const void* quality, const void* custom,
                 const void* own) const {
    if (!P.is_visual) return {boxes, nullptr, nullptr, nullptr, custom, nullptr};
    return {boxes, feat, feat ? hasf : nullptr, quality, custom, own};
  }
  template <auto F> static void to_frame(sb::Frame& f, const void* p) { f.*F = static_cast<std::remove_reference_t<decltype(f.*F)>>(const_cast<void*>(p)); }
  struct InCol { void (*bind)(sb::Frame&, const void*); size_t w; const char* name; };   // w: bytes per row
  std::array<InCol, kInCols> in_cols() const {
    using F = sb::Frame;
    return {{{to_frame<&F::in_boxes>, 24, "S.boxes"}, {to_frame<&F::in_feat>, (size_t)P.feature_dim * feat_bytes(), "S.feat"},
             {to_frame<&F::in_hasf>, 1, "S.hasf"}, {to_frame<&F::in_quality>, 4, "S.quality"},
             {to_frame<&F::in_custom>, 8, "S.custom"}, {to_frame<&F::in_own>, 4, "S.own"}}};
  }
  // The output columns (sb200_predict_out), device or staged in o_col.
  static constexpr int kOutCols = 6;
  struct OutCol { void* host; void (*bind)(sb::Frame&, const void*); size_t w; const char* name; };
  static std::array<OutCol, kOutCols> out_cols(const sb200_predict_out& o) {
    using F = sb::Frame;
    return {{{o.ids, to_frame<&F::o_ids>, 8, "o_ids"}, {o.epochs, to_frame<&F::o_epochs>, 4, "o_epochs"},
             {o.lengths, to_frame<&F::o_lengths>, 4, "o_lengths"}, {o.voting_types, to_frame<&F::o_vt>, 1, "o_vt"},
             {o.predicted_boxes, to_frame<&F::o_pred>, 24, "o_pred"}, {o.observed_boxes, to_frame<&F::o_obs>, 24, "o_obs"}}};
  }
  // rows of the per-detection frame buffers and of the staging sets: the request's detections, or what the capacity
  // hints allow for (n_scenes 0 when the scene count is not known), so that steady-state frames never reallocate
  long long hint_dets(int n_scenes) const { return (long long)std::max(opts.max_scenes_hint, n_scenes) * opts.max_dets_per_scene_hint; }
  size_t frame_rows(int total, int n_scenes) const { return (size_t)std::max<long long>(std::max(total, 1), hint_dets(n_scenes)); }
  int hint_tracks() const { return opts.max_tracks_per_scene_hint > 0 ? track_cap : 0; }   // the store's rows per scene: hint + pipeline room
  // two input staging sets: sb200_prefetch_inputs() fills one while the kernels of the previous frame read the other
  struct Staging {
    DBuf col[kInCols];
    InPtrs key{};   // the host columns of the prefetch
    int total = -1;
    int type = sb::kFeatF32;   // element type of the prefetched features column
    bool pending = false;   // holds a prefetched request that no predict call has consumed yet
    cudaEvent_t ev = nullptr;
    cudaEvent_t ev0 = nullptr;   // start of the set's prefetch copy (SB200_TRACE timing)
    cudaEvent_t ev_read = nullptr;   // end of the last frame that read this set (a prefetch into it waits for that)
    bool read_pending = false;
  } stg[2];
  int stg_last = 1;   // staging set used by the most recent predict
  struct CandBufs { DBuf box, radius, conf, vert, flags, norm2, bf16, decided, fp8, scale; } cand[2];   // candidate side, two sets
  DBuf f_winner, f_cvt, f_pos, f_vis, f_scenes, f_newcount,
      f_status, f_featdst, f_apprank, f_appmeta, f_frameout, f_excl, f_prewin, f_own, f_ownovf, f_dyn, f_ws, f_tmeta, f_rowinfo, f_slabc, f_slabm, f_slabmask,
      f_dscene, f_maxc, f_maxcval, f_drowb, f_dcolb, f_slabk, f_scene_max, f_tiles, f_pairs, f_colmeta, f_colgeo, f_colb, f_colvalid, f_rowmeta, f_poslist, f_counters, f_visval, f_colsb;
  int num_sms = 132;
  DBuf o_col[kOutCols];
  HBuf h_small;
  bool adapt_dense = false;     // a nominally selective threshold whose survivor lists overflow: treat it as non-selective
  unsigned long long acc_dense_scenes = 0;   // scenes the exact SIMT fallback had to take (over all absorbed frames)
  int last_dense_scenes = 0;
  bool seen_features = false;   // a request has carried feature rows (the feature dimension is fixed from then on)
  // element type of the features column of the calls that follow (sb200_set_feature_type): an input format, not state --
  // each frame copies it at enqueue, and it is not part of the state blob
  int feat_type = sb::kFeatF32;
  size_t feat_bytes() const { return feat_type == sb::kFeatF32 ? 4 : 2; }
  bool transferred = false;     // built by sb200_tracker_load or filled by sb200_scenes_import: holds state without a frame
  int last_n_scenes = 0;   // scenes of the last frame (sb200_last_costs reads its scene table back from the device)

  // The buffers free themselves after this body, so every stream the tracker owns is drained first (a caller's stream,
  // which the tracker only joins, is not).
  ~sb200_tracker() {
    cudaSetDevice(device);
    for (cudaStream_t s : {stream, prep_stream, side_stream, copy_stream}) if (s) cudaStreamSynchronize(s);
    for (auto& g : stg)
      for (cudaEvent_t e : {g.ev, g.ev0, g.ev_read}) if (e) cudaEventDestroy(e);
    for (auto& q : pend) {
      if (q.done) cudaEventDestroy(q.done);
      for (auto& e : q.ev) if (e) cudaEventDestroy(e);
      for (auto& e : q.ev_k) if (e) cudaEventDestroy(e);
      for (auto& e : q.ev_pos) if (e) cudaEventDestroy(e);
    }
    if (copy_stream) cudaStreamDestroy(copy_stream);
    if (side_stream) cudaStreamDestroy(side_stream);
    if (prep_stream) cudaStreamDestroy(prep_stream);
    for (cudaEvent_t e : {ev_user_in, ev_user_out, ev_prep_done, ev_set_free[0], ev_set_free[1], ev_inputs, ev_join_req, ev_cost_done}) if (e) cudaEventDestroy(e);
    for (auto& e : ev_fork) if (e) cudaEventDestroy(e);
    if (ev_join) cudaEventDestroy(ev_join);
    if (stream) cudaStreamDestroy(stream);
  }

  template <auto F> static void in_ts(sb200_tracker& t, void* p) { t.ts.*F = static_cast<std::remove_reference_t<decltype(t.ts.*F)>>(p); }
  template <auto F> static void in_wb(sb200_tracker& t, void* p) { t.wb.*F = static_cast<std::remove_reference_t<decltype(t.wb.*F)>>(p); }

  // The device track store: scene_cap x track_cap rows per column, in blob order.
  std::vector<Col> store_table() {
    using TS = sb::TrackStore;
    const size_t K = (size_t)P.max_obs, d8 = (size_t)P.d8, H = (size_t)hist_len;
    std::vector<Col> c = {{&b_id, in_ts<&TS::id>, 8}, {&b_epoch, in_ts<&TS::epoch>, 4}, {&b_length, in_ts<&TS::length>, 4},
                          {&b_custom, in_ts<&TS::custom>, 8}, {&b_vt, in_ts<&TS::vt>, 1}, {&b_pred, in_ts<&TS::pred>, 24},
                          {&b_obs, in_ts<&TS::obs>, 24}, {&b_radius, in_ts<&TS::radius>, 4},
                          {&b_kst, in_ts<&TS::kst>, 4 * (size_t)sb::kStateStride}};
    if (P.positional_kind == SB200_POS_IOU) c.push_back({&b_vert, in_ts<&TS::vert>, 64});
    if (H > 1) {
      c.push_back({&b_hpred, in_ts<&TS::hist_pred>, 24 * H, true});
      c.push_back({&b_hobs, in_ts<&TS::hist_obs>, 24 * H, true});
    }
    if (P.is_visual) {
      c.push_back({&b_obs_phys, in_ts<&TS::obs_phys>, K, false, kRowTrack, kBlobAll, kTagObsPhys});
      c.push_back({&b_obs_hasf, in_ts<&TS::obs_hasf>, K});
      c.push_back({&b_obs_q, in_ts<&TS::obs_q>, 4 * K});
      c.push_back({&b_obs_n, in_ts<&TS::obs_n>, 1, false, kRowTrack, kBlobAll, kTagObsN});
      c.push_back({&b_feat_cnt, in_ts<&TS::feat_cnt>, 1});
      c.push_back({&b_fblk, in_ts<&TS::fblk>, 4, false, kRowTrack, kBlobAll, kTagFblk});
      // the history pool is not indexed by slot: only the tracks' block indices move with the store.  A scene blob carries
      // the history rows themselves (renumbered on import), a tracker blob the pool and the indices.
      if (fhist_on) c.push_back({&b_hblk, in_ts<&TS::hblk>, 4, false, kRowTrack, kBlobTrackerOnly, kTagHblk});
      // zeroed: a block's rows past its track's observations are in the blob, and a full BF16 conversion reads them
      c.push_back({&b_feat, in_ts<&TS::feat>, 4 * K * d8, true, kRowBlock});
      c.push_back({&b_feat_bf16, in_ts<&TS::feat_bf16>, 2 * K * d8, true, kRowBlock});
      c.push_back({&b_fnorm2, in_ts<&TS::fnorm2>, 4 * K, false, kRowBlock});
      // the e4m3 copies: only the A-stationary screen (d8 <= 512) reads them.  Not in the blob: a load converts the f32
      // rows again (regen_fp8).
      if (P.d8 <= sb::kFp8MaxD8) {
        c.push_back({&b_feat_fp8, in_ts<&TS::feat_fp8>, K * sb::fp8_pitch(P.d8), false, kRowBlock, kBlobNo});
        c.push_back({&b_fscale, in_ts<&TS::fscale>, 4 * K, false, kRowBlock, kBlobNo});
      }
      c.push_back({&b_blk_owner, in_ts<&TS::blk_owner>, 4, false, kRowBlock, kBlobAll, kTagOwner});
      c.push_back({&b_blk_free, in_ts<&TS::blk_free>, 4, false, kRowFree, kBlobAll, kTagFree});
    }
    return c;
  }

  // per-slot arrays (scene_cap rows; not in the blob): live tracks, the epochs and scene ids run_waste uploads, free
  // blocks, arena top
  std::vector<Col> slot_table() {
    using TS = sb::TrackStore;
    return {{&b_ntracks, nullptr, 4, true}, {&b_cur_epoch, nullptr, 4, true}, {&b_scene_ids, nullptr, 8, true},
            {&b_nfree, in_ts<&TS::n_free>, 4, true}, {&b_atop, in_ts<&TS::arena_top>, 4, true}};
  }

  // the wasted-track buffer: one row per record, in blob order
  std::vector<Col> wasted_table() {
    using WB = sb::WastedBuf;
    const size_t H = (size_t)hist_len;
    std::vector<Col> c = {{&w_id, in_wb<&WB::id>, 8, false, kRowWasted}, {&w_scene, in_wb<&WB::scene>, 8, false, kRowWasted},
                          {&w_epoch, in_wb<&WB::epoch>, 4, false, kRowWasted}, {&w_length, in_wb<&WB::length>, 4, false, kRowWasted},
                          {&w_pred, in_wb<&WB::pred>, 24, false, kRowWasted}, {&w_obs, in_wb<&WB::obs>, 24, false, kRowWasted}};
    if (H > 1) {
      c.push_back({&w_hpred, in_wb<&WB::hist_pred>, 24 * H, false, kRowWasted});
      c.push_back({&w_hobs, in_wb<&WB::hist_obs>, 24 * H, false, kRowWasted});
    }
    if (fhist_on) c.push_back({&w_hblk, in_wb<&WB::hblk>, 4, false, kRowWasted, kBlobAll, kTagHblk});
    return c;
  }

  // the feature-history pool (only with the feature history on): one row per block, in blob order
  std::vector<Col> pool_table() {
    using TS = sb::TrackStore;
    const size_t H = (size_t)hist_len;
    return {{&b_hrows, in_ts<&TS::hrows>, H * (size_t)P.d8 * 4, false, kRowHistTop},
            {&b_hpresent, in_ts<&TS::hpresent>, H, true, kRowHistTop},
            {&b_hfree, in_ts<&TS::hfree>, 4, false, kRowHistFree, kBlobAll, kTagHblk}};
  }

  // Re-creates column `b` with `groups` x `rows` rows of `w` bytes, keeping the first `old_rows` rows of each of the first
  // `old_groups` groups (old pitch: `old_rows` rows).  Allocate, zero-fill if asked, copy, synchronise, free the old one.
  int regrow(DBuf& b, size_t w, size_t groups, size_t rows, size_t old_groups, size_t old_rows, bool zero) {
    const size_t bytes = std::max<size_t>(1, groups * rows * w);
    DBuf nb;
    int rc = nb.ensure(bytes);
    if (rc) return rc;
    if (zero) CU(cudaMemsetAsync(nb.p, 0, bytes, stream));
    if (b.p && old_groups > 0 && old_rows > 0) {
      if (old_groups == 1)   // one contiguous run: a plain copy, which has no pitch limit
        CU(cudaMemcpyAsync(nb.p, b.p, old_rows * w, cudaMemcpyDeviceToDevice, stream));
      else
        CU(cudaMemcpy2DAsync(nb.p, rows * w, b.p, old_rows * w, old_rows * w, old_groups, cudaMemcpyDeviceToDevice, stream));
      CU(cudaStreamSynchronize(stream));
    }
    b = std::move(nb);
    return 0;
  }

  // Grows every column of `cols` (see regrow) and re-points it.  One column at a time: memory peaks at the old columns
  // plus one, where allocating all first would hold two whole stores at once.
  int grow(const std::vector<Col>& cols, size_t groups, size_t rows, size_t old_groups, size_t old_rows) {
    for (const Col& c : cols) {
      // Rows and row tails that no kernel has written yet travel in the state blob (the squared norms of a block's unused
      // rows, the history rings of a short wasted record): every column a blob carries starts zeroed, so that trackers in
      // the same state give the same blob whatever the allocation held before.
      const int rc = regrow(*c.buf, c.w, groups, rows, old_groups, old_rows, c.zero || c.blob != kBlobNo);
      if (rc) return rc;
      if (c.point) c.point(*this, c.buf->p);
    }
    return 0;
  }

  // The e4m3 copies of the feature rows are not part of the state blob: after a load / import they are converted again from
  // the f32 rows of the arena blocks [0, top) of each listed slot (one launch per slot).
  int regen_fp8(int slot, int top) {
    if (!ts.feat_fp8 || top <= 0) return 0;
    const long long r0 = (long long)slot * track_cap * P.max_obs, rows = (long long)top * P.max_obs;
    sb::launch_to_fp8(ts.feat + r0 * P.d8, P.d8, P.d8, P.d8, rows, ts.feat_fp8 + r0 * sb::fp8_pitch(P.d8), ts.fscale + r0, stream);
    return cudaGetLastError() == cudaSuccess ? 0 : fail(SB200_ERR_CUDA, "e4m3 row conversion failed");
  }

  // The BF16 rows the e4m3 frames skip (sb::Frame::skip_bf16).  Each such frame appends the rows it stores to a log of
  // row indices; past its capacity every arena row counts as stale.  regen_bf16 converts them, in stream order, before
  // anything reads the BF16 rows or the row indices change: a frame on the BF16 screen or the dense path, a blob, a regrow
  // of the store.  The host decides a frame's precision while earlier frames are in flight: stream order alone makes the
  // rows those frames store part of the conversion, with no wait for the device.
  static constexpr long long kBf16LogCap = 1 << 18;
  DBuf b_bf16log;
  long long bf16_log_n = 0;     // entries in the log (each e4m3 frame adds one per detection, -1 where nothing is stored)
  bool bf16_stale_all = false;  // the log overflowed
  int regen_bf16() {
    if (bf16_stale_all) sb::launch_bf16_regen(ts, P.d8, P.max_obs, nullptr, 0, scene_cap, stream);
    else if (bf16_log_n > 0) sb::launch_bf16_regen(ts, P.d8, P.max_obs, b_bf16log.as<int>(), bf16_log_n, 0, stream);
    else return 0;
    bf16_log_n = 0;
    bf16_stale_all = false;
    return cudaGetLastError() == cudaSuccess ? 0 : fail(SB200_ERR_CUDA, "BF16 row conversion failed");
  }

  // (re)allocates the track store for scene_cap x track_cap rows, preserving the live rows
  int ensure_store(int need_scenes, int need_tracks) {
    if (need_scenes <= scene_cap && need_tracks <= track_cap) return 0;
    int ns = scene_cap, nt = track_cap;
    if (need_scenes > ns) ns = std::max(need_scenes, std::max(4, ns * 2));
    if (need_tracks > nt) nt = std::max(need_tracks, std::max(64, nt * 2));
    int rc = regen_bf16();   // the log's row indices hold for the old row pitch only
    if (rc) return rc;
    rc = grow(store_table(), ns, nt, scene_cap, track_cap);
    if (rc) return rc;
    if (ns != scene_cap && (rc = grow(slot_table(), ns, 1, scene_cap, 1))) return rc;
    ts.kst_stride = sb::kStateStride;
    if (hist_len > 1) ts.hist_len = hist_len;
    scene_cap = ns;
    track_cap = nt;
    ts.track_cap = nt;
    return 0;
  }

  int slot_for(uint64_t scene_id, bool create) {
    auto it = slot_of.find(scene_id);
    if (it != slot_of.end()) return it->second;
    if (!create) return -1;
    int s = (int)scene_of_slot.size();
    slot_of[scene_id] = s;
    scene_of_slot.push_back(scene_id);
    epoch.push_back(0);
    n_tracks.push_back(0);
    n_hidden.push_back(0);
    arena_top.push_back(0);
    pending_add.push_back(0);
    return s;
  }

  int ensure_wasted(int64_t need) {
    if (need <= wb.cap) return 0;
    int64_t ncap = std::max<int64_t>(need, std::max<int64_t>(1024, (int64_t)wb.cap * 3));
    // wasted records are drained by sb200_wasted; growing preserves the pending ones
    int rc = grow(wasted_table(), 1, (size_t)ncap, 1, (size_t)wasted_count);
    if (rc) return rc;
    if (!w_count.p) {
      if ((rc = w_count.ensure(sizeof(int)))) return rc;
      CU(cudaMemsetAsync(w_count.p, 0, sizeof(int), stream));
    }
    wb.cap = (int)ncap;
    wb.count = w_count.as<int>();
    return 0;
  }

  // TrackerAPI::auto_waste (src/trackers/tracker_api.rs:81-88)
  int run_waste() {
    int n_slots = (int)scene_of_slot.size();
    if (n_slots == 0) return 0;
    int64_t active = 0;
    int max_n = 0;
    for (int v : n_tracks) { active += v; max_n = std::max(max_n, v); }
    if (active == 0) {
      revealed = wasted_count;
      std::fill(n_hidden.begin(), n_hidden.end(), 0);
      return 0;
    }
    int rc = ensure_wasted(wasted_count + active);
    if (rc) return rc;
    if ((rc = h_small.ensure((size_t)n_slots * 16))) return rc;
    unsigned int* he = h_small.as<unsigned int>();
    for (int s = 0; s < n_slots; ++s) he[s] = epoch[s];
    CU(cudaMemcpyAsync(b_cur_epoch.p, he, sizeof(unsigned int) * n_slots, cudaMemcpyHostToDevice, stream));
    CU(cudaStreamSynchronize(stream));
    unsigned long long* hs = h_small.as<unsigned long long>();
    for (int s = 0; s < n_slots; ++s) hs[s] = scene_of_slot[s];
    CU(cudaMemcpyAsync(b_scene_ids.p, hs, sizeof(unsigned long long) * n_slots, cudaMemcpyHostToDevice, stream));
    sb::launch_waste(P, ts, n_slots, b_cur_epoch.as<unsigned int>(), b_scene_ids.as<unsigned long long>(),
                     b_ntracks.as<int>(), wb, max_n, stream);
    CU(cudaGetLastError());
    int* hn = h_small.as<int>();
    CU(cudaStreamSynchronize(stream));
    CU(cudaMemcpyAsync(hn, b_ntracks.p, sizeof(int) * n_slots, cudaMemcpyDeviceToHost, stream));
    int hc = 0;
    CU(cudaMemcpyAsync(&hc, w_count.p, sizeof(int), cudaMemcpyDeviceToHost, stream));
    CU(cudaStreamSynchronize(stream));
    for (int s = 0; s < n_slots; ++s) n_tracks[s] = hn[s];
    wasted_count = hc;
    // this is one of the reference's collection points: everything swept early becomes visible now
    revealed = wasted_count;
    std::fill(n_hidden.begin(), n_hidden.end(), 0);
    return 0;
  }

  // removes the first n records of the wasted buffer (the rest, hidden ones included, shift to the front)
  int drop_wasted_front(int64_t n) {
    if (n <= 0 || !w_count.p) return 0;
    n = std::min(n, wasted_count);
    const int64_t rest = wasted_count - n;
    cudaStream_t st = stream;
    int rc = 0;
    if (fhist_on) {
      // the collected records' history blocks go back on the pool's free list.  Every caller has drained: no frame in
      // flight reads the list, and a block pushed here is handed out only by a frame enqueued after this point.
      int nf = 0;
      CU(cudaMemcpyAsync(&nf, ts.hpool, sizeof(int), cudaMemcpyDeviceToHost, st));
      CU(cudaStreamSynchronize(st));
      CU(cudaMemcpyAsync(ts.hfree + nf, wb.hblk, 4 * (size_t)n, cudaMemcpyDeviceToDevice, st));
      nf += (int)n;
      CU(cudaMemcpyAsync(ts.hpool, &nf, sizeof(int), cudaMemcpyHostToDevice, st));
      CU(cudaStreamSynchronize(st));
      hpool_free = nf;
    }
    if (rest > 0) {
      const std::vector<Col> cols = wasted_table();
      size_t wmax = 0;
      for (const Col& c : cols) wmax = std::max(wmax, c.w);
      DBuf tmp;   // overlapping device-to-device moves are done through a temporary
      if ((rc = tmp.ensure((size_t)rest * wmax))) return rc;
      for (const Col& c : cols) {
        char* base = c.buf->as<char>();
        CU(cudaMemcpyAsync(tmp.p, base + n * c.w, rest * c.w, cudaMemcpyDeviceToDevice, st));
        CU(cudaMemcpyAsync(base, tmp.p, rest * c.w, cudaMemcpyDeviceToDevice, st));
      }
      CU(cudaStreamSynchronize(st));
    }
    int newc = (int)rest;
    CU(cudaMemcpyAsync(w_count.p, &newc, sizeof(int), cudaMemcpyHostToDevice, st));
    CU(cudaStreamSynchronize(st));
    wasted_count = rest;
    revealed = std::max<int64_t>(0, revealed - n);
    return 0;
  }

  // (re)allocates the feature-history pool for exactly `need` blocks (at least 256), preserving the blocks handed out so
  // far [0, hpool_top) and the free list (never longer than that).  Nothing may be in flight.
  int ensure_hpool(long long need) {
    if (need <= hpool_cap) return 0;
    const long long ncap = std::max<long long>(need, 256);
    int rc = grow(pool_table(), 1, (size_t)ncap, 1, (size_t)hpool_top);
    if (rc) return rc;
    hpool_cap = ncap;
    return 0;
  }

  // Adds or drops the feature history: the block index of every store row and wasted record (the entries of those tables
  // tagged kTagHblk), the pool's counters; the pool itself comes with the first frame that needs it (ensure_hpool).  An
  // add that fails drops what it added.
  int set_feature_history(bool on) {
    if (on == fhist_on) return 0;
    CU(cudaSetDevice(device));
    CU(cudaStreamSynchronize(stream));
    fhist_on = true;   // the tables list the history columns while they are added or dropped
    const int rc = on ? add_feature_history() : 0;
    if (on && rc == 0) return 0;
    std::vector<Col> cols = pool_table();
    for (const Col& c : store_table()) if (c.tag == kTagHblk) cols.push_back(c);
    for (const Col& c : wasted_table()) if (c.tag == kTagHblk) cols.push_back(c);
    for (const Col& c : cols) { c.buf->release(); c.point(*this, nullptr); }
    b_hpool.release();
    f_histdst.release();
    ts.hpool = nullptr;
    ts.fhist_len = 0;
    fhist_on = false;
    hpool_cap = hpool_top = hpool_free = hpool_pend = 0;
    return rc;
  }
  int add_feature_history() {
    int rc;
    if ((rc = b_hpool.ensure(2 * sizeof(int)))) return rc;
    CU(cudaMemsetAsync(b_hpool.p, 0, 2 * sizeof(int), stream));
    for (const Col& c : store_table())
      if (c.tag == kTagHblk && scene_cap > 0 && (rc = grow({c}, scene_cap, track_cap, 0, 0))) return rc;
    for (const Col& c : wasted_table())   // no record exists before the first frame
      if (c.tag == kTagHblk && wb.cap > 0 && (rc = grow({c}, 1, wb.cap, 0, 0))) return rc;
    CU(cudaStreamSynchronize(stream));
    ts.hpool = b_hpool.as<int>();
    ts.fhist_len = hist_len;
    return 0;
  }

  int predict(int32_t n_scenes, const uint64_t* scene_ids, const int32_t* det_offsets, const float* boxes,
              const float* features, const uint8_t* has_feature, const float* quality, const int64_t* custom_ids,
              const float* own_area, const sb200_predict_out* out, bool device_io, bool wait);
  int absorb_oldest(bool block);
  int poll();
  int drain(const char* why = nullptr);
  int ens(DBuf& b, size_t need, const char* name = "") {   // ensure() that never reallocates under a frame in flight
    if (need <= b.bytes) return 0;
    static const bool trace_ens = getenv("SB200_TRACE") != nullptr;
    if (trace_ens) fprintf(stderr, "[sb200] %s grows: %zu -> %zu bytes\n", name, b.bytes, need);
    int rc = drain("frame buffer grows");
    if (rc) return rc;
    return b.ensure(need);
  }
  template <class T> int ens(DBuf& b, size_t need, T*& to, const char* name) {   // ... and points `to` at the buffer
    const int rc = ens(b, need, name);
    if (rc == 0) to = static_cast<T*>(b.p);
    return rc;
  }
  static constexpr int kDenseVoteCap = 8192;   // visual entries per scene of the voting kernel on the dense path (power of two)

  struct Request {   // the arguments of one predict call
    int n_scenes = 0, total = 0;
    const uint64_t* scene_ids = nullptr;
    const int32_t* det_offsets = nullptr;
    InPtrs in{};   // input columns (device pointers with device_io), null: not given
    sb200_predict_out out{};
    bool device_io = false, same_req = false;   // same_req (set by check_request): the previous request's scene list
  };
  struct FramePlan {   // what the stages derive from the request and the tracker's state
    // bounds(): upper bounds of what the device sizes exactly (tracks per scene with frames still in flight)
    std::vector<int> m_of, nb_ub;
    int max_m = 0, max_n = 0, max_nb = 0, need_tracks = 0;
    long long live_ub = 0, pos_total = 0, vis_total = 0, col_total = 0, work = 0;
    // plan_frame: the frame's own positional elements, the list totals, the buffer rows, the visual path
    long long pos_ub = 0, posl_total = 0, visl_total = 0;
    size_t T = 0;
    int cset = 0, vote_cap = 0, mstep = 0, cstep = 256;
    bool want_tc = false, want_dense = false, want_fp8 = false;
    // bind_frame: the staging set, whether a prefetch filled it, the lazy positional stage, derived own-area shares
    Staging* sin = nullptr;
    bool prefetched = false, fork = false, derive_own = false;
  };
  // takes a frame's share out of the bounds of the frames in flight (absorbed, or rolled back by a failed enqueue)
  void unbook(Pending& q) {
    for (int s = 0; s < q.n_scenes; ++s) pending_add[q.slots[s]] -= q.m[s];
    inflight_live_ub -= q.live_ub;
    if (fhist_on) hpool_pend -= q.total;
    q.active = false;
    pend_count -= 1;
  }
  // a CUDA failure while the frame is being enqueued takes it out of the ring again (the context is lost anyway)
  struct Rollback { sb200_tracker* t; Pending* q; bool armed; ~Rollback() { if (armed) t->unbook(*q); } };
  // Refuses a malformed request, or one the on-chip assignment solver cannot hold, before any tracker state changes (a
  // drain is allowed).  Sets rq.total and rq.same_req (the slots of the previous request's scene list are reused).
  int check_request(Request& rq) {
    const int n_scenes = rq.n_scenes;
    const uint64_t* scene_ids = rq.scene_ids;
    const int32_t* det_offsets = rq.det_offsets;
    if (n_scenes < 0) return fail(SB200_ERR_INVALID, "n_scenes must be >= 0");
    if (n_scenes > 0 && (!scene_ids || !det_offsets)) return fail(SB200_ERR_INVALID, "scene_ids / det_offsets are NULL");
    rq.total = n_scenes > 0 ? det_offsets[n_scenes] : 0;
    if (n_scenes > 0 && det_offsets[0] != 0) return fail(SB200_ERR_INVALID, "det_offsets[0] must be 0");
    for (int s = 0; s < n_scenes; ++s)
      if (det_offsets[s + 1] < det_offsets[s]) return fail(SB200_ERR_INVALID, "det_offsets must be non-decreasing");
    if (rq.total > 0 && !rq.in[kBoxes]) return fail(SB200_ERR_INVALID, "boxes is NULL");
    int rc = 0;
    // frames that have completed since the last call hand over their results; an error of an earlier asynchronous frame
    // is reported now
    poll();
    if (async_rc) { if ((rc = drain("error of an earlier frame"))) return rc; }
    rq.same_req = (int)last_req_scenes.size() == n_scenes && n_scenes > 0 &&
                memcmp(last_req_scenes.data(), scene_ids, sizeof(uint64_t) * (size_t)n_scenes) == 0;
    if (!rq.same_req && n_scenes > 0) {
      std::unordered_map<uint64_t, int> seen;
      for (int s = 0; s < n_scenes; ++s)
        if (!seen.emplace(scene_ids[s], s).second) return fail(SB200_ERR_INVALID, "scene %llu appears twice in one request", (unsigned long long)scene_ids[s]);
    }
    // the host epochs already count the frames in flight
    for (int s = 0; s < n_scenes; ++s) {
      const int slot = rq.same_req ? last_req_slots[s] : slot_for(scene_ids[s], false);
      if (slot >= 0 && epoch[slot] == UINT32_MAX)
        return fail(SB200_ERR_INVALID, "scene %llu is at the last epoch %u", (unsigned long long)scene_ids[s], UINT32_MAX);
    }
    // the on-chip assignment solver holds a scene's rows and columns in shared memory
    int max_m0 = 0, max_n0 = 0;
    auto fits = [&] {
      max_m0 = max_n0 = 0;
      for (int s = 0; s < n_scenes; ++s) {
        int slot = -1;
        if (rq.same_req) slot = last_req_slots[s];
        else { auto it = slot_of.find(scene_ids[s]); if (it != slot_of.end()) slot = it->second; }
        max_m0 = std::max(max_m0, det_offsets[s + 1] - det_offsets[s]);
        max_n0 = std::max(max_n0, slot >= 0 ? n_tracks[slot] + pending_add[slot] : 0);
      }
      return sb::voting_smem_need(max_m0, max_n0, P.is_visual ? kDenseVoteCap : 0) <= sb::kVotingSmemLimit;
    };
    // the bound counts every detection in flight as a new track: get the exact counts first
    bool ok = fits();
    if (!ok && pend_count > 0) { if ((rc = drain("assignment solver bound"))) return rc; ok = fits(); }
    if (!ok) return fail(SB200_ERR_CAPACITY, "scene too large for the on-chip assignment solver (m=%d, n=%d)", max_m0, max_n0);
    return 0;
  }

  // upper bounds of everything the device will size exactly (tracks per scene with frames still in flight)
  void bounds(const Request& rq, FramePlan& pl) const {
    const int n_scenes = rq.n_scenes, K = P.max_obs;
    pl.m_of.resize(n_scenes);
    pl.nb_ub.resize(n_scenes);
    pl.max_m = pl.max_n = pl.max_nb = pl.need_tracks = 0;
    pl.live_ub = pl.pos_total = pl.vis_total = pl.col_total = pl.work = 0;
    for (int s = 0; s < n_scenes; ++s) {
      const int slot = last_req_slots[s];
      const int m = rq.det_offsets[s + 1] - rq.det_offsets[s];
      const int n = n_tracks[slot] + pending_add[slot];
      pl.m_of[s] = m;
      pl.nb_ub[s] = P.is_visual ? arena_top[slot] + pending_add[slot] : 0;
      pl.live_ub += n;
      pl.pos_total += (long long)m * n;
      if (P.is_visual) pl.vis_total += (long long)m * n * K;
      pl.col_total += ((long long)pl.nb_ub[s] * K + 127) / 128 * 128;
      pl.work += (long long)m * n * K;
      pl.max_m = std::max(pl.max_m, m);
      pl.max_n = std::max(pl.max_n, n);
      pl.max_nb = std::max(pl.max_nb, pl.nb_ub[s]);
      pl.need_tracks = std::max(pl.need_tracks, n + m);
    }
  }

  int reserve_state(const Request& rq, FramePlan& pl) {
    const int n_scenes = rq.n_scenes, total = rq.total;
    int rc = 0;
    bounds(rq, pl);
    // Capacity has to hold the UPPER BOUNDS: with frames in flight every queued detection counts as a possible new track.
    // So the store is sized for the pipeline once -- the caller's hint (or what this frame needs) plus the detections of
    // kDepth frames -- and later frames neither wait for the device nor reallocate.
    const int pipe_room = kDepth * std::max(pl.max_m, opts.max_dets_per_scene_hint);
    int hint_s = std::max((int)scene_of_slot.size(), opts.max_scenes_hint);
    if (hint_s > scene_cap || pl.need_tracks > track_cap) {
      // the store has to grow: meet the device first (the exact counts are the ones to grow from)
      if ((rc = drain("track store bound"))) return rc;
      bounds(rq, pl);
      // grow generously (a regrow copies the whole feature arena: tens of milliseconds): what is needed now plus the
      // pipeline's room, and at least half again as much as before
      const int want_t = std::max(pl.need_tracks, opts.max_tracks_per_scene_hint) + pipe_room;
      if (hint_s > scene_cap || pl.need_tracks > track_cap)
        if ((rc = ensure_store(hint_s, std::max(want_t, track_cap + track_cap / 2)))) return rc;
    }
    // room for every live track of the frames in flight and of this one in the wasted buffer: the end-of-frame sweep
    // appends without a host check
    if (wasted_count + inflight_live_ub + pl.live_ub + 1 > wb.cap) {
      // the bound that failed is the pipeline's (frames in flight + this one): grow for twice that, or the next frame meets
      // the same bound again -- after the wait the exact counts alone would fit and nothing would grow
      const long long pipe_need = inflight_live_ub + pl.live_ub;
      if ((rc = drain("wasted buffer bound"))) return rc;
      bounds(rq, pl);
      // a full ring: kDepth frames in flight plus this one, each bounded by the live tracks plus every detection queued before it
      const long long dets = std::max<long long>(total, hint_dets(n_scenes));
      const long long ring_need = (long long)(kDepth + 1) * (pl.live_ub + (long long)kDepth * dets);
      // and the records already waiting for collection doubled: a caller that collects rarely pays for few regrows
      // and several times that while it is cheap (<= ~2 GB of records): a regrow drains the ring and reallocates
      const long long rec_bytes = 72 + (hist_len > 1 ? 48ll * hist_len : 0);
      const long long base_need = std::max<long long>(ring_need, 2 * pipe_need);
      const long long mult = std::max<long long>(1, std::min<long long>(8, (2ll << 30) / std::max<long long>(1, base_need * rec_bytes)));
      if ((rc = ensure_wasted(2 * wasted_count + mult * base_need + 1))) return rc;
    }
    // Feature-history pool.  New tracks take free blocks first, so the blocks handed out after this frame are at most
    //   top + max(0, detections queued since - free)      (top, free: as of the last absorbed frame or collection).
    // When that bound exceeds the pool, meet the device (the counts become exact) and grow, if needed, to
    //   top + max(0, f * detections of this frame - free),   f = the frames the bound covered (in flight + this one),
    // and at least half again as much as before.  So the pool is at most 1.5 x (live + uncollected wasted tracks + the
    // detections of the frames actually queued together, less the free blocks): a caller that waits for every frame (the
    // Python API) has f = 1, and only a caller that really queues f frames gets room for f frames of new tracks.
    if (fhist_on && total > 0 && hpool_top + std::max<long long>(0, hpool_pend + total - hpool_free) > hpool_cap) {
      const long long frames = pend_count + 1;
      if ((rc = drain("feature history pool bound"))) return rc;   // hpool_top / hpool_free are exact from here on
      const long long want = hpool_top + std::max<long long>(0, frames * total - hpool_free);
      if (want > hpool_cap && (rc = ensure_hpool(std::max<long long>(want, hpool_cap + hpool_cap / 2)))) return rc;
    }
    if (!b_idc.p) {
      if ((rc = b_idc.ensure(8))) return rc;
      CU(cudaMemsetAsync(b_idc.p, 0, 8, stream));
    }
    return 0;
  }

  // The ring slot's host tables, the visual cost path, the scenes' list slices (into the request table) and the sizes.
  int plan_frame(const Request& rq, Pending& q, FramePlan& pl) {
    const int n_scenes = rq.n_scenes, total = rq.total, K = P.max_obs;
    int rc = 0;
    if ((rc = q.h_req.ensure(sizeof(sb::SceneReq) * (size_t)n_scenes)) ||
        (rc = q.h_out.ensure(back_offset(n_scenes) + sizeof(FrameBack))))
      return rc;
    // visual cost path of this frame: tensor-core screen + exact refinement for large frames with a selective threshold, the
    // dense tensor-core weight sums for thresholds that cut nothing, the exact SIMT kernel otherwise (small frames, and as the
    // device-side fallback of single scenes)
    if (P.is_visual && rq.in[kFeat] != nullptr && total > 0) {
      const sb::VisKernel vk = sb::vis_kernel_env();
      const bool selective = sb::vis_selective(P.visual_kind == SB200_VIS_EUCLIDEAN, P.visual_threshold);
      const bool big = sb::vis_tc_worth(P.d8, pl.work);
      // features wider than kDenseMaxD have no proven dense bound (dense_f32_err is infinite): never the dense path
      const bool dense_ok = P.n_constraints == 0 && std::isfinite(P.vis_dense_f32) && std::isfinite(P.vis_sample_margin);
      pl.want_dense = big && dense_ok && (!selective || adapt_dense);
      pl.want_tc = selective && big && !pl.want_dense;
      if (vk == sb::kVisSimt) { pl.want_tc = false; pl.want_dense = false; }
      else if (vk == sb::kVisTc || vk == sb::kVisTc8 || vk == sb::kVisTc16) { pl.want_tc = pl.work > 0; pl.want_dense = false; }
      else if (vk == sb::kVisDense) { pl.want_dense = pl.work > 0 && dense_ok; pl.want_tc = pl.work > 0 && !pl.want_dense; }
      // screen precision (d8 <= 512): e4m3 unless a recent e4m3 frame showed its slack to be too wide; tc8 / tc16 force one
      const bool can8 = pl.want_tc && P.d8 <= sb::kFp8MaxD8 && ts.feat_fp8 != nullptr;
      const bool forced = vk == sb::kVisTc8 || vk == sb::kVisTc16;
      pl.want_fp8 = can8 && (forced ? vk == sb::kVisTc8 : fp8_hold == 0);
      if (!forced && can8 && fp8_hold > 0) fp8_hold -= 1;
    }
    pl.vote_cap = pl.want_dense ? kDenseVoteCap : sb::kVoteVisCap;
    sb::SceneReq* hreq = q.h_req.as<sb::SceneReq>();
    for (int s = 0; s < n_scenes; ++s) {
      sb::SceneReq& r = hreq[s];
      r.slot = last_req_slots[s];
      r.m = pl.m_of[s];
      r.det_base = rq.det_offsets[s];
      r.epoch = epoch[r.slot] + 1;   // EpochDb::next_epoch, src/trackers/epoch_db.rs:35-49 (committed by commit())
      r.scene_id = rq.scene_ids[s];
      r.pos_lbase = (int)pl.posl_total;
      r.pos_lcap = sb::pos_lcap(r.m);
      pl.posl_total += r.pos_lcap;
      r.vis_lbase = (int)pl.visl_total;
      r.vis_lcap = P.is_visual ? sb::vis_lcap(r.m, pl.vote_cap) : 0;
      pl.visl_total += r.vis_lcap;
    }
    // ---- frame buffers (sized once from the capacity hints when given, so steady-state frames never reallocate)
    pl.T = frame_rows(total, n_scenes);
    pl.pos_ub = pl.pos_total;
    const long long hint_pos = hint_dets(n_scenes) * hint_tracks();
    pl.pos_total = std::max(pl.pos_total, hint_pos);
    if (P.is_visual) pl.vis_total = std::max(pl.vis_total, hint_pos * K);
    // candidate-side buffers: the set of this frame (the other one may still be read by the frame in front of it)
    pl.cset = (int)(frame_seq & 1);
    if (!pl.want_tc && !pl.want_dense) return 0;
    pl.mstep = 256;   // a cluster covers two 128-row candidate tiles
    // dense: column tiles end at block boundaries, a track's observations stay together
    pl.cstep = pl.want_dense ? (256 / K) * K : sb::vis_screen_ucols(P.d8, num_sms, n_scenes, pl.m_of.data(), pl.nb_ub.data(), K);
    return 0;
  }

#define ENS(b, ...) ens(b, __VA_ARGS__, #b)
  // Grows the frame buffers (each growth waits for the frames in flight) and points the kernels' arguments at them.
  int bind_frame(const Request& rq, FramePlan& pl, sb::Frame& f, sb::TcArgs& tc) {
    const int n_scenes = rq.n_scenes, total = rq.total, K = P.max_obs;
    const size_t T = pl.T;
    CandBufs& cb = cand[pl.cset];
    int rc = 0;
    if ((rc = ENS(cb.box, T * 24, f.c_box)) || (rc = ENS(cb.radius, T * 4, f.c_radius)) || (rc = ENS(cb.conf, T * 4, f.c_conf)) ||
        (rc = ENS(f_winner, T * 4, f.winner)) || (rc = ENS(f_cvt, T, f.c_vt)) ||
        (rc = ENS(f_scenes, sizeof(sb::SceneDesc) * n_scenes, f.scenes)) || (rc = ENS(f_newcount, 4 * (size_t)n_scenes, f.new_count)) ||
        (rc = ENS(f_dyn, sizeof(sb::FrameDyn), f.dyn)) || (rc = ENS(f_apprank, T * 8, f.app_rank)) ||
        (rc = ENS(f_appmeta, 16 * (size_t)n_scenes, f.app_meta)) || (rc = ENS(f_pos, std::max<size_t>(4, (size_t)pl.pos_total * 4), f.pos)))
      return rc;
    if (P.positional_kind == SB200_POS_IOU && (rc = ENS(cb.vert, T * 64, f.c_vert))) return rc;
    if (P.is_visual) {
      if (fhist_on && (rc = ENS(f_histdst, T * 4, f.hist_dst))) return rc;
      if ((rc = ENS(cb.flags, T, f.c_flags)) || (rc = ENS(cb.norm2, T * 4, f.c_norm2)) || (rc = ENS(f_featdst, T * 4, f.feat_dst)) ||
          (rc = ENS(f_vis, std::max<size_t>(4, (size_t)pl.vis_total * 4), f.vis)) ||
          (rc = ENS(f_scene_max, 4 * (size_t)n_scenes, f.scene_max)))
        return rc;
    }
    tc.num_sms = num_sms;
    const int hint_tr = hint_tracks();
    const long long hs = std::max(opts.max_scenes_hint, n_scenes), visl_alloc = std::max(pl.visl_total, hint_dets(n_scenes) * 64);
    if (pl.want_tc || pl.want_dense) {
      tc.use_tc = true;
      tc.dense = pl.want_dense;
      const int mstep = pl.mstep, cstep = tc.cstep = pl.cstep;
      long long tiles_ub = 0, slabs_ub = 0, ws_ub = 0, blk_ub = 0;
      for (int s = 0; s < n_scenes; ++s) {
        const long long ct = ((long long)pl.nb_ub[s] * K + cstep - 1) / cstep;
        tiles_ub += (long long)((pl.m_of[s] + mstep - 1) / mstep) * ct;
        slabs_ub += ct;
        ws_ub += ct * (cstep / K) * ((pl.m_of[s] + 127) / 128 * 128);   // blocks padded to whole column tiles
        blk_ub += ct * (cstep / K);
      }
      tc.n_tiles = (int)tiles_ub;   // an upper bound: the list is built on the device
      // the tile list is sized from the hints like the other frame buffers (the bound grows with the frames in flight: a
      // list sized for this frame alone would be outgrown, and wait for the device, again and again)
      const long long hd = std::max(opts.max_dets_per_scene_hint, pl.max_m), ht = std::max(hint_tr, pl.max_nb);
      long long tiles_alloc = std::max(tiles_ub, hs * ((hd + mstep - 1) / mstep) * ((ht * K + cstep - 1) / cstep + 1));
      if (f_tiles.bytes > 0 && sizeof(sb::TcTile) * (size_t)tiles_alloc > f_tiles.bytes) tiles_alloc += tiles_alloc / 2;
      // both operand copies of the candidates whenever the e4m3 screen can run: a switch between the precisions must not
      // allocate (and synchronise) in the middle of a stream of frames
      const bool alloc8 = !pl.want_dense && P.d8 <= sb::kFp8MaxD8 && ts.feat_fp8 != nullptr;
      if (alloc8 && ((rc = ENS(cb.fp8, T * sb::fp8_pitch(P.d8))) || (rc = ENS(cb.scale, T * 4)) || (rc = ENS(b_bf16log, kBf16LogCap * 4))))
        return rc;
      if ((rc = ENS(cb.bf16, T * P.d8 * 2)) ||
          (rc = ENS(f_tiles, sizeof(sb::TcTile) * (size_t)std::max<long long>(1, tiles_alloc), tc.d_tiles)) ||
          (rc = ENS(f_rowmeta, sizeof(sb::VisRowMeta) * (T + 256), tc.rowmeta)))
        return rc;
      tc.max_rows = pl.max_nb * K;
      tc.d_n_tiles = &f_dyn.as<sb::FrameDyn>()->n_tiles;
      tc.a_rows = total;
      tc.b_rows = (long long)scene_cap * track_cap * K;
      if (!tc.dense) {
        const size_t cols = (size_t)std::max(pl.col_total, hs * (((long long)hint_tr * K + 127) / 128 * 128));
        if ((rc = ENS(f_colmeta, sizeof(sb::VisColMeta) * (cols + 256), tc.colmeta)) || (rc = ENS(f_colb, 4 * (cols + 256), tc.colb)) ||
            (rc = ENS(f_colvalid, (cols + 256) / 8 + 16, tc.colvalid)) ||
            (rc = ENS(f_colgeo, sizeof(sb::VisColGeo) * std::max<size_t>(1, P.n_constraints > 0 ? cols : 1), tc.colgeo)))
          return rc;
        tc.total_cols = (int)pl.col_total;
        if (alloc8 && P.visual_kind != SB200_VIS_COSINE) {
          if ((rc = ENS(f_colsb, 4 * (cols + 256)))) return rc;
          if (pl.want_fp8) tc.colsb = f_colsb.as<float>();
        }
        tc.fp8 = pl.want_fp8;
      } else {
        // sized from the hints like the other frame buffers, so steady-state frames never reallocate
        const long long hd0 = std::max(opts.max_dets_per_scene_hint, 0);
        ws_ub = std::max(ws_ub, hs * (hint_tr + 256) * ((hd0 + 127) / 128 * 128));
        blk_ub = std::max(blk_ub, hs * (hint_tr + 256));
        slabs_ub = std::max(slabs_ub, hs * (((long long)hint_tr * K + cstep - 1) / cstep + 1));
        const size_t slabs = (size_t)std::max<long long>(1, slabs_ub), blks = (size_t)std::max<long long>(1, blk_ub);
        const size_t visl = (size_t)std::max<long long>(1, visl_alloc);
        if ((rc = ENS(f_drowb, 4 * 5 * T, tc.d_rowb)) || (rc = ENS(f_dcolb, 4 * blks, tc.d_colb)) ||
            (rc = ENS(f_slabk, 4 * 256 * slabs, tc.slab_ktf)) || (rc = ENS(f_ws, 4 * (size_t)std::max<long long>(1, ws_ub), tc.ws)) ||
            (rc = ENS(f_tmeta, sizeof(sb::DenseTrackMeta) * blks, tc.tmeta)) ||
            (rc = ENS(f_rowinfo, 8 * (size_t)std::max<long long>(1, blk_ub * K), tc.rowinfo)) ||
            (rc = ENS(f_slabc, 4 * 256 * slabs, tc.slab_colc)) || (rc = ENS(f_slabm, 4 * 256 * slabs, tc.slab_cmax)) ||
            (rc = ENS(f_slabmask, 2 * 32 * slabs, tc.slab_vmask)) || (rc = ENS(f_dscene, dscene_bytes(n_scenes))) ||
            (rc = ENS(f_maxc, sizeof(sb::VisPair) * visl, tc.maxc)) || (rc = ENS(f_maxcval, 4 * visl, tc.maxc_val)))
          return rc;
        tc.max_blocks = pl.max_nb;
        tc.n_slabs_ub = (int)slabs_ub;
        tc.blk_ub = blk_ub;
        tc.slab_bmask = tc.slab_vmask + (size_t)slabs_ub * 8;
        carve_dscene(f_dscene.p, n_scenes, tc);
      }
    }
    f.total = total;
    f.pos_total = pl.pos_ub;
    f.id_counter = b_idc.as<unsigned long long>();
    f.id_add = P.is_batch ? (long long)total : -1;
    f.dense_bad = tc.dense ? tc.dense_bad : nullptr;
    // dense positional matrices for every scene only on request (SB200_FULL_COSTS: parity of sb200_last_costs)
    f.pos_dense_all = getenv("SB200_FULL_COSTS") != nullptr;
    f.feat_type = feat_type;
    // inputs: the caller's device columns, or a staging set.  A set already filled by sb200_prefetch_inputs() for exactly
    // these host columns is used as is; otherwise enqueue() issues the H2D copies.  Boxes are always staged.
    const std::array<InCol, kInCols> ic = in_cols();
    if (rq.device_io) {
      for (int c = 0; c < kInCols; ++c) ic[c].bind(f, rq.in[c]);
    } else {
      int use = -1;
      for (int k = 0; k < 2; ++k)
        if (stg[k].pending && stg[k].total == total && stg[k].type == feat_type && stg[k].key == rq.in)
          use = k;
      if (use >= 0) {
        pl.prefetched = true;
        stg[use].pending = false;
        CU(cudaStreamWaitEvent(stream, stg[use].ev, 0));
      } else {
        use = stg[0].pending ? 1 : (stg[1].pending ? 0 : 1 - stg_last);
        stg[use].pending = false;
      }
      stg_last = use;
      Staging& S = stg[use];
      pl.sin = &S;
      for (int c = 0; c < kInCols; ++c) {
        if (c != kBoxes && !(rq.in[c] && total > 0)) continue;
        // a filled set smaller than this frame's sizing rule (hints changed?): re-copy instead of reallocating
        if (S.col[c].bytes < T * ic[c].w) pl.prefetched = false;
        if ((rc = ens(S.col[c], T * ic[c].w, ic[c].name))) return rc;
        ic[c].bind(f, S.col[c].p);
      }
    }
    f.new_count_all = f.new_count;
    if ((rc = ENS(f_frameout, sizeof(int) * 3 * (size_t)n_scenes, f.frame_out))) return rc;
    f.c_bf16 = tc.use_tc && !tc.fp8 ? cb.bf16.p : nullptr;
    f.c_fp8 = tc.fp8 ? cb.fp8.as<unsigned char>() : nullptr;
    f.c_scale = tc.fp8 ? cb.scale.as<float>() : nullptr;
    if ((rc = ENS(f_poslist, sizeof(sb::PosEntry) * (size_t)std::max<long long>(1, std::max(pl.posl_total, hint_dets(n_scenes) * 32)), f.pos_list)) ||
        (rc = ENS(f_counters, sizeof(int) * sb::counter_ints(n_scenes))))
      return rc;
    if (P.is_visual && ((rc = ENS(f_pairs, sizeof(sb::VisPair) * (size_t)std::max<long long>(1, visl_alloc), f.vis_pairs)) ||
                        (rc = ENS(f_visval, sizeof(float) * (size_t)std::max<long long>(1, visl_alloc), f.vis_val))))
      return rc;
    sb::carve_counters(f_counters.as<int>(), n_scenes, f);
    if (!tc.use_tc || tc.dense) f.screen_cnt = nullptr;   // only the screen counts its survivors
    // outputs: the caller's device columns, or staged and copied back by enqueue()
    const std::array<OutCol, kOutCols> oc = out_cols(rq.out);
    for (int c = 0; c < kOutCols; ++c) {
      if (!oc[c].host) continue;
      if (rq.device_io) { oc[c].bind(f, oc[c].host); continue; }
      if ((rc = ens(o_col[c], T * oc[c].w, oc[c].name))) return rc;
      oc[c].bind(f, o_col[c].p);
    }
    // Visual trackers on the tensor-core path evaluate the positional metric lazily: VisualVoting only consults it for
    // candidates the visual BestFit pass left undecided, against tracks it did not claim, so the order is
    // screen -> refine -> BestFit pre-pass (masks) -> culled scan of what is still open -> full voting.
    // SB200_FULL_COSTS=1 (every pair is evaluated, sb200_last_costs is complete) keeps the plain order.
    pl.fork = P.is_visual && tc.use_tc && tc.n_tiles > 0 && !f.pos_dense_all;
    if (pl.fork && ((rc = ENS(cb.decided, T, f.decided)) || (rc = ENS(f_excl, (size_t)scene_cap * track_cap + 16, f.excl)) ||
                    (rc = ENS(f_prewin, T * 4, f.pre_winner))))
      return rc;
    pl.derive_own = P.is_visual && P.use_own_area && f.in_own == nullptr && total > 0;
    if (pl.derive_own && ((rc = ENS(f_own, T * 4)) || (rc = ENS(f_ownovf, 16 + T * sizeof(int2))))) return rc;
    return 0;
  }
#undef ENS

  // The scenes' epochs, the ring slot and the in-flight bounds; the guard undoes the slot unless enqueue() completes.
  Rollback commit(const Request& rq, const FramePlan& pl, Pending& q) {
    const int n_scenes = rq.n_scenes;
    for (int s = 0; s < n_scenes; ++s) epoch[last_req_slots[s]] += 1;
    if (rq.in[kFeat] != nullptr && rq.total > 0) seen_features = true;
    frame_seq += 1;
    q.active = true;
    q.n_scenes = n_scenes;
    q.total = rq.total;
    q.slots.assign(last_req_slots.begin(), last_req_slots.end());
    q.m = pl.m_of;
    q.live_ub = pl.live_ub;
    q.tc_timed = false;
    q.pos_forked = false;
    q.mode = pl.want_dense ? 2 : (pl.want_tc ? 1 : 0);
    q.fp8 = pl.want_fp8;
    for (int s = 0; s < n_scenes; ++s) pending_add[last_req_slots[s]] += pl.m_of[s];
    inflight_live_ub += pl.live_ub;
    if (fhist_on) hpool_pend += rq.total;
    pend_count += 1;
    last_n_scenes = n_scenes;
    return Rollback{this, &q, true};
  }

  // The stream joins, input copies, launches (prep -> costs -> voting -> apply -> store / sweep) and the read-back.
  int enqueue(const Request& rq, const FramePlan& pl, Pending& q, sb::Frame& f, sb::TcArgs& tc) {
    const int n_scenes = rq.n_scenes, total = rq.total, max_m = pl.max_m, max_n = pl.max_n, cset = pl.cset;
    sb::Params Pf = P;
    Pf.vote_vis_cap = pl.vote_cap;
    if (has_user_stream) {   // everything the caller's stream holds now comes first
      CU(cudaEventRecord(ev_user_in, user_stream));
      CU(cudaStreamWaitEvent(stream, ev_user_in, 0));
    }
    if (!rq.device_io && !pl.prefetched && total > 0) {
      const std::array<InCol, kInCols> ic = in_cols();
      for (int c = 0; c < kInCols; ++c)
        if (rq.in[c]) CU(cudaMemcpyAsync(pl.sin->col[c].p, rq.in[c], (size_t)total * ic[c].w, cudaMemcpyHostToDevice, stream));
    }
    if (q.fp8 && f.in_feat) {
      f.skip_bf16 = true;
      if (!bf16_stale_all && bf16_log_n + total <= kBf16LogCap) {
        f.bf16_log = b_bf16log.as<int>() + bf16_log_n;
        bf16_log_n += total;
      } else {
        bf16_stale_all = true;
      }
    } else if (tc.use_tc && !tc.fp8) {   // the BF16 screen or the dense path reads the BF16 rows
      if (const int rc = regen_bf16()) return rc;
    }
    const bool prep_ahead = !pl.derive_own && total > 0;
    // The frame's tables (scene descriptors, tile list, frame scalars; counters zeroed) come from one small CTA: with no
    // own-area derivation (which reads them) it runs on the side stream beside the candidate preparation -- on the work
    // stream it would move the next frame's preparation under the screen kernel -- and the main stream joins later.
    const bool side_setup = !pl.derive_own && total > 0;
    cudaStream_t s_setup = stream;
    if (side_setup) {
      CU(cudaEventRecord(ev_fork[0], stream));
      CU(cudaStreamWaitEvent(side_stream, ev_fork[0], 0));
      s_setup = side_stream;
    }
    sb::launch_frame_setup(P, ts, f, reinterpret_cast<const sb::SceneReq*>(q.h_req.dp), n_scenes, b_ntracks.as<int>(), pl.mstep,
                           pl.cstep, tc.dense, f_tiles.as<sb::TcTile>(), f_dyn.as<sb::FrameDyn>(), f_counters.as<int>(),
                           (int)sb::counter_ints(n_scenes), s_setup);
    tc.max_init_done = 1;   // frame_setup resets scene_max
    if (side_setup && Pf.is_visual && tc.use_tc && !tc.dense && tc.n_tiles > 0 && max_m > 0 && max_n > 0 && f.in_feat) {
      // the screen's column metadata reads the tables and the store only: it follows the setup on the side stream
      sb::launch_vis_colmeta(Pf, ts, f, n_scenes, max_n, tc, side_stream);
      tc.colmeta_done = 1;
    }
    if (side_setup) CU(cudaEventRecord(ev_join, side_stream));
    CU(cudaEventRecord(q.ev[0], stream));
    if (pl.derive_own) {
      // visual_sort/simple_api.rs:110-127: with an own-area threshold and no shares supplied by the caller, the shares come
      // from the scene's observation boxes (exclusively_owned_areas_normalized_shares)
      sb::launch_own_area(f, n_scenes, max_m, f.in_boxes, f_own.as<float>(), f_ownovf.as<int>(),
                          reinterpret_cast<int2*>(f_ownovf.as<char>() + 16), stream);
      f.in_own = f_own.as<float>();
    }
    // Candidate preparation needs the request only (boxes, features): it runs on its own stream as soon as the inputs are there
    // and the frame that read this set of candidate buffers (two frames back) has ended -- in the steady state under the
    // tensor-core kernel of the frame in front.  (With derived own-area shares it needs the frame tables: main stream.)
    if (prep_ahead) {
      if (has_user_stream) CU(cudaStreamWaitEvent(prep_stream, ev_user_in, 0));
      if (!rq.device_io) {   // staged inputs: the prefetch copy, or the copies issued above on the work stream
        if (pl.prefetched) CU(cudaStreamWaitEvent(prep_stream, pl.sin->ev, 0));
        else { CU(cudaEventRecord(ev_inputs, stream)); CU(cudaStreamWaitEvent(prep_stream, ev_inputs, 0)); }
      }
      if (set_busy[cset]) CU(cudaStreamWaitEvent(prep_stream, ev_set_free[cset], 0));
      // ... and not before the frame in front has left its cost kernels: the preparation is HBM traffic that would slow that
      // frame's tensor-core screen.  Waiting keeps the tensor-core kernel undisturbed and the step time reproducible.
      if (cost_done_valid) CU(cudaStreamWaitEvent(prep_stream, ev_cost_done, 0));
      sb::launch_prep(Pf, f, n_scenes, max_m, prep_stream);
      CU(cudaEventRecord(ev_prep_done, prep_stream));
      CU(cudaStreamWaitEvent(stream, ev_prep_done, 0));
    } else {
      sb::launch_prep(Pf, f, n_scenes, max_m, stream);
    }
    if (side_setup) CU(cudaStreamWaitEvent(stream, ev_join, 0));
    CU(cudaEventRecord(q.ev[1], stream));
    sb::TcArgs tcc = tc;
    if (tc.use_tc && tc.n_tiles > 0) { tcc.ev_screen0 = q.ev_k[0]; tcc.ev_screen1 = q.ev_k[1]; tcc.ev_refine1 = q.ev_k[2]; q.tc_timed = true; }
    if (!pl.fork) {
      sb::launch_pos_cost(Pf, ts, f, n_scenes, max_m, max_n, stream);
      CU(cudaEventRecord(q.ev[2], stream));
      int vr0 = sb::launch_vis_cost(Pf, ts, f, n_scenes, max_m, max_n, tcc, stream);
      if (vr0 != 0) return fail(SB200_ERR_CUDA, "visual cost launch failed (%d)", vr0);
      // scenes whose entry list overflowed vote on the dense matrix: it is filled and scanned for them alone, now
      if (!f.pos_dense_all) sb::launch_pos_scan_lazy(Pf, ts, f, n_scenes, max_m, max_n, /*pass=*/1, stream);
    } else {
      CU(cudaEventRecord(q.ev[2], stream));
      {
        int vr0 = sb::launch_vis_cost_a(Pf, ts, f, n_scenes, max_m, max_n, tcc, stream);   // metadata, screen, vis_mode, refinement
        if (vr0 != 0) return fail(SB200_ERR_CUDA, "visual cost launch failed (%d)", vr0);
        vr0 = sb::launch_vote_masks(Pf, ts, f, n_scenes, max_m, max_n, stream);            // who is still open positionally
        if (vr0 != 0) return fail(SB200_ERR_CUDA, "voting launch failed: %s", cudaGetErrorString((cudaError_t)vr0));
      }
      CU(cudaEventRecord(q.ev_pos[0], stream));
      sb::launch_pos_scan_lazy(Pf, ts, f, n_scenes, max_m, max_n, /*pass=*/0, stream);
      CU(cudaEventRecord(q.ev_pos[1], stream));
      int vr1 = sb::launch_vis_cost_b(Pf, ts, f, n_scenes, max_m, max_n, tcc, stream);     // final scene mode, dense fallbacks
      if (vr1 != 0) return fail(SB200_ERR_CUDA, "visual cost launch failed (%d)", vr1);
      sb::launch_pos_scan_lazy(Pf, ts, f, n_scenes, max_m, max_n, /*pass=*/1, stream);     // scenes that fell back to dense voting
      q.pos_forked = true;
    }
    CU(cudaEventRecord(q.ev[3], stream));
    CU(cudaEventRecord(ev_cost_done, stream));
    cost_done_valid = true;
    int vr = sb::launch_voting(Pf, ts, f, n_scenes, max_m, max_n, stream);
    if (vr != 0) return fail(SB200_ERR_CUDA, "voting launch failed: %s", cudaGetErrorString((cudaError_t)vr));
    CU(cudaEventRecord(q.ev[4], stream));
    sb::launch_apply(Pf, ts, f, n_scenes, max_m, 0ull, b_ntracks.as<int>(), stream);
    // The sweep (latency-bound, one CTA per scene) and the feature store (HBM-bound) touch disjoint arrays -- a track's feature
    // block is not moved by the compaction -- so the sweep runs on the side stream beside the store; the frame ends at the join.
    const bool side_sweep = Pf.is_visual && f.in_feat && total > 0;
    if (side_sweep) {
      CU(cudaEventRecord(ev_fork[1], stream));
      CU(cudaStreamWaitEvent(side_stream, ev_fork[1], 0));
      sb::launch_frame_sweep(Pf, ts, f, n_scenes, b_ntracks.as<int>(), wb, side_stream);
      CU(cudaEventRecord(ev_join, side_stream));
      sb::launch_feat_store(Pf, ts, f, stream);
      CU(cudaStreamWaitEvent(stream, ev_join, 0));
    } else {
      sb::launch_feat_store(Pf, ts, f, stream);
      sb::launch_frame_sweep(Pf, ts, f, n_scenes, b_ntracks.as<int>(), wb, stream);
    }
    CU(cudaEventRecord(q.ev[5], stream));
    CU(cudaGetLastError());

    if (!rq.device_io && total > 0) {
      const std::array<OutCol, kOutCols> oc = out_cols(rq.out);
      for (int c = 0; c < kOutCols; ++c)
        if (oc[c].host) CU(cudaMemcpyAsync(oc[c].host, o_col[c].p, (size_t)total * oc[c].w, cudaMemcpyDeviceToHost, stream));
    }
    FrameBack* back = q.back();
    sb::Frame cnt{};   // the counters, screen_cnt included on every path (zeros where nothing counts)
    sb::carve_counters(f_counters.as<int>(), n_scenes, cnt);
    CU(cudaMemcpyAsync(q.h_out.p, f.frame_out, 12 * (size_t)n_scenes, cudaMemcpyDeviceToHost, stream));
    CU(cudaMemcpyAsync(q.h_out.as<char>() + 12 * (size_t)n_scenes, cnt.status, 4 * (size_t)n_scenes, cudaMemcpyDeviceToHost, stream));
    CU(cudaMemcpyAsync(&back->dyn, f_dyn.p, sizeof(back->dyn), cudaMemcpyDeviceToHost, stream));
    CU(cudaMemcpyAsync(&back->dense_scenes, cnt.dense_cnt, sizeof(back->dense_scenes), cudaMemcpyDeviceToHost, stream));
    if (fhist_on) CU(cudaMemcpyAsync(back->hpool, ts.hpool, sizeof(back->hpool), cudaMemcpyDeviceToHost, stream));
    CU(cudaMemcpyAsync(back->screen, cnt.screen_cnt, sizeof(back->screen), cudaMemcpyDeviceToHost, stream));
    static const bool trace_dense = getenv("SB200_TRACE") != nullptr && atoi(getenv("SB200_TRACE")) >= 2;   // synchronises: level 2 only
    if (trace_dense && tc.dense && tc.n_tiles > 0) {
      int hc[8] = {0};
      CU(cudaMemcpyAsync(hc, tc.dbg_counts, sizeof(hc), cudaMemcpyDeviceToHost, stream));
      CU(cudaStreamSynchronize(stream));
      std::vector<int> vcnt((size_t)n_scenes);
      CU(cudaMemcpy(vcnt.data(), f.vis_cnt, 4 * (size_t)n_scenes, cudaMemcpyDeviceToHost));
      long long tot = 0; int mx = 0;
      for (int v : vcnt) { tot += v; mx = std::max(mx, v); }
      fprintf(stderr, "[sb200] dense frame: fallback reasons threshold %d, max-list overflow %d, no maximum %d; max candidates %d; pairs to refine %lld (largest scene %d)\n",
              hc[0], hc[1], hc[2], hc[3], tot, mx);
    }
    CU(cudaEventRecord(q.done, stream));
    CU(cudaEventRecord(ev_set_free[cset], stream));   // this frame's candidate buffers may be rewritten after this point
    set_busy[cset] = true;
    if (has_user_stream && join_per_call) {   // the caller's stream continues after the frame
      CU(cudaEventRecord(ev_user_out, stream));
      CU(cudaStreamWaitEvent(user_stream, ev_user_out, 0));
    }
    return 0;
  }

  // The per-scene block of the dense path (f_dscene): maxc_cnt | maxc_next | dense_bad | zeros ([n] ints each, zeroed
  // together), scene_l0 | scene_cmax ([n] floats each), 4 unused ints, dbg_counts[8].
  static size_t dscene_bytes(int n) { return 4 * 6 * (size_t)n + 128; }
  static void carve_dscene(void* p, int n, sb::TcArgs& tc) {
    using A = sb::TcArgs;
    int* A::* const ints[] = {&A::maxc_cnt, &A::maxc_next, &A::dense_bad, &A::zeros};
    for (int i = 0; i < 4; ++i) tc.*ints[i] = static_cast<int*>(p) + (size_t)i * n;
    tc.scene_l0 = reinterpret_cast<float*>(tc.maxc_cnt + 4 * (size_t)n);
    tc.scene_cmax = tc.scene_l0 + n;
    tc.dbg_counts = reinterpret_cast<int*>(tc.scene_cmax + n) + 4;
  }
};

// Reads back what the oldest frame in flight left for the host: per scene {live tracks, arena blocks, newly expired} and
// the status word, plus the frame scalars.  block == false: only if the frame has completed.  Returns 1 when nothing was
// absorbed.  Errors of an asynchronous frame are kept (async_rc / async_err) for the next call that reports status.
int sb200_tracker::absorb_oldest(bool block) {
  if (pend_count == 0) return 1;
  Pending& q = pend[pend_head];
  cudaError_t e;
  if (block) {
    const auto w0 = std::chrono::steady_clock::now();
    e = cudaEventSynchronize(q.done);
    host_ms_blocked += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - w0).count();
  } else {
    e = cudaEventQuery(q.done);
  }
  if (e == cudaErrorNotReady) { cudaGetLastError(); return 1; }
  const int n = q.n_scenes;
  if (e != cudaSuccess) {
    cudaGetLastError();
    if (!async_rc) { async_rc = SB200_ERR_CUDA; async_err = std::string("a frame in flight failed: ") + cudaGetErrorString(e); }
  } else {
    const int* h_fo = q.h_out.as<int>();            // [n][3] live tracks, arena blocks, newly expired
    const int* h_status = h_fo + 3 * (size_t)n;
    const FrameBack& back = *q.back();
    for (int s = 0; s < n; ++s) {
      const int slot = q.slots[s];
      if (h_status[s] && !async_rc) {
        async_rc = (h_status[s] & 2) ? SB200_ERR_CAPACITY : SB200_ERR_INTERNAL;
        char buf[160];
        snprintf(buf, sizeof(buf), (h_status[s] & 2) ? "more than 2800 boxes overlap one detection of scene %llu (own-area shares)"
                                                      : "track store overflow in scene %llu",
                 (unsigned long long)scene_of_slot[slot]);
        async_err = buf;
      }
      n_tracks[slot] = h_fo[3 * s];
      arena_top[slot] = h_fo[3 * s + 1];
      n_hidden[slot] += h_fo[3 * s + 2];   // swept from the device store, not yet collected in the reference's sense
      wasted_count += h_fo[3 * s + 2];
    }
    if (fhist_on) {   // the history pool's counters {free, handed out} as the frame's sweep left them
      hpool_free = back.hpool[0];
      hpool_top = back.hpool[1];
    }
    acc_units_mn += back.dyn.units_mn;
    acc_units_rows += back.dyn.units_rows;
    acc_frames += 1;
    {
      const int dense_scenes = back.dense_scenes;
      if (q.mode != 0) acc_dense_scenes += (unsigned long long)dense_scenes;   // mode 0 IS the exact kernel: not a fallback
      last_dense_scenes = dense_scenes;
      // most scenes of a screened frame overflowed their survivor lists: the threshold cuts (almost) nothing, so the
      // following frames take the dense tensor-core path; and back, if that path's precondition keeps failing
      // (an overflow of the e4m3 screen says that its slack is too wide, not that the threshold cuts nothing)
      if (q.mode == 1 && !q.fp8 && n >= 1 && dense_scenes * 4 > n) adapt_dense = true;
      if (q.mode == 2 && n >= 1 && dense_scenes * 4 > n) adapt_dense = false;
      if (q.mode == 1) {
        const unsigned long long kept = (unsigned int)back.screen[0], cut = (unsigned int)back.screen[1],
                                 ovf = (unsigned int)back.screen[2];
        acc_screen[q.fp8 ? 0 : 1] += 1;
        acc_screen[2] += kept;
        acc_screen[3] += cut;
        if (q.fp8 && (ovf > 0 || 2 * cut > kept)) fp8_hold = kFp8Hold;
      }
    }
    for (int i = 0; i < 5; ++i) cudaEventElapsedTime(&stage_ms[i], q.ev[i], q.ev[i + 1]);
    if (q.pos_forked) {
      // lazy frame: the culled scan sits inside the visual span (after the BestFit pre-pass): report it on its own
      float fill_ms = stage_ms[1], scan_ms = 0.0f;
      cudaEventElapsedTime(&scan_ms, q.ev_pos[0], q.ev_pos[1]);
      stage_ms[1] = scan_ms;
      stage_ms[2] += fill_ms - scan_ms;
    }
    tc_timed = q.tc_timed;
    kernel_ms[0] = kernel_ms[1] = 0.0f;
    if (tc_timed) { cudaEventElapsedTime(&kernel_ms[0], q.ev_k[0], q.ev_k[1]); cudaEventElapsedTime(&kernel_ms[1], q.ev_k[1], q.ev_k[2]); }
    for (int i = 0; i < 5; ++i) acc_stage_ms[i] += stage_ms[i];
    if (tc_timed) { acc_kernel_ms[0] += kernel_ms[0]; acc_kernel_ms[1] += kernel_ms[1]; acc_tc_frames += 1; }
    static const bool trace_abs = getenv("SB200_TRACE") != nullptr;
    if (trace_abs)
      fprintf(stderr, "[sb200] frame absorbed: mode %d, %d of %d scenes on the exact SIMT fallback; prep %.3f pos %.3f vis %.3f vote %.3f apply %.3f ms (main kernel %.3f, refine %.3f)\n",
              q.mode, last_dense_scenes, n, stage_ms[0], stage_ms[1], stage_ms[2], stage_ms[3], stage_ms[4], kernel_ms[0], kernel_ms[1]);
    cudaGetLastError();   // an event that was never recorded in this frame leaves cudaErrorInvalidResourceHandle behind
  }
  unbook(q);
  pend_head = (pend_head + 1) % kDepth;
  return 0;
}

int sb200_tracker::poll() {
  while (pend_count > 0 && absorb_oldest(false) == 0) {}
  return 0;
}

int sb200_tracker::drain(const char* why) {
  static const bool trace_dr = getenv("SB200_TRACE") != nullptr;
  if (trace_dr && why && pend_count > 0) fprintf(stderr, "[sb200] predict waits for %d frame(s) in flight: %s\n", pend_count, why);
  while (pend_count > 0) absorb_oldest(true);
  if (async_rc) {
    const int rc = async_rc;
    async_rc = 0;
    return fail(rc, "%s", async_err.c_str());
  }
  return 0;
}

// enqueues one request as a frame, in the stages above (DESIGN.md §3a)
int sb200_tracker::predict(int32_t n_scenes, const uint64_t* scene_ids, const int32_t* det_offsets, const float* boxes,
                           const float* features, const uint8_t* has_feature, const float* quality,
                           const int64_t* custom_ids, const float* own_area, const sb200_predict_out* out,
                           bool device_io, bool wait) {
  CU(cudaSetDevice(device));
  static const bool trace = getenv("SB200_TRACE") != nullptr;
  const auto t_begin = std::chrono::steady_clock::now();
  auto since = [&] { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_begin).count(); };
  Request rq{n_scenes, 0, scene_ids, det_offsets, in_ptrs(boxes, features, has_feature, quality, custom_ids, own_area),
             out ? *out : sb200_predict_out{}, device_io};
  int rc = check_request(rq);
  if (rc) return rc;
  // auto-waste tick (src/trackers/sort/simple_api.rs:115-120): a collection point of the reference, host and device meet
  if (auto_waste_counter == 0) {
    if ((rc = drain("auto-waste tick"))) return rc;
    if ((rc = run_waste())) return rc;
    auto_waste_counter = auto_waste_periodicity;
  } else auto_waste_counter -= 1;
  if (n_scenes == 0) return wait ? drain() : 0;

  if (!rq.same_req) {
    last_req_slots.resize(n_scenes);
    for (int s = 0; s < n_scenes; ++s) last_req_slots[s] = slot_for(scene_ids[s], true);
    last_req_scenes.assign(scene_ids, scene_ids + n_scenes);
  }
  if (pend_count == kDepth) {
    if (trace) fprintf(stderr, "[sb200] predict waits: ring of %d frames full\n", kDepth);
    absorb_oldest(true);
  }   // back-pressure: at most kDepth frames in flight

  FramePlan pl;
  if ((rc = reserve_state(rq, pl))) return rc;
  Pending& q = pend[(pend_head + pend_count) % kDepth];
  if ((rc = plan_frame(rq, q, pl))) return rc;
  sb::Frame f{};   // bind_frame sets what the frame uses, the rest stays zero
  sb::TcArgs tc{};
  if ((rc = bind_frame(rq, pl, f, tc))) return rc;
  // ==================================================== nothing below can fail for capacity reasons: the request is committed
  Rollback rollback = commit(rq, pl, q);
  const double ms_setup = since();
  if ((rc = enqueue(rq, pl, q, f, tc))) return rc;
  rollback.armed = false;
  if (pl.sin) { CU(cudaEventRecord(pl.sin->ev_read, stream)); pl.sin->read_pending = true; }
  const double ms_launch = since();
  if (wait) rc = drain();
  host_ms_total += since();
  host_calls += 1;
  if (trace && pl.prefetched && wait) {
    float cms = 0.0f;
    if (cudaEventElapsedTime(&cms, pl.sin->ev0, pl.sin->ev) == cudaSuccess)
      fprintf(stderr, "[sb200] prefetch copy of this frame took %.3f ms on the copy stream\n", cms);
  }
  if (trace) fprintf(stderr, "[sb200] predict: setup %.3f ms, launched at %.3f ms, returned at %.3f ms (total dets %d, %d in flight)\n", ms_setup, ms_launch, since(), rq.total, pend_count);
  return rc;
}

// =============================================================================================== C ABI
extern "C" {

const char* sb200_last_error(void) { return sb::g_err.c_str(); }

int sb200_device_count(void) { return sb::device_count(); }

void sb200_options_default(sb200_options* o) {
  if (!o) return;
  memset(o, 0, sizeof(*o));
  o->kind = SB200_KIND_SORT;
  o->positional_kind = SB200_POS_MAHA;
  o->iou_threshold = 0.3f;
  o->min_confidence = 0.05f;
  o->max_idle_epochs = 5;
  o->history_length = 1;
  o->kalman_position_weight = 1.0f / 20.0f;
  o->kalman_velocity_weight = 1.0f / 160.0f;
  o->visual_kind = SB200_VIS_EUCLIDEAN;
  o->visual_threshold = 3.402823466e+38f;
  o->visual_max_observations = 5;
  o->visual_min_votes = 1;
  o->visual_minimal_track_length = 3;
}

int sb200_tracker_create(const sb200_options* opts, sb200_tracker** out) {
  if (!opts || !out) return fail(SB200_ERR_INVALID, "opts / out is NULL");
  *out = nullptr;
  int rc = sb::check_device(opts->device);
  if (rc) return rc;
  sb::Params P;
  rc = make_params(*opts, &P);
  if (rc) return rc;
  CU(cudaSetDevice(opts->device));
  sb200_tracker* t = new sb200_tracker();
  t->opts = *opts;
  t->P = P;
  t->device = opts->device;
  // history_length 0 means "unlimited" in the reference (sort.rs:166); the device keeps at most kMaxHist boxes per track
  t->hist_len = opts->history_length <= 0 ? sb::kMaxHist : std::min<int>(opts->history_length, sb::kMaxHist);
  {
    int sms = 0;
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, opts->device) == cudaSuccess && sms > 0) t->num_sms = sms;
  }
  int prio_lo = 0, prio_hi = 0;
  cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);
  // numerically lower = more urgent: side stream (prio_hi) > work stream > candidate preparation (prio_lo)
  cudaError_t e = cudaStreamCreateWithPriority(&t->stream, cudaStreamNonBlocking, prio_hi < prio_lo ? prio_hi + 1 : prio_lo);
  if (e != cudaSuccess) { delete t; return fail(SB200_ERR_CUDA, "cudaStreamCreate failed: %s", cudaGetErrorString(e)); }
  for (auto& g : t->stg) {
    e = cudaEventCreate(&g.ev);
    if (e == cudaSuccess) e = cudaEventCreate(&g.ev0);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&g.ev_read, cudaEventDisableTiming);
    if (e != cudaSuccess) { delete t; return fail(SB200_ERR_CUDA, "cudaEventCreate failed: %s", cudaGetErrorString(e)); }
  }
  // the internal streams, and the events of the frame ring, of the fork / join points and of the caller-stream joins
  e = cudaStreamCreateWithPriority(&t->side_stream, cudaStreamNonBlocking, prio_hi);
  if (e == cudaSuccess) e = cudaStreamCreateWithPriority(&t->prep_stream, cudaStreamNonBlocking, prio_lo);
  for (cudaEvent_t* p : {&t->ev_fork[0], &t->ev_fork[1], &t->ev_join, &t->ev_prep_done, &t->ev_inputs, &t->ev_cost_done,
                         &t->ev_set_free[0], &t->ev_set_free[1], &t->ev_user_in, &t->ev_user_out})
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(p, cudaEventDisableTiming);
  for (auto& q : t->pend) {
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&q.done, cudaEventDisableTiming);
    for (auto& x : q.ev) if (e == cudaSuccess) e = cudaEventCreate(&x);
    for (auto& x : q.ev_k) if (e == cudaSuccess) e = cudaEventCreate(&x);
    for (auto& x : q.ev_pos) if (e == cudaSuccess) e = cudaEventCreate(&x);
  }
  if (e != cudaSuccess) { delete t; return fail(SB200_ERR_CUDA, "stream / event creation failed: %s", cudaGetErrorString(e)); }
  if (opts->max_scenes_hint > 0 || opts->max_tracks_per_scene_hint > 0) {
    // + room for the tracks the frames in flight may add (see predict())
    rc = t->ensure_store(std::max(1, opts->max_scenes_hint),
                         std::max(64, opts->max_tracks_per_scene_hint + sb200_tracker::kDepth * std::max(0, opts->max_dets_per_scene_hint)));
    if (rc) { delete t; return rc; }
  }
  *out = t;
  return 0;
}

void sb200_tracker_destroy(sb200_tracker* t) { delete t; }

int sb200_tracker_set_stream(sb200_tracker* t, void* cuda_stream) {
  if (!t) return fail(SB200_ERR_INVALID, "tracker is NULL");
  CU(cudaSetDevice(t->device));
  int rc = t->drain();
  if (rc) return rc;
  CU(cudaStreamSynchronize(t->stream));
  // the tracker keeps its own work stream; the caller's stream is joined by events at every call (see `user_stream`)
  t->user_stream = reinterpret_cast<cudaStream_t>(cuda_stream);
  t->has_user_stream = true;
  return 0;
}

int sb200_set_stream_join(sb200_tracker* t, int32_t per_call) {
  if (!t) return fail(SB200_ERR_INVALID, "tracker is NULL");
  t->join_per_call = per_call != 0;
  return 0;
}

int sb200_stream_join(sb200_tracker* t, void* cuda_stream) {
  if (!t) return fail(SB200_ERR_INVALID, "tracker is NULL");
  CU(cudaSetDevice(t->device));
  if (!t->ev_join_req) CU(cudaEventCreateWithFlags(&t->ev_join_req, cudaEventDisableTiming));
  CU(cudaEventRecord(t->ev_join_req, t->stream));
  CU(cudaStreamWaitEvent(reinterpret_cast<cudaStream_t>(cuda_stream), t->ev_join_req, 0));
  return 0;
}

int sb200_predict_batch(sb200_tracker* t, int32_t n_scenes, const uint64_t* scene_ids, const int32_t* det_offsets,
                        const float* boxes, const float* features, const uint8_t* has_feature, const float* quality,
                        const int64_t* custom_ids, const float* own_area, const sb200_predict_out* out) {
  if (!t) return fail(SB200_ERR_INVALID, "tracker is NULL");
  return t->predict(n_scenes, scene_ids, det_offsets, boxes, features, has_feature, quality, custom_ids, own_area, out, false, true);
}

int sb200_predict_batch_async(sb200_tracker* t, int32_t n_scenes, const uint64_t* scene_ids, const int32_t* det_offsets,
                              const float* boxes, const float* features, const uint8_t* has_feature, const float* quality,
                              const int64_t* custom_ids, const float* own_area, const sb200_predict_out* out) {
  if (!t) return fail(SB200_ERR_INVALID, "tracker is NULL");
  return t->predict(n_scenes, scene_ids, det_offsets, boxes, features, has_feature, quality, custom_ids, own_area, out, false, false);
}

int sb200_set_feature_dim(sb200_tracker* t, int32_t feature_dim) {
  if (!t || feature_dim <= 0) return fail(SB200_ERR_INVALID, "bad arguments");
  if (!t->P.is_visual) return fail(SB200_ERR_INVALID, "not a visual tracker");
  if (feature_dim == t->P.feature_dim) return 0;
  if (t->seen_features) return fail(SB200_ERR_INVALID, "features of dimension %d are already stored", t->P.feature_dim);
  CU(cudaSetDevice(t->device));
  int rc = t->drain();
  if (rc) return rc;
  CU(cudaStreamSynchronize(t->stream));
  // No track holds a feature yet (obs_hasf == 0 everywhere): the columns whose rows depend on d8 are simply re-created for
  // the new row size -- the feature rows with their BF16 and e4m3 copies (the latter exist for d8 <= 512 only) and the
  // history rows of the pool.  The present bytes (all zero so far) and the tracks' blocks stay.
  auto d8_cols = [t] {   // (column, rows it holds)
    std::vector<std::pair<Col, size_t>> v;
    for (const Col& c : t->store_table())
      if (c.buf == &t->b_feat || c.buf == &t->b_feat_bf16 || c.buf == &t->b_feat_fp8 || c.buf == &t->b_fscale)
        v.push_back({c, (size_t)t->scene_cap * t->track_cap});
    if (t->fhist_on)
      for (const Col& c : t->pool_table()) if (c.buf == &t->b_hrows) v.push_back({c, (size_t)t->hpool_cap});
    return v;
  };
  for (const auto& [c, rows] : d8_cols()) { c.buf->release(); c.point(*t, nullptr); }
  for (auto& cb : t->cand) { cb.bf16.release(); cb.fp8.release(); }
  t->P.feature_dim = feature_dim;
  t->P.d8 = (feature_dim + 7) / 8 * 8;
  t->P.vis_rel_err = sb::screen_rel_err(feature_dim);
  t->P.vis_rel_err8 = sb::screen_rel_err_fp8(feature_dim);
  t->P.vis_dense_f32 = sb::dense_f32_err(feature_dim);
  t->P.vis_sample_margin = sb::dense_sample_margin(feature_dim);
  t->opts.feature_dim = feature_dim;
  for (const auto& [c, rows] : d8_cols()) {
    if (rows == 0) continue;
    if ((rc = c.buf->ensure(rows * c.w))) return rc;
    c.point(*t, c.buf->p);
  }
  for (auto& g : t->stg) g.col[sb200_tracker::kFeat].release();   // the staged features: their row width changed
  return 0;
}

int sb200_feature_history_pool(sb200_tracker* t, int64_t* out3) {
  if (!t || !out3) return fail(SB200_ERR_INVALID, "bad arguments");
  if (!t->fhist_on) return fail(SB200_ERR_INVALID, "the feature history is off (sb200_set_feature_history)");
  CU(cudaSetDevice(t->device));
  { int rc_ = t->drain(); if (rc_) return rc_; }
  int h[2] = {0, 0};
  CU(cudaMemcpyAsync(h, t->ts.hpool, sizeof(h), cudaMemcpyDeviceToHost, t->stream));
  CU(cudaStreamSynchronize(t->stream));
  out3[0] = t->hpool_cap;
  out3[1] = h[1];
  out3[2] = h[0];
  return 0;
}

int sb200_set_feature_history(sb200_tracker* t, int32_t on) {
  if (!t) return fail(SB200_ERR_INVALID, "tracker is NULL");
  if (!t->P.is_visual) return fail(SB200_ERR_INVALID, "the feature history belongs to the visual trackers");
  // tracks (and their history blocks) exist once a frame has run or a blob has been loaded / imported
  if (t->frame_seq > 0 || t->transferred)
    return fail(SB200_ERR_INVALID, "the feature history is switched before the first predict, load or import");
  return t->set_feature_history(on != 0);
}

static_assert(SB200_FEATURE_F32 == sb::kFeatF32 && SB200_FEATURE_F16 == sb::kFeatF16 && SB200_FEATURE_BF16 == sb::kFeatBF16,
              "feature type codes of the ABI and the kernels differ");

int sb200_set_feature_type(sb200_tracker* t, int32_t type) {
  if (!t) return fail(SB200_ERR_INVALID, "tracker is NULL");
  if (!t->P.is_visual) return fail(SB200_ERR_INVALID, "the feature type belongs to the visual trackers");
  if (type != SB200_FEATURE_F32 && type != SB200_FEATURE_F16 && type != SB200_FEATURE_BF16)
    return fail(SB200_ERR_INVALID, "unknown feature type %d", (int)type);
  t->feat_type = type;   // frames already enqueued keep the type they were enqueued with (Frame::feat_type)
  return 0;
}

int sb200_sync(sb200_tracker* t) {
  if (!t) return fail(SB200_ERR_INVALID, "tracker is NULL");
  CU(cudaSetDevice(t->device));
  return t->drain();
}

int sb200_frames_in_flight(sb200_tracker* t) {
  if (!t) return fail(SB200_ERR_INVALID, "tracker is NULL");
  CU(cudaSetDevice(t->device));
  t->poll();
  return t->pend_count;
}

int sb200_work_counters(sb200_tracker* t, uint64_t* out3 /* [4] */, double* ms7 /* [8] */) {
  if (!t) return fail(SB200_ERR_INVALID, "tracker is NULL");
  CU(cudaSetDevice(t->device));
  int rc = t->drain();
  if (rc) return rc;
  if (out3) { out3[0] = t->acc_units_mn; out3[1] = t->acc_units_rows; out3[2] = t->acc_frames; out3[3] = t->acc_dense_scenes; }
  if (ms7) {
    for (int i = 0; i < 5; ++i) ms7[i] = t->acc_stage_ms[i];
    ms7[5] = t->acc_kernel_ms[0]; ms7[6] = t->acc_kernel_ms[1]; ms7[7] = (double)t->acc_tc_frames;
  }
  return 0;
}

int sb200_screen_counters(sb200_tracker* t, uint64_t* out4) {
  if (!t || !out4) return fail(SB200_ERR_INVALID, "bad arguments");
  CU(cudaSetDevice(t->device));
  int rc = t->drain();
  if (rc) return rc;
  for (int i = 0; i < 4; ++i) out4[i] = t->acc_screen[i];
  return 0;
}

uint64_t sb200_launch_count(void) { return sb::launch_count(); }

int sb200_host_counters(sb200_tracker* t, double* out3 /* [3] */) {
  if (!t || !out3) return fail(SB200_ERR_INVALID, "bad arguments");
  out3[0] = (double)t->host_calls; out3[1] = t->host_ms_total; out3[2] = t->host_ms_blocked;
  return 0;
}

int sb200_prefetch_inputs(sb200_tracker* t, int32_t total, const float* boxes, const float* features,
                          const uint8_t* has_feature, const float* quality, const int64_t* custom_ids,
                          const float* own_area) {
  if (!t || total < 0 || (total > 0 && !boxes)) return fail(SB200_ERR_INVALID, "bad arguments");
  CU(cudaSetDevice(t->device));
  if (total == 0) return 0;
  if (!t->copy_stream) CU(cudaStreamCreateWithFlags(&t->copy_stream, cudaStreamNonBlocking));
  // a free set: not holding an unconsumed prefetch; with nothing pending, the one the last predict did not read
  if (t->stg[0].pending && t->stg[1].pending)
    return fail(SB200_ERR_INVALID, "two prefetched requests are already waiting for their predict call");
  const int k = t->stg[0].pending ? 1 : (t->stg[1].pending ? 0 : 1 - t->stg_last);
  sb200_tracker::Staging& S = t->stg[k];
  const sb200_tracker::InPtrs in = t->in_ptrs(boxes, features, has_feature, quality, custom_ids, own_area);
  const auto ic = t->in_cols();
  // rows as predict() sizes them (the scene count is not known yet), so the predict call never reallocates a filled set
  const size_t T = t->frame_rows(total, 0);
  int rc = 0;
  cudaStream_t cs = t->copy_stream;
  // the set's previous reader (a frame that may still be in flight) finishes first; a reallocation meets the device
  bool grows = false;
  for (int c = 0; c < sb200_tracker::kInCols; ++c) grows |= in[c] && S.col[c].bytes < T * ic[c].w;
  if (grows && (rc = t->drain())) return rc;
  if (S.read_pending) { CU(cudaStreamWaitEvent(cs, S.ev_read, 0)); S.read_pending = false; }
  for (int c = 0; c < sb200_tracker::kInCols; ++c)
    if (in[c] && (rc = S.col[c].ensure(T * ic[c].w))) return rc;
  CU(cudaEventRecord(S.ev0, cs));
  for (int c = 0; c < sb200_tracker::kInCols; ++c)
    if (in[c]) CU(cudaMemcpyAsync(S.col[c].p, in[c], (size_t)total * ic[c].w, cudaMemcpyHostToDevice, cs));
  CU(cudaEventRecord(S.ev, cs));
  S.key = in;
  S.total = total; S.type = t->feat_type; S.pending = true;
  return 0;
}

int sb200_predict_batch_device(sb200_tracker* t, int32_t n_scenes, const uint64_t* scene_ids,
                               const int32_t* det_offsets, const float* boxes, const float* features,
                               const uint8_t* has_feature, const float* quality, const int64_t* custom_ids,
                               const float* own_area, const sb200_predict_out* out) {
  if (!t) return fail(SB200_ERR_INVALID, "tracker is NULL");
  return t->predict(n_scenes, scene_ids, det_offsets, boxes, features, has_feature, quality, custom_ids, own_area, out, true, false);
}

int sb200_skip_epochs(sb200_tracker* t, uint64_t scene_id, int32_t n) {
  if (!t || n < 0) return fail(SB200_ERR_INVALID, "bad arguments");
  CU(cudaSetDevice(t->device));
  { int rc_ = t->drain(); if (rc_) return rc_; }
  const int old = t->slot_for(scene_id, false);   // a new scene is at epoch 0: n < 2^31 always fits
  if (old >= 0 && (uint64_t)t->epoch[old] + (uint64_t)n > UINT32_MAX)
    return fail(SB200_ERR_INVALID, "scene %llu: epoch %u + %d is past the last epoch %u", (unsigned long long)scene_id,
                t->epoch[old], n, UINT32_MAX);
  int slot = t->slot_for(scene_id, true);
  int rc = t->ensure_store((int)t->scene_of_slot.size(), std::max(t->track_cap, 64));
  if (rc) return rc;
  t->epoch[slot] += (uint32_t)n;
  return t->run_waste();  // skip_epochs_for_scene ends with auto_waste (tracker_api.rs:48-51)
}

int64_t sb200_current_epoch(sb200_tracker* t, uint64_t scene_id) {
  if (!t) return fail(SB200_ERR_INVALID, "tracker is NULL");
  int slot = t->slot_for(scene_id, false);
  return slot < 0 ? 0 : (int64_t)t->epoch[slot];
}

int64_t sb200_active_tracks(sb200_tracker* t) {
  if (!t) return fail(SB200_ERR_INVALID, "tracker is NULL");
  { int rc_ = t->drain(); if (rc_) return rc_; }
  int64_t n = 0;   // the reference's store still holds the expired tracks it has not collected yet
  for (int v : t->n_tracks) n += v;
  for (int v : t->n_hidden) n += v;
  return n;
}

int sb200_scene_track_counts(sb200_tracker* t, int32_t n_scenes, const uint64_t* scene_ids, int32_t* out) {
  if (!t || n_scenes < 0 || (n_scenes > 0 && (!scene_ids || !out))) return fail(SB200_ERR_INVALID, "bad arguments");
  { int rc_ = t->drain(); if (rc_) return rc_; }
  for (int s = 0; s < n_scenes; ++s) {
    int slot = t->slot_for(scene_ids[s], false);
    out[s] = slot < 0 ? 0 : t->n_tracks[slot] + t->n_hidden[slot];
  }
  return 0;
}

int sb200_scene_live_counts(sb200_tracker* t, int32_t n_scenes, const uint64_t* scene_ids, int32_t* live, int32_t* blocks) {
  if (!t || n_scenes < 0 || (n_scenes > 0 && !scene_ids)) return fail(SB200_ERR_INVALID, "bad arguments");
  { int rc_ = t->drain(); if (rc_) return rc_; }
  for (int s = 0; s < n_scenes; ++s) {
    int slot = t->slot_for(scene_ids[s], false);
    if (live) live[s] = slot < 0 ? 0 : t->n_tracks[slot];
    if (blocks) blocks[s] = slot < 0 ? 0 : (t->P.is_visual ? t->arena_top[slot] : t->n_tracks[slot]);
  }
  return 0;
}

int sb200_set_auto_waste(sb200_tracker* t, int32_t periodicity) {
  if (!t || periodicity < 0) return fail(SB200_ERR_INVALID, "bad arguments");
  t->auto_waste_periodicity = periodicity;
  t->auto_waste_counter = 0;  // set_auto_waste resets the counter (tracker_api.rs:29-33)
  return 0;
}

int sb200_clear_wasted(sb200_tracker* t) {
  if (!t) return fail(SB200_ERR_INVALID, "tracker is NULL");
  CU(cudaSetDevice(t->device));
  { int rc_ = t->drain(); if (rc_) return rc_; }
  // TrackerAPI::clear_wasted (src/trackers/tracker_api.rs:94-100) empties the wasted store; tracks swept early that the
  // reference has not collected yet are not in it and stay pending
  return t->drop_wasted_front(t->revealed);
}

int64_t sb200_wasted(sb200_tracker* t, int64_t cap, uint64_t* ids, uint64_t* scene_ids, uint32_t* epochs,
                     uint32_t* lengths, float* predicted_boxes, float* observed_boxes) {
  if (!t || cap < 0) return fail(SB200_ERR_INVALID, "bad arguments");
  CU(cudaSetDevice(t->device));
  { int rc_ = t->drain(); if (rc_) return rc_; }
  int rc = t->run_waste();  // wasted() starts with auto_waste (tracker_api.rs:90-91)
  if (rc) return rc;
  int64_t n = std::min<int64_t>(cap, t->wasted_count);
  if (n == 0) return 0;
  cudaStream_t st = t->stream;
  if (ids) CU(cudaMemcpyAsync(ids, t->wb.id, 8 * n, cudaMemcpyDeviceToHost, st));
  if (scene_ids) CU(cudaMemcpyAsync(scene_ids, t->wb.scene, 8 * n, cudaMemcpyDeviceToHost, st));
  if (epochs) CU(cudaMemcpyAsync(epochs, t->wb.epoch, 4 * n, cudaMemcpyDeviceToHost, st));
  if (lengths) CU(cudaMemcpyAsync(lengths, t->wb.length, 4 * n, cudaMemcpyDeviceToHost, st));
  if (predicted_boxes) CU(cudaMemcpyAsync(predicted_boxes, t->wb.pred, 24 * n, cudaMemcpyDeviceToHost, st));
  if (observed_boxes) CU(cudaMemcpyAsync(observed_boxes, t->wb.obs, 24 * n, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  if ((rc = t->drop_wasted_front(n))) return rc;   // drain
  return n;
}

// the first n records of the wasted buffer and their box histories into `o`, as sb200_wasted_history returns them
static int read_wasted(sb200_tracker* t, int64_t n, const sb::WastedOut& o) {
  cudaStream_t st = t->stream;
  const int32_t history_cap = o.history_cap;
  std::vector<uint32_t> hlen((size_t)n);
  if (o.ids) CU(cudaMemcpyAsync(o.ids, t->wb.id, 8 * n, cudaMemcpyDeviceToHost, st));
  if (o.scene_ids) CU(cudaMemcpyAsync(o.scene_ids, t->wb.scene, 8 * n, cudaMemcpyDeviceToHost, st));
  if (o.epochs) CU(cudaMemcpyAsync(o.epochs, t->wb.epoch, 4 * n, cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(hlen.data(), t->wb.length, 4 * n, cudaMemcpyDeviceToHost, st));
  std::vector<float> lastp((size_t)n * 6), lasto((size_t)n * 6);
  CU(cudaMemcpyAsync(lastp.data(), t->wb.pred, 24 * n, cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(lasto.data(), t->wb.obs, 24 * n, cudaMemcpyDeviceToHost, st));
  const int H = t->hist_len;
  std::vector<float> hp, ho;
  if (H > 1 && history_cap > 0) {
    hp.resize((size_t)n * H * 6); ho.resize((size_t)n * H * 6);
    CU(cudaMemcpyAsync(hp.data(), t->wb.hist_pred, sizeof(float) * hp.size(), cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(ho.data(), t->wb.hist_obs, sizeof(float) * ho.size(), cudaMemcpyDeviceToHost, st));
  }
  CU(cudaStreamSynchronize(st));
  if (o.lengths) memcpy(o.lengths, hlen.data(), 4 * (size_t)n);
  if (o.predicted_boxes) memcpy(o.predicted_boxes, lastp.data(), 24 * (size_t)n);
  if (o.observed_boxes) memcpy(o.observed_boxes, lasto.data(), 24 * (size_t)n);
  // rings -> chronological order (oldest first), at most history_cap boxes per track
  for (int64_t i = 0; i < n; ++i) {
    const uint32_t len = hlen[(size_t)i];
    int cnt = (int)std::min<uint32_t>(len, (uint32_t)H);
    cnt = std::min(cnt, (int)history_cap);
    if (o.history_counts) o.history_counts[i] = history_cap > 0 ? cnt : 0;
    for (int c = 0; c < cnt; ++c) {
      const uint32_t j = len - (uint32_t)cnt + (uint32_t)c;   // observation number
      const float* sp; const float* so;
      if (H > 1) { sp = &hp[((size_t)i * H + j % H) * 6]; so = &ho[((size_t)i * H + j % H) * 6]; }
      else { sp = &lastp[(size_t)i * 6]; so = &lasto[(size_t)i * 6]; }
      if (o.predicted_history) memcpy(o.predicted_history + ((size_t)i * history_cap + c) * 6, sp, 24);
      if (o.observed_history) memcpy(o.observed_history + ((size_t)i * history_cap + c) * 6, so, 24);
    }
  }
  return 0;
}

// sb200_wasted_history, and sb200_wasted_visual when `features` / `feature_present` are given
static int64_t wasted_records(sb200_tracker* t, int64_t cap, uint64_t* ids, uint64_t* scene_ids, uint32_t* epochs,
                              uint32_t* lengths, float* predicted_boxes, float* observed_boxes, int32_t history_cap,
                              float* predicted_history, float* observed_history, int32_t* history_counts, float* features,
                              uint8_t* feature_present) {
  if (!t || cap < 0 || history_cap < 0) return fail(SB200_ERR_INVALID, "bad arguments");
  const bool want_feat = features != nullptr || feature_present != nullptr;
  if (want_feat && !(features && feature_present)) return fail(SB200_ERR_INVALID, "features and feature_present go together");
  if (want_feat && !t->fhist_on) return fail(SB200_ERR_INVALID, "the feature history is off (sb200_set_feature_history)");
  CU(cudaSetDevice(t->device));
  { int rc_ = t->drain(); if (rc_) return rc_; }
  int rc = t->run_waste();  // wasted() starts with auto_waste (tracker_api.rs:90-91)
  if (rc) return rc;
  const int64_t n = std::min<int64_t>(cap, t->wasted_count);
  if (n == 0) return 0;
  cudaStream_t st = t->stream;
  if ((rc = read_wasted(t, n, {ids, scene_ids, epochs, lengths, predicted_boxes, observed_boxes, history_cap,
                               predicted_history, observed_history, history_counts})))
    return rc;
  if (want_feat && history_cap > 0) {
    // the records' rings are gathered on the device in the same order, a chunk of records at a time, and copied back once
    const size_t rec_bytes = (size_t)history_cap * t->P.d8 * 4;
    const int64_t chunk = std::max<int64_t>(1, std::min<int64_t>(n, (int64_t)((64u << 20) / rec_bytes)));
    DBuf rows, pres;
    if ((rc = rows.ensure((size_t)chunk * rec_bytes)) || (rc = pres.ensure((size_t)chunk * history_cap))) return rc;
    for (int64_t i0 = 0; i0 < n; i0 += chunk) {
      const int c = (int)std::min<int64_t>(chunk, n - i0);
      sb::launch_hist_gather(t->ts, t->P.d8, t->wb.hblk + i0, t->wb.length + i0, c, history_cap, rows.as<float>(),
                             pres.as<unsigned char>(), st);
      CU(cudaGetLastError());
      CU(cudaMemcpyAsync(features + (size_t)i0 * history_cap * t->P.d8, rows.p, (size_t)c * rec_bytes, cudaMemcpyDeviceToHost, st));
      CU(cudaMemcpyAsync(feature_present + (size_t)i0 * history_cap, pres.p, (size_t)c * history_cap, cudaMemcpyDeviceToHost, st));
      CU(cudaStreamSynchronize(st));
    }
  }
  if ((rc = t->drop_wasted_front(n))) return rc;   // drain
  return n;
}

int64_t sb200_wasted_history(sb200_tracker* t, int64_t cap, uint64_t* ids, uint64_t* scene_ids, uint32_t* epochs, uint32_t* lengths,
                             float* predicted_boxes, float* observed_boxes, int32_t history_cap, float* predicted_history,
                             float* observed_history, int32_t* history_counts) {
  return wasted_records(t, cap, ids, scene_ids, epochs, lengths, predicted_boxes, observed_boxes, history_cap,
                        predicted_history, observed_history, history_counts, nullptr, nullptr);
}

int64_t sb200_wasted_visual(sb200_tracker* t, int64_t cap, uint64_t* ids, uint64_t* scene_ids, uint32_t* epochs, uint32_t* lengths,
                            float* predicted_boxes, float* observed_boxes, int32_t history_cap, float* predicted_history,
                            float* observed_history, int32_t* history_counts, float* features, uint8_t* feature_present) {
  if (!t) return fail(SB200_ERR_INVALID, "tracker is NULL");
  if (!t->fhist_on) return fail(SB200_ERR_INVALID, "the feature history is off (sb200_set_feature_history)");
  if (!features || !feature_present) return fail(SB200_ERR_INVALID, "features / feature_present is NULL");
  return wasted_records(t, cap, ids, scene_ids, epochs, lengths, predicted_boxes, observed_boxes, history_cap,
                        predicted_history, observed_history, history_counts, features, feature_present);
}

static int64_t dump_scene(sb200_tracker* t, uint64_t scene_id, int64_t cap, bool idle_only, uint64_t* ids,
                          uint32_t* epochs, uint32_t* lengths, float* pred, float* obs, float* states30,
                          int32_t* feat_counts) {
  if (!t || cap < 0) return fail(SB200_ERR_INVALID, "bad arguments");
  CU(cudaSetDevice(t->device));
  { int rc_ = t->drain(); if (rc_) return rc_; }
  int slot = t->slot_for(scene_id, false);
  if (slot < 0) return 0;
  int n = t->n_tracks[slot];
  if (n == 0) return 0;
  size_t base = (size_t)slot * t->track_cap;
  std::vector<uint64_t> hid(n);
  std::vector<uint32_t> hep(n), hle(n);
  std::vector<float> hpr((size_t)n * 6), hob((size_t)n * 6), hst((size_t)n * 30);
  std::vector<unsigned char> hfc(n, 0);
  cudaStream_t st = t->stream;
  CU(cudaMemcpyAsync(hid.data(), t->ts.id + base, 8 * (size_t)n, cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(hep.data(), t->ts.epoch + base, 4 * (size_t)n, cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(hle.data(), t->ts.length + base, 4 * (size_t)n, cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(hpr.data(), t->ts.pred + base * 6, 24 * (size_t)n, cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(hob.data(), t->ts.obs + base * 6, 24 * (size_t)n, cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpy2DAsync(hst.data(), 120, t->ts.kst + base * sb::kStateStride, 4 * (size_t)sb::kStateStride, 120, (size_t)n, cudaMemcpyDeviceToHost, st));
  if (t->P.is_visual) CU(cudaMemcpyAsync(hfc.data(), t->ts.feat_cnt + base, (size_t)n, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  int64_t k = 0;
  for (int j = 0; j < n && k < cap; ++j) {
    // SortLookup::IdleLookup (src/trackers/sort.rs:190-208): last_updated_epoch != current epoch of the scene
    if (idle_only && hep[j] == t->epoch[slot]) continue;
    if (ids) ids[k] = hid[j];
    if (epochs) epochs[k] = hep[j];
    if (lengths) lengths[k] = hle[j];
    if (pred) memcpy(pred + k * 6, &hpr[(size_t)j * 6], 24);
    if (obs) memcpy(obs + k * 6, &hob[(size_t)j * 6], 24);
    if (states30) memcpy(states30 + k * 30, &hst[(size_t)j * 30], 120);
    if (feat_counts) feat_counts[k] = hfc[j];
    ++k;
  }
  return k;
}

// expired tracks of `scene_id` swept early: the reference's store still holds them (they are idle by definition)
static int64_t append_hidden(sb200_tracker* t, uint64_t scene_id, int64_t k, int64_t cap, uint64_t* ids, uint32_t* epochs,
                             uint32_t* lengths, float* pred, float* obs) {
  const int64_t h0 = t->revealed, hn = t->wasted_count - t->revealed;
  if (hn <= 0 || k >= cap) return k;
  std::vector<uint64_t> hid(hn), hsc(hn);
  std::vector<uint32_t> hep(hn), hle(hn);
  std::vector<float> hpr((size_t)hn * 6), hob((size_t)hn * 6);
  cudaStream_t st = t->stream;
  CU(cudaMemcpyAsync(hid.data(), t->wb.id + h0, 8 * (size_t)hn, cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(hsc.data(), t->wb.scene + h0, 8 * (size_t)hn, cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(hep.data(), t->wb.epoch + h0, 4 * (size_t)hn, cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(hle.data(), t->wb.length + h0, 4 * (size_t)hn, cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(hpr.data(), t->wb.pred + h0 * 6, 24 * (size_t)hn, cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(hob.data(), t->wb.obs + h0 * 6, 24 * (size_t)hn, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  for (int64_t j = 0; j < hn && k < cap; ++j) {
    if (hsc[j] != scene_id) continue;
    if (ids) ids[k] = hid[j];
    if (epochs) epochs[k] = hep[j];
    if (lengths) lengths[k] = hle[j];
    if (pred) memcpy(pred + k * 6, &hpr[(size_t)j * 6], 24);
    if (obs) memcpy(obs + k * 6, &hob[(size_t)j * 6], 24);
    ++k;
  }
  return k;
}

int64_t sb200_idle_tracks(sb200_tracker* t, uint64_t scene_id, int64_t cap, uint64_t* ids, uint32_t* epochs,
                          uint32_t* lengths, float* predicted_boxes, float* observed_boxes) {
  int64_t k = dump_scene(t, scene_id, cap, true, ids, epochs, lengths, predicted_boxes, observed_boxes, nullptr, nullptr);
  if (k < 0) return k;
  return append_hidden(t, scene_id, k, cap, ids, epochs, lengths, predicted_boxes, observed_boxes);
}

int64_t sb200_scene_tracks(sb200_tracker* t, uint64_t scene_id, int64_t cap, uint64_t* ids, float* boxes,
                           float* states30, int32_t* feature_counts) {
  return dump_scene(t, scene_id, cap, false, ids, nullptr, nullptr, boxes, nullptr, states30, feature_counts);
}

int64_t sb200_last_costs(sb200_tracker* t, uint64_t scene_id, int64_t cap, float* out, int32_t* m, int32_t* n) {
  if (!t || !out || !m || !n) return fail(SB200_ERR_INVALID, "bad arguments");
  CU(cudaSetDevice(t->device));
  { int rc_ = t->drain(); if (rc_) return rc_; }
  *m = 0; *n = 0;
  if (t->last_n_scenes <= 0) return 0;
  // the scene table of the last frame was built on the device: read it back
  std::vector<sb::SceneDesc> sd((size_t)t->last_n_scenes);
  CU(cudaMemcpyAsync(sd.data(), t->f_scenes.p, sizeof(sb::SceneDesc) * sd.size(), cudaMemcpyDeviceToHost, t->stream));
  CU(cudaStreamSynchronize(t->stream));
  for (size_t si = 0; si < sd.size(); ++si) {
    const sb::SceneDesc& d = sd[si];
    if (d.scene_id != scene_id) continue;
    *m = d.m; *n = d.n;
    const int64_t full = (int64_t)d.m * d.n;
    const int64_t cnt = std::min<int64_t>(cap, full);
    if (cnt <= 0) return 0;
    // the dense matrix exists for scenes in dense voting mode and in SB200_FULL_COSTS runs; elsewhere the entry list is
    // the matrix (None wherever no entry is listed)
    int h[2] = {0, 0};   // pos_cnt, scene_mode
    sb::Frame ctr{};
    sb::carve_counters(t->f_counters.as<int>(), t->last_n_scenes, ctr);
    CU(cudaMemcpyAsync(&h[0], ctr.pos_cnt + si, 4, cudaMemcpyDeviceToHost, t->stream));
    CU(cudaMemcpyAsync(&h[1], ctr.scene_mode + si, 4, cudaMemcpyDeviceToHost, t->stream));
    CU(cudaStreamSynchronize(t->stream));
    const bool dense_exists = h[1] != 0 || getenv("SB200_FULL_COSTS") != nullptr;
    if (dense_exists) {
      CU(cudaMemcpyAsync(out, t->f_pos.as<float>() + d.pos_off, 4 * (size_t)cnt, cudaMemcpyDeviceToHost, t->stream));
      CU(cudaStreamSynchronize(t->stream));
      return cnt;
    }
    const int ne = std::min(h[0], d.pos_lcap);
    std::vector<sb::PosEntry> ents((size_t)std::max(ne, 0));
    if (ne > 0) {
      CU(cudaMemcpyAsync(ents.data(), t->f_poslist.as<sb::PosEntry>() + d.pos_lbase, sizeof(sb::PosEntry) * (size_t)ne,
                         cudaMemcpyDeviceToHost, t->stream));
      CU(cudaStreamSynchronize(t->stream));
    }
    const float qnan = std::nanf("");
    for (int64_t i = 0; i < cnt; ++i) out[i] = qnan;
    for (const sb::PosEntry& e : ents) {
      const int64_t idx = (int64_t)e.m * d.n + e.n;
      if (idx < cnt) out[idx] = e.v;
    }
    return cnt;
  }
  return 0;
}

int sb200_last_stage_ms(sb200_tracker* t, float* out5) {
  if (!t || !out5) return fail(SB200_ERR_INVALID, "bad arguments");
  { int rc_ = t->drain(); if (rc_) return rc_; }
  memcpy(out5, t->stage_ms, sizeof(float) * 5);
  return 0;
}

int sb200_last_kernel_ms(sb200_tracker* t, float* out2) {
  if (!t || !out2) return fail(SB200_ERR_INVALID, "bad arguments");
  { int rc_ = t->drain(); if (rc_) return rc_; }
  out2[0] = t->kernel_ms[0];
  out2[1] = t->kernel_ms[1];
  return 0;
}

}  // extern "C"

// =============================================================================================== state blob
// One versioned format for sb200_tracker_save / _load (the whole tracker) and sb200_scenes_export / _import (the live
// tracks of some scenes).  Layout: BlobHeader, then sections at 256-byte aligned offsets: the scene table (BlobScene per
// scene, in slot order for a tracker blob), one section per store column holding the listed scenes' rows back to back
// (live tracks, arena blocks or free-list entries: scene i's rows start at the prefix of the counts before it), then,
// for a tracker blob, the wasted buffer's records [0, wasted_count) and the feature-history pool (blocks [0, top), free
// stack [0, free)), or, for a scene blob with the feature history on, the history block of every live track in the
// order of the track columns.  Rows are copied as they are (BF16 copies, norms, permutations and vertex caches included),
// so a loaded tracker continues bit for bit.
namespace {

constexpr uint32_t kBlobMagic = 0x42534253u;   // "SBSB"
constexpr uint32_t kBlobVersion = 1;
constexpr uint32_t kBlobTracker = 1, kBlobScenes = 2;
constexpr int kMaxSections = 48;

struct BlobHeader {
  uint32_t magic, version, type, n_sections;
  uint64_t total_bytes;
  sb200_options opts;
  int32_t feature_history, hist_len, d8, n_scenes;
  int32_t seen_features, adapt_dense, auto_waste_counter, auto_waste_periodicity;
  int32_t scene_cap, track_cap, pad0, pad1;
  int64_t live_total, blk_total, free_total, wasted_count, revealed, hpool_top, hpool_free, hpool_cap;
  uint64_t id_counter;   // ids handed out by the source (at export, for a scene blob)
  uint64_t sec_off[kMaxSections], sec_bytes[kMaxSections];
};
struct BlobScene { uint64_t scene_id; uint32_t epoch; int32_t n_tracks, n_hidden, arena_top; };

// the columns of the sections after the scene table, in blob order
std::vector<Col> blob_cols(sb200_tracker* t, uint32_t type) {
  const bool tracker_blob = type == kBlobTracker;
  std::vector<Col> b;
  for (const Col& c : t->store_table())
    if (c.blob == kBlobAll || (c.blob == kBlobTrackerOnly && tracker_blob)) b.push_back(c);
  if (tracker_blob) {
    for (const Col& c : t->wasted_table()) b.push_back(c);
    if (t->fhist_on) for (const Col& c : t->pool_table()) b.push_back(c);
  } else if (t->fhist_on) {
    for (const Col& c : t->pool_table())   // the history rows of each live track, gathered from the pool
      if (c.rows == kRowHistTop) b.push_back({c.buf, nullptr, c.w, false, kRowTrackHist});
  }
  return b;
}

// byte sizes of every section, in blob order (the structure depends on the options only)
std::vector<uint64_t> section_bytes(sb200_tracker* t, uint32_t type, int64_t n_scenes, int64_t live, int64_t blk,
                                    int64_t fre, int64_t wasted, int64_t top, int64_t hfree) {
  std::vector<uint64_t> b = {(uint64_t)n_scenes * sizeof(BlobScene)};
  const int64_t cnt[] = {live, blk, fre, wasted, top, hfree, live};   // rows, by ColRows
  for (const Col& c : blob_cols(t, type)) b.push_back((uint64_t)cnt[c.rows] * c.w);
  return b;
}

// rows of a section that covers the whole tracker (kRowWasted, kRowHistTop, kRowHistFree)
int64_t tracker_rows(const BlobHeader& h, int rows) {
  return rows == kRowWasted ? h.wasted_count : (rows == kRowHistTop ? h.hpool_top : h.hpool_free);
}

struct SlotRows { int slot, n, blk, fre; };

// Pack (dir 0: store -> blob) or unpack (dir 1: blob -> store) of the store columns of `rows` (one per scene, in blob
// order) and, for a tracker blob, of the wasted buffer and the history pool; `dblob` is on the tracker's device.  For a
// scene blob with the feature history on, unpack hands the tracks the fresh pool blocks [hist_base, hist_base + live).
int move_store(sb200_tracker* t, int dir, uint32_t type, const BlobHeader& h, char* dblob, const std::vector<SlotRows>& rows,
               int hist_base) {
  const size_t tc = (size_t)t->track_cap;
  std::vector<sb::XferSeg> segs;
  const std::vector<Col> cols = blob_cols(t, type);
  size_t hist_sec = 0;   // scene blob: the history rows, then the present bytes, of the live tracks (launch_xfer_hist)
  for (size_t c = 0; c < cols.size(); ++c) {
    const Col& col = cols[c];
    char* sec = dblob + h.sec_off[1 + c];
    if (col.rows == kRowTrackHist) {
      if (!hist_sec) hist_sec = 1 + c;
      continue;
    }
    if (col.rows >= kRowWasted) {
      sb::add_segment(segs, dir, col.buf->as<char>(), sec, (uint64_t)tracker_rows(h, col.rows) * col.w);
      continue;
    }
    int64_t pre = 0;
    for (const SlotRows& r : rows) {
      const int64_t cnt = col.rows == kRowTrack ? r.n : (col.rows == kRowBlock ? r.blk : r.fre);
      sb::add_segment(segs, dir, col.buf->as<char>() + (size_t)r.slot * tc * col.w, sec + (uint64_t)pre * col.w,
                      (uint64_t)cnt * col.w);
      pre += cnt;
    }
  }
  const cudaStream_t st = t->stream;
  if (int rc = sb::copy_segments(segs, t->num_sms, st)) return rc;
  if (type == kBlobScenes && t->fhist_on && h.live_total > 0) {
    std::vector<int> tab(2 * rows.size() + 1, 0);   // slots | prefix of the live tracks
    for (size_t i = 0; i < rows.size(); ++i) { tab[i] = rows[i].slot; tab[rows.size() + i + 1] = tab[rows.size() + i] + rows[i].n; }
    DBuf d_tab;
    int rc = d_tab.ensure(tab.size() * sizeof(int));
    if (rc) return rc;
    CU(cudaMemcpyAsync(d_tab.p, tab.data(), tab.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    const int e = sb::launch_xfer_hist(t->ts, t->P.d8, d_tab.as<int>(), d_tab.as<int>() + rows.size(), (int)rows.size(),
                                       (int)h.live_total, dir, reinterpret_cast<float*>(dblob + h.sec_off[hist_sec]),
                                       reinterpret_cast<unsigned char*>(dblob + h.sec_off[hist_sec + 1]), hist_base, t->num_sms, st);
    if (e) return fail(SB200_ERR_CUDA, "history copy launch failed: %s", cudaGetErrorString((cudaError_t)e));
    CU(cudaStreamSynchronize(st));
  }
  return 0;
}

// Checks, on the device, every index a blob carries before anything is copied into the store: a track's arena block,
// the free list and the block owners against the scene's arena, observation counts and permutations against K, history
// block indices against the pool.  A damaged blob is refused instead of turning into out-of-bounds accesses later.
int check_indices(sb200_tracker* t, uint32_t type, const BlobHeader& h, const char* dblob,
                  const std::vector<BlobScene>& table) {
  std::vector<sb::XferCheck> ck;
  const std::vector<Col> cols = blob_cols(t, type);
  const int K = t->P.max_obs;
  const char* obs_n_sec = nullptr;
  for (size_t c = 0; c < cols.size(); ++c)
    if (cols[c].tag == kTagObsN) obs_n_sec = dblob + h.sec_off[1 + c];
  for (size_t c = 0; c < cols.size(); ++c) {
    const Col& col = cols[c];
    if (col.tag == kTagNone) continue;
    const char* sec = dblob + h.sec_off[1 + c];
    if (col.rows >= kRowWasted) {   // history block indices of the wasted records / the pool's free stack
      ck.push_back({sec, nullptr, tracker_rows(h, col.rows), 0, (int)h.hpool_top, 0});
      continue;
    }
    int64_t pre = 0;
    for (const BlobScene& s : table) {
      const int fre = s.arena_top - s.n_tracks;
      const int64_t cnt = col.rows == kRowTrack ? s.n_tracks : (col.rows == kRowBlock ? s.arena_top : fre);
      const char* p = sec + (uint64_t)pre * col.w;
      switch (col.tag) {
        case kTagFblk: case kTagFree: ck.push_back({p, nullptr, cnt, 0, s.arena_top, 0}); break;
        case kTagOwner: ck.push_back({p, nullptr, cnt, -1, s.n_tracks, 0}); break;
        case kTagHblk: ck.push_back({p, nullptr, cnt, 0, (int)h.hpool_top, 0}); break;
        case kTagObsN: ck.push_back({p, nullptr, cnt, 0, K + 1, 1}); break;
        case kTagObsPhys: ck.push_back({p, reinterpret_cast<const unsigned char*>(obs_n_sec) + pre, cnt, 0, K, 2}); break;
        default: break;
      }
      pre += cnt;
    }
  }
  ck.erase(std::remove_if(ck.begin(), ck.end(), [](const sb::XferCheck& x) { return x.n <= 0; }), ck.end());
  if (ck.empty()) return 0;
  DBuf d;
  int rc = d.ensure(ck.size() * sizeof(sb::XferCheck) + 16);
  if (rc) return rc;
  int* d_bad = reinterpret_cast<int*>(d.as<char>() + ck.size() * sizeof(sb::XferCheck));
  CU(cudaMemcpyAsync(d.p, ck.data(), ck.size() * sizeof(sb::XferCheck), cudaMemcpyHostToDevice, t->stream));
  CU(cudaMemsetAsync(d_bad, 0, sizeof(int), t->stream));
  const int e = sb::launch_xfer_check(d.as<sb::XferCheck>(), (int)ck.size(), K, d_bad, t->stream);
  if (e) return fail(SB200_ERR_CUDA, "index check launch failed: %s", cudaGetErrorString((cudaError_t)e));
  int bad = 0;
  CU(cudaMemcpyAsync(&bad, d_bad, sizeof(int), cudaMemcpyDeviceToHost, t->stream));
  CU(cudaStreamSynchronize(t->stream));
  if (bad) return fail(SB200_ERR_INVALID, "the blob holds %d out-of-range block or observation indices", bad);
  return 0;
}

// sets the device counters of the listed slots (and, for removed scenes, frees their history blocks); see XferSlot
int set_slots(sb200_tracker* t, const std::vector<sb::XferSlot>& tab, int free0, int free_add, int top_add,
              unsigned long long id_min, bool raise_ids) {
  if (tab.empty()) return 0;
  DBuf d_tab;
  int rc = d_tab.ensure(tab.size() * sizeof(sb::XferSlot));
  if (rc) return rc;
  CU(cudaMemcpyAsync(d_tab.p, tab.data(), tab.size() * sizeof(sb::XferSlot), cudaMemcpyHostToDevice, t->stream));
  const int e = sb::launch_xfer_slots(d_tab.as<sb::XferSlot>(), (int)tab.size(), t->b_ntracks.as<int>(), t->ts.n_free,
                                      t->ts.arena_top, t->ts, free0, free_add, top_add,
                                      raise_ids ? t->b_idc.as<unsigned long long>() : nullptr, id_min, t->stream);
  if (e) return fail(SB200_ERR_CUDA, "slot update launch failed: %s", cudaGetErrorString((cudaError_t)e));
  CU(cudaStreamSynchronize(t->stream));
  return 0;
}

uint64_t read_id_counter(sb200_tracker* t, int* rc) {
  uint64_t v = 0;
  *rc = 0;
  if (!t->b_idc.p) return 0;
  cudaError_t e = cudaMemcpyAsync(&v, t->b_idc.p, 8, cudaMemcpyDeviceToHost, t->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(t->stream);
  if (e != cudaSuccess) *rc = fail(SB200_ERR_CUDA, "id counter read failed: %s", cudaGetErrorString(e));
  return v;
}

// Writes the blob of `slots` (type kBlobScenes) or of the whole tracker to `dst` (host, or device memory on any device).
int save_blob(sb200_tracker* t, uint32_t type, const std::vector<int>& slots, void* dst, size_t cap, size_t* bytes) {
  if (int rc = t->regen_bf16()) return rc;   // the blob carries the BF16 rows
  BlobHeader h;
  memset(&h, 0, sizeof(h));
  h.magic = kBlobMagic; h.version = kBlobVersion; h.type = type;
  h.opts = t->opts;
  h.feature_history = t->fhist_on; h.hist_len = t->hist_len; h.d8 = t->P.d8; h.n_scenes = (int32_t)slots.size();
  h.seen_features = t->seen_features;
  if (type == kBlobTracker) {   // tracker-wide state: a scene blob carries the scenes alone
    h.adapt_dense = t->adapt_dense;
    h.auto_waste_counter = t->auto_waste_counter; h.auto_waste_periodicity = t->auto_waste_periodicity;
    h.scene_cap = t->scene_cap; h.track_cap = t->track_cap;
  }
  std::vector<BlobScene> table(slots.size());
  std::vector<SlotRows> rows(slots.size());
  for (size_t i = 0; i < slots.size(); ++i) {
    const int s = slots[i];
    const int blk = t->P.is_visual ? t->arena_top[s] : 0;
    table[i] = {t->scene_of_slot[s], t->epoch[s], t->n_tracks[s], type == kBlobTracker ? t->n_hidden[s] : 0, blk};
    rows[i] = {s, t->n_tracks[s], blk, t->P.is_visual ? blk - t->n_tracks[s] : 0};
    h.live_total += rows[i].n; h.blk_total += rows[i].blk; h.free_total += rows[i].fre;
  }
  if (type == kBlobTracker) {
    h.wasted_count = t->wasted_count; h.revealed = t->revealed;
    h.hpool_top = t->fhist_on ? t->hpool_top : 0; h.hpool_free = t->fhist_on ? t->hpool_free : 0;
    h.hpool_cap = t->fhist_on ? t->hpool_cap : 0;
  }
  int rc = 0;
  h.id_counter = read_id_counter(t, &rc);
  if (rc) return rc;
  const std::vector<uint64_t> sec = section_bytes(t, type, h.n_scenes, h.live_total, h.blk_total, h.free_total,
                                                  h.wasted_count, h.hpool_top, h.hpool_free);
  h.n_sections = (uint32_t)sec.size();
  sb::lay_out(h, sec.data(), h.n_sections);
  *bytes = (size_t)h.total_bytes;
  if (!dst || cap < h.total_bytes)
    return fail(SB200_ERR_CAPACITY, "the blob needs %llu bytes", (unsigned long long)h.total_bytes);
  return sb::write_blob(dst, t->device, t->stream, h, h.n_sections, [&](char* p) {
    if (!table.empty())
      CU(cudaMemcpyAsync(p + h.sec_off[0], table.data(), table.size() * sizeof(BlobScene), cudaMemcpyHostToDevice,
                         t->stream));
    return move_store(t, 0, type, h, p, rows, 0);
  });
}

// Orders the tracker's work after what the caller's stream (sb200_tracker_set_stream) holds now, as predict does: a device
// blob that the caller's stream is still writing (a receive) or reading (a send) is complete before the blob calls touch it.
int join_caller(sb200_tracker* t) {
  if (!t->has_user_stream) return 0;
  CU(cudaEventRecord(t->ev_user_in, t->user_stream));
  CU(cudaStreamWaitEvent(t->stream, t->ev_user_in, 0));
  return 0;
}

// every option an import compares: all but the capacity hints and the device; the constraints up to n_constraints
bool same_options(const sb200_options& a, const sb200_options& b) {
  auto f = [](float x, float y) { return x == y || (x != x && y != y); };
  if (a.kind != b.kind || a.positional_kind != b.positional_kind || !f(a.iou_threshold, b.iou_threshold) ||
      !f(a.min_confidence, b.min_confidence) || a.max_idle_epochs != b.max_idle_epochs || a.history_length != b.history_length ||
      !f(a.kalman_position_weight, b.kalman_position_weight) || !f(a.kalman_velocity_weight, b.kalman_velocity_weight) ||
      a.n_constraints != b.n_constraints || a.visual_kind != b.visual_kind || !f(a.visual_threshold, b.visual_threshold) ||
      a.feature_dim != b.feature_dim || a.visual_max_observations != b.visual_max_observations ||
      a.visual_min_votes != b.visual_min_votes || a.visual_minimal_track_length != b.visual_minimal_track_length ||
      !f(a.visual_minimal_area, b.visual_minimal_area) || !f(a.visual_minimal_quality_use, b.visual_minimal_quality_use) ||
      !f(a.visual_minimal_quality_collect, b.visual_minimal_quality_collect) ||
      !f(a.visual_minimal_own_area_percentage_use, b.visual_minimal_own_area_percentage_use) ||
      !f(a.visual_minimal_own_area_percentage_collect, b.visual_minimal_own_area_percentage_collect))
    return false;
  const int n = std::min(std::max(a.n_constraints, 0), SB200_MAX_CONSTRAINTS);
  for (int i = 0; i < n; ++i)
    if (a.constraint_epochs[i] != b.constraint_epochs[i] || !f(a.constraint_max_dist[i], b.constraint_max_dist[i])) return false;
  return true;
}

// Reads and checks the header and the scene table of a blob (host or device memory): magic, version, type, the
// section table against the sizes the counts imply, and the bounds of every section.
int parse_blob(const void* src, size_t bytes, uint32_t want_type, cudaStream_t st, BlobHeader* h,
               std::vector<BlobScene>* table) {
  if (bytes < sizeof(BlobHeader)) return fail(SB200_ERR_INVALID, "the blob is truncated (%zu bytes)", bytes);
  CU(cudaMemcpyAsync(h, src, sizeof(BlobHeader), cudaMemcpyDefault, st));
  CU(cudaStreamSynchronize(st));
  if (h->magic != kBlobMagic) return fail(SB200_ERR_INVALID, "not a state blob (bad magic)");
  if (h->version != kBlobVersion) return fail(SB200_ERR_INVALID, "state blob version %u (this library reads %u)", h->version, kBlobVersion);
  if (h->type != want_type)
    return fail(SB200_ERR_INVALID, h->type == kBlobTracker ? "a whole-tracker blob: use sb200_tracker_load"
                                                           : "a scene blob: use sb200_scenes_import");
  if (h->total_bytes > bytes) return fail(SB200_ERR_INVALID, "the blob is truncated (%zu of %llu bytes)", bytes, (unsigned long long)h->total_bytes);
  if (h->n_sections < 1 || h->n_sections > (uint32_t)kMaxSections) return fail(SB200_ERR_INVALID, "bad section count");
  if (int rc = sb::check_section_table(*h, h->n_sections)) return rc;
  if (h->n_scenes < 0 || h->live_total < 0 || h->blk_total < 0 || h->free_total < 0 || h->wasted_count < 0 ||
      h->revealed < 0 || h->revealed > h->wasted_count || h->hpool_top < 0 || h->hpool_free < 0 || h->hpool_free > h->hpool_top ||
      h->hpool_cap < 0 || (h->hpool_cap > 0 && h->hpool_cap < h->hpool_top) ||
      h->sec_bytes[0] != (uint64_t)h->n_scenes * sizeof(BlobScene))
    return fail(SB200_ERR_INVALID, "inconsistent blob counts");
  table->resize((size_t)h->n_scenes);
  if (h->n_scenes > 0)
  {
    CU(cudaMemcpyAsync(table->data(), static_cast<const char*>(src) + h->sec_off[0], h->sec_bytes[0], cudaMemcpyDefault, st));
    CU(cudaStreamSynchronize(st));
  }
  int64_t live = 0, blk = 0, hidden = 0;
  const bool visual = h->opts.kind == SB200_KIND_VISUAL_SORT || h->opts.kind == SB200_KIND_BATCH_VISUAL_SORT;
  std::unordered_map<uint64_t, int> seen;
  for (const BlobScene& s : *table) {
    if (s.n_tracks < 0 || s.n_hidden < 0 || (visual ? s.arena_top < s.n_tracks : s.arena_top != 0))
      return fail(SB200_ERR_INVALID, "inconsistent counts of scene %llu", (unsigned long long)s.scene_id);
    if (!seen.emplace(s.scene_id, 1).second) return fail(SB200_ERR_INVALID, "scene %llu appears twice in the blob", (unsigned long long)s.scene_id);
    live += s.n_tracks; blk += s.arena_top; hidden += s.n_hidden;
  }
  if (live != h->live_total || blk != h->blk_total || (visual && h->free_total != blk - live) ||
      (h->type == kBlobScenes && hidden != 0) || hidden > h->wasted_count - h->revealed)
    return fail(SB200_ERR_INVALID, "inconsistent blob counts");
  return 0;
}

// the section sizes the tracker `t` (built with the blob's options) expects for the blob's counts
int check_sections(sb200_tracker* t, const BlobHeader& h) {
  const std::vector<uint64_t> sec = section_bytes(t, h.type, h.n_scenes, h.live_total, h.blk_total, h.free_total,
                                                  h.wasted_count, h.hpool_top, h.hpool_free);
  if (sec.size() != h.n_sections) return fail(SB200_ERR_INVALID, "the blob has %u sections, %zu expected", h.n_sections, sec.size());
  for (size_t i = 0; i < sec.size(); ++i)
    if (sec[i] != h.sec_bytes[i]) return fail(SB200_ERR_INVALID, "section %zu holds %llu bytes, %llu expected", i,
                                              (unsigned long long)h.sec_bytes[i], (unsigned long long)sec[i]);
  return 0;
}

}  // namespace

extern "C" {

int sb200_tracker_save(sb200_tracker* t, void* dst, size_t cap, size_t* bytes) {
  if (!t || !bytes) return fail(SB200_ERR_INVALID, "tracker / bytes is NULL");
  int rc = sb::check_device(0);   // any device at all, before `t` is read
  if (rc) return rc;
  CU(cudaSetDevice(t->device));
  if ((rc = t->drain())) return rc;
  if ((rc = join_caller(t))) return rc;   // the caller's pending work on the destination comes first
  std::vector<int> slots(t->scene_of_slot.size());
  for (size_t i = 0; i < slots.size(); ++i) slots[i] = (int)i;
  return save_blob(t, kBlobTracker, slots, dst, cap, bytes);
}

int sb200_tracker_load(const void* src, size_t bytes, int32_t device, sb200_tracker** out) {
  if (!src || !out) return fail(SB200_ERR_INVALID, "src / out is NULL");
  *out = nullptr;
  int rc = sb::check_device(device);
  if (rc) return rc;
  BlobHeader h;
  std::vector<BlobScene> table;
  // no tracker (and no caller stream) yet: a device blob must be complete when the call is made
  rc = parse_blob(src, bytes, kBlobTracker, nullptr, &h, &table);
  if (rc) return rc;
  // created without the capacity hints, then sized to the source's store exactly (a save of the loaded tracker is the
  // same blob), then the hints restored for the growth of later frames
  sb200_options o = h.opts;
  o.device = device;
  o.max_scenes_hint = o.max_tracks_per_scene_hint = o.max_dets_per_scene_hint = 0;
  sb200_tracker* t = nullptr;
  if ((rc = sb200_tracker_create(&o, &t))) return rc;
  struct Guard { sb200_tracker* t; ~Guard() { if (t) sb200_tracker_destroy(t); } } guard{t};
  t->opts = h.opts;
  t->opts.device = device;
  if (h.feature_history && !t->P.is_visual) return fail(SB200_ERR_INVALID, "feature history on a non-visual tracker");
  if (h.feature_history && (rc = t->set_feature_history(true))) return rc;
  if (h.hist_len != t->hist_len || h.d8 != t->P.d8) return fail(SB200_ERR_INVALID, "the blob's row sizes do not match its options");
  if ((rc = check_sections(t, h))) return rc;
  int max_rows = 0;
  for (const BlobScene& s : table) max_rows = std::max(max_rows, std::max(s.n_tracks, s.arena_top));
  if ((h.scene_cap > 0 || !table.empty()) &&
      (rc = t->ensure_store(std::max<int>(h.scene_cap, (int)table.size()), std::max(std::max(h.track_cap, max_rows), 64))))
    return rc;
  if (h.wasted_count > 0 && (rc = t->ensure_wasted(h.wasted_count))) return rc;
  if (t->fhist_on && h.hpool_cap > 0 && (rc = t->ensure_hpool(std::max(h.hpool_cap, h.hpool_top)))) return rc;
  if ((rc = t->b_idc.ensure(8))) return rc;
  const char* dblob = nullptr;
  DBuf tmp;
  if ((rc = sb::blob_on_device(src, h.total_bytes, t->device, t->stream, tmp, &dblob))) return rc;
  if ((rc = check_indices(t, h.type, h, dblob, table))) return rc;
  std::vector<SlotRows> rows(table.size());
  std::vector<sb::XferSlot> st(table.size());
  for (size_t i = 0; i < table.size(); ++i) {
    const BlobScene& s = table[i];
    const int fre = t->P.is_visual ? s.arena_top - s.n_tracks : 0;
    rows[i] = {(int)i, s.n_tracks, s.arena_top, fre};
    st[i] = {(int)i, s.n_tracks, fre, s.arena_top, 0, 0};
  }
  if ((rc = move_store(t, 1, kBlobTracker, h, const_cast<char*>(dblob), rows, 0))) return rc;
  if ((rc = set_slots(t, st, 0, 0, 0, 0, false))) return rc;
  for (size_t i = 0; i < table.size(); ++i)
    if ((rc = t->regen_fp8((int)i, table[i].arena_top))) return rc;
  CU(cudaMemcpyAsync(t->b_idc.p, &h.id_counter, 8, cudaMemcpyHostToDevice, t->stream));
  if (h.wasted_count > 0) {
    const int wc = (int)h.wasted_count;
    CU(cudaMemcpyAsync(t->w_count.p, &wc, sizeof(int), cudaMemcpyHostToDevice, t->stream));
  }
  if (t->fhist_on) {
    const int hp[2] = {(int)h.hpool_free, (int)h.hpool_top};
    CU(cudaMemcpyAsync(t->ts.hpool, hp, sizeof(hp), cudaMemcpyHostToDevice, t->stream));
  }
  CU(cudaStreamSynchronize(t->stream));
  // host side: the scene table in slot order and the scalars
  for (const BlobScene& s : table) {
    const int slot = t->slot_for(s.scene_id, true);
    t->epoch[slot] = s.epoch; t->n_tracks[slot] = s.n_tracks; t->n_hidden[slot] = s.n_hidden; t->arena_top[slot] = s.arena_top;
  }
  t->wasted_count = h.wasted_count; t->revealed = h.revealed;
  t->hpool_top = h.hpool_top; t->hpool_free = h.hpool_free;
  t->auto_waste_counter = h.auto_waste_counter; t->auto_waste_periodicity = h.auto_waste_periodicity;
  t->adapt_dense = h.adapt_dense != 0; t->seen_features = h.seen_features != 0;
  t->transferred = true;
  guard.t = nullptr;
  *out = t;
  return 0;
}

int sb200_scenes_export(sb200_tracker* t, int32_t n_scenes, const uint64_t* scene_ids, int32_t remove, void* dst,
                        size_t cap, size_t* bytes) {
  if (!t || !bytes || n_scenes < 1 || !scene_ids) return fail(SB200_ERR_INVALID, "bad arguments");
  int rc = sb::check_device(0);   // any device at all, before `t` is read
  if (rc) return rc;
  CU(cudaSetDevice(t->device));
  if ((rc = t->drain())) return rc;
  std::vector<int> slots((size_t)n_scenes);
  std::unordered_map<uint64_t, int> seen;
  for (int i = 0; i < n_scenes; ++i) {
    if (!seen.emplace(scene_ids[i], i).second) return fail(SB200_ERR_INVALID, "scene %llu is listed twice", (unsigned long long)scene_ids[i]);
    slots[i] = t->slot_for(scene_ids[i], false);
    if (slots[i] < 0) return fail(SB200_ERR_INVALID, "unknown scene %llu", (unsigned long long)scene_ids[i]);
  }
  if ((rc = join_caller(t))) return rc;   // the caller's pending work on the destination comes first
  if ((rc = save_blob(t, kBlobScenes, slots, dst, cap, bytes))) return rc;
  if (!remove) return 0;
  // the slots start over: no tracks, no arena, epoch 0; the live tracks' history blocks go back on the pool's free list
  // (the hidden records of the scenes stay here, with their blocks, until this tracker's next collection point)
  std::vector<sb::XferSlot> st((size_t)n_scenes);
  int pushed = 0;
  for (int i = 0; i < n_scenes; ++i) {
    const int n = t->fhist_on ? t->n_tracks[slots[i]] : 0;
    st[i] = {slots[i], 0, 0, 0, n, pushed};
    pushed += n;
  }
  if ((rc = set_slots(t, st, (int)t->hpool_free, pushed, 0, 0, false))) return rc;
  for (int s : slots) { t->n_tracks[s] = 0; t->arena_top[s] = 0; t->epoch[s] = 0; }
  t->hpool_free += pushed;
  return 0;
}

int sb200_scenes_import(sb200_tracker* t, const void* src, size_t bytes) {
  if (!t || !src) return fail(SB200_ERR_INVALID, "tracker / src is NULL");
  int rc = sb::check_device(0);   // any device at all, before `t` is read
  if (rc) return rc;
  CU(cudaSetDevice(t->device));
  if ((rc = t->drain())) return rc;
  BlobHeader h;
  std::vector<BlobScene> table;
  if ((rc = join_caller(t))) return rc;   // a blob the caller's stream is still writing is complete from here on
  if ((rc = parse_blob(src, bytes, kBlobScenes, t->stream, &h, &table))) return rc;
  if (!same_options(h.opts, t->opts)) return fail(SB200_ERR_INVALID, "the blob's tracker options differ from this tracker's");
  if ((h.feature_history != 0) != t->fhist_on)
    return fail(SB200_ERR_INVALID, "the feature history is %s in the blob and %s here", h.feature_history ? "on" : "off", t->fhist_on ? "on" : "off");
  if ((rc = check_sections(t, h))) return rc;
  // a scene id that exists here is refused, unless its slot is empty (epoch 0, no tracks: a scene exported with `remove`)
  std::vector<int> dst_slot(table.size());
  int next = (int)t->scene_of_slot.size(), max_rows = 0;
  for (size_t i = 0; i < table.size(); ++i) {
    const int s = t->slot_for(table[i].scene_id, false);
    if (s >= 0 && (t->epoch[s] != 0 || t->n_tracks[s] != 0 || t->arena_top[s] != 0))
      return fail(SB200_ERR_INVALID, "scene %llu already exists in this tracker", (unsigned long long)table[i].scene_id);
    dst_slot[i] = s >= 0 ? s : next++;
    max_rows = std::max(max_rows, std::max(table[i].n_tracks, table[i].arena_top));
  }
  // ---- checks done: from here on only growth (which preserves the state) can fail before the copies
  if ((rc = t->ensure_store(std::max(next, t->scene_cap), std::max(std::max(max_rows, t->track_cap), 64)))) return rc;
  if (!t->b_idc.p) {
    if ((rc = t->b_idc.ensure(8))) return rc;
    CU(cudaMemsetAsync(t->b_idc.p, 0, 8, t->stream));
  }
  const long long hist_base = t->fhist_on ? t->hpool_top : 0;
  if (t->fhist_on && hist_base + h.live_total > t->hpool_cap &&
      (rc = t->ensure_hpool(std::max(hist_base + h.live_total, t->hpool_cap + t->hpool_cap / 2))))
    return rc;
  const char* dblob = nullptr;
  DBuf tmp;
  if ((rc = sb::blob_on_device(src, h.total_bytes, t->device, t->stream, tmp, &dblob))) return rc;
  if ((rc = check_indices(t, h.type, h, dblob, table))) return rc;
  std::vector<SlotRows> rows(table.size());
  std::vector<sb::XferSlot> st(table.size());
  for (size_t i = 0; i < table.size(); ++i) {
    const BlobScene& s = table[i];
    const int fre = t->P.is_visual ? s.arena_top - s.n_tracks : 0;
    rows[i] = {dst_slot[i], s.n_tracks, s.arena_top, fre};
    st[i] = {dst_slot[i], s.n_tracks, fre, s.arena_top, 0, 0};
  }
  if ((rc = move_store(t, 1, kBlobScenes, h, const_cast<char*>(dblob), rows, (int)hist_base))) return rc;
  if ((rc = set_slots(t, st, 0, 0, t->fhist_on ? (int)h.live_total : 0, h.id_counter, true))) return rc;
  for (size_t i = 0; i < table.size(); ++i)
    if ((rc = t->regen_fp8(dst_slot[i], table[i].arena_top))) return rc;
  for (size_t i = 0; i < table.size(); ++i) {
    const int slot = t->slot_for(table[i].scene_id, true);
    t->epoch[slot] = table[i].epoch; t->n_tracks[slot] = table[i].n_tracks; t->arena_top[slot] = table[i].arena_top;
  }
  if (t->fhist_on) t->hpool_top += h.live_total;
  if (h.seen_features) t->seen_features = true;
  t->transferred = true;
  return 0;
}

int sb200_tracker_options(sb200_tracker* t, sb200_options* out, int32_t* feature_dim_fixed) {
  if (!t || !out) return fail(SB200_ERR_INVALID, "tracker / out is NULL");
  *out = t->opts;
  if (feature_dim_fixed) *feature_dim_fixed = t->seen_features ? 1 : 0;
  return 0;
}

void* sb200_host_alloc(size_t bytes) {
  void* p = nullptr;
  if (cudaMallocHost(&p, bytes) != cudaSuccess) { cudaGetLastError(); fail(SB200_ERR_CUDA, "cudaMallocHost failed"); return nullptr; }
  return p;
}
void sb200_host_free(void* p) { if (p) cudaFreeHost(p); }

}  // extern "C"

// =============================================================================================== sb200_fstore_associate_wasted
// The tracker's side of that call (sb_wstore.cuh); wasted_store.cu holds the call itself.
namespace sb {

TrackerFeatureInfo tracker_feature_info(sb200_tracker* t) {
  return {t->device, t->P.is_visual, t->fhist_on, t->P.feature_dim, t->seen_features};
}

int64_t tracker_collect_wasted(sb200_tracker* t, int64_t cap, const WastedOut& out, std::vector<uint64_t>* ids,
                               WastedFeatures* feat) {
  CU(cudaSetDevice(t->device));
  { int rc_ = t->drain(); if (rc_) return rc_; }
  int rc = t->run_waste();  // wasted() starts with auto_waste (tracker_api.rs:90-91)
  if (rc) return rc;
  const int64_t n = std::min<int64_t>(cap, t->wasted_count);
  if (n == 0) return 0;
  ids->resize((size_t)n);
  WastedOut o = out;
  o.ids = ids->data();
  if ((rc = read_wasted(t, n, o))) return rc;
  if (out.ids) memcpy(out.ids, ids->data(), 8 * (size_t)n);
  *feat = {t->wb.hblk, t->wb.length, t->ts.hrows, t->ts.hpresent, t->hist_len, t->P.d8, t->stream};
  return n;
}

int tracker_drop_wasted(sb200_tracker* t, int64_t n) { return t->drop_wasted_front(n); }

// The tracker's side of sb200_scene_observations and sb200_fstore_search_tracks (live_store.cu).
int tracker_live(sb200_tracker* t, int n, const uint64_t* scene_ids, LiveTracks* lt, std::vector<LiveScene>* scenes) {
  CU(cudaSetDevice(t->device));
  { int rc_ = t->drain(); if (rc_) return rc_; }
  const TrackStore& ts = t->ts;
  *lt = {ts.id, ts.fblk, ts.obs_phys, ts.obs_hasf, ts.obs_n, ts.obs_q, ts.feat, t->track_cap, t->P.max_obs, t->P.d8,
         t->P.feature_dim, t->stream};
  scenes->resize((size_t)n);
  for (int i = 0; i < n; ++i) {
    const int slot = t->slot_for(scene_ids[i], false);
    (*scenes)[(size_t)i] = slot < 0 ? LiveScene{-1, 0} : LiveScene{(long long)slot * t->track_cap, t->n_tracks[slot]};
  }
  return 0;
}

}  // namespace sb
