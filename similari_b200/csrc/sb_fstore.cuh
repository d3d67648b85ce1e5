// sb_fstore.cuh -- device side of the feature track store (csrc/kernels_fstore.cu), shared with its host side
// (csrc/fstore.cu).  The store is the reference's TrackStore specialised to feature-only tracks: one feature class, the
// newest `max_observations` (K) observations of each track (src/track/store.rs, benches/feature_tracker.rs), and, in a
// gated store only, the CamTrackingAttributes of examples/track_merging.rs as track attributes (FsAttrCols, FsGate).  A
// quality store keeps each track's best observations instead, in its order from the ring start, with a quality per
// slot (examples/track_merging.rs:279-297, sb200_fstore_set_retention; the fs_launch_q* calls below).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <climits>
#include <vector>

#include "../../include/similari_b200.h"

namespace sb {

constexpr int kFsMaxTopn = 64;
constexpr int kFsMaxObs = 64;
constexpr int kFsMaxDim = 8192;
constexpr long long kFsMaxPairs = 1LL << 30;   // observation pairs of one call's distance matrix (4 B each)
constexpr int kFsMaxClasses = 16;   // SB200_FSTORE_MAX_CLASSES

// The store's device columns, in store order (insertion order; removal is a stable compaction).  Observation j (oldest
// first) of track t lives in ring slot (start[t] + j) % K of feat[t][.][.]; rows are zero-padded from D to d8 as
// Feature::from_vec pads (src/track/utils.rs:45-71).  Rows are stored as f32, binary16 or bfloat16 (stype, an
// SB200_FEATURE_*); every kernel that touches them is instantiated per storage type, picked by its launcher, and widens a
// stored element to f32 where it loads it.  stype sits in what was the struct's tail padding, so the layout the existing
// f32 kernels read is unchanged.
struct FsStore {
  void* feat;                 // [cap][K][d8] elements of stype
  int* cnt;                   // [cap] observations held (1..K)
  int* start;                 // [cap] ring slot of the oldest observation
  unsigned long long* ids;    // [cap]
  int* run;                   // [cap] scratch of the apply stage; zero between calls
  int K, d8, live;
  int stype;                  // storage type of feat (SB200_FEATURE_*); host side only
};

// One request on the device.  Items are the queries of search / associate, or the single observations of add.
struct FsCall {
  const float* rows;              // [R][d8] the items' observations (a query's newest K only), item by item
  const unsigned long long* qid;  // [Q]
  const int* qoff;                // [Q + 1] row ranges
  const int* row_q;               // [R] item of each row
  int* dest;                      // [Q] apply: store position to merge into, or -1 = new track at the end
  int* maxkey;                    // max_dist of the call, as an order-preserving int (fs_key)
  int4* plan;                     // [Q] apply: {position, first combined index, combined total, old ring start}
  float* qnorm;                   // [R] squared norms (cosine)
  float* snorm;                   // [live * K]
  float* dist;                    // [R][live * K] NaN == dropped (filtered, empty slot or same id)
  int* out_cnt;                   // [Q] results of TopN
  int* out_pos;                   // [Q][topn] store positions
  double* out_w;                  // [Q][topn]
  int Q, R;
};

// Track attributes of a gated store (sb200_fstore_set_gate): per stored track a source id and a [t0, t1] window, in
// columns of their own so that FsStore and FsCall keep their layout (CamTrackingAttributes, examples/track_merging.rs:
// 218-245).  An ungated store has none, and its kernels never see these structs.
struct FsAttrCols {
  unsigned long long* src;   // [cap]
  long long* t0;             // [cap]
  long long* t1;             // [cap]
};
// What the gated instances read: the stored columns, one triple per query of the call ([Q], indexed through row_q for
// a request row) and the rule (SB200_FSTORE_GATE_SAME_SOURCE or _ANY_SOURCE).
struct FsGate {
  FsAttrCols st;
  const unsigned long long* qsrc;
  const long long* qt0;
  const long long* qt1;
  int rule;
};

// CamTrackingAttributes::compatible (examples/track_merging.rs:222-225): the windows are disjoint, touching windows
// counting as disjoint, and under SB200_FSTORE_GATE_SAME_SOURCE (1) the sources are equal.  Symmetric in a and b.
__host__ __device__ __forceinline__ bool fs_compatible(int rule, unsigned long long as, long long a0, long long a1,
                                                       unsigned long long bs, long long b0, long long b1) {
  return (a0 >= b1 || a1 <= b0) && (rule != 1 || as == bs);
}

// The reference's `baked` (examples/track_merging.rs:240-247, compared in u128): now > t_end + period, exact for every
// int64 value.  The sum leaves the int64 range only where its sign alone decides the answer.
__host__ __device__ __forceinline__ bool fs_baked(long long now, long long t_end, long long period) {
  if (period >= 0) return t_end <= LLONG_MAX - period && now > t_end + period;
  return t_end < LLONG_MIN - period || now > t_end + period;
}

// How an owned search (sb200_fstore_search_owned) differs from a search of foreign queries, as template parameters of
// the distance and TopN kernels: kFsForeign is the search / associate path; kFsOwnedGroup drops the entries of the
// tracks marked in excl[live] (the queried ones); kFsOwnedEach folds max_dist per query into maxkey[Q].
enum { kFsForeign = 0, kFsOwnedGroup = 1, kFsOwnedEach = 2 };

// order-preserving map of an f32 onto an int (negative values included); NaN never reaches it
__host__ __device__ __forceinline__ int fs_key(float f) {
  int b;
  memcpy(&b, &f, 4);
  return b >= 0 ? b : (b ^ 0x7fffffff);
}

// The rows of the caller's feature column that take part in a search / associate call: the newest K of each query, query
// by query, oldest first (a track built by TrackBuilder keeps its newest K, src/track/builder.rs:168-179).  row_src[r] is
// the column row behind request row r, qoff[q] .. qoff[q + 1] the request rows of query q.  offs is the caller's CSR
// (offs[0] == 0, every query with at least one row: checked by the caller).
inline void fs_row_table(int Q, const int32_t* offs, int K, std::vector<int>* row_src, std::vector<int>* qoff) {
  row_src->clear();
  qoff->assign(1, 0);
  for (int q = 0; q < Q; ++q) {
    for (int r = std::max(offs[q], offs[q + 1] - K); r < offs[q + 1]; ++r) row_src->push_back(r);
    qoff->push_back((int)row_src->size());
  }
}

// rows[r][0 .. d8) = column row row_src[r] widened to f32 and zero-padded from D; `type` is the column's SB200_FEATURE_*
void fs_launch_stage(int type, const void* col, const int* row_src, int R, int D, int d8, float* rows, cudaStream_t st);
// rows[r][0 .. d8) = observation r - qoff[q] (oldest first) of the stored track at qpos[q], q = row_q[r]
void fs_launch_owned_stage(const FsStore& s, const FsCall& c, const int* qpos, float* rows, cudaStream_t st);
// mode: kFsForeign, kFsOwnedGroup (excl[live] marks the queried tracks) or kFsOwnedEach
// gate: a gated store's attributes; the pairs it finds incompatible are dropped like filtered ones (NaN)
void fs_launch_dist(int metric, float filter, const FsStore& s, const FsCall& c, cudaStream_t st, int mode = kFsForeign,
                    const unsigned char* excl = nullptr, const FsGate* gate = nullptr);
void fs_launch_topn(float max_distance, int min_votes, int topn, bool want_dest, const FsStore& s, const FsCall& c,
                    cudaStream_t st, int mode = kFsForeign);
// BestFit voting, after fs_launch_topn on the same call (the call's max_dist in maxkey[0]): every group of the call claims
// its track, the heaviest group, lower query on ties, winning it; a reported element whose track another query claimed
// gets position -2 (the host reports the query's id), and with want_dest dest[q] = the first element's track if q
// claimed it, else -1.  wmax / qmin: [live] scratch, initialised here.  Returns the error of that initialisation.
cudaError_t fs_launch_claim(float max_distance, int min_votes, int topn, bool want_dest, const FsStore& s,
                            const FsCall& c, unsigned long long* wmax, int* qmin, cudaStream_t st);
// out[2 i] = cnt[pos[i]], out[2 i + 1] = start[pos[i]]: the ring state of the tracks an owned call touches
void fs_launch_peek(const FsStore& s, const int* pos, int n, int* out, cudaStream_t st);
// merge_owned: scratch[m] = stored row src[m], then stored row dst[m] = scratch[m] (rows index feat as [cap * K][d8];
// scratch rows are in the storage type), and cnt / start of the tracks hdr[3 j] set to hdr[3 j + 1] / hdr[3 j + 2]
void fs_launch_move_rows(const FsStore& s, const int* src, const int* dst, int n_moves, const int* hdr, int n_hdr,
                         void* scratch, cudaStream_t st);
// merge / append; the f32 request rows are rounded to the storage type here (round to nearest even), and nowhere else
void fs_launch_apply(const FsStore& s, const FsCall& c, cudaStream_t st);
// out[i][b][.] = observation b (oldest first) of the track at pos[i] (-1: none), widened to f32, out_cnt[i] its count (0
// for -1)
void fs_launch_gather(const FsStore& s, const int* pos, int n, float* out, int* out_cnt, cudaStream_t st);
// dst[i] = src[from[i]] for the i < n kept tracks (stable compaction into fresh columns)
void fs_launch_compact(const FsStore& src, const FsStore& dst, const int* from, int n, cudaStream_t st);
// gated associate, between TopN and apply: in query order, a query stays with its first winner (dest[q]) only if it is
// compatible with that track's window as extended by the queries kept with it before; else dest[q] = -1 (a new track).
// The kept queries' hulls are written into the stored windows.
void fs_launch_gate_resolve(const FsCall& c, const FsGate& g, cudaStream_t st);
// gated associate, after apply: the triple of every query that became a new track (dest[q] >= live) into its position
void fs_launch_attr_new(int live, const FsCall& c, const FsGate& g, cudaStream_t st);
// out[i] = the triple at pos[i] (0 for pos[i] < 0): read-back of touched tracks, the triples of owned queries and the
// compaction of fetch(remove) (out = fresh columns, pos = the kept positions)
void fs_launch_attr_gather(const FsAttrCols& a, const int* pos, int n, const FsAttrCols& out, cudaStream_t st);
// the triple at pos[i] = in[i]
void fs_launch_attr_scatter(const FsAttrCols& a, const int* pos, int n, const FsAttrCols& in, cudaStream_t st);
// store blob of a gated store, before anything is copied: bad[0] counts the windows with t0 > t1
void fs_launch_attr_check(const long long* t0, const long long* t1, int n, int* bad, cudaStream_t st);
// store blob, after its rows are copied: zeroes, in feat[n][K][d8] (elements of stype), the ring slots that hold no
// observation
void fs_launch_blob_scrub(int stype, void* feat, const int* cnt, const int* start, int n, int K, int d8, cudaStream_t st);

// ---- feature classes (sb200_fstore_set_classes): each class has its own feat, cnt, start (and qual) columns, over the
// shared ids, run and capacity, so every kernel above runs on one class's FsStore unchanged.  The cnt and start columns
// of every class, in declared order:
struct FsClassCols {
  const int* cnt[kFsMaxClasses];
  const int* start[kFsMaxClasses];
  int n;
};
// out[i][k] = cnt of class k at pos[i] (0 for pos[i] < 0)
void fs_launch_class_counts(const FsClassCols& cc, const int* pos, int n, int* out, cudaStream_t st);
// store blob of any version, before anything is copied (the columns: the blob's sections): bad[0] counts the cnt outside
// [0, K], bad[1] the start outside [0, K), bad[2] the tracks without a row in any class (of one class: the cnt of 0)
void fs_launch_class_check(const FsClassCols& cc, int n, int K, int* bad, cudaStream_t st);

// ---- a quality store (sb200_fstore_set_retention): observations kept in the track's order in ring slots 0, 1, ... (the
// ring start is always 0), qual[cap][K] the quality of the row in each slot (0 where a slot holds none) and hlen[cap]
// each track's merge history length.
// What associate and add on a quality store read besides FsStore and FsCall (a struct of its own, so that FsStore and
// FsCall keep their layout): the quality and history-length columns, c(h) for h < ntab (c(h) = cap_tab[ntab - 1]
// beyond), the request rows' qualities [R], and whether the call merges queries (associate: each adds a history of
// length 1) or appends rows (add).
struct FsQCall {
  float* qual;
  int* hlen;
  const int* cap_tab;
  int ntab;
  const float* rq;
  int assoc;
};
// associate / add: new positions for dest[q] == -1, then each destination's merges and appends in item order, each
// truncated at its own capacity, and the rows, qualities, counts, history lengths and new ids written.  hq: the history
// length of each query (associate_store, whose queries are stored tracks of another store), else every query adds 1.
void fs_launch_qmerge(const FsStore& s, const FsCall& c, const FsQCall& qc, cudaStream_t st, const int* hq = nullptr);
// associate_store on a quality store: rq[r] = the quality of the stored observation fs_launch_owned_stage copies into
// request row r (of the track at qpos[row_q[r]] of the store s, with its qualities qual)
void fs_launch_qual_stage(const FsStore& s, const FsCall& c, const float* qual, const int* qpos, float* rq,
                          cudaStream_t st);
// find_baked: out[0] = the number of the n tracks with fs_baked(now, t_end[i], period), out[1 ..] their positions in
// store order
void fs_launch_baked(const long long* t_end, int n, long long now, long long period, int* out, cudaStream_t st);
// out[2 i] = cnt, out[2 i + 1] = start of the track at pos[i]; oq[i][j] = the quality of its observation j (0 past cnt)
void fs_launch_qpeek(const FsStore& s, const float* qual, const int* pos, int n, int* out, float* oq, cudaStream_t st);
// qual[pos[i]][0 .. K) = vals[i][0 .. K), hlen[pos[i]] = hl[i]
void fs_launch_qual_set(float* qual, int* hlen, const int* pos, const float* vals, const int* hl, int n, int K,
                        cudaStream_t st);
// dst[i][.] = src[from[i]][.], i < n, w 32-bit words per track: the qualities and history lengths of a compaction
void fs_launch_words_compact(const void* src, void* dst, const int* from, int n, int w, cudaStream_t st);
// store blob, before anything is copied: bad[0] counts the NaN qualities in filled slots, bad[1] the observations whose
// quality is above the one before
void fs_launch_qual_check(const float* qual, const int* cnt, const int* start, int n, int K, int* bad, cudaStream_t st);
// store blob, after its sections are copied: zeroes the qualities of the slots that hold no observation
void fs_launch_qual_scrub(float* qual, const int* cnt, const int* start, int n, int K, cudaStream_t st);

// ---- the store blob's sections (layouts: include/similari_b200.h).  What a section holds:
enum {
  kFsSecIds, kFsSecSource, kFsSecTStart, kFsSecTEnd, kFsSecHistLen, kFsSecHistory, kFsSecClassIds, kFsSecClassDims,
  kFsSecCnt, kFsSecStart, kFsSecFeat, kFsSecQuality
};
struct FsSection {
  const char* name;
  uint64_t bytes;
  int role;   // kFsSec*
  int cls;    // the class index of a per-class section (cnt, start, feat, quality), else 0
};

// The sections of a blob of `version` (1 to 4), in blob order, for a store of `live` tracks of K observations stored as
// `stype`, with gate rule `gate`, retention rule `keep`, n classes of dims[] and hist_total merge history entries.
// Versions 1 to 3 are one class's; a version-2 blob is gated, and a version-3 one keeps by quality.  Host code only.
inline std::vector<FsSection> fs_blob_sections(int version, uint64_t live, int K, int stype, int gate, int keep, int n,
                                               const int32_t* dims, uint64_t hist_total) {
  static const char* const kNames[] = {"ids",        "source",     "t_start", "t_end", "history_length", "history",
                                       "class_ids",  "class_dims", "cnt",     "start", "feat",           "quality"};
  std::vector<FsSection> out;
  auto add = [&](int role, uint64_t bytes, int k = 0) { out.push_back({kNames[role], bytes, role, k}); };
  const uint64_t g = gate ? live * 8 : 0, hl = keep ? live * 4 : 0, h = keep ? hist_total * 8 : 0;
  const uint64_t q = keep ? live * K * 4 : 0, elem = stype == SB200_FEATURE_F32 ? 4 : 2;
  auto feat = [&](int k) { return live * K * ((uint64_t)(dims[k] + 7) / 8 * 8) * elem; };
  auto attrs = [&] { add(kFsSecSource, g); add(kFsSecTStart, g); add(kFsSecTEnd, g); };
  add(kFsSecIds, live * 8);
  if (version < 4) {
    add(kFsSecCnt, live * 4);
    add(kFsSecStart, live * 4);
    add(kFsSecFeat, feat(0));
    if (version >= 2) attrs();
    if (version == 3) {
      add(kFsSecQuality, q);
      add(kFsSecHistLen, hl);
      add(kFsSecHistory, h);
    }
    return out;
  }
  attrs();
  add(kFsSecHistLen, hl);
  add(kFsSecHistory, h);
  add(kFsSecClassIds, (uint64_t)n * 8);
  add(kFsSecClassDims, (uint64_t)n * 4);
  for (int k = 0; k < n; ++k) {
    add(kFsSecCnt, live * 4, k);
    add(kFsSecStart, live * 4, k);
    add(kFsSecFeat, feat(k), k);
    add(kFsSecQuality, q, k);
  }
  return out;
}

// the index in `plan` of the section of `role` (and class k), or -1
inline int fs_blob_section(const std::vector<FsSection>& plan, int role, int k = 0) {
  for (size_t i = 0; i < plan.size(); ++i)
    if (plan[i].role == role && plan[i].cls == k) return (int)i;
  return -1;
}

}  // namespace sb
