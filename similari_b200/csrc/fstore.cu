// fstore.cu -- host side of the feature track store (sb200_fstore_*): argument checks, device memory, the launch
// sequence of a call (distances -> TopN -> apply, kernels_fstore.cu) and the host copy of the store's id order.
// A call stages its request in one pinned buffer, uploads it once, runs its kernels back to back on the handle's stream
// and downloads its results once.  Everything a call can reject is checked before anything is launched or changed.
// The request rows reach the device in one of two ways: an f32 host column is staged row by row in the pinned buffer; a
// 2-byte host column (uploaded raw) and a device column (read in place) go through fs_stage_kernel.  The store blob
// (sb200_fstore_save / _load) shares the trackers' section layout, placement and copy machinery (sb_blob.cuh); all four
// of its versions go through one section plan (sb::fs_blob_sections), one writer (save) and one loader (load_blob, then
// the member load, whose device check is fs_class_check_kernel for every version).  The
// owned calls (search_owned, merge_owned) take stored tracks: their rows never leave the device, and the host reads back
// only the counts and ring starts of the tracks they touch.  The stored rows are f32, binary16 or bfloat16 (stype,
// sb200_fstore_set_storage_type); row_bytes() is the size of one stored row, and nothing else on the host depends on the
// storage type.  A gated store (sb200_fstore_set_gate) also keeps a source and a window per track in three device
// columns of its own; a call reads back the triples of the tracks it touches, and an ungated store allocates none.
// Allocation, growth, compaction, the gate switch and the blob sections all go by one table of columns (kCols).
// A quality store (sb200_fstore_set_retention) keeps each track's rows in the track's order (best first) from ring slot
// 0, so the search, fetch and owned kernels walk it unchanged, plus a quality per slot (qual) and a history length per
// track (hlen) on the device and the merge histories on the host (hist, beside hid, updated from each call's
// read-back).  Associate and add plan and apply their merges on the device (fs_launch_qmerge), with one read-back as on
// a newest store; merge_owned plans on the host from the qualities of the tracks it touches, as it plans rings.
// associate_store takes stored tracks of another store as the queries of one associate call: its row source
// (StoreRows) stages their rows, triples, qualities and history lengths from the source store's columns on the
// destination's stream, so the rows never leave the device; find_baked selects tracks by their t_end on the device and
// reads back only the selected positions.
#include <cuda_runtime.h>

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstddef>
#include <cstring>
#include <numeric>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "../../include/similari_b200.h"
#include "sb_blob.cuh"
#include "sb_fstore.cuh"
#include "sb_host.cuh"
#include "sb_wstore.cuh"

namespace {

using sb::DBuf;
using sb::fail;

size_t align16(size_t v) { return (v + 15) & ~size_t(15); }

// byte offsets of one request in the staging buffer (the device copy has the same layout)
struct ReqLayout {
  size_t rows, qid, qoff, row_q, dest, maxkey, row_src, qpos, excl, total;
  // with_src: the request carries the row-index table of fs_stage_kernel instead of host-staged rows.  An owned search
  // (owned_live >= 0) carries nkey max_dist keys (one per query in the each mode), the store position of each query and
  // an exclusion byte per stored track (owned_live of them; 0 in the each mode).
  ReqLayout(int Q, int R, int d8, bool with_src, int nkey = 1, long long owned_live = -1) {
    size_t o = 0;
    rows = o; o = align16(o + (size_t)R * d8 * 4);
    qid = o; o = align16(o + (size_t)Q * 8);
    qoff = o; o = align16(o + (size_t)(Q + 1) * 4);
    row_q = o; o = align16(o + (size_t)R * 4);
    dest = o; o = align16(o + (size_t)Q * 4);
    maxkey = o; o = align16(o + (size_t)nkey * 4);
    row_src = o;
    if (with_src) o = align16(o + (size_t)R * 4);
    qpos = excl = o;
    if (owned_live >= 0) {
      o = align16(o + (size_t)Q * 4);
      excl = o; o = align16(o + (size_t)owned_live);
    }
    total = o;
  }
};
// Stages what every request carries at hq, the host address of offset L.qid: ids, offsets, row -> query, dest (nullptr:
// -1 for every query) and nkey initial max_dist keys.
void stage_request(const ReqLayout& L, char* hq, int Q, const uint64_t* qids, const int* qoff, const int* dest, int nkey) {
  auto at = [&](size_t off) { return hq + (off - L.qid); };
  memcpy(at(L.qid), qids, (size_t)Q * 8);
  memcpy(at(L.qoff), qoff, (size_t)(Q + 1) * 4);
  int* row_q = reinterpret_cast<int*>(at(L.row_q));
  for (int q = 0; q < Q; ++q)
    for (int r = qoff[q]; r < qoff[q + 1]; ++r) row_q[r] = q;
  int* d = reinterpret_cast<int*>(at(L.dest));
  if (dest) memcpy(d, dest, (size_t)Q * 4);
  else std::fill_n(d, Q, -1);
  std::fill_n(reinterpret_cast<int*>(at(L.maxkey)), nkey, sb::fs_key(-1.0f));   // max_dist starts at -1.0 (topn.rs:78)
}

struct ResLayout {
  size_t w, cnt, pos, total;
  ResLayout(int Q, int topn) {
    size_t o = 0;
    w = o; o = align16(o + (size_t)Q * topn * 8);
    cnt = o; o = align16(o + (size_t)Q * 4);
    pos = o; o = align16(o + (size_t)Q * topn * 4);
    total = o;
  }
};

// the feature column of a call: a host pointer, or a device pointer with the caller's stream
struct Column {
  const void* p;
  bool on_device;
  cudaStream_t caller;
};

using BlobHeader = sb200_fstore_blob_header;
using BlobHeaderV2 = sb200_fstore_blob_header_v2;
using BlobHeaderV3 = sb200_fstore_blob_header_v3;
using BlobHeaderV4 = sb200_fstore_blob_header_v4;
static_assert(offsetof(BlobHeaderV2, live) == offsetof(BlobHeader, live), "version 2 repeats version 1's fields");
static_assert(offsetof(BlobHeaderV3, gate) == offsetof(BlobHeaderV2, gate), "version 3 repeats version 2's fields");
static_assert(offsetof(BlobHeaderV4, merge_extension) == offsetof(BlobHeaderV3, merge_extension),
              "version 4 repeats version 3's fields");
static_assert(SB200_FSTORE_MAX_CLASSES == sb::kFsMaxClasses, "the class bound of the kernels");

// The header of each blob version; `version` (1 to 4) names the blob's, and visit(f) calls f on it.
struct BlobHeaders {
  uint32_t version;
  BlobHeader v1;
  BlobHeaderV2 v2;
  BlobHeaderV3 v3;
  BlobHeaderV4 v4;
  template <class F> auto visit(F&& f) {
    switch (version) {
      case 1: return f(v1);
      case 2: return f(v2);
      case 3: return f(v3);
    }
    return f(v4);
  }
};

// What load reads from a blob's header besides the fields every version shares: a version-1 blob is an ungated newest
// store, a version-2 blob a gated newest one, and versions 1 to 3 hold one class
struct BlobView {
  uint32_t version;
  int gate = SB200_FSTORE_GATE_NONE, keep = SB200_FSTORE_KEEP_NEWEST, init_cap = 0;
  float ext = 0.0f;
  int n_classes = 1;
  const uint64_t* sec_off = nullptr;
  const uint64_t* sec_bytes = nullptr;
};
// the gate and retention rules a blob of each version may carry (bit r: rule r), by version
constexpr unsigned kBlobGates[5] = {0, 1u << SB200_FSTORE_GATE_NONE,
                                    1u << SB200_FSTORE_GATE_SAME_SOURCE | 1u << SB200_FSTORE_GATE_ANY_SOURCE, 7u, 7u};
constexpr unsigned kBlobKeeps[5] = {0, 1u << SB200_FSTORE_KEEP_NEWEST, 1u << SB200_FSTORE_KEEP_NEWEST,
                                    1u << SB200_FSTORE_KEEP_BEST_QUALITY, 3u};
bool allowed(unsigned rules, int r) { return r >= 0 && r < 32 && (rules >> r & 1u); }

// the store kinds that have a column (sb200_fstore::Col::need)
enum { kNeedAll, kNeedGate, kNeedQuality };
// which columns a step of alloc / swap_columns handles: every one, the shared ones, or the selected class's
enum { kPartAll, kPartShared, kPartClass };

// The queries of associate_store, which its row source puts on the device besides the rows: their triples in qattr (a
// gated store) and their rows' qualities in dqr (a quality store).  hq[Q]: their history lengths on the device, and
// hist[q] their merge histories (a quality store; else nullptr).
struct TrackQueries {
  const int* hq;
  const std::vector<std::vector<uint64_t>>* hist;
};

// a gated call's triples on the host: n entries of each column
struct Triples {
  std::vector<uint64_t> src;
  std::vector<int64_t> t0, t1;
  explicit Triples(size_t n = 0) : src(n), t0(n), t1(n) {}
};

bool known_type(int t) { return t == SB200_FEATURE_F32 || t == SB200_FEATURE_F16 || t == SB200_FEATURE_BF16; }
size_t type_bytes(int t) { return t == SB200_FEATURE_F32 ? 4 : 2; }

// c(h) = min(K, (u64)((float)init * powf(ext, (float)h))) for h = 0 .. the first h with c(h) == K (h = 0 alone for a
// constant capacity, ext == 1), as examples/track_merging.rs:257-265 computes it: f32 arithmetic with the C library's
// powf (what Rust's f32::powf calls), then the truncating cast of `as u64`.  Refuses what the store does not take.
int capacity_table(int K, int init, float ext, std::vector<int>* tab) {
  if (init < 1) return fail(SB200_ERR_INVALID, "initial_capacity %d < 1", init);
  if (!std::isfinite(ext) || ext < 1.0f) return fail(SB200_ERR_INVALID, "merge_extension %g is not finite or is below 1", ext);
  auto c = [&](int h) {
    const float v = (float)init * powf(ext, (float)h);
    return v >= (float)K ? K : (int)(uint64_t)v;
  };
  tab->assign(1, c(0));
  while (tab->back() < K && ext != 1.0f) {
    if (tab->size() > 65536)
      return fail(SB200_ERR_INVALID, "initial_capacity %d and merge_extension %g do not reach max_observations %d by a "
                  "merge history of 65536", init, ext, K);
    tab->push_back(c((int)tab->size()));
  }
  return 0;
}

// the first NaN of n qualities, or -1
int first_nan(int n, const float* q) {
  for (int i = 0; i < n; ++i)
    if (std::isnan(q[i])) return i;
  return -1;
}

int check_options(const sb200_fstore_options& o) {
  if (o.metric != SB200_VIS_EUCLIDEAN && o.metric != SB200_VIS_COSINE) return fail(SB200_ERR_INVALID, "unknown metric");
  if (o.max_observations < 1 || o.max_observations > SB200_FSTORE_MAX_OBS)
    return fail(SB200_ERR_INVALID, "max_observations must lie in 1..64");
  if (o.feature_dim < 1 || o.feature_dim > SB200_FSTORE_MAX_DIM)
    return fail(SB200_ERR_INVALID, "feature_dim must lie in 1..8192");
  if (o.topn < 1 || o.topn > SB200_FSTORE_MAX_TOPN) return fail(SB200_ERR_INVALID, "topn must lie in 1..64");
  if (o.min_votes < 0) return fail(SB200_ERR_INVALID, "min_votes < 0");
  return 0;
}

}  // namespace

struct sb200_fstore {
  sb200_fstore_options o{};
  int d8 = 8;
  int ftype = SB200_FEATURE_F32;   // element type of the calls' feature columns
  int stype = SB200_FEATURE_F32;   // element type of the stored rows
  int num_sms = 1;
  cudaStream_t st = nullptr;
  cudaEvent_t ev[4] = {};
  cudaEvent_t ev_in = nullptr;     // what the caller's stream held when a device-column call was made
  float stage_ms[3] = {0, 0, 0};
  // store columns (kCols)
  size_t cap = 0;
  DBuf feat, cnt, start, ids, run;
  int gate = SB200_FSTORE_GATE_NONE;
  int voting = SB200_FSTORE_VOTING_TOPN;     // how calls read the store; handle state, not saved in the blob
  DBuf asrc, at0, at1;                       // gated store: [cap] source, t_start, t_end
  int keep = SB200_FSTORE_KEEP_NEWEST;       // retention rule, and its parameters for a quality store
  int init_cap = 4;
  float ext = 1.5f;
  std::vector<int> cap_tab;                  // quality store: c(h) (capacity_table), and its device copy
  DBuf dcap;
  DBuf qual, hlen;                           // quality store: [cap][K] quality of the row in each slot, [cap] history length
  DBuf dqr;                                  // quality store: the request rows' qualities of a call
  std::vector<std::vector<uint64_t>> hist;   // quality store: merge history of each track, in store order
  // A store column: its buffer, bytes per track (0: K stored rows) or per slot (per_obs), the kind of store that has it
  // (kNeed*), whether allocation zero-fills it, and what its blob sections hold (sb::kFsSec*).  Without a section (-1)
  // it is scratch, which growth and compaction start afresh.
  // Per-class columns (per_class) exist once per declared feature class; the selected class's sit in the members above
  // and the others' in cls (select).
  struct Col {
    DBuf sb200_fstore::*buf; uint32_t w; bool per_obs; int need; bool zero; int sec; bool per_class;
  };
  static constexpr int kNumCols = 10;
  static const Col kCols[kNumCols];
  // Feature classes (sb200_fstore_set_classes), in declared order.  Capacity is shared, so every class holds its feat
  // [cap][K][d8_c], cnt, start and (quality store) qual columns; cls[sel]'s buffers are empty while it is selected, its
  // columns being the members feat, cnt, start and qual, and d8 / o.feature_dim being its own.
  struct ClassCols { uint64_t id; int dim, d8; DBuf feat, cnt, start, qual; };
  std::vector<ClassCols> cls;
  int sel = 0;
  DBuf qattr;                                // a gated call's triples, [n] of each column
  DBuf sq;                                   // associate_store: the queried src positions [n], history lengths [n]
  DBuf dinc;                                 // associate_store, quality store of classes: history increments [n]
  std::vector<uint64_t> hid;                 // ids in store order
  std::unordered_map<uint64_t, int> hpos;    // id -> store position
  // per-call buffers
  DBuf dreq, dres, plan, qnorm, snorm, dist, gpos, gout, dcol;
  DBuf claim;                                // BestFit voting: [live] u64 column maxima, then [live] i32 claimants
  sb::PinnedBuf<cudaHostAllocDefault> hreq, hres, hcol;   // staging, contents not kept

  ~sb200_fstore() {
    if (st) cudaStreamSynchronize(st);
    for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e);
    if (ev_in) cudaEventDestroy(ev_in);
    if (st) cudaStreamDestroy(st);
  }

  sb::FsStore view() const {
    sb::FsStore s;
    s.feat = feat.p;
    s.cnt = cnt.as<int>();
    s.start = start.as<int>();
    s.ids = ids.as<unsigned long long>();
    s.run = run.as<int>();
    s.K = o.max_observations;
    s.d8 = d8;
    s.live = (int)hid.size();
    s.stype = stype;
    return s;
  }

  // bytes of one stored row (observation)
  size_t row_bytes() const { return (size_t)d8 * type_bytes(stype); }
  size_t track_bytes(const Col& c) const {
    const size_t K = o.max_observations;
    return c.w ? (c.per_obs ? K * c.w : c.w) : K * row_bytes();
  }
  // the store (its gate rule and retention) has column c
  bool has(const Col& c) const {
    return c.need == kNeedAll || (c.need == kNeedGate && gate) || (c.need == kNeedQuality && keep);
  }
  static bool in_part(const Col& c, int part) {
    return part == kPartAll || (part == kPartClass) == c.per_class;
  }

  // fresh columns of this store for max(n, 1) tracks in nw[] (one per kCols entry; only != kNeedAll: the columns of
  // that kind of store alone; part: kPartShared / kPartClass, the shared ones or the selected class's alone),
  // zero-filled where the table says so; the caller copies what it keeps
  int alloc(size_t n, DBuf* nw, int only = kNeedAll, int part = kPartAll) {
    n = std::max<size_t>(n, 1);
    for (int k = 0; k < kNumCols; ++k) {
      const Col& c = kCols[k];
      if (!has(c) || (only != kNeedAll && c.need != only) || !in_part(c, part)) continue;
      const size_t bytes = n * track_bytes(c);
      if (int rc = nw[k].ensure(bytes)) return rc;
      if (c.zero) CU(cudaMemsetAsync(nw[k].p, 0, bytes, st));
    }
    return 0;
  }

  // exchanges the store's columns with nw[] (only, part: as for alloc)
  void swap_columns(DBuf* nw, int only = kNeedAll, int part = kPartAll) {
    for (int k = 0; k < kNumCols; ++k)
      if ((only == kNeedAll || kCols[k].need == only) && in_part(kCols[k], part)) std::swap(this->*kCols[k].buf, nw[k]);
  }

  // ---- feature classes
  // exchanges the per-class members with class k's parked buffers
  void swap_class(int k) {
    ClassCols& c = cls[k];
    std::swap(feat, c.feat);
    std::swap(cnt, c.cnt);
    std::swap(start, c.start);
    std::swap(qual, c.qual);
  }
  // makes class k the one whose columns the members (and view()) are
  void select(int k) {
    if (k == sel) return;
    swap_class(sel);
    swap_class(k);
    sel = k;
    d8 = cls[k].d8;
    o.feature_dim = cls[k].dim;
  }
  // runs f(k) with each class k selected in turn, in `order` (default: declared order), then selects the class
  // selected before; stops at the first nonzero return
  template <class F> int each_class(F f, const std::vector<int>* order = nullptr) {
    const int s0 = sel;
    int rc = 0;
    for (int i = 0; i < (int)cls.size() && !rc; ++i) {
      const int k = order ? (*order)[i] : i;
      select(k);
      rc = f(k);
    }
    select(s0);
    return rc;
  }
  // the class indices in ascending class id: the order in which a merge walks a source's classes
  std::vector<int> ascending_classes() const {
    std::vector<int> ix(cls.size());
    std::iota(ix.begin(), ix.end(), 0);
    std::sort(ix.begin(), ix.end(), [&](int a, int b) { return cls[a].id < cls[b].id; });
    return ix;
  }
  int class_index(uint64_t id) const {
    for (size_t k = 0; k < cls.size(); ++k)
      if (cls[k].id == id) return (int)k;
    return -1;
  }
  // the store holds one class, id 0: the blob is a version 1 to 3 one
  bool plain_classes() const { return cls.size() == 1 && cls[0].id == 0; }

  int set_classes(int n, const uint64_t* idv, const int32_t* dims) {
    if (n < 1 || n > SB200_FSTORE_MAX_CLASSES) return fail(SB200_ERR_INVALID, "n must lie in 1..%d", SB200_FSTORE_MAX_CLASSES);
    if (!idv || !dims) return fail(SB200_ERR_INVALID, "class_ids / feature_dims is NULL");
    for (int i = 0; i < n; ++i) {
      if (dims[i] < 1 || dims[i] > SB200_FSTORE_MAX_DIM)
        return fail(SB200_ERR_INVALID, "class %llu: feature_dim %d outside 1..%d", (unsigned long long)idv[i], dims[i],
                    SB200_FSTORE_MAX_DIM);
      for (int j = 0; j < i; ++j)
        if (idv[j] == idv[i]) return fail(SB200_ERR_INVALID, "class id %llu appears twice", (unsigned long long)idv[i]);
    }
    if (!hid.empty()) return fail(SB200_ERR_INVALID, "the classes are fixed while the store holds tracks (%zu)", hid.size());
    CU(cudaSetDevice(o.device));
    CU(cudaStreamSynchronize(st));
    // no track is stored: every class starts without columns, and the next reserve allocates all columns afresh
    swap_class(sel);
    std::vector<ClassCols> nc(n);
    for (int i = 0; i < n; ++i) {
      nc[i].id = idv[i];
      nc[i].dim = dims[i];
      nc[i].d8 = (dims[i] + 7) / 8 * 8;
    }
    cls.swap(nc);
    sel = 0;
    swap_class(0);
    d8 = cls[0].d8;
    o.feature_dim = cls[0].dim;
    cap = 0;
    return 0;
  }

  int use_class(uint64_t id) {
    const int k = class_index(id);
    if (k < 0) return fail(SB200_ERR_INVALID, "the store declares no class %llu", (unsigned long long)id);
    select(k);
    return 0;
  }

  // every class's cnt and start columns, in declared order, as the class kernels read them
  sb::FsClassCols class_cols() {
    sb::FsClassCols cc{};
    cc.n = (int)cls.size();
    each_class([&](int k) {
      cc.cnt[k] = cnt.as<int>();
      cc.start[k] = start.as<int>();
      return 0;
    });
    return cc;
  }

  // counts[i][k]: the rows of track ids[i] in class k (0 for an id that is not stored); returns the ids found
  int64_t class_counts(int n, const uint64_t* idv, int32_t* counts) {
    if (n < 0) return fail(SB200_ERR_INVALID, "n < 0");
    if (n > 0 && (!idv || !counts)) return fail(SB200_ERR_INVALID, "ids / counts is NULL");
    if (int rc = begin()) return rc;
    if (n == 0) return 0;
    std::vector<int> pos(n, -1);
    int64_t found = 0;
    for (int i = 0; i < n; ++i) {
      auto it = hpos.find(idv[i]);
      if (it != hpos.end()) { pos[i] = it->second; ++found; }
    }
    const size_t out = (size_t)n * cls.size();
    if (int rc = gpos.ensure((size_t)n * 4)) return rc;
    if (int rc = gout.ensure(out * 4)) return rc;
    CU(cudaMemcpyAsync(gpos.p, pos.data(), (size_t)n * 4, cudaMemcpyHostToDevice, st));
    sb::fs_launch_class_counts(class_cols(), gpos.as<int>(), n, gout.as<int>(), st);
    CU(cudaMemcpyAsync(counts, gout.p, out * 4, cudaMemcpyDeviceToHost, st));
    if (int rc = finish()) return rc;
    return found;
  }

  // the tracks every column holds as allocated, at most cap (after a storage type change: in rows of the new type)
  size_t held() {
    size_t n = cap;
    each_class([&](int) {
      for (const Col& c : kCols) if (has(c)) n = std::min(n, (this->*c.buf).bytes / track_bytes(c));
      return 0;
    });
    return n;
  }

  sb::FsAttrCols attr_cols() const {
    return {asrc.as<unsigned long long>(), at0.as<long long>(), at1.as<long long>()};
  }

  // capacity for `need` tracks: grows by at least 1.5x, keeping the live tracks
  int reserve(size_t need) {
    if (need <= cap) return 0;
    const size_t nc = std::max(need, cap + cap / 2);
    if (int rc = each_class([&](int) { return grow(nc, kPartClass); })) return rc;
    if (int rc = grow(nc, kPartShared)) return rc;
    cap = nc;
    return 0;
  }
  // reserve's step for the columns of `part`
  int grow(size_t nc, int part) {
    DBuf nw[kNumCols];
    if (int rc = alloc(nc, nw, kNeedAll, part)) return rc;
    const size_t live = hid.size();
    for (int k = 0; k < kNumCols; ++k)   // the live tracks of the state columns
      if (live && kCols[k].sec >= 0 && has(kCols[k]) && in_part(kCols[k], part))
        CU(cudaMemcpyAsync(nw[k].p, (this->*kCols[k].buf).p, live * track_bytes(kCols[k]), cudaMemcpyDeviceToDevice, st));
    CU(cudaStreamSynchronize(st));   // the old columns are freed with nw
    swap_columns(nw, kNeedAll, part);
    return 0;
  }

  // ---- track attributes (gated store)
  int refuse_gated() const {
    if (gate) return fail(SB200_ERR_INVALID, "the store is gated (rule %d): use the _attr calls, with a source and a window per row", gate);
    return 0;
  }

  // checks of the triples of an _attr call with n rows / queries
  int check_attrs(int n, const sb200_fstore_attrs* a) const {
    if (!gate) return fail(SB200_ERR_INVALID, "the store has no gate (sb200_fstore_set_gate): the _attr calls need one");
    if (n <= 0) return 0;
    if (!a || !a->source || !a->t_start || !a->t_end) return fail(SB200_ERR_INVALID, "attrs or one of its columns is NULL");
    for (int i = 0; i < n; ++i)
      if (a->t_start[i] > a->t_end[i])
        return fail(SB200_ERR_INVALID, "row %d: t_start %lld > t_end %lld", i, (long long)a->t_start[i],
                    (long long)a->t_end[i]);
    return 0;
  }

  // the device triples of a call (n of each column, in qattr) as the gated kernels read them
  sb::FsGate gate_view(int n) const {
    const unsigned long long* q = qattr.as<unsigned long long>();
    return {attr_cols(), q, reinterpret_cast<const long long*>(q + n), reinterpret_cast<const long long*>(q + 2 * (size_t)n),
            gate};
  }
  // n triples in b, as the column of each field
  static sb::FsAttrCols triples(const DBuf& b, int n) {
    unsigned long long* q = b.as<unsigned long long>();
    return {q, reinterpret_cast<long long*>(q + n), reinterpret_cast<long long*>(q + 2 * (size_t)n)};
  }

  // uploads n triples into qattr
  int upload_triples(int n, const uint64_t* src, const int64_t* t0, const int64_t* t1) {
    if (int rc = qattr.ensure(std::max(n, 1) * 24)) return rc;
    if (n == 0) return 0;
    char* d = qattr.as<char>();
    CU(cudaMemcpyAsync(d, src, (size_t)n * 8, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(d + (size_t)n * 8, t0, (size_t)n * 8, cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(d + (size_t)n * 16, t1, (size_t)n * 8, cudaMemcpyHostToDevice, st));
    return 0;
  }

  // the stored triples at pos[] (-1: zeros), read back; changes nothing
  int peek_attrs(const std::vector<int>& pos, Triples* out) {
    const int n = (int)pos.size();
    *out = Triples(pos.size());
    if (n == 0) return 0;
    if (int rc = gpos.ensure((size_t)n * 4)) return rc;
    if (int rc = gout.ensure((size_t)n * 24)) return rc;
    CU(cudaMemcpyAsync(gpos.p, pos.data(), (size_t)n * 4, cudaMemcpyHostToDevice, st));
    const unsigned long long* g = gout.as<unsigned long long>();
    sb::fs_launch_attr_gather(attr_cols(), gpos.as<int>(), n, triples(gout, n), st);
    CU(cudaMemcpyAsync(out->src.data(), g, (size_t)n * 8, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(out->t0.data(), g + n, (size_t)n * 8, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(out->t1.data(), g + 2 * (size_t)n, (size_t)n * 8, cudaMemcpyDeviceToHost, st));
    if (int rc = finish()) return rc;
    return 0;
  }

  // writes the triples `v` to the stored positions pos[]
  int write_attrs(const std::vector<int>& pos, const Triples& v) {
    const int n = (int)pos.size();
    if (n == 0) return 0;
    if (int rc = gpos.ensure((size_t)n * 4)) return rc;
    if (int rc = upload_triples(n, v.src.data(), v.t0.data(), v.t1.data())) return rc;
    CU(cudaMemcpyAsync(gpos.p, pos.data(), (size_t)n * 4, cudaMemcpyHostToDevice, st));
    sb::fs_launch_attr_scatter(attr_cols(), gpos.as<int>(), n, triples(qattr, n), st);
    if (int rc = finish()) return rc;
    return 0;
  }

  int set_gate(int rule) {
    if (rule != SB200_FSTORE_GATE_NONE && rule != SB200_FSTORE_GATE_SAME_SOURCE && rule != SB200_FSTORE_GATE_ANY_SOURCE)
      return fail(SB200_ERR_INVALID, "unknown gate rule %d", rule);
    if (!hid.empty()) return fail(SB200_ERR_INVALID, "the gate is fixed while the store holds tracks (%zu)", hid.size());
    CU(cudaSetDevice(o.device));
    gate = rule;
    DBuf nw[kNumCols];   // no track is stored: the columns start empty, sized to the capacity
    if (cap)
      if (int rc = alloc(cap, nw, kNeedGate)) return rc;
    CU(cudaStreamSynchronize(st));
    swap_columns(nw, kNeedGate);
    return 0;
  }

  // ---- retention by quality
  int set_retention(int rule, int init, float ex) {
    if (rule != SB200_FSTORE_KEEP_NEWEST && rule != SB200_FSTORE_KEEP_BEST_QUALITY)
      return fail(SB200_ERR_INVALID, "unknown retention rule %d", rule);
    if (!hid.empty()) return fail(SB200_ERR_INVALID, "the retention is fixed while the store holds tracks (%zu)", hid.size());
    std::vector<int> tab;
    if (rule == SB200_FSTORE_KEEP_BEST_QUALITY)
      if (int rc = capacity_table(o.max_observations, init, ex, &tab)) return rc;
    CU(cudaSetDevice(o.device));
    if (!tab.empty()) {
      if (int rc = dcap.ensure(tab.size() * 4)) return rc;
      CU(cudaMemcpy(dcap.p, tab.data(), tab.size() * 4, cudaMemcpyHostToDevice));
    }
    keep = rule;
    if (rule == SB200_FSTORE_KEEP_BEST_QUALITY) { init_cap = init; ext = ex; }
    cap_tab.swap(tab);
    // as set_gate: the quality columns start empty, sized to the capacity
    auto fresh = [&](int part) {
      DBuf nw[kNumCols];
      if (cap)
        if (int rc = alloc(cap, nw, kNeedQuality, part)) return rc;
      CU(cudaStreamSynchronize(st));
      swap_columns(nw, kNeedQuality, part);
      return 0;
    };
    if (int rc = each_class([&](int) { return fresh(kPartClass); })) return rc;
    return fresh(kPartShared);
  }

  int refuse_quality() const {
    if (keep) return fail(SB200_ERR_INVALID, "the store keeps its best observations by quality: use the _quality calls");
    return 0;
  }

  // checks of a _quality call with n rows: a quality store, a quality per row and none NaN, attrs as the gate needs them
  int check_quality(int n, const float* q, const sb200_fstore_attrs* attrs) const {
    if (!keep) return fail(SB200_ERR_INVALID, "the store keeps its newest observations: the _quality calls need "
                                              "sb200_fstore_set_retention(SB200_FSTORE_KEEP_BEST_QUALITY)");
    if (!gate && attrs) return fail(SB200_ERR_INVALID, "attrs must be NULL on an ungated store");
    if (n > 0 && !q) return fail(SB200_ERR_INVALID, "quality is NULL");
    const int bad = n > 0 ? first_nan(n, q) : -1;
    if (bad >= 0) return fail(SB200_ERR_INVALID, "row %d: the quality is NaN", bad);
    return 0;
  }

  int capacity(size_t h) const { return cap_tab[std::min(h, cap_tab.size() - 1)]; }

  // A track's list while a call is planned: ref[j] is its observation j, a pre-call stored row (position * K + slot,
  // >= 0) or request row r (-(r + 1)), q[j] its quality; h its merge history; dirty once the call changes it.
  struct QTrack {
    int pos;
    std::vector<int> ref;
    std::vector<float> q;
    std::vector<uint64_t> h;
    bool dirty;
  };

  // optimize (examples/track_merging.rs:279-297): the stable sort by quality, descending, then the truncation to c(h)
  void keep_best(QTrack& t) const {
    std::vector<int> ix(t.ref.size());
    std::iota(ix.begin(), ix.end(), 0);
    std::stable_sort(ix.begin(), ix.end(), [&](int a, int b) { return t.q[a] > t.q[b]; });
    ix.resize(std::min(ix.size(), (size_t)capacity(t.h.size())));
    std::vector<int> ref;
    std::vector<float> q;
    for (int i : ix) { ref.push_back(t.ref[i]); q.push_back(t.q[i]); }
    t.ref.swap(ref);
    t.q.swap(q);
  }
  // Track::merge with merge_history = true (src/track.rs:522-588): dest ++ src, then optimize at dest's new capacity
  void merge_into(QTrack& d, const QTrack& src) const {
    d.ref.insert(d.ref.end(), src.ref.begin(), src.ref.end());
    d.q.insert(d.q.end(), src.q.begin(), src.q.end());
    d.h.insert(d.h.end(), src.h.begin(), src.h.end());
    keep_best(d);
    d.dirty = true;
  }

  // the lists of the stored tracks at pos[] as they are: their rows, qualities and histories.  Changes nothing.
  int peek_tracks(const std::vector<int>& pos, std::vector<QTrack>* out) {
    const size_t n = pos.size();
    const int K = o.max_observations;
    out->clear();
    if (n == 0) return 0;
    if (int rc = gpos.ensure(n * 4)) return rc;
    if (int rc = gout.ensure(n * (2 + (size_t)K) * 4)) return rc;
    CU(cudaMemcpyAsync(gpos.p, pos.data(), n * 4, cudaMemcpyHostToDevice, st));
    sb::fs_launch_qpeek(view(), qual.as<float>(), gpos.as<int>(), (int)n, gout.as<int>(), gout.as<float>() + 2 * n, st);
    std::vector<int> ring(2 * n);
    std::vector<float> qv(n * K);
    CU(cudaMemcpyAsync(ring.data(), gout.p, n * 8, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(qv.data(), gout.as<float>() + 2 * n, n * K * 4, cudaMemcpyDeviceToHost, st));
    if (int rc = finish()) return rc;
    for (size_t i = 0; i < n; ++i) {
      QTrack t{pos[i], {}, {}, hist[pos[i]], false};
      for (int j = 0; j < ring[2 * i]; ++j) {
        t.ref.push_back(pos[i] * K + (ring[2 * i + 1] + j) % K);
        t.q.push_back(qv[i * K + j]);
      }
      out->push_back(std::move(t));
    }
    return 0;
  }

  // merge_owned: writes the planned lists of the dirty tracks of t[] (every ref a stored row): observation j of a track
  // at position p goes to slot j, by the two-launch move (every row read from its pre-call slot before any is written),
  // then each track's K qualities (0 past its count) and its history length
  int apply_tracks(const std::vector<QTrack>& t) {
    const int K = o.max_observations;
    std::vector<int> mv_src, mv_dst, hdr, qpos, hl;
    std::vector<float> qv;
    for (const QTrack& tr : t) {
      if (!tr.dirty) continue;
      const int c1 = (int)tr.ref.size();
      hdr.insert(hdr.end(), {tr.pos, c1, 0});
      for (int j = 0; j < c1; ++j) {
        const int dst = tr.pos * K + j;
        if (tr.ref[j] != dst) { mv_src.push_back(tr.ref[j]); mv_dst.push_back(dst); }
      }
      qpos.push_back(tr.pos);
      hl.push_back((int)tr.h.size());
      for (int j = 0; j < K; ++j) qv.push_back(j < c1 ? tr.q[j] : 0.0f);
    }
    const int nm = (int)mv_src.size(), nh = (int)hdr.size() / 3, nq = (int)qpos.size();
    std::vector<int> tab;
    tab.reserve(2 * (size_t)nm + hdr.size() + qpos.size() + hl.size() + qv.size());
    for (const std::vector<int>* v : {&mv_src, &mv_dst, &hdr, &qpos, &hl}) tab.insert(tab.end(), v->begin(), v->end());
    const size_t qoff = tab.size();
    tab.resize(qoff + qv.size());
    if (!qv.empty()) memcpy(tab.data() + qoff, qv.data(), qv.size() * 4);
    if (int rc = gpos.ensure(std::max<size_t>(tab.size(), 1) * 4)) return rc;
    if (int rc = gout.ensure(std::max<size_t>((size_t)nm * row_bytes(), 16))) return rc;
    CU(cudaMemcpyAsync(gpos.p, tab.data(), tab.size() * 4, cudaMemcpyHostToDevice, st));
    const int* dtab = gpos.as<int>();
    const int* dq = dtab + 2 * nm + 3 * nh;
    CU(cudaEventRecord(ev[2], st));
    sb::fs_launch_move_rows(view(), dtab, dtab + nm, nm, dtab + 2 * nm, nh, gout.p, st);
    sb::fs_launch_qual_set(qual.as<float>(), hlen.as<int>(), dq, reinterpret_cast<const float*>(dtab + qoff), dq + nq, nq,
                           K, st);
    CU(cudaEventRecord(ev[3], st));
    return finish(2, 3);
  }

  // The device view of a quality store's associate (assoc) or add, with rq[R] the request rows' qualities uploaded
  int qcall(const std::vector<float>& rq, bool assoc, sb::FsQCall* qc) {
    if (int rc = dqr.ensure(std::max<size_t>(rq.size(), 1) * 4)) return rc;
    if (!rq.empty()) CU(cudaMemcpyAsync(dqr.p, rq.data(), rq.size() * 4, cudaMemcpyHostToDevice, st));
    *qc = {qual.as<float>(), hlen.as<int>(), dcap.as<int>(), (int)cap_tab.size(), dqr.as<float>(), assoc ? 1 : 0};
    return 0;
  }

  // The best c(1) rows of each query in quality order, ties to the earlier row (a query is a fresh track, h = 1):
  // row_src / qoff as fs_row_table makes them
  void quality_row_table(int Q, const int32_t* offs, const float* q, std::vector<int>* row_src,
                         std::vector<int>* qoff) const {
    row_src->clear();
    qoff->assign(1, 0);
    for (int i = 0; i < Q; ++i) {
      std::vector<int> ix(offs[i + 1] - offs[i]);
      std::iota(ix.begin(), ix.end(), offs[i]);
      std::stable_sort(ix.begin(), ix.end(), [&](int a, int b) { return q[a] > q[b]; });
      ix.resize(std::min(ix.size(), (size_t)capacity(1)));
      row_src->insert(row_src->end(), ix.begin(), ix.end());
      qoff->push_back((int)row_src->size());
    }
  }

  int begin() {
    CU(cudaSetDevice(o.device));
    stage_ms[0] = stage_ms[1] = stage_ms[2] = 0.0f;
    return 0;
  }

  size_t elem() const { return ftype == SB200_FEATURE_F32 ? 4 : 2; }

  // a device column must be device memory on the store's device
  int check_column(const Column& col) const {
    if (!col.on_device || !col.p) return 0;
    if (sb::blob_device(col.p) != o.device)
      return fail(SB200_ERR_INVALID, "d_features is not device memory on device %d", o.device);
    return 0;
  }

  // Puts the request on the device: rows [R][d8] (zero-padded), ids, offsets, row -> item, dest (nullptr: -1 for every
  // item) and the initial max_dist.
  // row_src[r] is the row of the caller's column behind request row r; col_rows the rows of a host column to upload.
  // With `rsrc` there is no column: rsrc writes the rows on the device (row_src gives only their number).
  int upload(const ReqLayout& L, int Q, const uint64_t* qids, const std::vector<int>& qoff, const std::vector<int>& row_src,
             const int* dest, const Column& col, size_t col_rows, const sb::FsRowSource* rsrc = nullptr) {
    const bool host_f32 = !rsrc && !col.on_device && ftype == SB200_FEATURE_F32;
    const bool staged = !rsrc && !host_f32;     // rows built by fs_stage_kernel from the column
    const size_t base = host_f32 ? 0 : L.qid;   // the rows of the other paths are written on the device
    const int D = o.feature_dim, R = (int)row_src.size();
    if (int rc = hreq.ensure(L.total - base)) return rc;
    if (int rc = dreq.ensure(L.total)) return rc;
    auto at = [&](size_t off) { return static_cast<char*>(hreq.p) + (off - base); };   // off: an offset of L >= base
    if (host_f32) {
      const float* feats = static_cast<const float*>(col.p);
      float* rows = reinterpret_cast<float*>(at(L.rows));
      for (int r = 0; r < R; ++r) {
        memcpy(rows + (size_t)r * d8, feats + (size_t)row_src[r] * D, (size_t)D * 4);
        for (int k = D; k < d8; ++k) rows[(size_t)r * d8 + k] = 0.0f;
      }
    } else if (staged) {
      memcpy(at(L.row_src), row_src.data(), (size_t)R * 4);
    }
    stage_request(L, at(L.qid), Q, qids, qoff.data(), dest, 1);
    const void* dev_col = col.p;
    if (staged && !col.on_device) {   // the raw 2-byte rows: half the bytes of the widened request
      const size_t bytes = col_rows * D * elem();
      if (int rc = hcol.ensure(bytes)) return rc;
      if (int rc = dcol.ensure(bytes)) return rc;
      memcpy(hcol.p, col.p, bytes);
      CU(cudaMemcpyAsync(dcol.p, hcol.p, bytes, cudaMemcpyHostToDevice, st));
      dev_col = dcol.p;
    }
    if (staged && col.on_device) {   // the column is complete once the caller's stream has reached this point
      CU(cudaEventRecord(ev_in, col.caller));
      CU(cudaStreamWaitEvent(st, ev_in, 0));
    }
    CU(cudaMemcpyAsync(dreq.as<char>() + base, hreq.p, L.total - base, cudaMemcpyHostToDevice, st));
    char* d = dreq.as<char>();
    if (staged)
      sb::fs_launch_stage(ftype, dev_col, reinterpret_cast<const int*>(d + L.row_src), R, D, d8,
                          reinterpret_cast<float*>(d + L.rows), st);
    if (rsrc)
      return rsrc->fill(rsrc->ctx, reinterpret_cast<float*>(d + L.rows), reinterpret_cast<const int*>(d + L.qoff),
                        reinterpret_cast<const int*>(d + L.row_q), R, st);
    return 0;
  }

  sb::FsCall call_view(const ReqLayout& L, int Q, int R, const ResLayout* RL) {
    char* d = dreq.as<char>();
    sb::FsCall c{};
    c.rows = reinterpret_cast<const float*>(d + L.rows);
    c.qid = reinterpret_cast<const unsigned long long*>(d + L.qid);
    c.qoff = reinterpret_cast<const int*>(d + L.qoff);
    c.row_q = reinterpret_cast<const int*>(d + L.row_q);
    c.dest = reinterpret_cast<int*>(d + L.dest);
    c.maxkey = reinterpret_cast<int*>(d + L.maxkey);
    c.plan = plan.as<int4>();
    c.qnorm = qnorm.as<float>();
    c.snorm = snorm.as<float>();
    c.dist = dist.as<float>();
    if (RL) {
      char* r = dres.as<char>();
      c.out_w = reinterpret_cast<double*>(r + RL->w);
      c.out_cnt = reinterpret_cast<int*>(r + RL->cnt);
      c.out_pos = reinterpret_cast<int*>(r + RL->pos);
    }
    c.Q = Q;
    c.R = R;
    return c;
  }

  // checks of a search / associate request; fills the newest-K row table
  // (quality: a quality store's qualities, one per row of the column, checked here; the row table is then its own)
  int check_queries(int Q, const uint64_t* qids, const int32_t* offs, const Column& col, bool assoc,
                    std::vector<int>* qoff, std::vector<int>* row_src, const float* quality = nullptr) {
    if (Q < 0) return fail(SB200_ERR_INVALID, "n_queries < 0");
    if (Q == 0) return 0;
    if (!qids || !offs) return fail(SB200_ERR_INVALID, "query_ids / obs_offsets is NULL");
    if (offs[0] != 0) return fail(SB200_ERR_INVALID, "obs_offsets[0] != 0");
    if (int rc = check_ids(Q, qids, "query id", assoc, offs)) return rc;
    if (!col.p) return fail(SB200_ERR_INVALID, "features is NULL");
    if (int rc = check_column(col)) return rc;
    if (keep) {
      if (!quality) return fail(SB200_ERR_INVALID, "quality is NULL");
      const int bad = first_nan(offs[Q], quality);
      if (bad >= 0) return fail(SB200_ERR_INVALID, "row %d: the quality is NaN", bad);
    }
    return plan_rows(Q, offs, qoff, row_src, quality);
  }

  // the newest-K row table of a request (with quality: quality_row_table), within the pair bound of one distance matrix
  int plan_rows(int Q, const int32_t* offs, std::vector<int>* qoff, std::vector<int>* row_src,
                const float* quality = nullptr) const {
    const int K = o.max_observations;
    if (quality) quality_row_table(Q, offs, quality, row_src, qoff);
    else sb::fs_row_table(Q, offs, K, row_src, qoff);
    const long long pairs = (long long)row_src->size() * (long long)hid.size() * K;
    if (pairs > sb::kFsMaxPairs)
      return fail(SB200_ERR_CAPACITY, "the call needs %lld observation pairs; one call holds at most 2^30", pairs);
    return 0;
  }

  // Refuses the first of a call's n ids that appears twice in it (`what`: "query id" or "id") or, with `fresh`, that is
  // already stored; with offs, the query of each id is first refused when it has no observations.
  int check_ids(int n, const uint64_t* ids, const char* what, bool fresh, const int32_t* offs = nullptr) const {
    std::unordered_set<uint64_t> seen;
    seen.reserve((size_t)n * 2);
    for (int q = 0; q < n; ++q) {
      if (offs && offs[q + 1] - offs[q] <= 0) return fail(SB200_ERR_INVALID, "query %d has no observations", q);
      if (!seen.insert(ids[q]).second)
        return fail(SB200_ERR_INVALID, "%s %llu appears twice in the call", what, (unsigned long long)ids[q]);
      if (fresh && hpos.count(ids[q]))
        return fail(SB200_ERR_INVALID, "%s %llu is already stored", what, (unsigned long long)ids[q]);
    }
    return 0;
  }

  // the per-call buffers of Q queries with R rows against S stored rows: results, plan, norms and distances
  int size_call(const ResLayout& RL, int Q, int R, long long S) {
    if (int rc = hres.ensure(RL.total)) return rc;
    if (int rc = dres.ensure(RL.total)) return rc;
    if (int rc = plan.ensure((size_t)Q * 16)) return rc;
    if (o.metric == SB200_VIS_COSINE) {
      if (int rc = qnorm.ensure((size_t)R * 4)) return rc;
      if (int rc = snorm.ensure((size_t)std::max<long long>(S, 1) * 4)) return rc;
    }
    return dist.ensure((size_t)std::max<long long>((long long)R * S, 1) * 4);
  }

  // waits for the stream and reports a failed kernel; then adds the times of stages [first, last) to stage_ms (stage i
  // runs from ev[i] to ev[i + 1])
  int finish(int first = 0, int last = 0) {
    CU(cudaStreamSynchronize(st));
    CU(cudaGetLastError());
    for (int i = first; i < last; ++i) {
      float ms = 0.0f;
      CU(cudaEventElapsedTime(&ms, ev[i], ev[i + 1]));
      stage_ms[i] += ms;
    }
    return 0;
  }

  // BestFit voting (sb200_fstore_set_voting), after TopN on the call c: the claims across its queries, rewriting the
  // results and, with want_dest, the destinations; nothing under TopN
  int claim_best_fit(const sb::FsStore& s, const sb::FsCall& c, bool want_dest) {
    if (voting != SB200_FSTORE_VOTING_BEST_FIT) return 0;
    if (int rc = claim.ensure((size_t)std::max(s.live, 1) * 12)) return rc;
    unsigned long long* wmax = claim.as<unsigned long long>();
    CU(sb::fs_launch_claim(o.max_distance, o.min_votes, o.topn, want_dest, s, c, wmax,
                           reinterpret_cast<int*>(wmax + s.live), st));
    return 0;
  }

  // the TopN results of Q queries (hres, layout RL) as counts[Q], winners[Q][topn] and weights[Q][topn], zero past a count;
  // an element BestFit rewrote (position -2) names the query's own id, qids[q]
  void read_results(const ResLayout& RL, int Q, const uint64_t* qids, int32_t* counts, uint64_t* winners,
                    double* weights) const {
    const char* h = static_cast<const char*>(hres.p);
    const double* w = reinterpret_cast<const double*>(h + RL.w);
    const int* cn = reinterpret_cast<const int*>(h + RL.cnt);
    const int* ps = reinterpret_cast<const int*>(h + RL.pos);
    for (int q = 0; q < Q; ++q) {
      counts[q] = cn[q];
      for (int e = 0; e < o.topn; ++e) {
        const size_t i = (size_t)q * o.topn + e;
        winners[i] = e < cn[q] ? (ps[i] == -2 ? qids[q] : hid[ps[i]]) : 0;
        weights[i] = e < cn[q] ? w[i] : 0.0;
      }
    }
  }

  // search (assoc == false) or associate
  // attrs: the queries' triples of a gated store's call (checked by the caller), else nullptr
  // quality: a quality store's qualities, one per row of the column
  int run_queries(int Q, const uint64_t* qids, const int32_t* offs, const Column& col, int32_t* counts,
                  uint64_t* winners, double* weights, uint64_t* track_ids, uint8_t* merged, bool assoc,
                  const sb200_fstore_attrs* attrs = nullptr, const float* quality = nullptr) {
    std::vector<int> qoff, src;
    if (int rc = check_queries(Q, qids, offs, col, assoc, &qoff, &src, quality)) return rc;
    if (Q > 0 && (!counts || !winners || !weights || (assoc && (!track_ids || !merged))))
      return fail(SB200_ERR_INVALID, "an output is NULL");
    if (int rc = begin()) return rc;
    if (Q == 0) return 0;
    return launch_queries(Q, qids, qoff, src, col, (size_t)offs[Q], nullptr, counts, winners, weights, track_ids, merged,
                          assoc, attrs, quality);
  }

  // associate whose request rows `rsrc` writes on the device (sb200_fstore_associate_wasted, and associate_store with
  // its queries `tq`); offs as for associate
  int associate_rows(int Q, const uint64_t* qids, const int32_t* offs, const sb::FsRowSource& rsrc, int32_t* counts,
                     uint64_t* winners, double* weights, uint64_t* track_ids, uint8_t* merged,
                     const TrackQueries* tq = nullptr, std::vector<int>* decided = nullptr) {
    if (int rc = check_ids(Q, qids, "query id", true)) return rc;
    std::vector<int> qoff, src;
    if (int rc = plan_rows(Q, offs, &qoff, &src)) return rc;
    if (int rc = begin()) return rc;
    if (Q == 0) return 0;
    return launch_queries(Q, qids, qoff, src, Column{nullptr, false, nullptr}, 0, &rsrc, counts, winners, weights,
                          track_ids, merged, true, nullptr, nullptr, tq, decided);
  }

  // search whose request rows `rsrc` writes on the device (sb200_fstore_search_tracks); quality / attrs as run_queries
  // takes them, the triples checked by the caller; *row_table receives the row table before rsrc runs
  int search_rows(int Q, const uint64_t* qids, const int32_t* offs, const float* quality, const sb200_fstore_attrs* attrs,
                  const sb::FsRowSource& rsrc, std::vector<int>* row_table, int32_t* counts, uint64_t* winners,
                  double* weights) {
    if (int rc = check_ids(Q, qids, "query id", false, offs)) return rc;
    const int bad = keep && Q > 0 ? first_nan(offs[Q], quality) : -1;
    if (bad >= 0) return fail(SB200_ERR_INVALID, "row %d: the quality is NaN", bad);
    std::vector<int> qoff;
    if (int rc = plan_rows(Q, offs, &qoff, row_table, keep ? quality : nullptr)) return rc;
    if (int rc = begin()) return rc;
    if (Q == 0) return 0;
    return launch_queries(Q, qids, qoff, *row_table, Column{nullptr, false, nullptr}, 0, &rsrc, counts, winners, weights,
                          nullptr, nullptr, false, attrs, quality);
  }

  // the device part of search / associate, after every check: upload, distances, TopN, apply, results
  int launch_queries(int Q, const uint64_t* qids, const std::vector<int>& qoff, const std::vector<int>& src,
                     const Column& col, size_t col_rows, const sb::FsRowSource* rsrc, int32_t* counts,
                     uint64_t* winners, double* weights, uint64_t* track_ids, uint8_t* merged, bool assoc,
                     const sb200_fstore_attrs* attrs = nullptr, const float* quality = nullptr,
                     const TrackQueries* tq = nullptr, std::vector<int>* decided = nullptr) {
    const int R = (int)src.size(), topn = o.topn, K = o.max_observations;
    const bool qa = assoc && keep;   // a quality store's merges are planned and applied by fs_launch_qmerge
    const bool gated = attrs || (tq && gate);   // the queries' triples are in qattr
    const long long live = (long long)hid.size(), S = live * K;
    const ReqLayout L(Q, R, d8, !rsrc && (col.on_device || ftype != SB200_FEATURE_F32));
    const ResLayout RL(Q, topn);
    if (int rc = size_call(RL, Q, R, S)) return rc;
    if (assoc)
      if (int rc = reserve(hid.size() + (size_t)Q)) return rc;
    if (int rc = upload(L, Q, qids, qoff, src, nullptr, col, col_rows, rsrc)) return rc;
    if (attrs)
      if (int rc = upload_triples(Q, attrs->source, attrs->t_start, attrs->t_end)) return rc;
    sb::FsQCall qc{};
    if (qa && tq) {   // the row source wrote the rows' qualities
      qc = {qual.as<float>(), hlen.as<int>(), dcap.as<int>(), (int)cap_tab.size(), dqr.as<float>(), 1};
    } else if (qa) {
      std::vector<float> rq(R);
      for (int r = 0; r < R; ++r) rq[r] = quality[src[r]];
      if (int rc = qcall(rq, true, &qc)) return rc;
    }
    const sb::FsGate g = gate_view(Q);
    const sb::FsStore s = view();
    const sb::FsCall c = call_view(L, Q, R, &RL);
    CU(cudaEventRecord(ev[0], st));
    sb::fs_launch_dist(o.metric, o.distance_filter, s, c, st, sb::kFsForeign, nullptr, gated ? &g : nullptr);
    CU(cudaEventRecord(ev[1], st));
    sb::fs_launch_topn(o.max_distance, o.min_votes, topn, assoc, s, c, st);
    if (int rc = claim_best_fit(s, c, assoc)) return rc;
    CU(cudaEventRecord(ev[2], st));
    // BestFit destinations are exclusive and every scored pair is compatible, so the gate keeps each of them
    if (assoc && gated) sb::fs_launch_gate_resolve(c, g, st);
    if (decided) {   // associate_store of several classes on a quality store: the caller applies every class
      decided->resize(Q);
      CU(cudaMemcpyAsync(hres.p, dres.p, RL.total, cudaMemcpyDeviceToHost, st));
      CU(cudaMemcpyAsync(decided->data(), c.dest, (size_t)Q * 4, cudaMemcpyDeviceToHost, st));
      if (int rc = finish(S > 0 ? 0 : 1, 2)) return rc;
      read_results(RL, Q, qids, counts, winners, weights);
      return 0;
    }
    if (qa) sb::fs_launch_qmerge(s, c, qc, st, tq ? tq->hq : nullptr);
    else if (assoc) sb::fs_launch_apply(s, c, st);
    if (assoc && gated) sb::fs_launch_attr_new(s.live, c, g, st);
    CU(cudaEventRecord(ev[3], st));
    CU(cudaMemcpyAsync(hres.p, dres.p, RL.total, cudaMemcpyDeviceToHost, st));
    // gated, quality or BestFit associate: the position each query ended up at (>= live: a new track)
    const bool best = voting == SB200_FSTORE_VOTING_BEST_FIT;
    std::vector<int> where;
    if (assoc && (gated || qa || best)) {
      where.resize(Q);
      CU(cudaMemcpyAsync(where.data(), c.dest, (size_t)Q * 4, cudaMemcpyDeviceToHost, st));
    }
    if (int rc = finish(S > 0 ? 0 : 1, assoc ? 3 : 2)) return rc;   // no distance stage on an empty store
    read_results(RL, Q, qids, counts, winners, weights);
    if (assoc) {
      // Track::merge with merge_history = true appends the query's history: [id], or a stored track's whole one
      auto qhist = [&](int q) { return tq ? (*tq->hist)[q] : std::vector<uint64_t>{qids[q]}; };
      for (int q = 0; q < Q; ++q) {
        // a first winner the gate refused, or another query claimed under BestFit, leaves a new track
        merged[q] = gated || qa || best ? where[q] < live : counts[q] > 0;
        track_ids[q] = merged[q] ? winners[(size_t)q * topn] : qids[q];
        if (qa && merged[q]) {
          const std::vector<uint64_t> h = qhist(q);
          hist[where[q]].insert(hist[where[q]].end(), h.begin(), h.end());
        }
      }
      for (int q = 0; q < Q; ++q)
        if (!merged[q]) {
          hpos[qids[q]] = (int)hid.size();
          hid.push_back(qids[q]);
          if (qa) hist.push_back(qhist(q));
        }
    }
    return 0;
  }

  // attrs: the rows' triples of a gated store's call (checked by the caller), else nullptr; quality: a quality store's
  // qualities, one per row (checked by the caller)
  int add(int n, const uint64_t* idv, const Column& col, const sb200_fstore_attrs* attrs = nullptr,
          const float* quality = nullptr) {
    if (n < 0) return fail(SB200_ERR_INVALID, "n < 0");
    if (n > 0 && (!idv || !col.p)) return fail(SB200_ERR_INVALID, "ids / features is NULL");
    if (int rc = check_column(col)) return rc;
    if (int rc = begin()) return rc;
    if (n == 0) return 0;
    // destination of every observation: a stored track, or a new one placed at the first appearance of its id
    std::vector<int> dest(n);
    std::vector<uint64_t> fresh;
    std::unordered_map<uint64_t, int> fresh_pos;
    const int live = (int)hid.size();
    for (int i = 0; i < n; ++i) {
      auto it = hpos.find(idv[i]);
      if (it != hpos.end()) { dest[i] = it->second; continue; }
      auto jt = fresh_pos.find(idv[i]);
      if (jt == fresh_pos.end()) {
        jt = fresh_pos.emplace(idv[i], live + (int)fresh.size()).first;
        fresh.push_back(idv[i]);
      }
      dest[i] = jt->second;
    }
    // gated: the final triple of every touched track, planned from the stored ones before anything changes
    std::vector<int> tpos;
    Triples fin;
    if (attrs)
      if (int rc = plan_add_attrs(n, idv, dest, live, *attrs, &tpos, &fin)) return rc;
    std::vector<int> qoff(n + 1), src(n);
    for (int i = 0; i <= n; ++i) qoff[i] = i;
    for (int i = 0; i < n; ++i) src[i] = i;
    const ReqLayout L(n, n, d8, col.on_device || ftype != SB200_FEATURE_F32);
    if (int rc = plan.ensure((size_t)n * 16)) return rc;
    if (int rc = reserve(hid.size() + fresh.size())) return rc;
    if (int rc = upload(L, n, idv, qoff, src, dest.data(), col, (size_t)n)) return rc;
    sb::FsQCall qc{};
    if (keep)   // each row appended to its track in order, and the track optimized at its capacity
      if (int rc = qcall(std::vector<float>(quality, quality + n), false, &qc)) return rc;
    const sb::FsStore s = view();
    const sb::FsCall c = call_view(L, n, n, nullptr);
    CU(cudaEventRecord(ev[2], st));
    if (keep) sb::fs_launch_qmerge(s, c, qc, st);
    else sb::fs_launch_apply(s, c, st);
    CU(cudaEventRecord(ev[3], st));
    if (int rc = finish(2, 3)) return rc;
    for (uint64_t id : fresh) {
      hpos[id] = (int)hid.size();
      hid.push_back(id);
      if (keep) hist.push_back({id});
    }
    return write_attrs(tpos, fin);
  }

  // add's attributes: a new track takes its first row's triple, a track takes the hull of its rows' windows, and a row
  // whose source differs from its track's is refused.  tpos = the touched positions, fin their final triples.
  int plan_add_attrs(int n, const uint64_t* idv, const std::vector<int>& dest, int live, const sb200_fstore_attrs& a,
                     std::vector<int>* tpos, Triples* fin) {
    std::unordered_map<int, int> at;   // position -> index into tpos
    std::vector<int> known;
    for (int i = 0; i < n; ++i)
      if (at.emplace(dest[i], (int)tpos->size()).second) {
        tpos->push_back(dest[i]);
        if (dest[i] < live) known.push_back(dest[i]);
      }
    Triples old;
    if (int rc = peek_attrs(known, &old)) return rc;
    *fin = Triples(tpos->size());
    std::vector<char> set(tpos->size(), 0);
    for (size_t k = 0; k < known.size(); ++k) {
      const int j = at[known[k]];
      fin->src[j] = old.src[k]; fin->t0[j] = old.t0[k]; fin->t1[j] = old.t1[k];
      set[j] = 1;
    }
    for (int i = 0; i < n; ++i) {
      const int j = at[dest[i]];
      if (!set[j]) {
        fin->src[j] = a.source[i]; fin->t0[j] = a.t_start[i]; fin->t1[j] = a.t_end[i];
        set[j] = 1;
        continue;
      }
      if (fin->src[j] != a.source[i])
        return fail(SB200_ERR_INVALID, "row %d: source %llu differs from track %llu's source %llu", i,
                    (unsigned long long)a.source[i], (unsigned long long)idv[i], (unsigned long long)fin->src[j]);
      fin->t0[j] = std::min<int64_t>(fin->t0[j], a.t_start[i]);
      fin->t1[j] = std::max<int64_t>(fin->t1[j], a.t_end[i]);
    }
    return 0;
  }

  int64_t fetch_attr(int n, const uint64_t* idv, uint64_t* src, int64_t* t0, int64_t* t1) {
    if (!gate) return fail(SB200_ERR_INVALID, "the store has no gate (sb200_fstore_set_gate): it keeps no attributes");
    if (n < 0) return fail(SB200_ERR_INVALID, "n < 0");
    if (n > 0 && (!idv || !src || !t0 || !t1)) return fail(SB200_ERR_INVALID, "ids or an output is NULL");
    if (int rc = begin()) return rc;
    std::vector<int> pos(n, -1);
    int64_t found = 0;
    for (int i = 0; i < n; ++i) {
      auto it = hpos.find(idv[i]);
      if (it != hpos.end()) { pos[i] = it->second; ++found; }
    }
    Triples v;
    if (int rc = peek_attrs(pos, &v)) return rc;
    std::copy(v.src.begin(), v.src.end(), src);
    std::copy(v.t0.begin(), v.t0.end(), t0);
    std::copy(v.t1.begin(), v.t1.end(), t1);
    return found;
  }

  // ---- store to store (examples/track_merging.rs:371-481)
  // TrackStore::find_usable with `baked` (now > t_end + period): the baked ids in store order, the first min(cap, total)
  // into ids; returns the total.  Only the count and the selected positions come back.
  int64_t find_baked(int64_t now, int64_t period, int64_t cap_ids, uint64_t* idv) {
    if (!gate) return fail(SB200_ERR_INVALID, "the store has no gate (sb200_fstore_set_gate): it keeps no windows");
    if (cap_ids < 0 || (cap_ids > 0 && !idv)) return fail(SB200_ERR_INVALID, "cap < 0, or ids is NULL with cap > 0");
    if (int rc = begin()) return rc;
    const int n = (int)hid.size();
    if (n == 0) return 0;
    if (int rc = gout.ensure(((size_t)n + 1) * 4)) return rc;
    sb::fs_launch_baked(at1.as<long long>(), n, (long long)now, (long long)period, gout.as<int>(), st);
    int total = 0;
    CU(cudaMemcpyAsync(&total, gout.p, 4, cudaMemcpyDeviceToHost, st));
    if (int rc = finish()) return rc;
    const int m = (int)std::min<int64_t>(cap_ids, total);
    if (m > 0) {
      std::vector<int> pos(m);
      CU(cudaMemcpyAsync(pos.data(), gout.as<int>() + 1, (size_t)m * 4, cudaMemcpyDeviceToHost, st));
      if (int rc = finish()) return rc;
      for (int i = 0; i < m; ++i) idv[i] = hid[pos[i]];
    }
    return total;
  }

  // associate_store's row source: the queried tracks of `src` (positions qpos[Q] on the device) staged on this store's
  // stream into the call's rows, and into the tables TrackQueries names
  struct StoreRows {
    sb200_fstore* src;
    const int* qpos;
    int Q;
    sb::FsAttrCols qattr;   // gated: the queries' triples
    float* rq;              // quality store: the rows' qualities
    int* hq;                // quality store: the queries' history lengths
  };
  static int stage_store_rows(void* ctx, float* rows, const int* qoff, const int* row_q, int R, cudaStream_t st) {
    const StoreRows& x = *static_cast<const StoreRows*>(ctx);
    const sb200_fstore& src = *x.src;
    sb::FsCall c{};
    c.qoff = qoff;
    c.row_q = row_q;
    c.Q = x.Q;
    c.R = R;
    const sb::FsStore s = src.view();   // each row widened exactly from src's storage type
    sb::fs_launch_owned_stage(s, c, x.qpos, rows, st);
    if (src.gate) sb::fs_launch_attr_gather(src.attr_cols(), x.qpos, x.Q, x.qattr, st);
    if (src.keep) {
      sb::fs_launch_qual_stage(s, c, src.qual.as<float>(), x.qpos, x.rq, st);
      sb::fs_launch_words_compact(src.hlen.p, x.hq, x.qpos, x.Q, 1, st);
    }
    CU(cudaGetLastError());
    return 0;
  }

  // fetch_tracks(ids) from src, then one associate call of this store with those tracks as its queries (merge_external
  // with merge_history = true, or add_track), then, with remove, the tracks taken out of src
  int associate_store(sb200_fstore* src, int n, const uint64_t* idv, int remove, int32_t* counts, uint64_t* winners,
                      double* weights, uint64_t* track_ids, uint8_t* merged) {
    if (src == this) return fail(SB200_ERR_INVALID, "dst and src are the same store (merge_owned merges within one)");
    const sb200_fstore_options& so = src->o;
    if (so.device != o.device) return fail(SB200_ERR_INVALID, "src is on device %d, dst on device %d", so.device, o.device);
    if (so.max_observations != o.max_observations)
      return fail(SB200_ERR_INVALID, "max_observations differ: %d in src, %d in dst", so.max_observations,
                  o.max_observations);
    bool same = src->cls.size() == cls.size();
    for (size_t k = 0; same && k < cls.size(); ++k) {
      const int j = src->class_index(cls[k].id);
      same = j >= 0 && src->cls[j].dim == cls[k].dim;
    }
    if (!same) return fail(SB200_ERR_INVALID, "feature classes or feature_dim differ between src and dst");
    if (src->gate != gate) return fail(SB200_ERR_INVALID, "gate rules differ: %d in src, %d in dst", src->gate, gate);
    if (src->keep != keep || (keep && (src->init_cap != init_cap || src->ext != ext)))
      return fail(SB200_ERR_INVALID, "retention rules or their parameters differ between src and dst");
    if (n < 0) return fail(SB200_ERR_INVALID, "n < 0");
    if (remove != 0 && remove != 1) return fail(SB200_ERR_INVALID, "remove must be 0 or 1");
    if (n > 0 && (!idv || !counts || !winners || !weights || !track_ids || !merged))
      return fail(SB200_ERR_INVALID, "ids or an output is NULL");
    if (int rc = check_ids(n, idv, "id", true)) return rc;
    std::vector<int> pos(n);
    for (int i = 0; i < n; ++i) {
      auto it = src->hpos.find(idv[i]);
      if (it == src->hpos.end())
        return fail(SB200_ERR_INVALID, "id %llu is not stored in src", (unsigned long long)idv[i]);
      pos[i] = it->second;
    }
    if (int rc = begin()) return rc;
    if (n == 0) return 0;
    // the queries are src's rows of the class this store has selected
    const int src_sel = src->sel;
    src->select(src->class_index(cls[sel].id));
    const int rc = associate_tracks(src, n, idv, pos, remove, counts, winners, weights, track_ids, merged);
    src->select(src_sel);
    return rc;
  }

  // associate_store once every check has passed, with src's class selected as this store's
  int associate_tracks(sb200_fstore* src, int n, const uint64_t* idv, const std::vector<int>& pos, int remove,
                       int32_t* counts, uint64_t* winners, double* weights, uint64_t* track_ids, uint8_t* merged) {
    // src's stream is idle once peek returns, so every column this call reads from src is complete
    std::vector<int> ring;
    if (int rc = src->peek(pos, &ring)) return rc;
    std::vector<int32_t> offs(n + 1, 0);
    for (int i = 0; i < n; ++i) offs[i + 1] = offs[i] + ring[2 * i];
    std::vector<std::vector<uint64_t>> qhist;
    if (keep)
      for (int p : pos) qhist.push_back(src->hist[p]);
    if (int rc = sq.ensure((size_t)n * 8)) return rc;
    if (gate)
      if (int rc = qattr.ensure((size_t)n * 24)) return rc;
    if (keep)
      if (int rc = dqr.ensure((size_t)offs[n] * 4)) return rc;
    CU(cudaMemcpyAsync(sq.p, pos.data(), (size_t)n * 4, cudaMemcpyHostToDevice, st));
    StoreRows ctx{src, sq.as<int>(), n, triples(qattr, n), dqr.as<float>(), sq.as<int>() + n};
    const TrackQueries tq{keep ? sq.as<int>() + n : nullptr, keep ? &qhist : nullptr};
    // a quality store of several classes decides the destinations here and applies every class below
    const bool qpasses = keep && cls.size() > 1;
    std::vector<int> dec;
    // returns once this store's stream has finished, so src's rows are read no more
    if (int rc = associate_rows(n, idv, offs.data(), {stage_store_rows, &ctx}, counts, winners, weights, track_ids,
                                merged, &tq, qpasses ? &dec : nullptr))
      return rc;
    if (qpasses) {
      if (int rc = qmerge_classes(src, ctx, n, idv, pos, qhist, dec, winners, track_ids, merged)) return rc;
    } else if (cls.size() > 1) {   // where each query went, and then its rows of the other classes
      std::vector<int> dpos(n);
      for (int q = 0; q < n; ++q) dpos[q] = hpos.at(merged[q] ? track_ids[q] : idv[q]);
      const int s0 = sel, src_sel = src->sel;
      const std::vector<int> asc = ascending_classes();
      const int rc = each_class([&](int k) {
        if (k == s0) return 0;
        src->select(src->class_index(cls[k].id));
        return append_class_rows(src, ctx, n, idv, pos, dpos);
      }, &asc);
      src->select(src_sel);
      if (rc) return rc;
    }
    if (!remove) return 0;
    std::vector<char> gone(src->hid.size(), 0);
    for (int p : pos) gone[p] = 1;
    return src->remove_marked(gone);
  }

  // associate_store on a quality store of several classes, once TopN and the gate have decided each query's
  // destination (dec[q]: a stored position, or -1 for a new track).  Track::merge walks the classes a query holds in
  // ascending id, each step appending the query's history h(q) before it optimizes that class; so one fs_qmerge_kernel
  // pass per class, in ascending id, over every query (a query without rows of the class truncates at a capacity no
  // smaller than its list's, which changes nothing), whose history increments make each item of a destination reach
  //   h0 + S(q) + le(q) h(q),   S(q) = the sum of |C(j)| h(j) over the destination's earlier items j,
  // le(q) = the classes q holds up to this pass's id, |C(j)| all the classes j holds.  A pass starts from the
  // history length the previous one left (h0 in the first); a new track is the query whole, h(q) in every pass.
  int qmerge_classes(sb200_fstore* src, const StoreRows& ctx0, int n, const uint64_t* idv, const std::vector<int>& pos,
                     const std::vector<std::vector<uint64_t>>& qhist, const std::vector<int>& dec,
                     const uint64_t* winners, uint64_t* track_ids, uint8_t* merged) {
    const int live = (int)hid.size(), nc = (int)cls.size(), src_sel = src->sel;
    std::vector<std::vector<int>> qcnt(nc);   // rows of each query in each class
    for (int k = 0; k < nc; ++k) {
      std::vector<int> ring;
      src->select(src->class_index(cls[k].id));
      if (int rc = src->peek(pos, &ring)) { src->select(src_sel); return rc; }
      for (int q = 0; q < n; ++q) qcnt[k].push_back(ring[2 * q]);
    }
    src->select(src_sel);
    std::vector<int> dpos(n), held(n, 0), prev(n, -1), last_of(n, -1);
    std::vector<long long> S(n, 0), h(n);
    std::unordered_map<int, int> last;
    std::unordered_map<int, long long> acc;
    for (int q = 0, fresh = 0; q < n; ++q) {
      for (int k = 0; k < nc; ++k) held[q] += qcnt[k][q] > 0;
      h[q] = (long long)qhist[q].size();
      dpos[q] = dec[q] >= 0 ? dec[q] : live + fresh++;
      if (dec[q] < 0) continue;
      auto it = last.find(dpos[q]);
      prev[q] = it == last.end() ? -1 : it->second;
      last[dpos[q]] = q;
      S[q] = acc[dpos[q]];
      acc[dpos[q]] += held[q] * h[q];
    }
    for (int q = 0; q < n; ++q)
      if (dec[q] >= 0) last_of[q] = last[dpos[q]];
    std::vector<long long> le(n, 0), r(n, 0), r_prev;
    std::vector<int> inc(n);
    for (int k : ascending_classes()) {
      std::vector<int> qoff(n + 1, 0);
      for (int q = 0; q < n; ++q) qoff[q + 1] = qoff[q] + qcnt[k][q];
      const int R = qoff[n];
      if (R == 0) continue;   // no query holds the class
      for (int q = 0; q < n; ++q) {
        le[q] += qcnt[k][q] > 0;
        r[q] = S[q] + le[q] * h[q];
      }
      for (int q = 0; q < n; ++q) {
        long long from = 0;   // the relative history length the kernel holds before item q
        if (prev[q] >= 0) from = r[prev[q]];
        else if (!r_prev.empty() && dec[q] >= 0) from = r_prev[last_of[q]];
        inc[q] = (int)(dec[q] >= 0 ? r[q] - from : h[q]);
      }
      r_prev = r;
      src->select(src->class_index(cls[k].id));
      const int s0 = sel;
      select(k);
      int rc = dqr.ensure((size_t)R * 4);
      if (!rc) rc = dinc.ensure((size_t)n * 4);
      if (!rc) {
        StoreRows ctx = ctx0;
        ctx.rq = dqr.as<float>();
        const sb::FsRowSource rs{stage_store_rows, &ctx};
        const ReqLayout L(n, R, d8, false);
        rc = upload(L, n, idv, qoff, std::vector<int>(R), dpos.data(), Column{nullptr, false, nullptr}, 0, &rs);
        if (!rc && cudaMemcpyAsync(dinc.p, inc.data(), (size_t)n * 4, cudaMemcpyHostToDevice, st) != cudaSuccess)
          rc = fail(SB200_ERR_CUDA, "history increment upload failed");
        if (!rc) {
          const sb::FsCall c = call_view(L, n, R, nullptr);
          const sb::FsQCall qc{qual.as<float>(), hlen.as<int>(), dcap.as<int>(), (int)cap_tab.size(), dqr.as<float>(), 1};
          sb::fs_launch_qmerge(view(), c, qc, st, dinc.as<int>());
          if (gate) sb::fs_launch_attr_new(live, c, gate_view(n), st);
          rc = finish();
        }
      }
      select(s0);
      src->select(src_sel);
      if (rc) return rc;
    }
    for (int q = 0; q < n; ++q) {
      merged[q] = dec[q] >= 0;
      track_ids[q] = merged[q] ? winners[(size_t)q * o.topn] : idv[q];
      for (int c = 0; merged[q] && c < held[q]; ++c)   // one history step per class the query holds
        hist[dpos[q]].insert(hist[dpos[q]].end(), qhist[q].begin(), qhist[q].end());
    }
    for (int q = 0; q < n; ++q)
      if (!merged[q]) {
        hpos[idv[q]] = (int)hid.size();
        hid.push_back(idv[q]);
        hist.push_back(qhist[q]);
      }
    return 0;
  }

  // associate_store on a newest store of several classes: the selected class's rows of the queried src tracks (at
  // src positions pos, staged by ctx) appended to the tracks they went to (dpos), as an add appends rows
  int append_class_rows(sb200_fstore* src, const StoreRows& ctx, int n, const uint64_t* idv, const std::vector<int>& pos,
                        const std::vector<int>& dpos) {
    std::vector<int> ring;
    if (int rc = src->peek(pos, &ring)) return rc;
    std::vector<int> qoff(n + 1, 0);
    for (int i = 0; i < n; ++i) qoff[i + 1] = qoff[i] + ring[2 * i];
    const int R = qoff[n];
    if (R == 0) return 0;
    const std::vector<int> rows(R);   // only their number: the row source writes them
    const ReqLayout L(n, R, d8, false);
    if (int rc = plan.ensure((size_t)n * 16)) return rc;
    const sb::FsRowSource rs{stage_store_rows, const_cast<StoreRows*>(&ctx)};
    if (int rc = upload(L, n, idv, qoff, rows, dpos.data(), Column{nullptr, false, nullptr}, 0, &rs)) return rc;
    sb::fs_launch_apply(view(), call_view(L, n, R, nullptr), st);
    return finish();
  }

  // qout: a quality store's qualities [n][K] of the rows returned (fetch_quality), else nullptr
  int64_t fetch(int n, const uint64_t* idv, int remove, int32_t* counts, float* feats, float* qout = nullptr) {
    if (n < 0) return fail(SB200_ERR_INVALID, "n < 0");
    if (n > 0 && (!idv || !counts || !feats)) return fail(SB200_ERR_INVALID, "ids / counts / features is NULL");
    if (qout && !keep) return fail(SB200_ERR_INVALID, "the store keeps no qualities (it keeps its newest observations)");
    if (int rc = begin()) return rc;
    if (n == 0) return 0;
    const int K = o.max_observations, D = o.feature_dim;
    std::vector<int> pos(n, -1);
    std::vector<char> gone(hid.size(), 0);
    int64_t found = 0;
    for (int i = 0; i < n; ++i) {
      auto it = hpos.find(idv[i]);
      if (it == hpos.end() || gone[it->second]) continue;   // fetch_tracks finds a removed id no more
      pos[i] = it->second;
      ++found;
      if (remove) gone[it->second] = 1;
    }
    if (qout) {
      std::vector<int> fpos;
      for (int p : pos) if (p >= 0) fpos.push_back(p);
      std::vector<QTrack> tl;
      if (int rc = peek_tracks(fpos, &tl)) return rc;
      std::fill(qout, qout + (size_t)n * K, 0.0f);
      for (int i = 0, f = 0; i < n; ++i)
        if (pos[i] >= 0) std::copy(tl[f].q.begin(), tl[f].q.end(), qout + (size_t)i * K), ++f;
    }
    const size_t out_bytes = (size_t)n * K * d8 * 4;
    if (int rc = gpos.ensure((size_t)n * 4)) return rc;
    if (int rc = gout.ensure(align16(out_bytes) + (size_t)n * 4)) return rc;
    if (int rc = hres.ensure(align16(out_bytes) + (size_t)n * 4)) return rc;
    CU(cudaMemcpyAsync(gpos.p, pos.data(), (size_t)n * 4, cudaMemcpyHostToDevice, st));
    const sb::FsStore s = view();
    float* dout = gout.as<float>();
    int* dcnt = reinterpret_cast<int*>(gout.as<char>() + align16(out_bytes));
    sb::fs_launch_gather(s, gpos.as<int>(), n, dout, dcnt, st);
    CU(cudaMemcpyAsync(hres.p, gout.p, align16(out_bytes) + (size_t)n * 4, cudaMemcpyDeviceToHost, st));
    if (int rc = finish()) return rc;
    const float* h = static_cast<const float*>(hres.p);
    const int* hc = reinterpret_cast<const int*>(static_cast<const char*>(hres.p) + align16(out_bytes));
    for (int i = 0; i < n; ++i) {
      counts[i] = hc[i];
      for (int b = 0; b < K; ++b)
        memcpy(feats + ((size_t)i * K + b) * D, h + ((size_t)i * K + b) * d8, (size_t)D * 4);
    }
    if (remove && found)
      if (int rc = remove_marked(gone)) return rc;
    return found;
  }

  // takes the tracks with gone[p] out of the store: a stable compaction into fresh columns
  int remove_marked(const std::vector<char>& gone) {
    std::vector<int> from;
    from.reserve(hid.size());
    for (size_t p = 0; p < hid.size(); ++p)
      if (!gone[p]) from.push_back((int)p);
    DBuf nws[kNumCols];
    if (int rc = alloc(cap, nws, kNeedAll, kPartShared)) return rc;
    if (int rc = gpos.ensure(std::max<size_t>(from.size(), 1) * 4)) return rc;
    CU(cudaMemcpyAsync(gpos.p, from.data(), from.size() * 4, cudaMemcpyHostToDevice, st));
    const unsigned long long* old_ids = ids.as<unsigned long long>();
    const sb::FsAttrCols sa = attr_cols();
    const void* sh = hlen.p;
    swap_columns(nws, kNeedAll, kPartShared);   // nws holds the old columns until the compaction below has read them
    if (gate) sb::fs_launch_attr_gather(sa, gpos.as<int>(), (int)from.size(), attr_cols(), st);
    if (keep) sb::fs_launch_words_compact(sh, hlen.p, gpos.as<int>(), (int)from.size(), 1, st);
    // each class's columns, the fresh ones zero past the kept tracks; every class writes the same ids
    if (int rc = each_class([&](int) {
          DBuf nw[kNumCols];
          if (int rc = alloc(cap, nw, kNeedAll, kPartClass)) return rc;
          sb::FsStore s = view();
          s.ids = const_cast<unsigned long long*>(old_ids);
          const void* sq = qual.p;
          swap_columns(nw, kNeedAll, kPartClass);
          sb::fs_launch_compact(s, view(), gpos.as<int>(), (int)from.size(), st);
          if (keep) sb::fs_launch_words_compact(sq, qual.p, gpos.as<int>(), (int)from.size(), o.max_observations, st);
          return finish();
        }))
      return rc;
    std::vector<uint64_t> kept;
    kept.reserve(from.size());
    for (int p : from) kept.push_back(hid[p]);
    hid.swap(kept);
    if (keep) {
      std::vector<std::vector<uint64_t>> kh;
      kh.reserve(from.size());
      for (int p : from) kh.push_back(std::move(hist[p]));
      hist.swap(kh);
    }
    hpos.clear();
    for (size_t p = 0; p < hid.size(); ++p) hpos[hid[p]] = (int)p;
    return 0;
  }

  // ---- owned calls: the queries / pairs are stored tracks
  // ring state of the stored tracks at pos[]: ring[2 i] = cnt, ring[2 i + 1] = start.  The host keeps neither, so an
  // owned call reads those of the tracks it touches back once, before it checks what depends on them.  Changes nothing.
  int peek(const std::vector<int>& pos, std::vector<int>* ring) {
    const size_t n = pos.size();
    ring->assign(n * 2, 0);
    if (n == 0) return 0;
    if (int rc = gpos.ensure(n * 4)) return rc;
    if (int rc = gout.ensure(n * 8)) return rc;
    CU(cudaMemcpyAsync(gpos.p, pos.data(), n * 4, cudaMemcpyHostToDevice, st));
    sb::fs_launch_peek(view(), gpos.as<int>(), (int)n, gout.as<int>(), st);
    CU(cudaMemcpyAsync(ring->data(), gout.p, n * 8, cudaMemcpyDeviceToHost, st));
    if (int rc = finish()) return rc;
    return 0;
  }

  // owned_track_distances + TopNVoting::winners.  each == 0: one group, whose members are not candidates of each other
  // and share one max_dist; each == 1: every query on its own (excluding only itself, its own max_dist), in chunks that
  // respect the pair bound.
  int search_owned(int n, const uint64_t* qids, int each, int32_t* counts, uint64_t* winners, double* weights) {
    if (n < 0) return fail(SB200_ERR_INVALID, "n < 0");
    if (each != 0 && each != 1) return fail(SB200_ERR_INVALID, "each must be 0 or 1");
    if (n > 0 && (!qids || !counts || !winners || !weights)) return fail(SB200_ERR_INVALID, "ids or an output is NULL");
    if (int rc = check_ids(n, qids, "id", false)) return rc;
    if (int rc = begin()) return rc;
    if (n == 0) return 0;
    const int topn = o.topn, K = o.max_observations;
    const long long live = (long long)hid.size(), S = live * K;
    std::vector<int> qpos(n, -1), found;
    for (int q = 0; q < n; ++q) {
      auto it = hpos.find(qids[q]);
      if (it != hpos.end()) { qpos[q] = it->second; found.push_back(it->second); }
    }
    std::vector<int> ring;
    if (int rc = peek(found, &ring)) return rc;
    std::vector<int> qcnt(n, 0);   // rows of each query: its stored observations (0 when it is not stored)
    for (int q = 0, f = 0; q < n; ++q)
      if (qpos[q] >= 0) qcnt[q] = ring[2 * f++];
    // chunks [chunk[i], chunk[i + 1]) of queries, each within the pair bound of one distance matrix
    std::vector<int> chunk(1, 0);
    long long rows = 0;
    for (int q = 0; q < n; ++q) {
      if ((long long)qcnt[q] * S > sb::kFsMaxPairs)
        return fail(SB200_ERR_CAPACITY, "query %d needs %lld observation pairs; one query holds at most 2^30", q,
                    (long long)qcnt[q] * S);
      if (each && (rows + qcnt[q]) * S > sb::kFsMaxPairs) { chunk.push_back(q); rows = 0; }
      rows += qcnt[q];
    }
    chunk.push_back(n);
    if (!each && rows * S > sb::kFsMaxPairs)
      return fail(SB200_ERR_CAPACITY, "the call needs %lld observation pairs; one call holds at most 2^30", rows * S);
    std::fill(counts, counts + n, 0);
    std::fill(winners, winners + (size_t)n * topn, 0);
    std::fill(weights, weights + (size_t)n * topn, 0.0);
    if (found.empty()) return 0;
    std::vector<unsigned char> excl;
    if (!each) {
      excl.assign((size_t)live, 0);
      for (int p : found) excl[p] = 1;
    }
    for (size_t i = 0; i + 1 < chunk.size(); ++i)
      if (int rc = owned_chunk(chunk[i], chunk[i + 1], qids, qpos, qcnt, excl, each, counts, winners, weights))
        return rc;
    return 0;
  }

  // queries [a, b) of an owned search: request rows staged on the device, distances, TopN, results into the outputs
  int owned_chunk(int a, int b, const uint64_t* qids, const std::vector<int>& qpos, const std::vector<int>& qcnt,
                  const std::vector<unsigned char>& excl, int each, int32_t* counts, uint64_t* winners,
                  double* weights) {
    const int Q = b - a, topn = o.topn, K = o.max_observations;
    const long long live = (long long)hid.size(), S = live * K;
    std::vector<int> qoff(Q + 1, 0);
    for (int q = 0; q < Q; ++q) qoff[q + 1] = qoff[q] + qcnt[a + q];
    const int R = qoff[Q];
    if (R == 0) return 0;
    const int nkey = each ? Q : 1;
    const ReqLayout L(Q, R, d8, false, nkey, (long long)excl.size());
    const ResLayout RL(Q, topn);
    if (int rc = hreq.ensure(L.total - L.qid)) return rc;
    if (int rc = dreq.ensure(L.total)) return rc;
    if (int rc = size_call(RL, Q, R, S)) return rc;
    auto at = [&](size_t off) { return static_cast<char*>(hreq.p) + (off - L.qid); };   // rows are written on the device
    stage_request(L, at(L.qid), Q, qids + a, qoff.data(), nullptr, nkey);
    int* qp = reinterpret_cast<int*>(at(L.qpos));
    for (int q = 0; q < Q; ++q) qp[q] = std::max(qpos[a + q], 0);   // a query that is not stored has no rows
    if (!excl.empty()) memcpy(at(L.excl), excl.data(), excl.size());
    CU(cudaMemcpyAsync(dreq.as<char>() + L.qid, hreq.p, L.total - L.qid, cudaMemcpyHostToDevice, st));
    const sb::FsStore s = view();
    const sb::FsCall c = call_view(L, Q, R, &RL);
    const int mode = each ? sb::kFsOwnedEach : sb::kFsOwnedGroup;
    const int* dqpos = reinterpret_cast<const int*>(dreq.as<char>() + L.qpos);
    if (gate)   // the queries' triples are their stored ones
      if (int rc = qattr.ensure((size_t)Q * 24)) return rc;
    const sb::FsGate g = gate_view(Q);
    CU(cudaEventRecord(ev[0], st));
    if (gate) sb::fs_launch_attr_gather(attr_cols(), dqpos, Q, triples(qattr, Q), st);
    sb::fs_launch_owned_stage(s, c, dqpos, reinterpret_cast<float*>(dreq.as<char>() + L.rows), st);
    sb::fs_launch_dist(o.metric, o.distance_filter, s, c, st, mode,
                       reinterpret_cast<const unsigned char*>(dreq.as<char>() + L.excl), gate ? &g : nullptr);
    CU(cudaEventRecord(ev[1], st));
    sb::fs_launch_topn(o.max_distance, o.min_votes, topn, false, s, c, st, mode);
    if (!each)   // each == 1 is one voting call per query: no claim crosses queries, and BestFit is TopN
      if (int rc = claim_best_fit(s, c, false)) return rc;
    CU(cudaEventRecord(ev[2], st));
    CU(cudaMemcpyAsync(hres.p, dres.p, RL.total, cudaMemcpyDeviceToHost, st));
    if (int rc = finish(0, 2)) return rc;   // summed over the chunks
    read_results(RL, Q, qids + a, counts + a, winners + (size_t)a * topn, weights + (size_t)a * topn);
    return 0;
  }

  // merge_owned for the pairs in order, each seeing the state the earlier ones left.  The final ring of every touched
  // destination is planned on the host as references to pre-call slots (the slots the sequential fetch + add emulation
  // leaves filled, with its ring starts); the rows that move are gathered into scratch and then scattered, so a chain
  // never reads a row already overwritten.
  int merge_owned(int n, const uint64_t* dids, const uint64_t* sids, int remove) {
    if (n < 0) return fail(SB200_ERR_INVALID, "n < 0");
    if (n > 0 && (!dids || !sids)) return fail(SB200_ERR_INVALID, "dest_ids / src_ids is NULL");
    std::vector<int> dp(n), sp(n);
    std::vector<char> gone(hid.size(), 0);
    for (int i = 0; i < n; ++i) {
      auto d = hpos.find(dids[i]), s = hpos.find(sids[i]);
      if (d == hpos.end()) return fail(SB200_ERR_INVALID, "pair %d: dest %llu is not stored", i, (unsigned long long)dids[i]);
      if (s == hpos.end()) return fail(SB200_ERR_INVALID, "pair %d: src %llu is not stored", i, (unsigned long long)sids[i]);
      if (d->second == s->second)
        return fail(SB200_ERR_INVALID, "pair %d: dest and src are the same track %llu", i, (unsigned long long)dids[i]);
      if (gone[d->second] || gone[s->second])
        return fail(SB200_ERR_INVALID, "pair %d names a track an earlier pair removed", i);
      dp[i] = d->second;
      sp[i] = s->second;
      if (remove) gone[s->second] = 1;
    }
    if (int rc = begin()) return rc;
    if (n == 0) return 0;
    const int K = o.max_observations;
    std::unordered_map<int, int> idx;   // store position -> touched track
    std::vector<int> touched;
    for (int i = 0; i < n; ++i)
      for (int p : {dp[i], sp[i]})
        if (idx.emplace(p, (int)touched.size()).second) touched.push_back(p);
    std::vector<int> wpos;   // gated: the destinations whose windows change, and their final triples
    Triples win;
    if (gate)
      if (int rc = plan_merge_attrs(n, dp, sp, idx, touched, &wpos, &win)) return rc;
    if (keep) {   // each pair's merge optimized at its destination's capacity, planned from the peeked lists
      // Track::merge walks the classes the source holds (ascending id here), and each class step appends the source's
      // history to the destination's before it optimizes that class's list at the new capacity
      const std::vector<int> asc = ascending_classes();
      std::vector<std::vector<QTrack>> tl(cls.size());
      if (int rc = each_class([&](int k) { return peek_tracks(touched, &tl[k]); })) return rc;
      std::vector<std::vector<uint64_t>> h(touched.size());
      for (size_t t = 0; t < touched.size(); ++t) h[t] = hist[touched[t]];
      for (int i = 0; i < n; ++i) {
        const int d = idx[dp[i]], sr = idx[sp[i]];
        for (int k : asc) {
          if (tl[k][sr].ref.empty()) continue;   // a class the source does not hold
          tl[k][d].h = h[d];
          tl[k][sr].h = h[sr];
          merge_into(tl[k][d], tl[k][sr]);
          h[d] = tl[k][d].h;
        }
      }
      std::vector<char> dirty(touched.size(), 0);
      for (std::vector<QTrack>& v : tl)
        for (size_t t = 0; t < touched.size(); ++t) {
          v[t].h = h[t];   // every class writes the track's final history length
          if (gone[v[t].pos]) v[t].dirty = false;
          dirty[t] |= v[t].dirty;
        }
      if (int rc = each_class([&](int k) { return apply_tracks(tl[k]); })) return rc;
      for (size_t t = 0; t < touched.size(); ++t)
        if (dirty[t]) hist[touched[t]] = h[t];
      if (int rc = write_attrs(wpos, win)) return rc;
      if (remove) return remove_marked(gone);
      return 0;
    }
    // a newest store: each class's rings planned and moved on their own
    if (int rc = each_class([&](int) { return merge_rings(n, dp, sp, idx, touched, gone); })) return rc;
    if (int rc = write_attrs(wpos, win)) return rc;
    if (remove) return remove_marked(gone);
    return 0;
  }

  // merge_owned on a newest store, for the selected class
  int merge_rings(int n, const std::vector<int>& dp, const std::vector<int>& sp, std::unordered_map<int, int>& idx,
                  const std::vector<int>& touched, const std::vector<char>& gone) {
    const int K = o.max_observations;
    std::vector<int> ring;
    if (int rc = peek(touched, &ring)) return rc;
    // per touched track: its rows oldest first as stored row indices (position * K + slot) of the pre-call store, and
    // how many rows its ring has taken since the call began (old ones included): virtual row v sits in slot (s0 + v) % K
    struct Plan { std::vector<int> rows; long long taken; bool dirty; };
    std::vector<Plan> pl(touched.size());
    for (size_t t = 0; t < touched.size(); ++t) {
      const int p = touched[t], c0 = ring[2 * t], s0 = ring[2 * t + 1];
      for (int j = 0; j < c0; ++j) pl[t].rows.push_back(p * K + (s0 + j) % K);
      pl[t].taken = c0;
      pl[t].dirty = false;
    }
    for (int i = 0; i < n; ++i) {
      Plan& d = pl[idx[dp[i]]];
      const Plan& s = pl[idx[sp[i]]];
      d.rows.insert(d.rows.end(), s.rows.begin(), s.rows.end());
      d.taken += (long long)s.rows.size();
      if ((int)d.rows.size() > K) d.rows.erase(d.rows.begin(), d.rows.end() - K);   // keep the newest K
      d.dirty = true;
    }
    std::vector<int> mv_src, mv_dst, hdr;
    for (size_t t = 0; t < touched.size(); ++t) {
      const int p = touched[t];
      if (!pl[t].dirty || gone[p]) continue;
      const int c1 = (int)pl[t].rows.size();
      const int s1 = (int)((ring[2 * t + 1] + std::max<long long>(0, pl[t].taken - K)) % K);
      hdr.insert(hdr.end(), {p, c1, s1});
      for (int j = 0; j < c1; ++j) {
        const int dst = p * K + (s1 + j) % K;
        if (pl[t].rows[j] != dst) { mv_src.push_back(pl[t].rows[j]); mv_dst.push_back(dst); }
      }
    }
    const int nm = (int)mv_src.size(), nh = (int)hdr.size() / 3;
    std::vector<int> tab;
    tab.reserve(2 * (size_t)nm + hdr.size());
    tab.insert(tab.end(), mv_src.begin(), mv_src.end());
    tab.insert(tab.end(), mv_dst.begin(), mv_dst.end());
    tab.insert(tab.end(), hdr.begin(), hdr.end());
    if (int rc = gpos.ensure(std::max<size_t>(tab.size(), 1) * 4)) return rc;
    if (int rc = gout.ensure(std::max<size_t>((size_t)nm * row_bytes(), 16))) return rc;
    CU(cudaMemcpyAsync(gpos.p, tab.data(), tab.size() * 4, cudaMemcpyHostToDevice, st));
    const int* dtab = gpos.as<int>();
    CU(cudaEventRecord(ev[2], st));
    sb::fs_launch_move_rows(view(), dtab, dtab + nm, nm, dtab + 2 * nm, nh, gout.p, st);
    CU(cudaEventRecord(ev[3], st));
    return finish(2, 3);
  }

  // merge_owned's attributes: each pair, in order, must be compatible with the windows the earlier pairs left (else the
  // call is refused); a destination takes the hull
  int plan_merge_attrs(int n, const std::vector<int>& dp, const std::vector<int>& sp,
                       std::unordered_map<int, int>& idx, const std::vector<int>& touched, std::vector<int>* wpos,
                       Triples* win) {
    Triples cur;
    if (int rc = peek_attrs(touched, &cur)) return rc;
    std::vector<char> dirty(touched.size(), 0);
    for (int i = 0; i < n; ++i) {
      const int d = idx[dp[i]], s = idx[sp[i]];
      if (!sb::fs_compatible(gate, cur.src[d], cur.t0[d], cur.t1[d], cur.src[s], cur.t0[s], cur.t1[s]))
        return fail(SB200_ERR_INVALID,
                    "pair %d: src %llu (source %llu, [%lld, %lld]) is not compatible with dest %llu (source %llu, "
                    "[%lld, %lld])", i, (unsigned long long)hid[sp[i]], (unsigned long long)cur.src[s],
                    (long long)cur.t0[s], (long long)cur.t1[s], (unsigned long long)hid[dp[i]],
                    (unsigned long long)cur.src[d], (long long)cur.t0[d], (long long)cur.t1[d]);
      cur.t0[d] = std::min(cur.t0[d], cur.t0[s]);
      cur.t1[d] = std::max(cur.t1[d], cur.t1[s]);
      dirty[d] = 1;
    }
    for (size_t t = 0; t < touched.size(); ++t)
      if (dirty[t]) {
        wpos->push_back(touched[t]);
        win->src.push_back(cur.src[t]); win->t0.push_back(cur.t0[t]); win->t1.push_back(cur.t1[t]);
      }
    return 0;
  }

  // ---- the store blob (layouts: include/similari_b200.h)
  // the device columns and the sections of `plan` at sec_off of a blob at dblob on this device: dir 0 packs, dir 1
  // unpacks.  Each class's columns are the members while it is selected; the class table and the histories, which have
  // no device column, are left to the caller.
  int move(int dir, const std::vector<sb::FsSection>& plan, const uint64_t* sec_off, char* dblob) {
    std::vector<sb::XferSeg> segs;
    each_class([&](int k) {
      for (size_t i = 0; i < plan.size(); ++i)
        for (const Col& c : kCols)
          if (c.sec == plan[i].role && (c.per_class ? plan[i].cls == k : k == 0))
            sb::add_segment(segs, dir, (this->*c.buf).as<char>(), dblob + sec_off[i], plan[i].bytes);
      return 0;
    });
    return sb::copy_segments(segs, num_sms, st);
  }

  int save(void* dst, uint64_t cap_bytes, uint64_t* bytes) {
    // a store of the single class 0 writes the version it wrote before classes existed
    const uint32_t version = !plain_classes() ? 4 : keep ? 3 : gate ? 2 : 1;
    const int nc = (int)cls.size(), K = o.max_observations, live = (int)hid.size();
    std::vector<uint64_t> hc, cid(nc);
    std::vector<int32_t> cdim(nc);
    for (const std::vector<uint64_t>& h : hist) hc.insert(hc.end(), h.begin(), h.end());
    for (int k = 0; k < nc; ++k) { cid[k] = cls[k].id; cdim[k] = cls[k].dim; }
    const std::vector<sb::FsSection> plan =
        sb::fs_blob_sections((int)version, live, K, stype, gate, keep, nc, cdim.data(), hc.size());
    std::vector<uint64_t> sec;
    for (const sb::FsSection& e : plan) sec.push_back(e.bytes);
    BlobHeaders hs{version};
    const uint64_t total = hs.visit([&](auto& h) {
      memset(&h, 0, sizeof(h));
      h.magic = SB200_FSTORE_BLOB_MAGIC; h.version = version;
      h.metric = o.metric; h.distance_filter = o.distance_filter; h.max_observations = K; h.topn = o.topn;
      h.max_distance = o.max_distance; h.min_votes = o.min_votes; h.feature_type = ftype; h.storage_type = stype;
      h.feature_dim = cls[0].dim;   // not the selected class's: the blob does not depend on the selection
      h.d8 = cls[0].d8;
      h.live = live;
      sb::lay_out(h, sec.data(), (uint32_t)sec.size());
      return h.total_bytes;
    });
    auto rules = [&](auto& h) {
      h.gate = gate;
      h.retention = keep;
      h.initial_capacity = init_cap;
      h.merge_extension = ext;
    };
    if (version == 2) hs.v2.gate = gate;
    if (version == 3) rules(hs.v3);
    if (version == 4) { rules(hs.v4); hs.v4.n_classes = nc; }
    *bytes = total;
    if (!dst) return 0;
    if (cap_bytes < total) return fail(SB200_ERR_CAPACITY, "the blob needs %llu bytes", (unsigned long long)total);
    CU(cudaSetDevice(o.device));
    return hs.visit([&](const auto& h) {
      return sb::write_blob(dst, o.device, st, h, (uint32_t)plan.size(), [&](char* p) {
        auto at = [&](int role, int k = 0) { return p + h.sec_off[sb::fs_blob_section(plan, role, k)]; };
        if (int rc = move(0, plan, h.sec_off, p)) return rc;
        each_class([&](int k) {
          sb::fs_launch_blob_scrub(stype, at(sb::kFsSecFeat, k), cnt.as<int>(), start.as<int>(), live, K, d8, st);
          if (keep)
            sb::fs_launch_qual_scrub(reinterpret_cast<float*>(at(sb::kFsSecQuality, k)), cnt.as<int>(), start.as<int>(),
                                     live, K, st);
          return 0;
        });
        if (version == 4) {
          CU(cudaMemcpyAsync(at(sb::kFsSecClassIds), cid.data(), nc * 8, cudaMemcpyHostToDevice, st));
          CU(cudaMemcpyAsync(at(sb::kFsSecClassDims), cdim.data(), nc * 4, cudaMemcpyHostToDevice, st));
        }
        if (!hc.empty()) CU(cudaMemcpyAsync(at(sb::kFsSecHistory), hc.data(), hc.size() * 8, cudaMemcpyHostToDevice, st));
        return finish();
      });
    });
  }

  // fills a store fresh from sb200_fstore_create, whose classes are the blob's, with the blob `h` / `v` at `src`, laid
  // out as `plan` (its host checks passed); refuses what its kernels find
  int load(const BlobHeader& h, const BlobView& v, const std::vector<sb::FsSection>& plan, const void* src,
           std::vector<uint64_t>&& blob_ids, std::vector<std::vector<uint64_t>>&& hists) {
    if (int rc = begin()) return rc;
    const int live = (int)h.live, K = o.max_observations, nc = (int)cls.size();
    ftype = h.feature_type;
    stype = h.storage_type;
    if (int rc = set_gate(v.gate)) return rc;
    if (int rc = set_retention(v.keep, v.init_cap, v.ext)) return rc;
    if (live == 0) return 0;
    if (int rc = reserve((size_t)live)) return rc;
    DBuf tmp;
    const char* dblob = nullptr;
    if (int rc = sb::blob_on_device(src, h.total_bytes, o.device, st, tmp, &dblob)) return rc;
    auto at = [&](int role, int k = 0) { return dblob + v.sec_off[sb::fs_blob_section(plan, role, k)]; };
    // counts and ring starts index the rows in every later kernel: checked before anything is copied into the store
    sb::FsClassCols cc{};
    cc.n = nc;
    for (int k = 0; k < nc; ++k) {
      cc.cnt[k] = reinterpret_cast<const int*>(at(sb::kFsSecCnt, k));
      cc.start[k] = reinterpret_cast<const int*>(at(sb::kFsSecStart, k));
    }
    int bad[6] = {0, 0, 0, 0, 0, 0};   // class check, windows, quality
    if (int rc = gpos.ensure(sizeof(bad))) return rc;
    CU(cudaMemsetAsync(gpos.p, 0, sizeof(bad), st));
    sb::fs_launch_class_check(cc, live, K, gpos.as<int>(), st);
    if (v.gate)
      sb::fs_launch_attr_check(reinterpret_cast<const long long*>(at(sb::kFsSecTStart)),
                               reinterpret_cast<const long long*>(at(sb::kFsSecTEnd)), live, gpos.as<int>() + 3, st);
    if (v.keep)
      for (int k = 0; k < nc; ++k)
        sb::fs_launch_qual_check(reinterpret_cast<const float*>(at(sb::kFsSecQuality, k)), cc.cnt[k], cc.start[k], live,
                                 K, gpos.as<int>() + 4, st);
    CU(cudaMemcpyAsync(bad, gpos.p, sizeof(bad), cudaMemcpyDeviceToHost, st));
    if (int rc = finish()) return rc;
    // versions 1 to 3 hold every track in their one class: a track without rows is a cnt outside their 1..K
    const int lo = v.version < 4 ? 1 : 0;
    if (lo) { bad[0] += bad[2]; bad[2] = 0; }
    if (bad[0]) return fail(SB200_ERR_INVALID, "the blob holds %d cnt entries outside %d..%d", bad[0], lo, K);
    if (bad[1]) return fail(SB200_ERR_INVALID, "the blob holds %d start entries outside 0..%d", bad[1], K - 1);
    if (bad[2]) return fail(SB200_ERR_INVALID, "the blob holds %d tracks without a row in any class", bad[2]);
    if (bad[3]) return fail(SB200_ERR_INVALID, "the blob holds %d windows with t_start > t_end", bad[3]);
    if (bad[4]) return fail(SB200_ERR_INVALID, "the blob holds %d NaN qualities in filled slots", bad[4]);
    if (bad[5])
      return fail(SB200_ERR_INVALID, "the blob holds %d observations out of the quality order (above the one before)",
                  bad[5]);
    hid = std::move(blob_ids);
    if (int rc = move(1, plan, v.sec_off, const_cast<char*>(dblob))) return rc;
    hist = std::move(hists);
    for (size_t p = 0; p < hid.size(); ++p) hpos[hid[p]] = (int)p;
    return 0;
  }
};

const sb200_fstore::Col sb200_fstore::kCols[kNumCols] = {
    {&sb200_fstore::feat, 0, false, kNeedAll, false, sb::kFsSecFeat, true},
    {&sb200_fstore::cnt, 4, false, kNeedAll, true, sb::kFsSecCnt, true},
    {&sb200_fstore::start, 4, false, kNeedAll, true, sb::kFsSecStart, true},
    {&sb200_fstore::ids, 8, false, kNeedAll, false, sb::kFsSecIds, false},
    {&sb200_fstore::run, 4, false, kNeedAll, true, -1, false},
    {&sb200_fstore::asrc, 8, false, kNeedGate, true, sb::kFsSecSource, false},
    {&sb200_fstore::at0, 8, false, kNeedGate, true, sb::kFsSecTStart, false},
    {&sb200_fstore::at1, 8, false, kNeedGate, true, sb::kFsSecTEnd, false},
    {&sb200_fstore::qual, 4, true, kNeedQuality, true, sb::kFsSecQuality, true},
    {&sb200_fstore::hlen, 4, false, kNeedQuality, true, sb::kFsSecHistLen, false},
};

// a call without a handle: SB200_ERR_CUDA when there is no device to have made one, else SB200_ERR_INVALID
int no_handle() {
  if (int rc = sb::check_device(0)) return rc;
  return fail(SB200_ERR_INVALID, "NULL handle");
}

extern "C" int sb200_fstore_create(const sb200_fstore_options* opts, sb200_fstore** out);

// sb200_fstore_load on `device`: every check the host can make from the header, the class table, the ids, the
// histories and (quality store) the counts and ring starts, then the store, whose kernels check the rest
static int load_blob(const void* buf, uint64_t bytes, int32_t device, sb200_fstore** out) {
  // no store (and no caller stream) yet: a device blob must be complete when the call is made
  auto truncated = [&] { return fail(SB200_ERR_INVALID, "the blob is truncated (%llu bytes)", (unsigned long long)bytes); };
  BlobHeaders hs;
  const BlobHeader& h = hs.v1;   // the fields every version shares
  if (bytes < sizeof(h)) return truncated();
  CU(cudaMemcpy(&hs.v1, buf, sizeof(h), cudaMemcpyDefault));
  if (h.magic != SB200_FSTORE_BLOB_MAGIC) return fail(SB200_ERR_INVALID, "not a feature store blob (bad magic)");
  if (h.version < SB200_FSTORE_BLOB_VERSION || h.version > SB200_FSTORE_BLOB_VERSION_CLASSES)
    return fail(SB200_ERR_INVALID, "feature store blob version %u (this library reads %u to %u)", h.version,
                SB200_FSTORE_BLOB_VERSION, SB200_FSTORE_BLOB_VERSION_CLASSES);
  hs.version = h.version;
  BlobView v;
  v.version = h.version;
  if (int rc = hs.visit([&](auto& x) {
        if (static_cast<const void*>(&x) != &h) {   // a version-1 header is read already
          if (bytes < sizeof(x)) return truncated();
          CU(cudaMemcpy(&x, buf, sizeof(x), cudaMemcpyDefault));
        }
        v.sec_off = x.sec_off;
        v.sec_bytes = x.sec_bytes;
        return 0;
      }))
    return rc;
  auto rules = [&](const auto& x) {
    v.gate = x.gate;
    v.keep = x.retention;
    v.init_cap = x.initial_capacity;
    v.ext = x.merge_extension;
  };
  if (v.version == 2) v.gate = hs.v2.gate;
  if (v.version == 3) rules(hs.v3);
  if (v.version == 4) { rules(hs.v4); v.n_classes = hs.v4.n_classes; }
  if (!allowed(kBlobGates[v.version], v.gate))
    return fail(SB200_ERR_INVALID, "a version-%u blob with unknown gate rule %d", v.version, v.gate);
  if (!allowed(kBlobKeeps[v.version], v.keep))
    return fail(SB200_ERR_INVALID, "a version-%u blob with unknown retention rule %d", v.version, v.keep);
  const int nc = v.n_classes;
  if (nc < 1 || nc > SB200_FSTORE_MAX_CLASSES)
    return fail(SB200_ERR_INVALID, "n_classes %d outside 1..%d", nc, SB200_FSTORE_MAX_CLASSES);
  if (h.total_bytes > bytes)
    return fail(SB200_ERR_INVALID, "the blob is truncated (%llu of total_bytes %llu)", (unsigned long long)bytes,
                (unsigned long long)h.total_bytes);
  sb200_fstore_options o = {h.metric, h.distance_filter, h.max_observations, h.feature_dim, h.topn, h.max_distance,
                            h.min_votes, device};
  if (int rc = check_options(o)) return rc;
  if (h.d8 != (h.feature_dim + 7) / 8 * 8) return fail(SB200_ERR_INVALID, "d8 is not feature_dim rounded up to 8");
  if (!known_type(h.feature_type)) return fail(SB200_ERR_INVALID, "unknown feature_type %d", h.feature_type);
  // before the section sizes, which depend on it
  if (!known_type(h.storage_type)) return fail(SB200_ERR_INVALID, "unknown storage_type %d", h.storage_type);
  // live * K indexes the distance matrix's columns as an int
  if (h.live < 0 || h.live > INT32_MAX / h.max_observations) return fail(SB200_ERR_INVALID, "live count out of range");
  const int K = h.max_observations;
  const uint64_t live = (uint64_t)h.live;
  std::vector<int> tab;   // quality store: c(h)
  if (v.keep)
    if (int rc = capacity_table(K, v.init_cap, v.ext, &tab)) return rc;
  // the section table (a version-4 blob's class dims are not read yet: only the names and the number count), then the
  // class table, then every section's size
  std::vector<uint64_t> cid(nc, 0);
  std::vector<int32_t> cdim(nc, h.feature_dim);
  std::vector<sb::FsSection> plan =
      sb::fs_blob_sections((int)v.version, live, K, h.storage_type, v.gate, v.keep, nc, cdim.data(), 0);
  std::vector<const char*> name;
  for (const sb::FsSection& e : plan) name.push_back(e.name);
  if (int rc = hs.visit([&](const auto& x) { return sb::check_section_table(x, (uint32_t)plan.size(), name.data()); }))
    return rc;
  auto at = [&](int role, int k = 0) {
    return static_cast<const char*>(buf) + v.sec_off[sb::fs_blob_section(plan, role, k)];
  };
  auto sec_bytes = [&](int role, int k = 0) { return v.sec_bytes[sb::fs_blob_section(plan, role, k)]; };
  if (v.version == SB200_FSTORE_BLOB_VERSION_CLASSES) {
    if (sec_bytes(sb::kFsSecClassIds) != (uint64_t)nc * 8 || sec_bytes(sb::kFsSecClassDims) != (uint64_t)nc * 4)
      return fail(SB200_ERR_INVALID, "the class table does not hold n_classes = %d entries", nc);
    CU(cudaMemcpy(cid.data(), at(sb::kFsSecClassIds), nc * 8, cudaMemcpyDefault));
    CU(cudaMemcpy(cdim.data(), at(sb::kFsSecClassDims), nc * 4, cudaMemcpyDefault));
    for (int k = 0; k < nc; ++k) {
      if (cdim[k] < 1 || cdim[k] > SB200_FSTORE_MAX_DIM)
        return fail(SB200_ERR_INVALID, "class %llu: feature_dim %d outside 1..%d", (unsigned long long)cid[k], cdim[k],
                    SB200_FSTORE_MAX_DIM);
      for (int j = 0; j < k; ++j)
        if (cid[j] == cid[k]) return fail(SB200_ERR_INVALID, "class id %llu appears twice", (unsigned long long)cid[k]);
    }
    if (cdim[0] != h.feature_dim) return fail(SB200_ERR_INVALID, "feature_dim is not the first class's dim");
    plan = sb::fs_blob_sections((int)v.version, live, K, h.storage_type, v.gate, v.keep, nc, cdim.data(), 0);
  }
  for (size_t i = 0; i < plan.size(); ++i)
    if (plan[i].role != sb::kFsSecHistory && v.sec_bytes[i] != plan[i].bytes)   // the history's: against its lengths
      return fail(SB200_ERR_INVALID, "section %s holds %llu bytes, %llu expected", plan[i].name,
                  (unsigned long long)v.sec_bytes[i], (unsigned long long)plan[i].bytes);
  std::vector<uint64_t> blob_ids(live);
  if (live) CU(cudaMemcpy(blob_ids.data(), at(sb::kFsSecIds), live * 8, cudaMemcpyDefault));
  std::unordered_set<uint64_t> seen;
  seen.reserve(live * 2);
  for (uint64_t id : blob_ids)
    if (!seen.insert(id).second) return fail(SB200_ERR_INVALID, "id %llu appears twice in the blob", (unsigned long long)id);
  std::vector<std::vector<uint64_t>> hists;   // quality store: every history non-empty and led by its track's id
  if (v.keep) {
    std::vector<int32_t> hl(live);
    if (live) CU(cudaMemcpy(hl.data(), at(sb::kFsSecHistLen), live * 4, cudaMemcpyDefault));
    uint64_t total = 0;
    for (uint64_t t = 0; t < live; ++t) {
      if (hl[t] < 1)
        return fail(SB200_ERR_INVALID, "track %llu has a merge history of length %d", (unsigned long long)blob_ids[t], hl[t]);
      total += (uint64_t)hl[t];
    }
    if (sec_bytes(sb::kFsSecHistory) != total * 8)
      return fail(SB200_ERR_INVALID, "section history holds %llu bytes, %llu expected (the sum of the history lengths)",
                  (unsigned long long)sec_bytes(sb::kFsSecHistory), (unsigned long long)(total * 8));
    // a state the rule produces: every list of every class from ring slot 0, and no longer than its capacity
    std::vector<int32_t> cn(live), sn(live);
    for (int k = 0; k < nc && live; ++k) {
      CU(cudaMemcpy(cn.data(), at(sb::kFsSecCnt, k), live * 4, cudaMemcpyDefault));
      CU(cudaMemcpy(sn.data(), at(sb::kFsSecStart, k), live * 4, cudaMemcpyDefault));
      for (uint64_t t = 0; t < live; ++t) {
        if (sn[t] != 0)
          return fail(SB200_ERR_INVALID, "track %llu has ring start %d; a quality store's lists start at slot 0",
                      (unsigned long long)blob_ids[t], sn[t]);
        const int c = tab[std::min<size_t>((size_t)hl[t], tab.size() - 1)];
        if (cn[t] > c)
          return fail(SB200_ERR_INVALID, "track %llu holds %d observations, above its capacity %d at history length %d",
                      (unsigned long long)blob_ids[t], cn[t], c, hl[t]);
      }
    }
    std::vector<uint64_t> hc(total);
    if (total) CU(cudaMemcpy(hc.data(), at(sb::kFsSecHistory), total * 8, cudaMemcpyDefault));
    hists.resize(live);
    for (uint64_t t = 0, a = 0; t < live; a += (uint64_t)hl[t], ++t) {
      hists[t].assign(hc.begin() + a, hc.begin() + a + hl[t]);
      if (hists[t][0] != blob_ids[t])
        return fail(SB200_ERR_INVALID, "the merge history of track %llu starts with %llu, not with its id",
                    (unsigned long long)blob_ids[t], (unsigned long long)hists[t][0]);
    }
  } else if (v.version == SB200_FSTORE_BLOB_VERSION_CLASSES && sec_bytes(sb::kFsSecHistory) != 0) {
    return fail(SB200_ERR_INVALID, "a newest store's blob with a history section");
  }
  sb200_fstore* s = nullptr;
  if (int rc = sb200_fstore_create(&o, &s)) return rc;
  // the fresh store holds the single class 0 of feature_dim, which versions 1 to 3 declare
  int rc = v.version == SB200_FSTORE_BLOB_VERSION_CLASSES ? s->set_classes(nc, cid.data(), cdim.data()) : 0;
  if (!rc) rc = s->load(h, v, plan, buf, std::move(blob_ids), std::move(hists));
  if (rc) {
    sb200_fstore_destroy(s);   // the handle owns every buffer made so far
    return rc;
  }
  *out = s;
  return 0;
}

extern "C" {

int sb200_fstore_create(const sb200_fstore_options* opts, sb200_fstore** out) {
  if (!opts || !out) return fail(SB200_ERR_INVALID, "opts / out is NULL");
  *out = nullptr;
  if (int rc = sb::check_device(0)) return rc;   // no device at all; the index is checked after the options
  const sb200_fstore_options& o = *opts;
  if (int rc = check_options(o)) return rc;
  if (int rc = sb::check_device(o.device)) return rc;
  CU(cudaSetDevice(o.device));
  sb200_fstore* s = new sb200_fstore();
  s->o = o;
  s->d8 = (o.feature_dim + 7) / 8 * 8;
  s->cls.resize(1);
  s->cls[0].id = 0;
  s->cls[0].dim = o.feature_dim;
  s->cls[0].d8 = s->d8;
  cudaError_t e = cudaStreamCreateWithFlags(&s->st, cudaStreamNonBlocking);
  for (int i = 0; i < 4 && e == cudaSuccess; ++i) e = cudaEventCreate(&s->ev[i]);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&s->ev_in, cudaEventDisableTiming);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&s->num_sms, cudaDevAttrMultiProcessorCount, o.device);
  if (e != cudaSuccess) {
    delete s;
    return fail(SB200_ERR_CUDA, "stream / event creation failed: %s", cudaGetErrorString(e));
  }
  *out = s;
  return 0;
}

void sb200_fstore_destroy(sb200_fstore* s) {
  if (!s) return;
  cudaSetDevice(s->o.device);
  delete s;
}

int sb200_fstore_add(sb200_fstore* s, int32_t n, const uint64_t* ids, const float* features) {
  if (!s) return no_handle();
  if (int rc = s->refuse_gated()) return rc;
  if (int rc = s->refuse_quality()) return rc;
  return s->add(n, ids, {features, false, nullptr});
}

int sb200_fstore_search(sb200_fstore* s, int32_t n_queries, const uint64_t* query_ids, const int32_t* obs_offsets,
                        const float* features, int32_t* counts, uint64_t* winners, double* weights) {
  if (!s) return no_handle();
  if (int rc = s->refuse_gated()) return rc;
  if (int rc = s->refuse_quality()) return rc;
  return s->run_queries(n_queries, query_ids, obs_offsets, {features, false, nullptr}, counts, winners, weights, nullptr,
                        nullptr, false);
}

int sb200_fstore_associate(sb200_fstore* s, int32_t n_queries, const uint64_t* query_ids, const int32_t* obs_offsets,
                           const float* features, int32_t* counts, uint64_t* winners, double* weights,
                           uint64_t* track_ids, uint8_t* merged) {
  if (!s) return no_handle();
  if (int rc = s->refuse_gated()) return rc;
  if (int rc = s->refuse_quality()) return rc;
  return s->run_queries(n_queries, query_ids, obs_offsets, {features, false, nullptr}, counts, winners, weights, track_ids,
                        merged, true);
}

int64_t sb200_fstore_fetch(sb200_fstore* s, int32_t n, const uint64_t* ids, int32_t remove, int32_t* counts,
                           float* features) {
  if (!s) return no_handle();
  return s->fetch(n, ids, remove, counts, features);
}

int64_t sb200_fstore_size(sb200_fstore* s) {
  if (!s) return no_handle();
  return (int64_t)s->hid.size();
}

int64_t sb200_fstore_ids(sb200_fstore* s, int64_t cap, uint64_t* ids) {
  if (!s) return no_handle();
  if (cap < 0 || (cap > 0 && !ids)) return fail(SB200_ERR_INVALID, "bad cap / ids");
  const int64_t n = (int64_t)s->hid.size();
  std::copy(s->hid.begin(), s->hid.begin() + std::min(n, cap), ids);
  return n;
}

int sb200_fstore_last_stage_ms(sb200_fstore* s, float* out3) {
  if (!s) return no_handle();
  if (!out3) return fail(SB200_ERR_INVALID, "out3 is NULL");
  std::copy(s->stage_ms, s->stage_ms + 3, out3);
  return 0;
}

int sb200_fstore_set_feature_type(sb200_fstore* s, int32_t type) {
  if (!s) return no_handle();
  if (!known_type(type)) return fail(SB200_ERR_INVALID, "unknown feature type %d", type);
  s->ftype = type;
  return 0;
}

int sb200_fstore_set_storage_type(sb200_fstore* s, int32_t type) {
  if (!s) return no_handle();
  if (!known_type(type)) return fail(SB200_ERR_INVALID, "unknown storage type %d", type);
  if (!s->hid.empty())
    return fail(SB200_ERR_INVALID, "the storage type is fixed while the store holds tracks (%zu)", s->hid.size());
  s->stype = type;
  // no track is stored, so nothing moves: the capacity is what the allocated columns hold in rows of the new type, and
  // the next reserve allocates when it needs more
  s->cap = s->held();
  return 0;
}

int sb200_fstore_get_storage_type(sb200_fstore* s, int32_t* out) {
  if (!s) return no_handle();
  if (!out) return fail(SB200_ERR_INVALID, "out is NULL");
  *out = s->stype;
  return 0;
}

int sb200_fstore_get_options(sb200_fstore* s, sb200_fstore_options* out, int32_t* feature_type) {
  if (!s) return no_handle();
  if (out) *out = s->o;
  if (feature_type) *feature_type = s->ftype;
  return 0;
}

int sb200_fstore_add_device(sb200_fstore* s, int32_t n, const uint64_t* ids, const void* d_features, void* cuda_stream) {
  if (!s) return no_handle();
  if (int rc = s->refuse_gated()) return rc;
  if (int rc = s->refuse_quality()) return rc;
  return s->add(n, ids, {d_features, true, static_cast<cudaStream_t>(cuda_stream)});
}

int sb200_fstore_search_device(sb200_fstore* s, int32_t n_queries, const uint64_t* query_ids,
                               const int32_t* obs_offsets, const void* d_features, int32_t* counts, uint64_t* winners,
                               double* weights, void* cuda_stream) {
  if (!s) return no_handle();
  if (int rc = s->refuse_gated()) return rc;
  if (int rc = s->refuse_quality()) return rc;
  return s->run_queries(n_queries, query_ids, obs_offsets, {d_features, true, static_cast<cudaStream_t>(cuda_stream)},
                        counts, winners, weights, nullptr, nullptr, false);
}

int sb200_fstore_associate_device(sb200_fstore* s, int32_t n_queries, const uint64_t* query_ids,
                                  const int32_t* obs_offsets, const void* d_features, int32_t* counts,
                                  uint64_t* winners, double* weights, uint64_t* track_ids, uint8_t* merged,
                                  void* cuda_stream) {
  if (!s) return no_handle();
  if (int rc = s->refuse_gated()) return rc;
  if (int rc = s->refuse_quality()) return rc;
  return s->run_queries(n_queries, query_ids, obs_offsets, {d_features, true, static_cast<cudaStream_t>(cuda_stream)},
                        counts, winners, weights, track_ids, merged, true);
}

int sb200_fstore_set_gate(sb200_fstore* s, int32_t rule) {
  if (!s) return no_handle();
  return s->set_gate(rule);
}

int sb200_fstore_get_gate(sb200_fstore* s, int32_t* out) {
  if (!s) return no_handle();
  if (!out) return fail(SB200_ERR_INVALID, "out is NULL");
  *out = s->gate;
  return 0;
}

int sb200_fstore_set_voting(sb200_fstore* s, int32_t rule) {
  if (!s) return no_handle();
  if (rule != SB200_FSTORE_VOTING_TOPN && rule != SB200_FSTORE_VOTING_BEST_FIT)
    return fail(SB200_ERR_INVALID, "unknown voting rule %d", rule);
  s->voting = rule;
  return 0;
}

int sb200_fstore_get_voting(sb200_fstore* s, int32_t* out) {
  if (!s) return no_handle();
  if (!out) return fail(SB200_ERR_INVALID, "out is NULL");
  *out = s->voting;
  return 0;
}

// the feature column of an _attr call: exactly one of a host and a device pointer
static int attr_column(int n, const float* features, const void* d_features, void* cuda_stream, Column* col) {
  if (n > 0 && (features == nullptr) == (d_features == nullptr))
    return fail(SB200_ERR_INVALID, "exactly one of features and d_features must be non-NULL");
  *col = d_features ? Column{d_features, true, static_cast<cudaStream_t>(cuda_stream)} : Column{features, false, nullptr};
  return 0;
}

int sb200_fstore_add_attr(sb200_fstore* s, int32_t n, const uint64_t* ids, const sb200_fstore_attrs* attrs,
                          const float* features, const void* d_features, void* cuda_stream) {
  if (!s) return no_handle();
  if (int rc = s->refuse_quality()) return rc;
  if (int rc = s->check_attrs(n, attrs)) return rc;
  Column col;
  if (int rc = attr_column(n, features, d_features, cuda_stream, &col)) return rc;
  return s->add(n, ids, col, attrs);
}

int sb200_fstore_search_attr(sb200_fstore* s, int32_t n_queries, const uint64_t* query_ids, const int32_t* obs_offsets,
                             const sb200_fstore_attrs* attrs, const float* features, const void* d_features,
                             int32_t* counts, uint64_t* winners, double* weights, void* cuda_stream) {
  if (!s) return no_handle();
  if (int rc = s->refuse_quality()) return rc;
  if (int rc = s->check_attrs(n_queries, attrs)) return rc;
  Column col;
  if (int rc = attr_column(n_queries, features, d_features, cuda_stream, &col)) return rc;
  return s->run_queries(n_queries, query_ids, obs_offsets, col, counts, winners, weights, nullptr, nullptr, false, attrs);
}

int sb200_fstore_associate_attr(sb200_fstore* s, int32_t n_queries, const uint64_t* query_ids,
                                const int32_t* obs_offsets, const sb200_fstore_attrs* attrs, const float* features,
                                const void* d_features, int32_t* counts, uint64_t* winners, double* weights,
                                uint64_t* track_ids, uint8_t* merged, void* cuda_stream) {
  if (!s) return no_handle();
  if (int rc = s->refuse_quality()) return rc;
  if (int rc = s->check_attrs(n_queries, attrs)) return rc;
  Column col;
  if (int rc = attr_column(n_queries, features, d_features, cuda_stream, &col)) return rc;
  return s->run_queries(n_queries, query_ids, obs_offsets, col, counts, winners, weights, track_ids, merged, true, attrs);
}

int64_t sb200_fstore_fetch_attr(sb200_fstore* s, int32_t n, const uint64_t* ids, uint64_t* source, int64_t* t_start,
                                int64_t* t_end) {
  if (!s) return no_handle();
  return s->fetch_attr(n, ids, source, t_start, t_end);
}

int sb200_fstore_set_retention(sb200_fstore* s, int32_t rule, int32_t initial_capacity, float merge_extension) {
  if (!s) return no_handle();
  return s->set_retention(rule, initial_capacity, merge_extension);
}

int sb200_fstore_get_retention(sb200_fstore* s, int32_t* rule, int32_t* initial_capacity, float* merge_extension) {
  if (!s) return no_handle();
  if (rule) *rule = s->keep;
  if (initial_capacity) *initial_capacity = s->init_cap;
  if (merge_extension) *merge_extension = s->ext;
  return 0;
}

int sb200_fstore_add_quality(sb200_fstore* s, int32_t n, const uint64_t* ids, const float* quality,
                             const sb200_fstore_attrs* attrs, const float* features, const void* d_features,
                             void* cuda_stream) {
  if (!s) return no_handle();
  if (n < 0) return fail(SB200_ERR_INVALID, "n < 0");
  if (int rc = s->check_quality(n, quality, attrs)) return rc;
  if (s->gate)
    if (int rc = s->check_attrs(n, attrs)) return rc;
  Column col;
  if (int rc = attr_column(n, features, d_features, cuda_stream, &col)) return rc;
  return s->add(n, ids, col, s->gate ? attrs : nullptr, quality);
}

int sb200_fstore_search_quality(sb200_fstore* s, int32_t n_queries, const uint64_t* query_ids,
                                const int32_t* obs_offsets, const float* quality, const sb200_fstore_attrs* attrs,
                                const float* features, const void* d_features, int32_t* counts, uint64_t* winners,
                                double* weights, void* cuda_stream) {
  if (!s) return no_handle();
  if (int rc = s->check_quality(0, quality, attrs)) return rc;   // the rows' qualities: once the offsets are checked
  if (s->gate)
    if (int rc = s->check_attrs(n_queries, attrs)) return rc;
  Column col;
  if (int rc = attr_column(n_queries, features, d_features, cuda_stream, &col)) return rc;
  return s->run_queries(n_queries, query_ids, obs_offsets, col, counts, winners, weights, nullptr, nullptr, false,
                        s->gate ? attrs : nullptr, quality);
}

int sb200_fstore_associate_quality(sb200_fstore* s, int32_t n_queries, const uint64_t* query_ids,
                                   const int32_t* obs_offsets, const float* quality, const sb200_fstore_attrs* attrs,
                                   const float* features, const void* d_features, int32_t* counts, uint64_t* winners,
                                   double* weights, uint64_t* track_ids, uint8_t* merged, void* cuda_stream) {
  if (!s) return no_handle();
  if (int rc = s->check_quality(0, quality, attrs)) return rc;
  if (s->gate)
    if (int rc = s->check_attrs(n_queries, attrs)) return rc;
  Column col;
  if (int rc = attr_column(n_queries, features, d_features, cuda_stream, &col)) return rc;
  return s->run_queries(n_queries, query_ids, obs_offsets, col, counts, winners, weights, track_ids, merged, true,
                        s->gate ? attrs : nullptr, quality);
}

int64_t sb200_fstore_fetch_quality(sb200_fstore* s, int32_t n, const uint64_t* ids, int32_t remove, int32_t* counts,
                                   float* features, float* quality) {
  if (!s) return no_handle();
  if (n > 0 && !quality) return fail(SB200_ERR_INVALID, "quality is NULL");
  if (!s->keep) return fail(SB200_ERR_INVALID, "the store keeps no qualities (it keeps its newest observations)");
  return s->fetch(n, ids, remove, counts, features, quality);
}

int64_t sb200_fstore_merge_history(sb200_fstore* s, int32_t n, const uint64_t* ids, int32_t* lengths, int64_t cap,
                                   uint64_t* out) {
  if (!s) return no_handle();
  if (!s->keep) return fail(SB200_ERR_INVALID, "the store keeps no merge histories (it keeps its newest observations)");
  if (n < 0 || cap < 0) return fail(SB200_ERR_INVALID, "n < 0 or cap < 0");
  if ((n > 0 && (!ids || !lengths)) || (cap > 0 && !out)) return fail(SB200_ERR_INVALID, "ids / lengths / out is NULL");
  int64_t total = 0;
  for (int i = 0; i < n; ++i) {
    auto it = s->hpos.find(ids[i]);
    lengths[i] = 0;
    if (it == s->hpos.end()) continue;
    const std::vector<uint64_t>& h = s->hist[it->second];
    for (uint64_t v : h) {
      if (total < cap) out[total] = v;
      ++total;
    }
    lengths[i] = (int32_t)h.size();
  }
  return total;
}

int64_t sb200_fstore_find_baked(sb200_fstore* s, int64_t now, int64_t baked_period, int64_t cap, uint64_t* ids) {
  if (!s) return no_handle();
  return s->find_baked(now, baked_period, cap, ids);
}

int sb200_fstore_associate_store(sb200_fstore* dst, sb200_fstore* src, int32_t n, const uint64_t* ids, int32_t remove,
                                 int32_t* counts, uint64_t* winners, double* weights, uint64_t* track_ids,
                                 uint8_t* merged) {
  if (!dst || !src) return no_handle();
  return dst->associate_store(src, n, ids, remove, counts, winners, weights, track_ids, merged);
}

int sb200_fstore_search_owned(sb200_fstore* s, int32_t n, const uint64_t* ids, int32_t each, int32_t* counts,
                              uint64_t* winners, double* weights) {
  if (!s) return no_handle();
  return s->search_owned(n, ids, each, counts, winners, weights);
}

int sb200_fstore_merge_owned(sb200_fstore* s, int32_t n, const uint64_t* dest_ids, const uint64_t* src_ids,
                             int32_t remove_src) {
  if (!s) return no_handle();
  return s->merge_owned(n, dest_ids, src_ids, remove_src);
}

int sb200_fstore_set_classes(sb200_fstore* s, int32_t n, const uint64_t* class_ids, const int32_t* feature_dims) {
  if (!s) return no_handle();
  return s->set_classes(n, class_ids, feature_dims);
}

int32_t sb200_fstore_get_classes(sb200_fstore* s, int32_t cap, uint64_t* class_ids, int32_t* feature_dims) {
  if (!s) return no_handle();
  if (cap < 0 || (cap > 0 && (!class_ids || !feature_dims))) return fail(SB200_ERR_INVALID, "bad cap / outputs");
  for (int k = 0; k < std::min(cap, (int32_t)s->cls.size()); ++k) {
    class_ids[k] = s->cls[k].id;
    feature_dims[k] = s->cls[k].dim;
  }
  return (int32_t)s->cls.size();
}

int sb200_fstore_use_class(sb200_fstore* s, uint64_t class_id) {
  if (!s) return no_handle();
  return s->use_class(class_id);
}

int64_t sb200_fstore_class_counts(sb200_fstore* s, int32_t n, const uint64_t* ids, int32_t* counts) {
  if (!s) return no_handle();
  return s->class_counts(n, ids, counts);
}

int sb200_fstore_save(sb200_fstore* s, void* buf, uint64_t cap, uint64_t* bytes) {
  if (!s) return no_handle();
  if (!bytes) return fail(SB200_ERR_INVALID, "bytes is NULL");
  return s->save(buf, cap, bytes);
}

int sb200_fstore_load(const void* buf, uint64_t bytes, int32_t device, sb200_fstore** out) {
  if (!buf || !out) return fail(SB200_ERR_INVALID, "buf / out is NULL");
  *out = nullptr;
  if (int rc = sb::check_device(device)) return rc;
  CU(cudaSetDevice(device));
  return load_blob(buf, bytes, device, out);
}

}  // extern "C"

// =============================================================================================== sb200_fstore_associate_wasted
// The store's side of that call (sb_wstore.cuh); wasted_store.cu holds the call itself.
namespace sb {

void fstore_info(sb200_fstore* s, int* device, int* feature_dim, int* topn) {
  *device = s->o.device;
  *feature_dim = s->o.feature_dim;
  *topn = s->o.topn;
}

int fstore_gate(sb200_fstore* s) { return s->gate; }

int fstore_retention(sb200_fstore* s) { return s->keep; }

int fstore_associate_rows(sb200_fstore* s, int Q, const uint64_t* qids, const int32_t* offs, const FsRowSource& src,
                          int32_t* counts, uint64_t* winners, double* weights, uint64_t* track_ids, uint8_t* merged) {
  return s->associate_rows(Q, qids, offs, src, counts, winners, weights, track_ids, merged);
}

int fstore_check_attrs(sb200_fstore* s, int n, const sb200_fstore_attrs* attrs) { return s->check_attrs(n, attrs); }

int fstore_search_rows(sb200_fstore* s, int Q, const uint64_t* qids, const int32_t* offs, const float* quality,
                       const sb200_fstore_attrs* attrs, const FsRowSource& src, std::vector<int>* row_table,
                       int32_t* counts, uint64_t* winners, double* weights) {
  return s->search_rows(Q, qids, offs, quality, attrs, src, row_table, counts, winners, weights);
}

}  // namespace sb
