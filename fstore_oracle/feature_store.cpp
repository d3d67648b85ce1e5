// feature_store.cpp -- CPU ORACLE of the feature track store (sb200_fstore_*), TEST INFRASTRUCTURE ONLY.
//
// A restatement of the reference's TrackStore for the feature-only tracks of benches/feature_tracker.rs and of
// TopNVoting::winners (src/track/voting/topn.rs:74-138), built on the distance code of oracle/liboracle.so (the scalar /
// AVX2 restatement of src/distance.rs, reached through its orc_euclidean_blocks / orc_cosine_blocks hooks).  It defines
// the orders the reference leaves to its shards and HashMaps:
//   - store order = insertion order; removal is a stable compaction;
//   - entries are enumerated as (query, stored track in store order, query observation, track observation), oldest
//     observations first; a group's f64 weight is summed in that order;
//   - TopN ties (equal weights) go to the group that appeared first, i.e. the lower store position;
//   - BestFit (ofs_set_voting) orders the call's elements by weight descending, then query (call order), then store
//     position: the group's first appearance again.
// It is the parity reference of tests/test_gpu_feature_store.py and the timed CPU baseline of
// tools/feature_store_bench.py; the product never links it.
// Track attributes (gate != 0): each track carries the CamTrackingAttributes of examples/track_merging.rs:218-245, a
// source (camera) id and a [t_start, t_end] window.  compatible = the windows are disjoint (touching counts as disjoint)
// and, under gate 1, the sources are equal; merge = the hull of the windows.  An incompatible (query, track) pair gives no
// entries (Track::distances' error, src/track.rs:604-652).  Associate merges a query into its first winner only if it is
// compatible with the winner's window as extended by the queries merged into it earlier in the call, else the query
// becomes a new track; merge_owned refuses a call with an incompatible pair (checked in pair order) before anything
// changes.
// Retention (retention != 0): the rule of examples/track_merging.rs's `optimize` (:279-297) instead of the bench's newest
// K.  Each observation carries an f32 quality and each track a merge history (Track::get_merge_history), [id] when it is
// created, to which every merge appends the source's whole history (Track::merge with merge_history = true,
// src/track.rs:522-588).  After an observation is appended or a merge concatenates dest ++ src, the list is stably sorted
// by quality, descending, and truncated to c(h) = min(K, (u64)((float)initial_capacity * powf(merge_extension, (float)h)))
// with h the track's history length (:257-265).  Queries are fresh tracks (h = 1) built the same way, or, in
// ofs_associate_store, stored tracks of another store, which bring their lists and histories whole.
// Feature classes (ofs_set_classes): each track keeps its rows by class (Track::observations, a class -> rows map).  The
// rows of the selected class (ofs_use_class) are the track's obs / q, the others wait in its `cls` map; every call that
// takes rows works on the selected class, and a track without rows of it gives no entries (Track::distances'
// ObservationForClassNotFound).  A merge (Track::merge with classes = None) walks the classes the source holds in
// ascending id; on a quality store each class step appends the source's history before it optimizes that class.
#include <algorithm>
#include <map>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <functional>
#include <thread>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "../oracle/similari_oracle.h"

namespace {

struct Ent {
  uint64_t from, to;
  float d;   // NaN == None
};
struct Elt {
  uint64_t query, winner;
  double weight;
};
struct PairHash {
  size_t operator()(const std::pair<uint64_t, uint64_t>& p) const {
    return std::hash<uint64_t>()(p.first) * 0x9E3779B97F4A7C15ull ^ std::hash<uint64_t>()(p.second);
  }
};

// The groups of TopNVoting::winners and BestFitVoting::winners (topn.rs:78-117, best.rs:56-104 compute them alike): the
// groups that reach min_votes, in order of first appearance, with their f64 weights
std::vector<Elt> vote_groups(float max_distance, size_t min_votes, const std::vector<Ent>& ents) {
  float max_dist = -1.0f;
  std::vector<std::pair<std::pair<uint64_t, uint64_t>, std::vector<float>>> groups;
  std::unordered_map<std::pair<uint64_t, uint64_t>, size_t, PairHash> gidx;
  for (const Ent& e : ents) {
    if (std::isnan(e.d)) continue;   // feature_distance None
    if (max_dist < e.d) max_dist = e.d;
    if (!(e.d <= max_distance)) continue;
    const auto key = std::make_pair(e.from, e.to);
    auto it = gidx.find(key);
    if (it == gidx.end()) {
      gidx.emplace(key, groups.size());
      groups.push_back({key, {e.d}});
    } else {
      groups[it->second].second.push_back(e.d);
    }
  }
  std::vector<Elt> out;
  for (auto& g : groups) {
    if (g.second.size() < min_votes) continue;
    double weight = 0.0;
    for (float d : g.second) weight += (double)(max_dist - d);
    out.push_back({g.first.first, g.first.second, weight});
  }
  return out;
}

// the index of each element's query, queries numbered in order of first appearance (appended to *queries)
std::vector<size_t> query_index(const std::vector<Elt>& el, std::vector<uint64_t>* queries) {
  std::unordered_map<uint64_t, size_t> qidx;
  std::vector<size_t> at;
  for (const Elt& e : el) {
    auto it = qidx.find(e.query);
    if (it == qidx.end()) {
      it = qidx.emplace(e.query, queries->size()).first;
      queries->push_back(e.query);
    }
    at.push_back(it->second);
  }
  return at;
}

// TopNVoting::winners.  Returns, per query in order of first appearance, its at most `topn` elements, weight
// descending, equal weights in order of the group's first appearance.
std::vector<std::vector<Elt>> topn_voting(float max_distance, size_t min_votes, size_t topn, const std::vector<Ent>& ents,
                                          std::vector<uint64_t>* queries) {
  const std::vector<Elt> el = vote_groups(max_distance, min_votes, ents);
  const std::vector<size_t> at = query_index(el, queries);
  std::vector<std::vector<Elt>> res(queries->size());
  for (size_t i = 0; i < el.size(); ++i) res[at[i]].push_back(el[i]);
  for (auto& r : res) {
    std::stable_sort(r.begin(), r.end(), [](const Elt& a, const Elt& b) { return a.weight > b.weight; });
    if (r.size() > topn) r.resize(topn);
  }
  return res;
}

// BestFitVoting::winners (best.rs:52-128) on TopN's groups: every element of the call, weight descending, equal weights
// in order of the group's first appearance (in a store's enumeration: query, then store position), wins its track
// unless an earlier element took it; the winner of one that does not is its own query (best.rs:112-120).  The claims
// run over all elements; then, per query in order of first appearance, its first `topn` elements in that order.
std::vector<std::vector<Elt>> bestfit_voting(float max_distance, size_t min_votes, size_t topn,
                                             const std::vector<Ent>& ents, std::vector<uint64_t>* queries) {
  std::vector<Elt> el = vote_groups(max_distance, min_votes, ents);
  const std::vector<size_t> at = query_index(el, queries);
  std::vector<size_t> ord(el.size());
  for (size_t i = 0; i < ord.size(); ++i) ord[i] = i;
  std::stable_sort(ord.begin(), ord.end(), [&](size_t a, size_t b) { return el[a].weight > el[b].weight; });
  std::unordered_set<uint64_t> taken;
  std::vector<std::vector<Elt>> res(queries->size());
  for (size_t i : ord) {
    if (!taken.insert(el[i].winner).second) el[i].winner = el[i].query;
    if (res[at[i]].size() < topn) res[at[i]].push_back(el[i]);
  }
  return res;
}

void parallel_for(int n, int threads, const std::function<void(int, int)>& fn) {
  if (threads <= 1 || n <= 1) { fn(0, n); return; }
  threads = std::min(threads, n);
  std::vector<std::thread> th;
  const int chunk = (n + threads - 1) / threads;
  for (int t = 0; t < threads; ++t) {
    const int b = t * chunk, e = std::min(n, b + chunk);
    if (b >= e) break;
    th.emplace_back(fn, b, e);
  }
  for (auto& x : th) x.join();
}

struct Rows {
  std::vector<std::vector<float>> obs;
  std::vector<float> q;
};

struct Track {
  uint64_t id;
  std::map<uint64_t, Rows> cls;          // the rows of the classes other than the selected one
  std::vector<std::vector<float>> obs;   // zero-padded to d8, oldest first (a quality store: the track's order)
  uint64_t src = 0;                      // attributes of a gated store
  int64_t t0 = 0, t1 = 0;
  std::vector<float> q;                  // a quality store: the quality of each observation
  std::vector<uint64_t> hist;            // a quality store: the merge history
};

}  // namespace

struct ofs_store {
  int metric, K, D, d8, topn, min_votes;
  float filter, max_distance;
  int gate = 0;   // 0: no attributes; 1: windows disjoint and sources equal; 2: windows disjoint
  int retention = 0;   // 0: newest K; 1: best by quality, capacity growing with the merge history
  int voting = 0;      // 0: TopNVoting; 1: BestFitVoting
  int init_cap = 0;           // retention 1: its parameters
  float ext = 0.0f;
  std::vector<int> cap_tab;   // retention 1: c(h) for h = 0 .. the first h with c(h) == K (or h = 0 alone when constant)
  std::vector<Track> tracks;
  std::unordered_map<uint64_t, size_t> pos;
  std::vector<std::pair<uint64_t, int>> classes{{0, 0}};   // declared (id, dim); {0, feature_dim} by default
  uint64_t cur = 0;                                         // the selected class

  // the rows of class k of track t (the selected class's are t.obs / t.q)
  std::pair<std::vector<std::vector<float>>*, std::vector<float>*> rows(Track& t, uint64_t k) const {
    if (k == cur) return {&t.obs, &t.q};
    Rows& r = t.cls[k];
    return {&r.obs, &r.q};
  }

  // CamTrackingAttributes::compatible (examples/track_merging.rs:222-225); always true without a gate
  bool compatible(const Track& a, const Track& b) const {
    if (!gate) return true;
    return (a.t0 >= b.t1 || a.t1 <= b.t0) && (gate == 2 || a.src == b.src);
  }
  // CamTrackingAttributes::merge: the hull of the windows (the destination keeps its source)
  static void hull(Track& d, const Track& s) {
    d.t0 = std::min(d.t0, s.t0);
    d.t1 = std::max(d.t1, s.t1);
  }

  std::vector<float> pad(const float* v) const {
    std::vector<float> out((size_t)d8, 0.0f);
    std::memcpy(out.data(), v, sizeof(float) * (size_t)D);
    return out;
  }
  // optimize: keep the newest K in their original order (the bench's reverse / truncate(K) / reverse)
  void keep_newest(std::vector<std::vector<float>>& o) const {
    if ((int)o.size() > K) o.erase(o.begin(), o.end() - K);
  }
  // retention 1: c(h), from the table the first h with c(h) == K ends (a constant capacity has one entry)
  int capacity(size_t h) const { return cap_tab[std::min(h, cap_tab.size() - 1)]; }
  // retention 1: optimize, the stable sort by quality, descending (-0.0 == +0.0), then the truncation to c(h)
  void keep_best(std::vector<std::vector<float>>& to, std::vector<float>& tq, size_t h) const {
    std::vector<size_t> ix(to.size());
    for (size_t i = 0; i < ix.size(); ++i) ix[i] = i;
    std::stable_sort(ix.begin(), ix.end(), [&](size_t a, size_t b) { return tq[a] > tq[b]; });
    ix.resize(std::min(ix.size(), (size_t)capacity(h)));
    std::vector<std::vector<float>> obs;
    std::vector<float> q;
    for (size_t i : ix) { obs.push_back(std::move(to[i])); q.push_back(tq[i]); }
    to.swap(obs);
    tq.swap(q);
  }
  void keep_best(Track& t) const { keep_best(t.obs, t.q, t.hist.size()); }
  // Track::merge with classes = None: for each class src holds, in ascending id, dest's rows ++ src's, then (a quality
  // store) the history dest ++ src and optimize of that class at the new capacity; a newest store keeps the newest K
  void merge_into(Track& d, const Track& src_track) const {
    Track src = src_track;
    std::vector<uint64_t> ids;
    for (const auto& c : classes) ids.push_back(c.first);
    std::sort(ids.begin(), ids.end());
    for (uint64_t k : ids) {
      auto so = rows(src, k);
      if (so.first->empty()) continue;
      auto dr = rows(d, k);
      dr.first->insert(dr.first->end(), so.first->begin(), so.first->end());
      if (!retention) { keep_newest(*dr.first); continue; }
      dr.second->insert(dr.second->end(), so.second->begin(), so.second->end());
      d.hist.insert(d.hist.end(), src.hist.begin(), src.hist.end());
      keep_best(*dr.first, *dr.second, d.hist.size());
    }
  }
  // rows of every declared class of t, in declared order
  void class_counts(Track& t, int32_t* out) const {
    for (size_t k = 0; k < classes.size(); ++k) out[k] = (int32_t)rows(t, classes[k].first).first->size();
  }
  // add_observation + optimize of one row
  void append(Track& t, const float* feat, float quality) const {
    t.obs.push_back(pad(feat));
    if (!retention) { keep_newest(t.obs); return; }
    t.q.push_back(quality);
    keep_best(t);
  }
  Track fresh(uint64_t id) const {
    Track t;
    t.id = id;
    if (retention) t.hist.push_back(id);
    return t;
  }
  float metric_of(const float* a, const float* b) const {
    if (metric == 0) return orc_euclidean_blocks(a, b, d8 / 8);
    return 1.0f - orc_cosine_blocks(a, b, d8 / 8);
  }
  void reindex() {
    pos.clear();
    for (size_t i = 0; i < tracks.size(); ++i) pos[tracks[i].id] = i;
  }

  // TrackBuilder: each observation through add_observation (and optimize), so only the newest K remain (a quality
  // store: the best c(1), with the qualities `qual`, one per row)
  std::vector<Track> build_queries(int Q, const uint64_t* ids, const int32_t* offs, const float* feats,
                                   const uint64_t* src = nullptr, const int64_t* t0 = nullptr,
                                   const int64_t* t1 = nullptr, const float* qual = nullptr) const {
    std::vector<Track> qs((size_t)Q);
    for (int q = 0; q < Q; ++q) {
      qs[q] = fresh(ids[q]);
      if (src) { qs[q].src = src[q]; qs[q].t0 = t0[q]; qs[q].t1 = t1[q]; }
      for (int r = offs[q]; r < offs[q + 1]; ++r) append(qs[q], feats + (size_t)r * D, qual ? qual[r] : 0.0f);
    }
    return qs;
  }

  int check(int Q, const uint64_t* ids, const int32_t* offs, bool assoc) const {
    if (Q < 0) return -1;
    if (Q == 0) return 0;
    if (offs[0] != 0) return -1;
    std::unordered_set<uint64_t> seen;
    for (int q = 0; q < Q; ++q) {
      if (offs[q + 1] <= offs[q]) return -1;
      if (!seen.insert(ids[q]).second) return -1;
      if (assoc && pos.count(ids[q])) return -1;
    }
    return 0;
  }

  // foreign_track_distances + postprocess_distances (d < filter) + the voting `rule` (-1: the store's)
  std::vector<std::vector<Elt>> search(const std::vector<Track>& qs, int threads, int rule = -1) const {
    std::vector<std::vector<Ent>> per((size_t)qs.size());
    parallel_for((int)qs.size(), threads, [&](int b, int e) {
      for (int q = b; q < e; ++q)
        for (const Track& t : tracks) {
          if (t.id == qs[q].id) continue;   // src/track/store.rs:206
          if (!compatible(qs[q], t)) continue;   // Track::distances returns IncompatibleAttributes
          for (const auto& a : qs[q].obs)
            for (const auto& o : t.obs) {
              const float d = metric_of(a.data(), o.data());
              if (d < filter) per[q].push_back({qs[q].id, t.id, d});
            }
        }
    });
    std::vector<Ent> ents;
    for (auto& p : per) ents.insert(ents.end(), p.begin(), p.end());
    std::vector<uint64_t> order;
    auto groups = (rule < 0 ? voting : rule) == 1
                      ? bestfit_voting(max_distance, (size_t)std::max(min_votes, 0), (size_t)topn, ents, &order)
                      : topn_voting(max_distance, (size_t)std::max(min_votes, 0), (size_t)topn, ents, &order);
    std::unordered_map<uint64_t, size_t> at;
    for (size_t i = 0; i < order.size(); ++i) at[order[i]] = i;
    std::vector<std::vector<Elt>> out(qs.size());
    for (size_t q = 0; q < qs.size(); ++q) {
      auto it = at.find(qs[q].id);
      if (it != at.end()) out[q] = groups[it->second];
    }
    return out;
  }

  void write(const std::vector<std::vector<Elt>>& r, int32_t* counts, uint64_t* winners, double* weights) const {
    for (size_t q = 0; q < r.size(); ++q) {
      counts[q] = (int32_t)r[q].size();
      for (int e = 0; e < topn; ++e) {
        const bool ok = e < (int)r[q].size();
        winners[q * topn + e] = ok ? r[q][e].winner : 0;
        weights[q * topn + e] = ok ? r[q][e].weight : 0.0;
      }
    }
  }
};

extern "C" {

// The classes (n ids, each with its dim) of an empty store; the first is selected.  -1 for a bad n, a repeated id, a
// dim out of 1..8192 or a store that holds tracks.
int ofs_set_classes(ofs_store* s, int n, const uint64_t* ids, const int32_t* dims) {
  if (n < 1 || n > 16 || !s->tracks.empty()) return -1;
  for (int i = 0; i < n; ++i) {
    if (dims[i] < 1 || dims[i] > 8192) return -1;
    for (int j = 0; j < i; ++j)
      if (ids[j] == ids[i]) return -1;
  }
  s->classes.clear();
  for (int i = 0; i < n; ++i) s->classes.push_back({ids[i], dims[i]});
  s->cur = ids[0];
  s->D = dims[0];
  s->d8 = (dims[0] + 7) / 8 * 8;
  return 0;
}

// selects class `id` for the calls that take rows; -1 for an id the store does not declare
int ofs_use_class(ofs_store* s, uint64_t id) {
  int dim = 0;
  for (const auto& c : s->classes)
    if (c.first == id) dim = c.second;
  if (!dim) return -1;
  if (id == s->cur) return 0;
  for (Track& t : s->tracks) {
    Rows& old = t.cls[s->cur];
    old.obs.swap(t.obs);
    old.q.swap(t.q);
    if (old.obs.empty()) t.cls.erase(s->cur);
    auto it = t.cls.find(id);
    t.obs.clear();
    t.q.clear();
    if (it != t.cls.end()) {
      t.obs.swap(it->second.obs);
      t.q.swap(it->second.q);
      t.cls.erase(it);
    }
  }
  s->cur = id;
  s->D = dim;
  s->d8 = (dim + 7) / 8 * 8;
  return 0;
}

// counts[i][k]: the rows of track ids[i] in declared class k (0 when not stored); returns the ids found
int64_t ofs_class_counts(ofs_store* s, int n, const uint64_t* ids, int32_t* counts) {
  int64_t found = 0;
  const size_t nc = s->classes.size();
  for (int i = 0; i < n; ++i) {
    auto it = s->pos.find(ids[i]);
    std::fill(counts + (size_t)i * nc, counts + (size_t)(i + 1) * nc, 0);
    if (it == s->pos.end()) continue;
    s->class_counts(s->tracks[it->second], counts + (size_t)i * nc);
    ++found;
  }
  return found;
}

ofs_store* ofs_create(int metric, float distance_filter, int max_observations, int feature_dim, int topn,
                      float max_distance, int min_votes) {
  if ((metric != 0 && metric != 1) || max_observations < 1 || feature_dim < 1 || topn < 1) return nullptr;
  ofs_store* s = new ofs_store();
  s->metric = metric;
  s->filter = distance_filter;
  s->K = max_observations;
  s->D = feature_dim;
  s->d8 = (feature_dim + 7) / 8 * 8;
  s->classes = {{0, feature_dim}};
  s->topn = topn;
  s->max_distance = max_distance;
  s->min_votes = min_votes;
  return s;
}

void ofs_destroy(ofs_store* s) { delete s; }

// TrackStore::add, src/track/store.rs:530-568, in call order
int ofs_add(ofs_store* s, int n, const uint64_t* ids, const float* feats) {
  if (s->gate || s->retention) return -1;
  for (int i = 0; i < n; ++i) {
    auto it = s->pos.find(ids[i]);
    if (it == s->pos.end()) {
      s->pos[ids[i]] = s->tracks.size();
      Track t = s->fresh(ids[i]);
      t.obs.push_back(s->pad(feats + (size_t)i * s->D));
      s->tracks.push_back(std::move(t));
    } else {
      auto& o = s->tracks[it->second].obs;
      o.push_back(s->pad(feats + (size_t)i * s->D));
      s->keep_newest(o);
    }
  }
  return 0;
}

int ofs_search(ofs_store* s, int Q, const uint64_t* ids, const int32_t* offs, const float* feats, int32_t* counts,
               uint64_t* winners, double* weights, int threads) {
  if (s->gate || s->retention || s->check(Q, ids, offs, false)) return -1;
  if (Q == 0) return 0;
  s->write(s->search(s->build_queries(Q, ids, offs, feats), threads), counts, winners, weights);
  return 0;
}

// one iteration of benches/feature_tracker.rs: search, then merge_external into results[0].winner_track or add_track
// (the queries qs: fresh tracks built from a request, or stored tracks of another store, ofs_associate_store); a first
// winner equal to the query's own id (BestFit: another query took the track) means add_track, as
// examples/middleware_sort_tracker.rs:76-81 reads it
static void associate_tracks(ofs_store* s, const std::vector<Track>& qs, int32_t* counts, uint64_t* winners,
                             double* weights, uint64_t* track_ids, uint8_t* merged, int threads) {
  const int Q = (int)qs.size();
  const auto r = s->search(qs, threads);
  s->write(r, counts, winners, weights);
  for (int q = 0; q < Q; ++q) {
    // with a gate, the window of the first winner as the queries merged into it earlier in this call extended it
    if (!r[q].empty() && r[q][0].winner != qs[q].id &&
        s->compatible(qs[q], s->tracks[s->pos.at(r[q][0].winner)])) {
      // Track::merge (src/track.rs:522-600): extend, then optimize keeps the newest K
      Track& dt = s->tracks[s->pos.at(r[q][0].winner)];
      s->merge_into(dt, qs[q]);
      if (s->gate) ofs_store::hull(dt, qs[q]);
      track_ids[q] = r[q][0].winner;
      merged[q] = 1;
    } else {
      s->pos[qs[q].id] = s->tracks.size();
      s->tracks.push_back(qs[q]);
      track_ids[q] = qs[q].id;
      merged[q] = 0;
    }
  }
}

static int associate(ofs_store* s, int Q, const uint64_t* ids, const int32_t* offs, const float* feats,
                     const uint64_t* src, const int64_t* t0, const int64_t* t1, int32_t* counts, uint64_t* winners,
                     double* weights, uint64_t* track_ids, uint8_t* merged, int threads, const float* qual = nullptr) {
  if (s->check(Q, ids, offs, true)) return -1;
  if (Q == 0) return 0;
  associate_tracks(s, s->build_queries(Q, ids, offs, feats, src, t0, t1, qual), counts, winners, weights, track_ids,
                   merged, threads);
  return 0;
}

int ofs_associate(ofs_store* s, int Q, const uint64_t* ids, const int32_t* offs, const float* feats, int32_t* counts,
                  uint64_t* winners, double* weights, uint64_t* track_ids, uint8_t* merged, int threads) {
  if (s->gate || s->retention) return -1;
  return associate(s, Q, ids, offs, feats, nullptr, nullptr, nullptr, counts, winners, weights, track_ids, merged,
                   threads);
}

// fetch_tracks (src/track/store.rs:388-401) when remove != 0, else a read-only lookup; features [n][K][D]
int64_t ofs_fetch(ofs_store* s, int n, const uint64_t* ids, int remove, int32_t* counts, float* feats) {
  int64_t found = 0;
  std::memset(feats, 0, sizeof(float) * (size_t)n * s->K * s->D);
  for (int i = 0; i < n; ++i) {
    counts[i] = 0;
    auto it = s->pos.find(ids[i]);
    if (it == s->pos.end()) continue;
    const Track& t = s->tracks[it->second];
    counts[i] = (int32_t)t.obs.size();
    for (size_t b = 0; b < t.obs.size(); ++b)
      std::memcpy(feats + ((size_t)i * s->K + b) * s->D, t.obs[b].data(), sizeof(float) * (size_t)s->D);
    ++found;
    if (remove) {
      s->tracks.erase(s->tracks.begin() + (std::ptrdiff_t)it->second);
      s->reindex();
    }
  }
  return found;
}

// owned_track_distances (src/track/store.rs:471-486) + the store's voting, written literally: fetch_tracks the queried
// set out of the store, search the remainder with the fetched tracks as queries, put the tracks back (at their store
// positions: the order rule that replaces the reference's HashMap).  each != 0: once per id, in order.  An id that is not
// stored gets count 0; an id twice is rejected (-1).
int ofs_search_owned(ofs_store* s, int n, const uint64_t* ids, int each, int32_t* counts, uint64_t* winners,
                     double* weights, int threads) {
  if (n < 0) return -1;
  std::unordered_set<uint64_t> seen;
  for (int q = 0; q < n; ++q)
    if (!seen.insert(ids[q]).second) return -1;
  auto owned = [&](int a, int b, int rule) {   // one owned_track_distances(ids[a .. b)) call
    const std::vector<Track> saved = s->tracks;
    std::vector<Track> qs;
    for (int q = a; q < b; ++q) {   // fetch_tracks
      auto it = std::find_if(s->tracks.begin(), s->tracks.end(), [&](const Track& t) { return t.id == ids[q]; });
      if (it == s->tracks.end()) continue;
      qs.push_back(*it);
      s->tracks.erase(it);
    }
    s->reindex();
    const auto r = s->search(qs, threads, rule);
    s->tracks = saved;   // add_track of every fetched track
    s->reindex();
    for (int q = a; q < b; ++q) {
      std::vector<Elt> none;
      const std::vector<Elt>* res = &none;
      for (size_t i = 0; i < qs.size(); ++i)
        if (qs[i].id == ids[q]) res = &r[i];
      counts[q] = (int32_t)res->size();
      for (int e = 0; e < s->topn; ++e) {
        const bool ok = e < (int)res->size();
        winners[(size_t)q * s->topn + e] = ok ? (*res)[e].winner : 0;
        weights[(size_t)q * s->topn + e] = ok ? (*res)[e].weight : 0.0;
      }
    }
  };
  if (each) {   // one voting call per query: BestFit has no other query to lose a track to, and is TopN
    for (int q = 0; q < n; ++q) owned(q, q + 1, 0);
  } else if (n > 0) {
    owned(0, n, -1);
  }
  return 0;
}

// merge_owned(dest, src, None, remove_src, false) (src/track/store.rs:584-611) for each pair in order: fetch src, extend
// dest by its observations and keep the newest K (Track::merge + optimize; a quality store: merge_history = true and the
// best c(h)), then put src back at its position or drop it.  Rejected (-1) before anything changes: dest == src, a dest or src that is not stored, and with remove_src a pair
// naming a track an earlier pair removed.
int ofs_merge_owned(ofs_store* s, int n, const uint64_t* dest, const uint64_t* src, int remove_src) {
  if (n < 0) return -1;
  std::unordered_set<uint64_t> removed;
  for (int i = 0; i < n; ++i) {
    if (dest[i] == src[i] || !s->pos.count(dest[i]) || !s->pos.count(src[i])) return -1;
    if (removed.count(dest[i]) || removed.count(src[i])) return -1;
    if (remove_src) removed.insert(src[i]);
  }
  const std::vector<Track> saved = s->tracks;   // a pair found incompatible refuses the whole call
  for (int i = 0; i < n; ++i) {
    const size_t at = s->pos.at(src[i]);
    const Track t = s->tracks[at];   // fetch_tracks([src])
    s->tracks.erase(s->tracks.begin() + (std::ptrdiff_t)at);
    s->reindex();
    Track& dt = s->tracks[s->pos.at(dest[i])];   // merge_external -> Track::merge
    if (!s->compatible(dt, t)) {
      s->tracks = saved;
      s->reindex();
      return -1;
    }
    if (s->gate) ofs_store::hull(dt, t);
    s->merge_into(dt, t);
    if (!remove_src) s->tracks.insert(s->tracks.begin() + (std::ptrdiff_t)at, t);   // add_track
    s->reindex();
  }
  return 0;
}

// ---- track attributes (gate != 0)
// The rule may change only while the store holds no tracks.
int ofs_set_gate(ofs_store* s, int rule) {
  if (rule < 0 || rule > 2 || !s->tracks.empty()) return -1;
  s->gate = rule;
  return 0;
}

static bool bad_windows(int n, const int64_t* t0, const int64_t* t1) {
  for (int i = 0; i < n; ++i)
    if (t0[i] > t1[i]) return true;
  return false;
}

// TrackStore::add with attributes: an unknown id creates a track with the row's triple, a known id takes the hull of
// the windows; a source that differs from the track's is refused (the reference's WrongCamID) before anything changes.
int ofs_add_attr(ofs_store* s, int n, const uint64_t* ids, const uint64_t* src, const int64_t* t0, const int64_t* t1,
                 const float* feats) {
  if (!s->gate || s->retention || n < 0 || bad_windows(n, t0, t1)) return -1;
  std::unordered_map<uint64_t, uint64_t> source;
  for (const Track& t : s->tracks) source[t.id] = t.src;
  for (int i = 0; i < n; ++i) {
    auto it = source.emplace(ids[i], src[i]).first;
    if (it->second != src[i]) return -1;
  }
  for (int i = 0; i < n; ++i) {
    auto it = s->pos.find(ids[i]);
    if (it == s->pos.end()) {
      s->pos[ids[i]] = s->tracks.size();
      Track t = s->fresh(ids[i]);
      t.obs.push_back(s->pad(feats + (size_t)i * s->D));
      t.src = src[i]; t.t0 = t0[i]; t.t1 = t1[i];
      s->tracks.push_back(std::move(t));
    } else {
      Track& t = s->tracks[it->second];
      t.obs.push_back(s->pad(feats + (size_t)i * s->D));
      s->keep_newest(t.obs);
      t.t0 = std::min(t.t0, t0[i]);
      t.t1 = std::max(t.t1, t1[i]);
    }
  }
  return 0;
}

int ofs_search_attr(ofs_store* s, int Q, const uint64_t* ids, const int32_t* offs, const uint64_t* src, const int64_t* t0,
                    const int64_t* t1, const float* feats, int32_t* counts, uint64_t* winners, double* weights,
                    int threads) {
  if (!s->gate || s->retention || s->check(Q, ids, offs, false) || bad_windows(Q, t0, t1)) return -1;
  if (Q == 0) return 0;
  s->write(s->search(s->build_queries(Q, ids, offs, feats, src, t0, t1), threads), counts, winners, weights);
  return 0;
}

int ofs_associate_attr(ofs_store* s, int Q, const uint64_t* ids, const int32_t* offs, const uint64_t* src,
                       const int64_t* t0, const int64_t* t1, const float* feats, int32_t* counts, uint64_t* winners,
                       double* weights, uint64_t* track_ids, uint8_t* merged, int threads) {
  if (!s->gate || s->retention || bad_windows(Q, t0, t1)) return -1;
  return associate(s, Q, ids, offs, feats, src, t0, t1, counts, winners, weights, track_ids, merged, threads);
}

// the triples of the tracks `ids` (0 for an id that is not stored); returns how many were found
int64_t ofs_fetch_attr(ofs_store* s, int n, const uint64_t* ids, uint64_t* src, int64_t* t0, int64_t* t1) {
  if (!s->gate) return -1;
  int64_t found = 0;
  for (int i = 0; i < n; ++i) {
    auto it = s->pos.find(ids[i]);
    const bool ok = it != s->pos.end();
    src[i] = ok ? s->tracks[it->second].src : 0;
    t0[i] = ok ? s->tracks[it->second].t0 : 0;
    t1[i] = ok ? s->tracks[it->second].t1 : 0;
    found += ok;
  }
  return found;
}

// ---- retention by quality (retention != 0)
// Sets the rule and its parameters while the store holds no tracks.  Refused (-1): an unknown rule, initial_capacity < 1,
// a merge_extension that is not finite or is below 1, and parameters whose capacity has not reached K by h = 65536
// unless merge_extension == 1.
int ofs_set_retention(ofs_store* s, int rule, int initial_capacity, float merge_extension) {
  if ((rule != 0 && rule != 1) || !s->tracks.empty()) return -1;
  if (rule == 0) {
    s->retention = 0;
    s->cap_tab.clear();
    return 0;
  }
  if (initial_capacity < 1 || !std::isfinite(merge_extension) || merge_extension < 1.0f) return -1;
  auto c = [&](int h) {   // f32 arithmetic, then Rust's saturating `as u64`, then min(K, .)
    const float v = (float)initial_capacity * powf(merge_extension, (float)h);
    return v >= (float)s->K ? s->K : (int)(uint64_t)v;
  };
  std::vector<int> tab{c(0)};
  while (tab.back() < s->K && merge_extension != 1.0f) {
    if (tab.size() > 65536) return -1;
    tab.push_back(c((int)tab.size()));
  }
  s->retention = 1;
  s->init_cap = initial_capacity;
  s->ext = merge_extension;
  s->cap_tab = tab;
  return 0;
}

static bool bad_quality(int n, const float* q) {
  for (int i = 0; i < n; ++i)
    if (std::isnan(q[i])) return true;
  return false;
}

// TrackStore::add of a quality store: an unknown id creates a track with history [id]; each row is appended and the
// track optimized at its capacity.  src == nullptr: an ungated store.
int ofs_add_quality(ofs_store* s, int n, const uint64_t* ids, const float* qual, const uint64_t* src, const int64_t* t0,
                    const int64_t* t1, const float* feats) {
  if (!s->retention || (s->gate != 0) != (src != nullptr) || n < 0 || bad_quality(n, qual)) return -1;
  if (src) {
    if (bad_windows(n, t0, t1)) return -1;
    std::unordered_map<uint64_t, uint64_t> source;
    for (const Track& t : s->tracks) source[t.id] = t.src;
    for (int i = 0; i < n; ++i)
      if (source.emplace(ids[i], src[i]).first->second != src[i]) return -1;
  }
  for (int i = 0; i < n; ++i) {
    auto it = s->pos.find(ids[i]);
    if (it == s->pos.end()) {
      Track t = s->fresh(ids[i]);
      if (src) { t.src = src[i]; t.t0 = t0[i]; t.t1 = t1[i]; }
      s->pos[ids[i]] = s->tracks.size();
      s->tracks.push_back(std::move(t));
      it = s->pos.find(ids[i]);
      s->tracks[it->second].obs.push_back(s->pad(feats + (size_t)i * s->D));
      s->tracks[it->second].q.push_back(qual[i]);
    } else {
      Track& t = s->tracks[it->second];
      s->append(t, feats + (size_t)i * s->D, qual[i]);
      if (src) { t.t0 = std::min(t.t0, t0[i]); t.t1 = std::max(t.t1, t1[i]); }
    }
  }
  return 0;
}

int ofs_search_quality(ofs_store* s, int Q, const uint64_t* ids, const int32_t* offs, const float* qual,
                       const uint64_t* src, const int64_t* t0, const int64_t* t1, const float* feats, int32_t* counts,
                       uint64_t* winners, double* weights, int threads) {
  if (!s->retention || (s->gate != 0) != (src != nullptr) || s->check(Q, ids, offs, false)) return -1;
  if (Q == 0) return 0;
  if (bad_quality(offs[Q], qual) || (src && bad_windows(Q, t0, t1))) return -1;
  s->write(s->search(s->build_queries(Q, ids, offs, feats, src, t0, t1, qual), threads), counts, winners, weights);
  return 0;
}

int ofs_associate_quality(ofs_store* s, int Q, const uint64_t* ids, const int32_t* offs, const float* qual,
                          const uint64_t* src, const int64_t* t0, const int64_t* t1, const float* feats,
                          int32_t* counts, uint64_t* winners, double* weights, uint64_t* track_ids, uint8_t* merged,
                          int threads) {
  if (!s->retention || (s->gate != 0) != (src != nullptr) || s->check(Q, ids, offs, true)) return -1;
  if (Q == 0) return 0;
  if (bad_quality(offs[Q], qual) || (src && bad_windows(Q, t0, t1))) return -1;
  return associate(s, Q, ids, offs, feats, src, t0, t1, counts, winners, weights, track_ids, merged, threads, qual);
}

// ofs_fetch plus the qualities [n][K] of the rows returned (0 past a count: an id that is not stored, or that an
// earlier entry of the same call removed, returns none)
int64_t ofs_fetch_quality(ofs_store* s, int n, const uint64_t* ids, int remove, int32_t* counts, float* feats,
                          float* qual) {
  if (!s->retention) return -1;
  std::memset(qual, 0, sizeof(float) * (size_t)n * s->K);
  std::unordered_set<uint64_t> gone;
  for (int i = 0; i < n; ++i) {
    auto it = s->pos.find(ids[i]);
    if (it == s->pos.end() || gone.count(ids[i])) continue;
    const Track& t = s->tracks[it->second];
    std::copy(t.q.begin(), t.q.end(), qual + (size_t)i * s->K);
    if (remove) gone.insert(ids[i]);
  }
  return ofs_fetch(s, n, ids, remove, counts, feats);
}

// Track::get_merge_history of the tracks `ids` in CSR form: lengths[i] (0: not stored), the histories concatenated into
// out (at most cap entries written); returns the total length
int64_t ofs_merge_history(ofs_store* s, int n, const uint64_t* ids, int32_t* lengths, int64_t cap, uint64_t* out) {
  if (!s->retention) return -1;
  int64_t total = 0;
  for (int i = 0; i < n; ++i) {
    auto it = s->pos.find(ids[i]);
    lengths[i] = 0;
    if (it == s->pos.end()) continue;
    for (uint64_t h : s->tracks[it->second].hist) {
      if (total < cap) out[total] = h;
      ++total;
    }
    lengths[i] = (int32_t)s->tracks[it->second].hist.size();
  }
  return total;
}

// ---- store to store (examples/track_merging.rs:371-481)
// TrackStore::find_usable with `baked` (:240-247): the ids of the tracks with now > t_end + baked_period, in store order,
// compared in 128-bit integers as the reference compares in u128.  The first min(cap, total) are written; returns the
// total, or -1 for an ungated store or cap < 0.
int64_t ofs_find_baked(ofs_store* s, int64_t now, int64_t baked_period, int64_t cap, uint64_t* ids) {
  if (!s->gate || cap < 0) return -1;
  int64_t total = 0;
  for (const Track& t : s->tracks)
    if ((__int128)now > (__int128)t.t1 + (__int128)baked_period) {
      if (total < cap) ids[total] = t.id;
      ++total;
    }
  return total;
}

// fetch_tracks(ids) of src, each track whole (its list, qualities, triple and merge history), then one associate of dst
// with those tracks as its queries in the order of ids: merge_external(winner, &track, .., true) merges the lists and
// appends the history (h + h_q), add_track keeps the track whole; then, with remove, the tracks leave src (a stable
// compaction).  Refused (-1) before either store changes: dst == src, a different feature_dim, max_observations, gate,
// retention or retention parameters, n < 0, remove not 0 / 1, an id twice, not stored in src, or stored in dst.
int ofs_associate_store(ofs_store* d, ofs_store* s, int n, const uint64_t* ids, int remove, int32_t* counts,
                        uint64_t* winners, double* weights, uint64_t* track_ids, uint8_t* merged, int threads) {
  auto sorted = [](std::vector<std::pair<uint64_t, int>> c) { std::sort(c.begin(), c.end()); return c; };
  if (d == s || sorted(d->classes) != sorted(s->classes) || d->cur != s->cur || d->K != s->K || d->gate != s->gate ||
      d->retention != s->retention)
    return -1;
  if (d->retention && (d->init_cap != s->init_cap || d->ext != s->ext)) return -1;
  if (n < 0 || (remove != 0 && remove != 1)) return -1;
  std::unordered_set<uint64_t> seen;
  for (int i = 0; i < n; ++i)
    if (!seen.insert(ids[i]).second || !s->pos.count(ids[i]) || d->pos.count(ids[i])) return -1;
  if (n == 0) return 0;
  std::vector<Track> qs;
  for (int i = 0; i < n; ++i) qs.push_back(s->tracks[s->pos.at(ids[i])]);
  associate_tracks(d, qs, counts, winners, weights, track_ids, merged, threads);
  if (remove) {
    std::vector<Track> kept;
    for (Track& t : s->tracks)
      if (!seen.count(t.id)) kept.push_back(std::move(t));
    s->tracks.swap(kept);
    s->reindex();
  }
  return 0;
}

// ---- voting (0: TopNVoting, 1: BestFitVoting): how search, associate, search_owned and associate_store vote; it may
// change at any time.  -1 for an unknown rule.
int ofs_set_voting(ofs_store* s, int rule) {
  if (rule != 0 && rule != 1) return -1;
  s->voting = rule;
  return 0;
}

int64_t ofs_size(ofs_store* s) { return (int64_t)s->tracks.size(); }

int64_t ofs_ids(ofs_store* s, int64_t cap, uint64_t* ids) {
  for (int64_t i = 0; i < std::min<int64_t>(cap, (int64_t)s->tracks.size()); ++i) ids[i] = s->tracks[i].id;
  return (int64_t)s->tracks.size();
}

static int write_voting(const std::vector<std::vector<Elt>>& groups, uint64_t* out_query, uint64_t* out_winner,
                        double* out_weight) {
  int n = 0;
  for (const auto& g : groups)
    for (const Elt& e : g) {
      out_query[n] = e.query;
      out_winner[n] = e.winner;
      out_weight[n] = e.weight;
      ++n;
    }
  return n;
}

// TopNVoting::winners on an entry list (feat NaN == None).  Writes n results (query, winner, weight): queries in order
// of first appearance, each query's results weight descending, equal weights in order of first appearance.
int ofs_topn_voting(float max_distance, int min_votes, int topn, int n_ent, const uint64_t* from, const uint64_t* to,
                    const float* feat, uint64_t* out_query, uint64_t* out_winner, double* out_weight) {
  std::vector<Ent> ents((size_t)n_ent);
  for (int i = 0; i < n_ent; ++i) ents[i] = {from[i], to[i], feat[i]};
  std::vector<uint64_t> order;
  return write_voting(topn_voting(max_distance, (size_t)std::max(min_votes, 0), (size_t)topn, ents, &order), out_query,
                      out_winner, out_weight);
}

// BestFitVoting::winners on an entry list, as bestfit_voting above (claims over every element, each query's list cut at
// topn); results written as ofs_topn_voting writes them.
int ofs_bestfit_voting(float max_distance, int min_votes, int topn, int n_ent, const uint64_t* from, const uint64_t* to,
                       const float* feat, uint64_t* out_query, uint64_t* out_winner, double* out_weight) {
  std::vector<Ent> ents((size_t)n_ent);
  for (int i = 0; i < n_ent; ++i) ents[i] = {from[i], to[i], feat[i]};
  std::vector<uint64_t> order;
  return write_voting(bestfit_voting(max_distance, (size_t)std::max(min_votes, 0), (size_t)topn, ents, &order),
                      out_query, out_winner, out_weight);
}

}  // extern "C"
