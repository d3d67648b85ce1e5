// fstore.cu -- host side of the feature track store (sb200_fstore_*): argument checks, device memory, the launch
// sequence of a call (distances -> TopN -> apply, kernels_fstore.cu) and the host copy of the store's id order.
// A call stages its request in one pinned buffer, uploads it once, runs its kernels back to back on the handle's stream
// and downloads its results once.  Everything a call can reject is checked before anything is launched or changed.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "../../include/similari_b200.h"
#include "sb_fstore.cuh"
#include "sb_host.cuh"

namespace {

using sb::DBuf;
using sb::fail;

size_t align16(size_t v) { return (v + 15) & ~size_t(15); }

// byte offsets of one request in the staging buffer (the device copy has the same layout)
struct ReqLayout {
  size_t rows, qid, qoff, row_q, dest, maxkey, total;
  ReqLayout(int Q, int R, int d8) {
    size_t o = 0;
    rows = o; o = align16(o + (size_t)R * d8 * 4);
    qid = o; o = align16(o + (size_t)Q * 8);
    qoff = o; o = align16(o + (size_t)(Q + 1) * 4);
    row_q = o; o = align16(o + (size_t)R * 4);
    dest = o; o = align16(o + (size_t)Q * 4);
    maxkey = o; o = align16(o + 4);
    total = o;
  }
};
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

}  // namespace

struct sb200_fstore {
  sb200_fstore_options o{};
  int d8 = 8;
  cudaStream_t st = nullptr;
  cudaEvent_t ev[4] = {};
  float stage_ms[3] = {0, 0, 0};
  // store columns
  size_t cap = 0;
  DBuf feat, cnt, start, ids, run;
  std::vector<uint64_t> hid;                 // ids in store order
  std::unordered_map<uint64_t, int> hpos;    // id -> store position
  // per-call buffers
  DBuf dreq, dres, plan, qnorm, snorm, dist, gpos, gout;
  sb::PinnedBuf<cudaHostAllocDefault> hreq, hres;   // staging, contents not kept

  ~sb200_fstore() {
    if (st) cudaStreamSynchronize(st);
    for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e);
    if (st) cudaStreamDestroy(st);
  }

  sb::FsStore view() const {
    sb::FsStore s;
    s.feat = feat.as<float>();
    s.cnt = cnt.as<int>();
    s.start = start.as<int>();
    s.ids = ids.as<unsigned long long>();
    s.run = run.as<int>();
    s.K = o.max_observations;
    s.d8 = d8;
    s.live = (int)hid.size();
    return s;
  }

  // fresh columns for `n` tracks; the caller copies what it keeps
  int alloc_columns(size_t n, DBuf* f, DBuf* c, DBuf* s, DBuf* i, DBuf* r) {
    n = std::max<size_t>(n, 1);
    if (int rc = f->ensure(n * o.max_observations * d8 * 4)) return rc;
    if (int rc = c->ensure(n * 4)) return rc;
    if (int rc = s->ensure(n * 4)) return rc;
    if (int rc = i->ensure(n * 8)) return rc;
    if (int rc = r->ensure(n * 4)) return rc;
    CU(cudaMemsetAsync(r->p, 0, n * 4, st));
    return 0;
  }

  // capacity for `need` tracks: grows by at least 1.5x, keeping the live tracks
  int reserve(size_t need) {
    if (need <= cap) return 0;
    const size_t nc = std::max(need, cap + cap / 2);
    DBuf f, c, s, i, r;
    if (int rc = alloc_columns(nc, &f, &c, &s, &i, &r)) return rc;
    const size_t live = hid.size();
    if (live) {
      CU(cudaMemcpyAsync(f.p, feat.p, live * o.max_observations * d8 * 4, cudaMemcpyDeviceToDevice, st));
      CU(cudaMemcpyAsync(c.p, cnt.p, live * 4, cudaMemcpyDeviceToDevice, st));
      CU(cudaMemcpyAsync(s.p, start.p, live * 4, cudaMemcpyDeviceToDevice, st));
      CU(cudaMemcpyAsync(i.p, ids.p, live * 8, cudaMemcpyDeviceToDevice, st));
    }
    CU(cudaStreamSynchronize(st));   // the old columns are freed below
    feat = std::move(f); cnt = std::move(c); start = std::move(s); ids = std::move(i); run = std::move(r);
    cap = nc;
    return 0;
  }

  int begin() {
    CU(cudaSetDevice(o.device));
    stage_ms[0] = stage_ms[1] = stage_ms[2] = 0.0f;
    return 0;
  }

  // stages rows [R][d8] (zero-padded) + ids + offsets + row -> item + dest + the initial max_dist into hreq
  void stage(const ReqLayout& L, int Q, const uint64_t* qids, const std::vector<int>& qoff,
             const std::vector<const float*>& src, const std::vector<int>& dest) {
    char* h = static_cast<char*>(hreq.p);
    const int D = o.feature_dim, R = (int)src.size();
    float* rows = reinterpret_cast<float*>(h + L.rows);
    for (int r = 0; r < R; ++r) {
      memcpy(rows + (size_t)r * d8, src[r], (size_t)D * 4);
      for (int k = D; k < d8; ++k) rows[(size_t)r * d8 + k] = 0.0f;
    }
    memcpy(h + L.qid, qids, (size_t)Q * 8);
    memcpy(h + L.qoff, qoff.data(), (size_t)(Q + 1) * 4);
    int* row_q = reinterpret_cast<int*>(h + L.row_q);
    for (int q = 0; q < Q; ++q)
      for (int r = qoff[q]; r < qoff[q + 1]; ++r) row_q[r] = q;
    memcpy(h + L.dest, dest.data(), (size_t)Q * 4);
    *reinterpret_cast<int*>(h + L.maxkey) = sb::fs_key(-1.0f);   // max_dist starts at -1.0 (topn.rs:78)
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

  // checks of a search / associate request; fills the newest-K row ranges
  int check_queries(int Q, const uint64_t* qids, const int32_t* offs, const float* feats, bool assoc,
                    std::vector<int>* qoff, std::vector<const float*>* src) {
    if (Q < 0) return fail(SB200_ERR_INVALID, "n_queries < 0");
    if (Q == 0) return 0;
    if (!qids || !offs) return fail(SB200_ERR_INVALID, "query_ids / obs_offsets is NULL");
    if (offs[0] != 0) return fail(SB200_ERR_INVALID, "obs_offsets[0] != 0");
    std::unordered_set<uint64_t> seen;
    seen.reserve((size_t)Q * 2);
    qoff->assign(1, 0);
    const int K = o.max_observations;
    for (int q = 0; q < Q; ++q) {
      const int n = offs[q + 1] - offs[q];
      if (n <= 0) return fail(SB200_ERR_INVALID, "query %d has no observations", q);
      if (!seen.insert(qids[q]).second)
        return fail(SB200_ERR_INVALID, "query id %llu appears twice in the call", (unsigned long long)qids[q]);
      if (assoc && hpos.count(qids[q]))
        return fail(SB200_ERR_INVALID, "query id %llu is already stored", (unsigned long long)qids[q]);
      for (int k = std::max(0, n - K); k < n; ++k) src->push_back(feats + (size_t)(offs[q] + k) * o.feature_dim);
      qoff->push_back((int)src->size());
    }
    if (!feats) return fail(SB200_ERR_INVALID, "features is NULL");
    const long long pairs = (long long)src->size() * (long long)hid.size() * K;
    if (pairs > sb::kFsMaxPairs)
      return fail(SB200_ERR_CAPACITY, "the call needs %lld observation pairs; one call holds at most 2^30", pairs);
    return 0;
  }

  int finish_timing(bool dist_ran, bool topn_ran, bool apply_ran) {
    float ms = 0.0f;
    if (dist_ran) { CU(cudaEventElapsedTime(&ms, ev[0], ev[1])); stage_ms[0] = ms; }
    if (topn_ran) { CU(cudaEventElapsedTime(&ms, ev[1], ev[2])); stage_ms[1] = ms; }
    if (apply_ran) { CU(cudaEventElapsedTime(&ms, ev[2], ev[3])); stage_ms[2] = ms; }
    return 0;
  }

  // search (assoc == false) or associate
  int run_queries(int Q, const uint64_t* qids, const int32_t* offs, const float* feats, int32_t* counts,
                  uint64_t* winners, double* weights, uint64_t* track_ids, uint8_t* merged, bool assoc) {
    std::vector<int> qoff;
    std::vector<const float*> src;
    if (int rc = check_queries(Q, qids, offs, feats, assoc, &qoff, &src)) return rc;
    if (Q > 0 && (!counts || !winners || !weights || (assoc && (!track_ids || !merged))))
      return fail(SB200_ERR_INVALID, "an output is NULL");
    if (int rc = begin()) return rc;
    if (Q == 0) return 0;
    const int R = (int)src.size(), topn = o.topn, K = o.max_observations;
    const long long live = (long long)hid.size(), S = live * K;
    const ReqLayout L(Q, R, d8);
    const ResLayout RL(Q, topn);
    if (int rc = hreq.ensure(L.total)) return rc;
    if (int rc = hres.ensure(RL.total)) return rc;
    if (int rc = dreq.ensure(L.total)) return rc;
    if (int rc = dres.ensure(RL.total)) return rc;
    if (int rc = plan.ensure((size_t)Q * 16)) return rc;
    if (o.metric == SB200_VIS_COSINE) {
      if (int rc = qnorm.ensure((size_t)R * 4)) return rc;
      if (int rc = snorm.ensure((size_t)std::max<long long>(S, 1) * 4)) return rc;
    }
    if (int rc = dist.ensure((size_t)std::max<long long>((long long)R * S, 1) * 4)) return rc;
    if (assoc)
      if (int rc = reserve(hid.size() + (size_t)Q)) return rc;
    stage(L, Q, qids, qoff, src, std::vector<int>(Q, -1));
    const sb::FsStore s = view();
    const sb::FsCall c = call_view(L, Q, R, &RL);
    CU(cudaMemcpyAsync(dreq.p, hreq.p, L.total, cudaMemcpyHostToDevice, st));
    CU(cudaEventRecord(ev[0], st));
    sb::fs_launch_dist(o.metric, o.distance_filter, s, c, st);
    CU(cudaEventRecord(ev[1], st));
    sb::fs_launch_topn(o.max_distance, o.min_votes, topn, assoc, s, c, st);
    CU(cudaEventRecord(ev[2], st));
    if (assoc) sb::fs_launch_apply(s, c, st);
    CU(cudaEventRecord(ev[3], st));
    CU(cudaMemcpyAsync(hres.p, dres.p, RL.total, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    CU(cudaGetLastError());
    if (int rc = finish_timing(S > 0, true, assoc)) return rc;
    const char* h = static_cast<const char*>(hres.p);
    const double* w = reinterpret_cast<const double*>(h + RL.w);
    const int* cn = reinterpret_cast<const int*>(h + RL.cnt);
    const int* ps = reinterpret_cast<const int*>(h + RL.pos);
    for (int q = 0; q < Q; ++q) {
      counts[q] = cn[q];
      for (int e = 0; e < topn; ++e) {
        const bool ok = e < cn[q];
        winners[(size_t)q * topn + e] = ok ? hid[ps[(size_t)q * topn + e]] : 0;
        weights[(size_t)q * topn + e] = ok ? w[(size_t)q * topn + e] : 0.0;
      }
    }
    if (assoc) {
      for (int q = 0; q < Q; ++q) {
        merged[q] = cn[q] > 0 ? 1 : 0;
        track_ids[q] = cn[q] > 0 ? winners[(size_t)q * topn] : qids[q];
      }
      for (int q = 0; q < Q; ++q)
        if (!merged[q]) {
          hpos[qids[q]] = (int)hid.size();
          hid.push_back(qids[q]);
        }
    }
    return 0;
  }

  int add(int n, const uint64_t* idv, const float* feats) {
    if (n < 0) return fail(SB200_ERR_INVALID, "n < 0");
    if (n > 0 && (!idv || !feats)) return fail(SB200_ERR_INVALID, "ids / features is NULL");
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
    std::vector<int> qoff(n + 1);
    std::vector<const float*> src(n);
    for (int i = 0; i <= n; ++i) qoff[i] = i;
    for (int i = 0; i < n; ++i) src[i] = feats + (size_t)i * o.feature_dim;
    const ReqLayout L(n, n, d8);
    if (int rc = hreq.ensure(L.total)) return rc;
    if (int rc = dreq.ensure(L.total)) return rc;
    if (int rc = plan.ensure((size_t)n * 16)) return rc;
    if (int rc = reserve(hid.size() + fresh.size())) return rc;
    stage(L, n, idv, qoff, src, dest);
    const sb::FsStore s = view();
    const sb::FsCall c = call_view(L, n, n, nullptr);
    CU(cudaMemcpyAsync(dreq.p, hreq.p, L.total, cudaMemcpyHostToDevice, st));
    CU(cudaEventRecord(ev[2], st));
    sb::fs_launch_apply(s, c, st);
    CU(cudaEventRecord(ev[3], st));
    CU(cudaStreamSynchronize(st));
    CU(cudaGetLastError());
    if (int rc = finish_timing(false, false, true)) return rc;
    for (uint64_t id : fresh) {
      hpos[id] = (int)hid.size();
      hid.push_back(id);
    }
    return 0;
  }

  int64_t fetch(int n, const uint64_t* idv, int remove, int32_t* counts, float* feats) {
    if (n < 0) return fail(SB200_ERR_INVALID, "n < 0");
    if (n > 0 && (!idv || !counts || !feats)) return fail(SB200_ERR_INVALID, "ids / counts / features is NULL");
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
    CU(cudaStreamSynchronize(st));
    CU(cudaGetLastError());
    const float* h = static_cast<const float*>(hres.p);
    const int* hc = reinterpret_cast<const int*>(static_cast<const char*>(hres.p) + align16(out_bytes));
    for (int i = 0; i < n; ++i) {
      counts[i] = hc[i];
      for (int b = 0; b < K; ++b)
        memcpy(feats + ((size_t)i * K + b) * D, h + ((size_t)i * K + b) * d8, (size_t)D * 4);
    }
    if (remove && found) {
      std::vector<int> from;
      from.reserve(hid.size());
      for (size_t p = 0; p < hid.size(); ++p)
        if (!gone[p]) from.push_back((int)p);
      DBuf f, c, st_, i, r;
      if (int rc = alloc_columns(cap, &f, &c, &st_, &i, &r)) return rc;
      if (int rc = gpos.ensure(std::max<size_t>(from.size(), 1) * 4)) return rc;
      CU(cudaMemcpyAsync(gpos.p, from.data(), from.size() * 4, cudaMemcpyHostToDevice, st));
      sb::FsStore d = s;
      d.feat = f.as<float>(); d.cnt = c.as<int>(); d.start = st_.as<int>(); d.ids = i.as<unsigned long long>();
      sb::fs_launch_compact(s, d, gpos.as<int>(), (int)from.size(), st);
      CU(cudaStreamSynchronize(st));
      CU(cudaGetLastError());
      feat = std::move(f); cnt = std::move(c); start = std::move(st_); ids = std::move(i); run = std::move(r);
      std::vector<uint64_t> kept;
      kept.reserve(from.size());
      for (int p : from) kept.push_back(hid[p]);
      hid.swap(kept);
      hpos.clear();
      for (size_t p = 0; p < hid.size(); ++p) hpos[hid[p]] = (int)p;
    }
    return found;
  }
};

// a call without a handle: SB200_ERR_CUDA when there is no device to have made one, else SB200_ERR_INVALID
int no_handle() {
  if (int rc = sb::check_device(0)) return rc;
  return fail(SB200_ERR_INVALID, "NULL handle");
}

extern "C" {

int sb200_fstore_create(const sb200_fstore_options* opts, sb200_fstore** out) {
  if (!opts || !out) return fail(SB200_ERR_INVALID, "opts / out is NULL");
  *out = nullptr;
  if (int rc = sb::check_device(0)) return rc;   // no device at all; the index is checked after the options
  const sb200_fstore_options& o = *opts;
  if (o.metric != SB200_VIS_EUCLIDEAN && o.metric != SB200_VIS_COSINE) return fail(SB200_ERR_INVALID, "unknown metric");
  if (o.max_observations < 1 || o.max_observations > SB200_FSTORE_MAX_OBS)
    return fail(SB200_ERR_INVALID, "max_observations must lie in 1..64");
  if (o.feature_dim < 1 || o.feature_dim > SB200_FSTORE_MAX_DIM)
    return fail(SB200_ERR_INVALID, "feature_dim must lie in 1..8192");
  if (o.topn < 1 || o.topn > SB200_FSTORE_MAX_TOPN) return fail(SB200_ERR_INVALID, "topn must lie in 1..64");
  if (o.min_votes < 0) return fail(SB200_ERR_INVALID, "min_votes < 0");
  if (int rc = sb::check_device(o.device)) return rc;
  CU(cudaSetDevice(o.device));
  sb200_fstore* s = new sb200_fstore();
  s->o = o;
  s->d8 = (o.feature_dim + 7) / 8 * 8;
  cudaError_t e = cudaStreamCreateWithFlags(&s->st, cudaStreamNonBlocking);
  for (int i = 0; i < 4 && e == cudaSuccess; ++i) e = cudaEventCreate(&s->ev[i]);
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
  return s->add(n, ids, features);
}

int sb200_fstore_search(sb200_fstore* s, int32_t n_queries, const uint64_t* query_ids, const int32_t* obs_offsets,
                        const float* features, int32_t* counts, uint64_t* winners, double* weights) {
  if (!s) return no_handle();
  return s->run_queries(n_queries, query_ids, obs_offsets, features, counts, winners, weights, nullptr, nullptr, false);
}

int sb200_fstore_associate(sb200_fstore* s, int32_t n_queries, const uint64_t* query_ids, const int32_t* obs_offsets,
                           const float* features, int32_t* counts, uint64_t* winners, double* weights,
                           uint64_t* track_ids, uint8_t* merged) {
  if (!s) return no_handle();
  return s->run_queries(n_queries, query_ids, obs_offsets, features, counts, winners, weights, track_ids, merged, true);
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

}  // extern "C"
