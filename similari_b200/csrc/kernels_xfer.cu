// kernels_xfer.cu -- the bulk copies of the state blob (sb200_tracker_save / _load, sb200_scenes_export / _import).
//
// Pack and unpack are the same operation with source and destination swapped: a list of contiguous segments (one per
// column and scene slot: the scene's rows of the track store, the blocks of its feature arena, its free list; the
// wasted buffer and the feature-history pool whole), each cut into 32 KB chunks that the CTAs of one grid take in turn.
// Every chunk moves with 16-byte accesses where both ends and the length allow it (feature rows, Kalman rows), with
// narrower ones otherwise (the 1-byte and 24-byte columns).  The feature-history blocks of moved scenes are not
// contiguous in the source pool: they go through a kernel of their own that follows each track's block index.
#include <cuda_runtime.h>
#include <stdint.h>

#include "sb_engine.cuh"

namespace sb {

namespace {

constexpr int kXferThreads = 256;

template <typename V>
__device__ __forceinline__ void copy_as(const char* __restrict__ s, char* __restrict__ d, size_t len) {
  const V* sv = reinterpret_cast<const V*>(s);
  V* dv = reinterpret_cast<V*>(d);
  const size_t n = len / sizeof(V);
  for (size_t i = threadIdx.x; i < n; i += kXferThreads) dv[i] = sv[i];
}

__global__ void __launch_bounds__(kXferThreads) xfer_copy_kernel(const XferSeg* __restrict__ segs,
                                                                  const long long* __restrict__ cpre, int n_seg) {
  const long long total = cpre[n_seg];
  for (long long c = blockIdx.x; c < total; c += gridDim.x) {
    int lo = 0, hi = n_seg - 1;   // last segment whose first chunk is at or before c
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (cpre[mid] <= c) lo = mid; else hi = mid - 1;
    }
    const XferSeg sg = segs[lo];
    const size_t off = (size_t)(c - cpre[lo]) * kXferChunk;
    const size_t len = sg.bytes - off < (size_t)kXferChunk ? sg.bytes - off : (size_t)kXferChunk;
    const char* s = sg.src + off;
    char* d = sg.dst + off;
    const uintptr_t a = (uintptr_t)s | (uintptr_t)d | (uintptr_t)len;
    if ((a & 15) == 0) copy_as<uint4>(s, d, len);
    else if ((a & 7) == 0) copy_as<uint2>(s, d, len);
    else if ((a & 3) == 0) copy_as<unsigned int>(s, d, len);
    else copy_as<unsigned char>(s, d, len);
  }
}

// flat track t -> (entry e of the scene list, index j in the scene's store order)
__device__ __forceinline__ int find_scene(const int* pre, int n, int t) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (pre[mid] <= t) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// dir 0 (pack):   rows[t] <- hrows[hblk[slot, j]],  pres[t] <- hpresent[hblk[slot, j]]
// dir 1 (unpack): hrows[base + t] <- rows[t], hpresent[base + t] <- pres[t], hblk[slot, j] = base + t
__global__ void __launch_bounds__(kXferThreads) xfer_hist_kernel(TrackStore ts, int d8, const int* __restrict__ slots,
                                                                  const int* __restrict__ pre, int n, int dir,
                                                                  float* rows, unsigned char* pres, int base) {
  const int total = pre[n];
  const int H = ts.fhist_len;
  const size_t rw = (size_t)H * d8;   // floats per block (a multiple of 8)
  for (int t = blockIdx.x; t < total; t += gridDim.x) {
    const int e = find_scene(pre, n, t);
    const size_t idx = (size_t)slots[e] * ts.track_cap + (size_t)(t - pre[e]);
    int blk;
    if (dir == 0) blk = ts.hblk[idx];
    else {
      blk = base + t;
      if (threadIdx.x == 0) ts.hblk[idx] = blk;
    }
    const float4* s = reinterpret_cast<const float4*>(dir == 0 ? ts.hrows + (size_t)blk * rw : rows + (size_t)t * rw);
    float4* d = reinterpret_cast<float4*>(dir == 0 ? rows + (size_t)t * rw : ts.hrows + (size_t)blk * rw);
    for (size_t i = threadIdx.x; i < rw / 4; i += kXferThreads) d[i] = s[i];
    const unsigned char* sp = dir == 0 ? ts.hpresent + (size_t)blk * H : pres + (size_t)t * H;
    unsigned char* dp = dir == 0 ? pres + (size_t)t * H : ts.hpresent + (size_t)blk * H;
    for (int i = threadIdx.x; i < H; i += kXferThreads) dp[i] = sp[i];
  }
}

// One CTA per listed slot: pushes the history blocks of its `push` first tracks onto the pool's free list (a removed
// scene), then sets the slot's device counters.  CTA 0 also raises the id counter and moves the pool's counters.
__global__ void xfer_slots_kernel(const XferSlot* __restrict__ tab, int n, int* n_tracks, int* n_free, int* arena_top,
                                  TrackStore ts, int free0, int free_add, int top_add, unsigned long long* id_counter,
                                  unsigned long long id_min) {
  const XferSlot e = tab[blockIdx.x];
  const size_t base = (size_t)e.slot * ts.track_cap;
  if (e.push > 0)
    for (int j = threadIdx.x; j < e.push; j += blockDim.x) ts.hfree[free0 + e.push_off + j] = ts.hblk[base + j];
  if (threadIdx.x == 0) {
    n_tracks[e.slot] = e.n_tracks;
    if (n_free) n_free[e.slot] = e.n_free;
    if (arena_top) arena_top[e.slot] = e.arena_top;
    if (blockIdx.x == 0) {
      if (id_counter && *id_counter < id_min) *id_counter = id_min;
      if (ts.hpool) { ts.hpool[0] += free_add; ts.hpool[1] += top_add; }
    }
  }
}

// one CTA per check: counts the entries outside their range
__global__ void xfer_check_kernel(const XferCheck* __restrict__ ck, int K, int* bad) {
  const XferCheck c = ck[blockIdx.x];
  int cnt = 0;
  for (long long i = threadIdx.x; i < c.n; i += blockDim.x) {
    if (c.kind == 0) {
      const int v = static_cast<const int*>(c.p)[i];
      cnt += (v < c.lo || v >= c.hi);
    } else if (c.kind == 1) {
      const int v = static_cast<const unsigned char*>(c.p)[i];
      cnt += (v < c.lo || v >= c.hi);
    } else {
      const unsigned char* row = static_cast<const unsigned char*>(c.p) + i * K;
      const int on = min((int)c.aux[i], K);   // obs_n itself is checked by its own entry
      for (int k = 0; k < on; ++k) cnt += (row[k] < c.lo || row[k] >= c.hi);
    }
  }
  if (cnt) atomicAdd(bad, cnt);
}

}  // namespace

int launch_xfer_check(const XferCheck* d_ck, int n, int K, int* bad, cudaStream_t st) {
  if (n <= 0) return 0;
  xfer_check_kernel<<<n, 256, 0, st>>>(d_ck, K, bad);
  note_launch();
  return (int)cudaGetLastError();
}

int launch_xfer_copy(const XferSeg* d_segs, const long long* d_cpre, int n_seg, long long chunks, int num_sms,
                     cudaStream_t st) {
  if (n_seg <= 0 || chunks <= 0) return 0;
  const long long grid = chunks < (long long)num_sms * 8 ? chunks : (long long)num_sms * 8;
  xfer_copy_kernel<<<(unsigned)grid, kXferThreads, 0, st>>>(d_segs, d_cpre, n_seg);
  note_launch();
  return (int)cudaGetLastError();
}

int launch_xfer_hist(const TrackStore& ts, int d8, const int* d_slots, const int* d_pre, int n, int total, int dir,
                     float* rows, unsigned char* pres, int base, int num_sms, cudaStream_t st) {
  if (n <= 0 || total <= 0) return 0;
  const int grid = total < num_sms * 8 ? total : num_sms * 8;
  xfer_hist_kernel<<<grid, kXferThreads, 0, st>>>(ts, d8, d_slots, d_pre, n, dir, rows, pres, base);
  note_launch();
  return (int)cudaGetLastError();
}

int launch_xfer_slots(const XferSlot* d_tab, int n, int* d_n_tracks, int* d_n_free, int* d_arena_top,
                      const TrackStore& ts, int free0, int free_add, int top_add, unsigned long long* id_counter,
                      unsigned long long id_min, cudaStream_t st) {
  if (n <= 0) return 0;
  xfer_slots_kernel<<<n, 128, 0, st>>>(d_tab, n, d_n_tracks, d_n_free, d_arena_top, ts, free0, free_add, top_add,
                                       id_counter, id_min);
  note_launch();
  return (int)cudaGetLastError();
}

}  // namespace sb
