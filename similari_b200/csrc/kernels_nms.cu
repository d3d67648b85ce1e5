// kernels_nms.cu -- greedy non-maximum suppression of (oriented) boxes, src/utils/nms.rs:32-72, applied independently to
// every set of a request (sb200_nms_batch); sb200_nms is the one-set case.
//
//   filter  : score.unwrap_or(MAX) > score_threshold.unwrap_or(f32::MIN) && height > 0 && aspect > 0
//   rank    : score.unwrap_or(height), stable sort descending
//   suppress: a kept box cb removes every later ob with (intersection(cb, ob) as f32) / ob.area() > nms_threshold
//
// Set s is rows [base_s, base_s + n_s) of the request.  Every per-row array is indexed base_s + k, and every set has its
// own mask slab of n_s x ceil(n_s / 64) words, so one fixed sequence of three launches serves any number of sets:
//   (1) nms_rank_kernel, grid (set, 256-row chunk): filter + rank by counting within the set (stable by construction,
//       O(n_s^2) compares, no library sort); the box that lands at rank k writes its geometry to row base_s + k;
//   (2) nms_mask_kernel, one CTA per 64 x 64 tile (set, ib, jb >= ib) of a host-built list: suppression bits from the f64
//       Sutherland-Hodgman clip of sb_math.cuh behind the circumscribed-circle gate.  The list is built from the set
//       sizes, which bound the valid counts; tiles beyond a set's valid rows exit;
//   (3) nms_sweep_kernel, one CTA per set, all sets at once: the `removed` bitmap stays in shared memory.  Each 64-row
//       block's mask words (columns from the block onward, in column chunks when the set is large) are staged into shared
//       memory with coalesced asynchronous copies -- double-buffered, the next chunk loads while the current one is used --
//       and one thread makes the block's 64 sequential keep / drop decisions from the staged diagonal words.  No global
//       load depends on a keep / drop decision.
#include <cuda_pipeline.h>

#include <algorithm>
#include <cstring>
#include <functional>
#include <memory>
#include <mutex>
#include <vector>

#include "../../include/similari_b200.h"
#include "sb_engine.cuh"
#include "sb_host.cuh"

namespace sb {
namespace {

constexpr size_t kSweepBitmapBytes = 200 * 1024;  // per-set limit: the removed bitmap, ceil(n / 64) * 8 bytes
constexpr int kSweepThreads = 256;
// Workspace memory a pool keeps reserved between calls: the host entries synchronise, and a pool with the default
// threshold (0) would hand its memory back to the driver at every call.
constexpr unsigned long long kPoolKeepBytes = 256ull << 20;

struct NmsSet { int base, n; long long moff; };  // rows [base, base + n) of the request; first word of the mask slab
struct NmsTile { int set; unsigned short ib, jb; };  // ib, jb < ceil(n / 64) <= 25600

__device__ __forceinline__ bool nms_key(const float* boxes, const float* scores, int g, float score_thr, float& rank) {
  const float* b = boxes + (size_t)g * 6;
  const bool has = scores != nullptr && !is_nan(scores[g]);
  const float s = has ? scores[g] : 3.402823466e+38f;
  rank = has ? scores[g] : b[4];
  return s > score_thr && b[4] > 0.0f && b[3] > 0.0f;
}

// Position of each valid box in the stable descending order of its set's valid boxes; also resets the set's outputs.
__global__ void __launch_bounds__(256) nms_rank_kernel(const NmsSet* sets, const float* boxes, const float* scores,
                                                       float score_thr, int* n_valid, int* order, float* sx, float* sy,
                                                       float* sr, float* sarea, double* vert, int* keep_idx,
                                                       unsigned char* keep_mask) {
  __shared__ float s_rank[256];
  __shared__ unsigned char s_valid[256];
  const NmsSet d = sets[blockIdx.x];
  if ((int)blockIdx.y * 256 >= d.n) return;
  const int i = blockIdx.y * 256 + threadIdx.x;
  float r = 0.0f;
  const bool mine = i < d.n && nms_key(boxes, scores, d.base + i, score_thr, r);
  if (i < d.n) {
    keep_idx[d.base + i] = -1;
    if (keep_mask) keep_mask[d.base + i] = 0;
  }
  int pos = 0;
  for (int base = 0; base < d.n; base += 256) {
    const int j = base + threadIdx.x;
    float rj = 0.0f;
    s_valid[threadIdx.x] = j < d.n && nms_key(boxes, scores, d.base + j, score_thr, rj);
    s_rank[threadIdx.x] = rj;
    __syncthreads();
    if (mine) {
      const int lim = min(256, d.n - base);
      for (int q = 0; q < lim; ++q) {
        if (!s_valid[q]) continue;
        const float rq = s_rank[q];
        if (rq > r || (rq == r && base + q < i)) ++pos;
      }
    }
    __syncthreads();
  }
  const int cnt = __syncthreads_count(mine);
  if (threadIdx.x == 0 && cnt) atomicAdd(n_valid + blockIdx.x, cnt);
  if (!mine) return;
  const int k = d.base + pos;
  const float* b = boxes + (size_t)(d.base + i) * 6;
  order[k] = i;
  sx[k] = b[0]; sy[k] = b[1];
  sr[k] = box_radius(b[3], b[4]);
  sarea[k] = box_area(b[3], b[4]);
  box_vertices(b[0], b[1], b[2], b[3], b[4], vert + (size_t)k * 8);
}

// slab[i][jb] bit t: box i suppresses box jb*64+t (only j > i); rows and columns in rank order
__global__ void __launch_bounds__(64) nms_mask_kernel(const NmsTile* tiles, const NmsSet* sets, const int* n_valid,
                                                      float nms_thr, const float* sx, const float* sy, const float* sr,
                                                      const float* sarea, const double* vert, unsigned long long* mask) {
  const NmsTile tl = tiles[blockIdx.x];
  const int nv = n_valid[tl.set];
  const int ib = tl.ib, jb = tl.jb;
  if (ib * 64 >= nv || jb * 64 >= nv) return;
  const NmsSet d = sets[tl.set];
  const int words = (d.n + 63) >> 6;
  sx += d.base; sy += d.base; sr += d.base; sarea += d.base;
  vert += (size_t)d.base * 8;
  __shared__ float cx[64], cy[64], cr[64], ca[64];
  __shared__ double cv[64][8];
  const int t = threadIdx.x;
  const int j = jb * 64 + t;
  if (j < nv) {
    cx[t] = sx[j]; cy[t] = sy[j]; cr[t] = sr[j]; ca[t] = sarea[j];
    for (int q = 0; q < 8; ++q) cv[t][q] = vert[(size_t)j * 8 + q];
  }
  __syncthreads();
  const int i = ib * 64 + t;
  if (i >= nv) return;
  const float ix = sx[i], iy = sy[i], ir = sr[i];
  double iv[8];
  for (int q = 0; q < 8; ++q) iv[q] = vert[(size_t)i * 8 + q];
  unsigned long long bits = 0;
  const int lim = min(64, nv - jb * 64);
  for (int q = 0; q < lim; ++q) {
    const int jj = jb * 64 + q;
    if (jj <= i) continue;
    // intersection(cb, ob): 0.0 behind the circumscribed-circle gate, else clip(subject = cb, clip = ob)
    const double a = too_far(ix, iy, ir, cx[q], cy[q], cr[q]) ? 0.0 : clip_area(iv, cv[q]);
    const float metric = (float)a / ca[q];
    if (metric > nms_thr) bits |= 1ull << q;
  }
  mask[d.moff + (size_t)i * words + jb] = bits;
}

// rows [r0, r0 + rows) x words [c0, c0 + cw) of a slab with row pitch `words` -> dst with row pitch `pitch`; one commit
__device__ __forceinline__ void nms_stage(unsigned long long* dst, int pitch, const unsigned long long* slab, int words,
                                          int r0, int rows, int c0, int cw) {
  const int lane = threadIdx.x & 31;
  for (int r = threadIdx.x >> 5; r < rows; r += kSweepThreads / 32) {
    const unsigned long long* src = slab + (size_t)(r0 + r) * words + c0;
    for (int c = lane; c < cw; c += 32) __pipeline_memcpy_async(dst + r * pitch + c, src + c, 8);
  }
  __pipeline_commit();
}

// One CTA per set.  A step is (64-row block b, chunk of columns starting at c0); the chunks of block b cover the columns
// [b, nw) -- a row carries no bits left of its own block -- and the first one starts with the diagonal word.
__global__ void __launch_bounds__(kSweepThreads) nms_sweep_kernel(const NmsSet* sets, const int* n_valid,
                                                                  const unsigned long long* mask, const int* order,
                                                                  int chunk, int* keep_idx, int* keep_counts,
                                                                  unsigned char* keep_mask) {
  extern __shared__ unsigned long long sm[];  // [2][64][chunk] staged mask words, then removed[nw]
  __shared__ unsigned long long s_keep;
  const NmsSet d = sets[blockIdx.x];
  const int nv = n_valid[blockIdx.x];
  const int words = (d.n + 63) >> 6;  // row pitch of the slab
  const int nw = (nv + 63) >> 6;      // 64-row blocks (and bitmap words) of the valid rows
  const unsigned long long* slab = mask + d.moff;
  unsigned long long* removed = sm + 2 * 64 * chunk;
  for (int w = threadIdx.x; w < nw; w += kSweepThreads) removed[w] = 0ull;
  int b = 0, c0 = 0, kept = 0;
  unsigned long long keep = 0;
  if (nw > 0) nms_stage(sm, chunk, slab, words, 0, min(64, nv), 0, min(chunk, nw));
  for (int step = 0; b < nw; ++step) {
    int nb = b, nc = c0 + chunk;
    if (nc >= nw) { nb = b + 1; nc = nb; }
    const unsigned long long* cur = sm + (step & 1) * 64 * chunk;
    if (nb < nw) {
      // the buffer of step - 1 is free: the barrier that ended step - 1 came after its last read
      nms_stage(sm + ((step + 1) & 1) * 64 * chunk, chunk, slab, words, nb * 64, min(64, nv - nb * 64), nc,
                min(chunk, nw - nc));
      __pipeline_wait_prior(1);
    } else {
      __pipeline_wait_prior(0);
    }
    const int t = threadIdx.x;
    int src = 0;   // issued before the barrier: the load completes under the decisions
    if (c0 == b && t < 64 && b * 64 + t < nv) src = order[d.base + b * 64 + t];
    __syncthreads();
    if (c0 == b) {
      if (t == 0) {
        // visit only the rows still alive: the lowest one is kept and removes the later rows of its diagonal word
        const int lim = min(64, nv - b * 64);
        unsigned long long alive = (lim == 64 ? ~0ull : (1ull << lim) - 1ull) & ~removed[b], kp = 0;
        while (alive) {
          const int r = __ffsll((long long)alive) - 1;
          kp |= 1ull << r;
          alive &= alive - 1ull;
          alive &= ~cur[r * chunk];
        }
        s_keep = kp;
      }
      __syncthreads();
      keep = s_keep;
      if (t < 64 && ((keep >> t) & 1ull)) {
        keep_idx[d.base + kept + __popcll(keep & ((1ull << t) - 1ull))] = src;
        if (keep_mask) keep_mask[d.base + src] = 1;
      }
      kept += __popcll(keep);
    }
    if (keep) {
      const int cw = min(chunk, nw - c0);
      for (int c = threadIdx.x; c < cw; c += kSweepThreads) {
        if (c0 + c <= b) continue;
        unsigned long long acc = 0, m = keep;
        while (m) {
          acc |= cur[(__ffsll((long long)m) - 1) * chunk + c];
          m &= m - 1;
        }
        removed[c0 + c] |= acc;
      }
    }
    __syncthreads();
    b = nb;
    c0 = nc;
  }
  if (threadIdx.x == 0) keep_counts[blockIdx.x] = kept;
}

// Stream-ordered workspace from a library-owned pool per device.
cudaError_t ws_alloc(void** p, size_t bytes, int device, cudaStream_t st) {
  static std::mutex mu;
  static std::vector<cudaMemPool_t> pools;
  cudaMemPool_t pool;
  {
    std::lock_guard<std::mutex> g(mu);
    if ((int)pools.size() <= device) pools.resize(device + 1, nullptr);
    if (!pools[device]) {
      cudaMemPoolProps props;
      memset(&props, 0, sizeof(props));
      props.allocType = cudaMemAllocationTypePinned;
      props.location.type = cudaMemLocationTypeDevice;
      props.location.id = device;
      cudaError_t e = cudaMemPoolCreate(&pools[device], &props);
      if (e != cudaSuccess) { pools[device] = nullptr; return e; }
      unsigned long long keep = kPoolKeepBytes;
      cudaMemPoolSetAttribute(pools[device], cudaMemPoolAttrReleaseThreshold, &keep);
    }
    pool = pools[device];
  }
  return cudaMallocFromPoolAsync(p, bytes, pool, st);
}

// Pinned staging of the per-request tables (set descriptors, tile list).  A copy from pageable memory may wait for the
// work already queued on the stream; a copy from pinned memory does not.  A slot is reused once the copy that last read
// it has run, so a call waits only when kStageSlots earlier requests on the device still have their copy queued.
constexpr int kStageSlots = 8;
struct StageSlot { unsigned char* host = nullptr; size_t cap = 0; cudaEvent_t copied = nullptr; };
struct StageRing { std::mutex mu; StageSlot slot[kStageSlots]; int next = 0; };

StageRing& stage_ring(int device) {
  static std::mutex mu;
  static std::vector<std::unique_ptr<StageRing>> rings;
  std::lock_guard<std::mutex> g(mu);
  if ((int)rings.size() <= device) rings.resize(device + 1);
  if (!rings[device]) rings[device].reset(new StageRing);
  return *rings[device];
}

// fill(host) writes `bytes` bytes of tables; they are copied to dst on st
cudaError_t stage_upload(int device, void* dst, size_t bytes, const std::function<void(unsigned char*)>& fill,
                         cudaStream_t st) {
  StageRing& ring = stage_ring(device);
  std::lock_guard<std::mutex> g(ring.mu);
  StageSlot& sl = ring.slot[ring.next];
  ring.next = (ring.next + 1) % kStageSlots;
  cudaError_t e = sl.copied ? cudaEventSynchronize(sl.copied) : cudaEventCreateWithFlags(&sl.copied, cudaEventDisableTiming);
  if (e != cudaSuccess) return e;
  if (sl.cap < bytes) {
    const size_t cap = std::max(bytes, 2 * sl.cap);
    if (sl.host) cudaFreeHost(sl.host);
    sl.host = nullptr;
    sl.cap = 0;
    if ((e = cudaHostAlloc((void**)&sl.host, cap, cudaHostAllocDefault)) != cudaSuccess) { sl.host = nullptr; return e; }
    sl.cap = cap;
  }
  fill(sl.host);
  if ((e = cudaMemcpyAsync(dst, sl.host, bytes, cudaMemcpyHostToDevice, st)) != cudaSuccess) return e;
  return cudaEventRecord(sl.copied, st);
}

size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

// The device workspace of one call, from the set sizes alone: [sets | n_valid | tiles] (uploaded in one copy), then
// order, sx, sy, sr, sarea, vert and every set's mask slab of n x ceil(n / 64) words.
struct NmsWorkspace {
  size_t total = 0;                 // boxes in the request
  int max_n = 0, max_words = 0;
  int big_set = 0;                  // the set with the largest mask slab
  size_t n_tiles = 0, mask_words = 0;
  size_t o_nvalid = 0, o_tiles = 0, up_bytes = 0, o_order = 0, o_f32 = 0, o_vert = 0, o_mask = 0, bytes = 0;
};

NmsWorkspace nms_workspace(int n_sets, const int* offsets) {
  NmsWorkspace w;
  w.total = (size_t)offsets[n_sets];
  size_t big = 0;
  for (int s = 0; s < n_sets; ++s) {
    const int n = offsets[s + 1] - offsets[s], nw = (n + 63) / 64;
    w.max_n = std::max(w.max_n, n);
    w.max_words = std::max(w.max_words, nw);
    const size_t slab = (size_t)n * nw;
    if (slab > big) { big = slab; w.big_set = s; }
    w.mask_words += slab;
    w.n_tiles += (size_t)nw * (nw + 1) / 2;
  }
  w.o_nvalid = align256(sizeof(NmsSet) * n_sets);
  w.o_tiles = w.o_nvalid + align256(sizeof(int) * n_sets);
  w.up_bytes = w.o_tiles + sizeof(NmsTile) * w.n_tiles;
  w.o_order = align256(w.up_bytes);
  w.o_f32 = w.o_order + align256(4 * w.total);  // sx, sy, sr, sarea
  w.o_vert = w.o_f32 + 4 * align256(4 * w.total);
  w.o_mask = w.o_vert + align256(64 * w.total);
  w.bytes = w.o_mask + 8 * w.mask_words;
  return w;
}

// Total memory of the device, read once per device.  A fixed property, so whether a call is refused does not depend on
// what other processes hold at the time.
int device_total_memory(int device, size_t* bytes) {
  static std::mutex mu;
  static std::vector<size_t> total;
  std::lock_guard<std::mutex> g(mu);
  if ((int)total.size() <= device) total.resize(device + 1, 0);
  if (!total[device]) {
    cudaDeviceProp p;
    cudaError_t e = cudaGetDeviceProperties(&p, device);
    if (e != cudaSuccess) return fail(SB200_ERR_CUDA, "cudaGetDeviceProperties failed: %s", cudaGetErrorString(e));
    total[device] = p.totalGlobalMem;
  }
  *bytes = total[device];
  return 0;
}

// Enqueues the three launches for every set on st.  offsets (validated, total > 0) is a host array and lay its
// workspace; every other pointer is a device pointer.  No host synchronisation beyond the staging ring's bound.
// Returns a cudaError_t.
int nms_enqueue(int n_sets, const int* offsets, const NmsWorkspace& lay, const float* boxes, const float* scores,
                float nms_thr, float score_thr, int* keep_idx, int* keep_counts, unsigned char* keep_mask, int device,
                cudaStream_t st) {
  const size_t total = lay.total, n_tiles = lay.n_tiles, up_bytes = lay.up_bytes;
  const size_t o_nvalid = lay.o_nvalid, o_tiles = lay.o_tiles, o_order = lay.o_order, o_f32 = lay.o_f32;
  const size_t o_vert = lay.o_vert, o_mask = lay.o_mask;
  const int max_n = lay.max_n, max_words = lay.max_words;
  unsigned char* ws = nullptr;
  cudaError_t e = ws_alloc((void**)&ws, lay.bytes, device, st);
  if (e != cudaSuccess) return (int)e;

  e = stage_upload(device, ws, up_bytes, [&](unsigned char* up) {
    memset(up, 0, up_bytes);  // n_valid = 0
    NmsSet* hs = reinterpret_cast<NmsSet*>(up);
    NmsTile* ht = reinterpret_cast<NmsTile*>(up + o_tiles);
    long long moff = 0;
    size_t t = 0;
    for (int s = 0; s < n_sets; ++s) {
      const int n = offsets[s + 1] - offsets[s], w = (n + 63) / 64;
      hs[s] = NmsSet{offsets[s], n, moff};
      moff += (long long)n * w;
      for (int ib = 0; ib < w; ++ib)
        for (int jb = ib; jb < w; ++jb) ht[t++] = NmsTile{s, (unsigned short)ib, (unsigned short)jb};
    }
  }, st);
  if (e != cudaSuccess) { cudaFreeAsync(ws, st); return (int)e; }

  const NmsSet* d_sets = reinterpret_cast<const NmsSet*>(ws);
  int* d_nvalid = reinterpret_cast<int*>(ws + o_nvalid);
  const NmsTile* d_tiles = reinterpret_cast<const NmsTile*>(ws + o_tiles);
  int* order = reinterpret_cast<int*>(ws + o_order);
  float* sx = reinterpret_cast<float*>(ws + o_f32);
  float* sy = reinterpret_cast<float*>(ws + o_f32 + align256(4 * total));
  float* sr = reinterpret_cast<float*>(ws + o_f32 + 2 * align256(4 * total));
  float* sa = reinterpret_cast<float*>(ws + o_f32 + 3 * align256(4 * total));
  double* vert = reinterpret_cast<double*>(ws + o_vert);
  unsigned long long* mask = reinterpret_cast<unsigned long long*>(ws + o_mask);

  // sweep: removed bitmap of the largest set + two stages of 64 rows x `chunk` words in the opt-in shared memory
  int optin = 0;
  cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device);
  const int avail_words = (optin - 64) / 8 - max_words;
  const int chunk = std::max(1, std::min(max_words, avail_words / 128));
  const size_t smem = 8 * ((size_t)2 * 64 * chunk + max_words);
  if (smem > 48 * 1024) {
    e = cudaFuncSetAttribute(nms_sweep_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { cudaFreeAsync(ws, st); return (int)e; }
  }

  nms_rank_kernel<<<dim3(n_sets, (max_n + 255) / 256), 256, 0, st>>>(d_sets, boxes, scores, score_thr, d_nvalid, order,
                                                                     sx, sy, sr, sa, vert, keep_idx, keep_mask);
  nms_mask_kernel<<<(unsigned)n_tiles, 64, 0, st>>>(d_tiles, d_sets, d_nvalid, nms_thr, sx, sy, sr, sa, vert, mask);
  nms_sweep_kernel<<<n_sets, kSweepThreads, smem, st>>>(d_sets, d_nvalid, mask, order, chunk, keep_idx, keep_counts,
                                                        keep_mask);
  note_launch(3);
  e = cudaGetLastError();
  cudaFreeAsync(ws, st);
  return (int)e;
}

// Checks shared by both batch entries, in the order of sb200_nms; nothing is read but `offsets`.  On success *lay is the
// call's workspace.
int nms_check(int n_sets, const int* offsets, const float* boxes, const int* keep_idx, const int* keep_counts, int device,
              NmsWorkspace* lay) {
  if (n_sets < 0 || !offsets) return fail(SB200_ERR_INVALID, "nms_batch: n_sets < 0 or offsets is NULL");
  if (offsets[0] != 0) return fail(SB200_ERR_INVALID, "nms_batch: offsets[0] != 0");
  for (int s = 0; s < n_sets; ++s)
    if (offsets[s + 1] < offsets[s])
      return fail(SB200_ERR_INVALID, "nms_batch: offsets decrease at set %d", s);
  if ((n_sets > 0 && !keep_counts) || (offsets[n_sets] > 0 && (!boxes || !keep_idx)))
    return fail(SB200_ERR_INVALID, "nms_batch: bad arguments");
  if (int rc = check_device(device)) return rc;
  for (int s = 0; s < n_sets; ++s) {
    const int n = offsets[s + 1] - offsets[s];
    if ((size_t)((n + 63) / 64) * 8 > kSweepBitmapBytes)
      return fail(SB200_ERR_CAPACITY, "nms: set %d has %d boxes, too many for the on-chip sweep", s, n);
  }
  // the mask slabs grow as n^2 / 8 bytes: a set the bitmap admits can still need more memory than the device has
  *lay = nms_workspace(n_sets, offsets);
  size_t mem = 0;
  if (int rc = device_total_memory(device, &mem)) return rc;
  if (lay->bytes > mem) {
    const int s = lay->big_set, n = offsets[s + 1] - offsets[s];
    return fail(SB200_ERR_CAPACITY, "nms: set %d has %d boxes; the call's workspace (%zu bytes, %zu of them the mask of "
                "that set) exceeds the device's %zu bytes", s, n, lay->bytes, (size_t)n * ((n + 63) / 64) * 8, mem);
  }
  return 0;
}

}  // namespace
}  // namespace sb

extern "C" int sb200_nms_batch_device(int32_t n_sets, const int32_t* offsets, const float* boxes, const float* scores,
                                      float nms_threshold, float score_threshold, int32_t has_score_threshold,
                                      int32_t* keep_idx, int32_t* keep_counts, uint8_t* keep_mask, int32_t device,
                                      void* cuda_stream) {
  sb::NmsWorkspace lay;
  int rc = sb::nms_check(n_sets, offsets, boxes, keep_idx, keep_counts, device, &lay);
  if (rc) return rc;
  CU(cudaSetDevice(device));
  cudaStream_t st = (cudaStream_t)cuda_stream;
  cudaError_t e = cudaSuccess;
  if (offsets[n_sets] == 0) {
    if (n_sets > 0) e = cudaMemsetAsync(keep_counts, 0, 4 * (size_t)n_sets, st);
  } else {
    const float sthr = has_score_threshold ? score_threshold : -3.402823466e+38f;  // f32::MIN
    e = (cudaError_t)sb::nms_enqueue(n_sets, offsets, lay, boxes, scores, nms_threshold, sthr, keep_idx, keep_counts,
                                     keep_mask, device, st);
  }
  if (e != cudaSuccess) return sb::fail(SB200_ERR_CUDA, "nms: CUDA error: %s", cudaGetErrorString(e));
  return 0;
}

extern "C" int64_t sb200_nms_batch(int32_t n_sets, const int32_t* offsets, const float* boxes, const float* scores,
                                   float nms_threshold, float score_threshold, int32_t has_score_threshold,
                                   int32_t* keep_idx, int32_t* keep_counts, uint8_t* keep_mask, int32_t device) {
  sb::NmsWorkspace lay;
  int rc = sb::nms_check(n_sets, offsets, boxes, keep_idx, keep_counts, device, &lay);
  if (rc) return rc;
  const size_t total = (size_t)offsets[n_sets];
  if (total == 0) {
    if (n_sets > 0) memset(keep_counts, 0, 4 * (size_t)n_sets);
    return 0;
  }
  CU(cudaSetDevice(device));
  cudaStream_t st;
  CU(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
  // device copies: boxes, scores, keep_idx, keep_counts, keep_mask
  const size_t o_sc = sb::align256(24 * total), o_idx = o_sc + sb::align256(4 * total);
  const size_t o_cnt = o_idx + sb::align256(4 * total), o_km = o_cnt + sb::align256(4 * (size_t)n_sets);
  unsigned char* io = nullptr;
  cudaError_t e = sb::ws_alloc((void**)&io, o_km + total, device, st);
  if (e == cudaSuccess) {
    float* db = reinterpret_cast<float*>(io);
    float* ds = scores ? reinterpret_cast<float*>(io + o_sc) : nullptr;
    int* didx = reinterpret_cast<int*>(io + o_idx);
    int* dcnt = reinterpret_cast<int*>(io + o_cnt);
    unsigned char* dkm = keep_mask ? io + o_km : nullptr;
    e = cudaMemcpyAsync(db, boxes, 24 * total, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess && ds) e = cudaMemcpyAsync(ds, scores, 4 * total, cudaMemcpyHostToDevice, st);
    const float sthr = has_score_threshold ? score_threshold : -3.402823466e+38f;  // f32::MIN
    if (e == cudaSuccess)
      e = (cudaError_t)sb::nms_enqueue(n_sets, offsets, lay, db, ds, nms_threshold, sthr, didx, dcnt, dkm, device, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(keep_idx, didx, 4 * total, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(keep_counts, dcnt, 4 * (size_t)n_sets, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess && dkm) e = cudaMemcpyAsync(keep_mask, dkm, total, cudaMemcpyDeviceToHost, st);
    cudaFreeAsync(io, st);
  }
  cudaError_t es = cudaStreamSynchronize(st);
  if (e == cudaSuccess) e = es;
  cudaStreamDestroy(st);
  if (e != cudaSuccess) return sb::fail(SB200_ERR_CUDA, "nms: CUDA error: %s", cudaGetErrorString(e));
  int64_t kept = 0;
  for (int s = 0; s < n_sets; ++s) kept += keep_counts[s];
  return kept;
}

extern "C" int64_t sb200_nms(const float* boxes, const float* scores, int32_t n, float nms_threshold, float score_threshold,
                             int32_t has_score_threshold, int32_t* out_idx, int32_t device) {
  if (n < 0 || (n > 0 && (!boxes || !out_idx))) return sb::fail(SB200_ERR_INVALID, "bad arguments");
  const int32_t offsets[2] = {0, n};
  std::vector<int32_t> idx(std::max(n, 1));
  int32_t count = 0;
  const int64_t kept = sb200_nms_batch(1, offsets, boxes, scores, nms_threshold, score_threshold, has_score_threshold,
                                       idx.data(), &count, nullptr, device);
  if (kept > 0) memcpy(out_idx, idx.data(), 4 * (size_t)kept);
  return kept;
}
