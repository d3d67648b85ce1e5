// sb_blob.cuh -- host-side tools shared by the state blobs of the trackers (engine.cu) and of the feature track store
// (fstore.cu): the section layout and its check, where a blob lives and whether a handle works on it in place, the
// host <-> device copy of one, and the segment copy (kernels_xfer.cu) that packs and unpacks device columns.  Each format
// keeps its own header, sections and index checks.  Host code only.
#pragma once
#include <cstdint>
#include <cstring>
#include <vector>

#include "sb_engine.cuh"
#include "sb_host.cuh"

namespace sb {

// Both formats: a header H (with total_bytes, sec_off[] and sec_bytes[]), then sections at kBlobAlign-byte offsets,
// every gap zeroed.
constexpr uint64_t kBlobAlign = 256;
static_assert(kBlobAlign == SB200_FSTORE_BLOB_ALIGN, "the store blob's published section alignment");

// lays out `n` sections of sec[i] bytes after the header: sets h.sec_off, h.sec_bytes and h.total_bytes
template <class H> void lay_out(H& h, const uint64_t* sec, uint32_t n) {
  auto up = [](uint64_t v) { return (v + kBlobAlign - 1) / kBlobAlign * kBlobAlign; };
  h.total_bytes = up(sizeof(H));
  for (uint32_t i = 0; i < n; ++i) {
    h.sec_off[i] = h.total_bytes;
    h.sec_bytes[i] = sec[i];
    h.total_bytes += up(sec[i]);
  }
}

// Checks the section table of `n` sections: in order after the header, disjoint, inside total_bytes and at kBlobAlign
// offsets, as lay_out places them (the kernels access them with 16-byte loads and stores).  `names` names the sections
// in the messages; without it they are numbered.
template <class H> int check_section_table(const H& h, uint32_t n, const char* const* names = nullptr) {
  uint64_t end = sizeof(H);
  for (uint32_t i = 0; i < n; ++i) {
    char num[12];
    snprintf(num, sizeof(num), "%u", i);
    const char* name = names ? names[i] : num;
    if (h.sec_off[i] < end || h.sec_off[i] > h.total_bytes || h.sec_bytes[i] > h.total_bytes - h.sec_off[i])
      return fail(SB200_ERR_INVALID, "section %s lies outside the blob or overlaps the one before", name);
    if (h.sec_off[i] % kBlobAlign != 0)
      return fail(SB200_ERR_INVALID, names ? "section %s is not 256-byte aligned" : "section %s is not aligned", name);
    end = h.sec_off[i] + h.sec_bytes[i];
  }
  return 0;
}

// where a blob lives: -1 host memory, else the ordinal of the device that holds it
inline int blob_device(const void* p) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return -1; }
  return (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged) ? a.device : -1;
}

// A handle on `device` works on a blob in place when the blob is on that device and 16-byte aligned: the kernels that
// read and write the sections use 16-byte accesses.  Any other blob goes through a device copy.
inline bool blob_in_place(const void* p, int where, int device) {
  return where == device && (reinterpret_cast<uintptr_t>(p) & 15) == 0;
}

// host <-> device copy of a blob through two pinned staging buffers (the copy of one chunk overlaps the host copy of the
// other); memory that is pinned already is copied in one piece
inline int host_copy(cudaStream_t st, void* host, void* dev, size_t n, bool to_host) {
  cudaPointerAttributes a;
  const bool pinned = cudaPointerGetAttributes(&a, host) == cudaSuccess && a.type == cudaMemoryTypeHost;
  cudaGetLastError();
  if (pinned || n <= (1u << 20)) {
    CU(to_host ? cudaMemcpyAsync(host, dev, n, cudaMemcpyDeviceToHost, st) : cudaMemcpyAsync(dev, host, n, cudaMemcpyHostToDevice, st));
    CU(cudaStreamSynchronize(st));
    return 0;
  }
  constexpr size_t kStage = 32u << 20;
  struct Stage {
    void* p[2] = {nullptr, nullptr};
    cudaEvent_t ev[2] = {nullptr, nullptr};
    ~Stage() { for (int i = 0; i < 2; ++i) { if (p[i]) cudaFreeHost(p[i]); if (ev[i]) cudaEventDestroy(ev[i]); } }
  } sg;
  for (int i = 0; i < 2; ++i) {
    CU(cudaHostAlloc(&sg.p[i], kStage, cudaHostAllocDefault));
    CU(cudaEventCreateWithFlags(&sg.ev[i], cudaEventDisableTiming));
  }
  char* h = static_cast<char*>(host);
  char* d = static_cast<char*>(dev);
  const size_t nch = (n + kStage - 1) / kStage;
  auto len = [&](size_t i) { return std::min(kStage, n - i * kStage); };
  if (to_host) {
    CU(cudaMemcpyAsync(sg.p[0], d, len(0), cudaMemcpyDeviceToHost, st));
    CU(cudaEventRecord(sg.ev[0], st));
    for (size_t i = 0; i < nch; ++i) {
      if (i + 1 < nch) {
        CU(cudaMemcpyAsync(sg.p[(i + 1) & 1], d + (i + 1) * kStage, len(i + 1), cudaMemcpyDeviceToHost, st));
        CU(cudaEventRecord(sg.ev[(i + 1) & 1], st));
      }
      CU(cudaEventSynchronize(sg.ev[i & 1]));
      memcpy(h + i * kStage, sg.p[i & 1], len(i));
    }
  } else {
    for (size_t i = 0; i < nch; ++i) {
      if (i >= 2) CU(cudaEventSynchronize(sg.ev[i & 1]));   // the copy out of this buffer two chunks ago has finished
      memcpy(sg.p[i & 1], h + i * kStage, len(i));
      CU(cudaMemcpyAsync(d + i * kStage, sg.p[i & 1], len(i), cudaMemcpyHostToDevice, st));
      CU(cudaEventRecord(sg.ev[i & 1], st));
    }
  }
  CU(cudaStreamSynchronize(st));
  return 0;
}

// Writes the blob of header `h` (`n` sections) to `dst` (host memory, or device memory on any device) for a handle on
// `device`, on its stream `st`.  The blob is placed at `dst` itself when blob_in_place allows, else in a temporary on
// `device`; there the header is uploaded, every gap after it and after each section zeroed (equal states give equal
// blobs), and pack(p) fills the sections of the blob at p.  A temporary then goes to `dst` by a peer or a host copy.
template <class H, class Pack>
int write_blob(void* dst, int device, cudaStream_t st, const H& h, uint32_t n, Pack&& pack) {
  const int where = blob_device(dst);
  DBuf tmp;
  char* p = static_cast<char*>(dst);
  if (!blob_in_place(dst, where, device)) {
    if (int rc = tmp.ensure(h.total_bytes)) return rc;
    p = tmp.as<char>();
  }
  CU(cudaMemcpyAsync(p, &h, sizeof(H), cudaMemcpyHostToDevice, st));
  uint64_t end = sizeof(H);
  for (uint32_t i = 0; i <= n; ++i) {
    const uint64_t next = i < n ? h.sec_off[i] : h.total_bytes;
    if (next > end) CU(cudaMemsetAsync(p + end, 0, next - end, st));
    if (i < n) end = h.sec_off[i] + h.sec_bytes[i];
  }
  if (int rc = pack(p)) return rc;
  if (p == dst) return 0;
  if (where >= 0) {
    CU(cudaMemcpyPeerAsync(dst, where, p, device, h.total_bytes, st));
    CU(cudaStreamSynchronize(st));
    return 0;
  }
  return host_copy(st, dst, p, h.total_bytes, true);
}

// The blob at `src` (host memory, or device memory on any device) where a handle on `device` can work on it: `src`
// itself when blob_in_place allows, else a copy of its `bytes` bytes in `tmp`.
inline int blob_on_device(const void* src, uint64_t bytes, int device, cudaStream_t st, DBuf& tmp, const char** out) {
  const int where = blob_device(src);
  if (blob_in_place(src, where, device)) { *out = static_cast<const char*>(src); return 0; }
  if (int rc = tmp.ensure(bytes)) return rc;
  if (where >= 0) {
    CU(cudaMemcpyPeerAsync(tmp.p, device, src, where, bytes, st));
    CU(cudaStreamSynchronize(st));
  } else if (int rc = host_copy(st, const_cast<void*>(src), tmp.p, bytes, false)) {
    return rc;
  }
  *out = tmp.as<const char>();
  return 0;
}

// appends the copy of `bytes` between a handle's column and a blob section: dir 0 packs (column -> section), dir 1 unpacks
inline void add_segment(std::vector<XferSeg>& segs, int dir, char* col, char* sec, uint64_t bytes) {
  if (bytes) segs.push_back(dir == 0 ? XferSeg{col, sec, bytes} : XferSeg{sec, col, bytes});
}

// Copies every segment (device memory on the current device) with launch_xfer_copy on `st` and waits for it.
inline int copy_segments(const std::vector<XferSeg>& segs, int num_sms, cudaStream_t st) {
  if (segs.empty()) return 0;
  std::vector<long long> cpre(segs.size() + 1, 0);
  for (size_t i = 0; i < segs.size(); ++i)
    cpre[i + 1] = cpre[i] + (long long)((segs[i].bytes + kXferChunk - 1) / kXferChunk);
  DBuf d_tab;
  const size_t sb_ = segs.size() * sizeof(XferSeg);
  if (int rc = d_tab.ensure(sb_ + cpre.size() * sizeof(long long))) return rc;
  CU(cudaMemcpyAsync(d_tab.p, segs.data(), sb_, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(d_tab.as<char>() + sb_, cpre.data(), cpre.size() * sizeof(long long), cudaMemcpyHostToDevice, st));
  const int e = launch_xfer_copy(d_tab.as<XferSeg>(), reinterpret_cast<const long long*>(d_tab.as<char>() + sb_),
                                 (int)segs.size(), cpre.back(), num_sms, st);
  if (e) return fail(SB200_ERR_CUDA, "state copy launch failed: %s", cudaGetErrorString((cudaError_t)e));
  CU(cudaStreamSynchronize(st));
  return 0;
}

}  // namespace sb
