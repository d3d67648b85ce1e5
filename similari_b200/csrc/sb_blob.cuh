// sb_blob.cuh -- host-side tools shared by the state blobs of the trackers (engine.cu) and of the feature track store
// (fstore.cu): where a blob lives, the host <-> device copy of one, and the segment copy (kernels_xfer.cu) that packs and
// unpacks device columns.  Host code only.
#pragma once
#include <cstring>
#include <vector>

#include "sb_engine.cuh"
#include "sb_host.cuh"

namespace sb {

// where a blob lives: -1 host memory, else the ordinal of the device that holds it
inline int blob_device(const void* p) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return -1; }
  return (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged) ? a.device : -1;
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
