// sb_host.cuh -- host-side tools of every translation unit behind the C ABI: the thread's last error, the error and CUDA
// checks, the device check, and the grow-only device and pinned host buffers.  Host code only.
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <string>
#include <utility>

#include "../../include/similari_b200.h"

namespace sb {

inline thread_local std::string g_err;   // what sb200_last_error returns

// sets the calling thread's last error and returns `code`
__attribute__((format(printf, 2, 3))) inline int fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_err = buf;
  return code;
}

#define CU(x)                                                                                  \
  do {                                                                                         \
    cudaError_t e_ = (x);                                                                      \
    if (e_ != cudaSuccess)                                                                     \
      return sb::fail(SB200_ERR_CUDA, "%s failed: %s (%s:%d)", #x, cudaGetErrorString(e_), __FILE__, __LINE__); \
  } while (0)

// CUDA devices visible to the process (0 when the runtime finds none, or no driver)
inline int device_count() {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}

// SB200_ERR_CUDA without a device (there is no CPU execution path), SB200_ERR_INVALID for a device index out of range.
// check_device(0) asks only whether there is a device at all: index 0 is in range whenever one exists.
inline int check_device(int device) {
  const int n = device_count();
  if (n <= 0) return fail(SB200_ERR_CUDA, "no CUDA device available (this library has no CPU execution path)");
  if (device < 0 || device >= n) return fail(SB200_ERR_INVALID, "device %d out of range (%d devices)", device, n);
  return 0;
}

// grow-only device buffer; it owns its memory (move-only, freed by the destructor)
struct DBuf {
  void* p = nullptr;
  size_t bytes = 0;
  DBuf() = default;
  DBuf(const DBuf&) = delete;
  DBuf& operator=(const DBuf&) = delete;
  DBuf(DBuf&& o) noexcept : p(o.p), bytes(o.bytes) { o.p = nullptr; o.bytes = 0; }
  DBuf& operator=(DBuf&& o) noexcept {
    if (this != &o) { release(); p = o.p; bytes = o.bytes; o.p = nullptr; o.bytes = 0; }
    return *this;
  }
  ~DBuf() { release(); }
  int ensure(size_t need) {
    if (need <= bytes) return 0;
    size_t nb = std::max(need, bytes + bytes / 2);
    void* np = nullptr;
    cudaError_t e = cudaMalloc(&np, nb);
    if (e != cudaSuccess) return fail(SB200_ERR_CUDA, "cudaMalloc(%zu) failed: %s", nb, cudaGetErrorString(e));
    if (p) cudaFree(p);
    p = np;
    bytes = nb;
    return 0;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    bytes = 0;
  }
  template <typename T> T* as() const { return reinterpret_cast<T*>(p); }
};

// grow-only pinned host buffer (cudaHostAlloc with kFlags); owns its memory like DBuf.  With cudaHostAllocMapped it is
// also mapped into the device address space (dp): kernels can read it over PCIe without a copy-engine transfer.
template <unsigned kFlags> struct PinnedBuf {
  void* p = nullptr;
  void* dp = nullptr;   // device-side alias (mapped buffers only)
  size_t bytes = 0;
  PinnedBuf() = default;
  PinnedBuf(const PinnedBuf&) = delete;
  PinnedBuf& operator=(const PinnedBuf&) = delete;
  PinnedBuf(PinnedBuf&& o) noexcept : p(o.p), dp(o.dp), bytes(o.bytes) { o.p = o.dp = nullptr; o.bytes = 0; }
  PinnedBuf& operator=(PinnedBuf&& o) noexcept {
    if (this != &o) { release(); p = o.p; dp = o.dp; bytes = o.bytes; o.p = o.dp = nullptr; o.bytes = 0; }
    return *this;
  }
  ~PinnedBuf() { release(); }
  int ensure(size_t need) {
    if (need <= bytes) return 0;
    PinnedBuf nb;   // freed on failure
    const size_t n = std::max(need, bytes + bytes / 2);
    void* np = nullptr;
    cudaError_t e = cudaHostAlloc(&np, n, kFlags);
    if (e != cudaSuccess) return fail(SB200_ERR_CUDA, "cudaHostAlloc(%zu) failed: %s", n, cudaGetErrorString(e));
    nb.p = np;
    if (kFlags & cudaHostAllocMapped) {
      e = cudaHostGetDevicePointer(&nb.dp, nb.p, 0);
      if (e != cudaSuccess) return fail(SB200_ERR_CUDA, "cudaHostGetDevicePointer failed: %s", cudaGetErrorString(e));
    }
    nb.bytes = n;
    *this = std::move(nb);
    return 0;
  }
  void release() {
    if (p) cudaFreeHost(p);
    p = nullptr;
    dp = nullptr;
    bytes = 0;
  }
  template <typename T> T* as() const { return reinterpret_cast<T*>(p); }
};
using HBuf = PinnedBuf<cudaHostAllocMapped>;

}  // namespace sb
