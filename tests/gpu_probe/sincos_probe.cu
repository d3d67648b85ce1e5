// Runs the product's sin / cos (sb::sc::sincos_cr, sb_sincos.cuh) and box vertices (sb::box_vertices, sb_math.cuh) on the
// device, next to the host build of the same headers in this executable, so that tests/test_gpu_sincos.py can compare the
// two bit for bit.  Compiled with the product's NVCC_FLAGS (and -ffp-contract=off for the host side).
//
//   sincos_probe sweep START STOP STRIDE
//       the f32 bit patterns START, START + STRIDE, ... < STOP (as 64-bit integers, STOP <= 2^32), widened to f64: sin and
//       cos on the device and on the host, the host's share split over every hardware thread.  stdout, one per line:
//       "count N", "mismatches N", up to 64 x "mismatch BITS" (hex f32 pattern), "seconds S" (wall time of the sweep).
//   sincos_probe args       stdin: int64 n, n f32 angles      stdout: n f64 sines, then n f64 cosines (device)
//   sincos_probe vertices   stdin: int64 n, n x 5 f32 boxes   stdout: n x 8 f64 vertices (device)
//                           (xc, yc, angle, aspect, height; NaN angle == axis-aligned, as in the product)
#include <algorithm>
#include <chrono>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <thread>
#include <vector>

#include "sb_math.cuh"

namespace {

__device__ __host__ __forceinline__ double widen(uint32_t bits) {
  float f;
  memcpy(&f, &bits, 4);
  return (double)f;
}

__global__ void sweep_kernel(uint64_t start, uint64_t stride, uint64_t n, double* s, double* c) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
    sb::sc::sincos_cr(widen((uint32_t)(start + i * stride)), &s[i], &c[i]);
}

__global__ void args_kernel(const float* a, int64_t n, double* s, double* c) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    sb::sc::sincos_cr((double)a[i], &s[i], &c[i]);
}

__global__ void vertices_kernel(const float* b, int64_t n, double* v) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    sb::box_vertices(b[5 * i], b[5 * i + 1], b[5 * i + 2], b[5 * i + 3], b[5 * i + 4], v + 8 * i);
}

int fail(const char* what, cudaError_t e = cudaSuccess) {
  fprintf(stderr, "sincos_probe: %s %s\n", what, e == cudaSuccess ? "" : cudaGetErrorString(e));
  return 1;
}

bool same_bits(double a, double b) { return memcmp(&a, &b, 8) == 0; }

int sweep(uint64_t start, uint64_t stop, uint64_t stride) {
  if (stride == 0 || start >= stop || stop > (1ull << 32)) return fail("bad sweep range");
  const uint64_t total = (stop - start + stride - 1) / stride;
  const uint64_t chunk = 1ull << 24;
  double *ds = nullptr, *dc = nullptr;
  cudaError_t e;
  if ((e = cudaMalloc(&ds, chunk * 8)) || (e = cudaMalloc(&dc, chunk * 8))) return fail("cudaMalloc", e);
  std::vector<double> hs(chunk), hc(chunk);
  const int nt = std::max(1u, std::thread::hardware_concurrency());
  std::vector<uint64_t> bad;
  uint64_t n_bad = 0;
  const auto t0 = std::chrono::steady_clock::now();
  for (uint64_t done = 0; done < total; done += chunk) {
    const uint64_t n = std::min(chunk, total - done);
    const uint64_t first = start + done * stride;
    sweep_kernel<<<132 * 16, 256>>>(first, stride, n, ds, dc);
    if ((e = cudaGetLastError()) || (e = cudaMemcpy(hs.data(), ds, n * 8, cudaMemcpyDeviceToHost)) ||
        (e = cudaMemcpy(hc.data(), dc, n * 8, cudaMemcpyDeviceToHost)))
      return fail("sweep kernel", e);
    std::vector<std::vector<uint64_t>> t_bad(nt);
    std::vector<uint64_t> t_n(nt, 0);
    std::vector<std::thread> pool;
    for (int t = 0; t < nt; ++t)
      pool.emplace_back([&, t] {
        for (uint64_t i = t * n / nt; i < (t + 1) * n / nt; ++i) {
          const uint64_t bits = first + i * stride;
          double s, c;
          sb::sc::sincos_cr(widen((uint32_t)bits), &s, &c);
          if (!same_bits(s, hs[i]) || !same_bits(c, hc[i])) {
            if (t_bad[t].size() < 64) t_bad[t].push_back(bits);
            ++t_n[t];
          }
        }
      });
    for (auto& th : pool) th.join();
    for (int t = 0; t < nt; ++t) {
      n_bad += t_n[t];
      for (uint64_t b : t_bad[t])
        if (bad.size() < 64) bad.push_back(b);
    }
  }
  const double secs = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  printf("count %llu\nmismatches %llu\n", (unsigned long long)total, (unsigned long long)n_bad);
  for (uint64_t b : bad) printf("mismatch %08llx\n", (unsigned long long)b);
  printf("threads %d\nseconds %.3f\n", nt, secs);
  cudaFree(ds);
  cudaFree(dc);
  return 0;
}

template <class T>
bool read_all(std::vector<T>& v) { return fread(v.data(), sizeof(T), v.size(), stdin) == v.size(); }

int args_or_vertices(bool vertices) {
  int64_t n = 0;
  if (fread(&n, 8, 1, stdin) != 1 || n <= 0) return fail("bad count");
  const int64_t in_w = vertices ? 5 : 1, out_w = vertices ? 8 : 2;
  std::vector<float> in(n * in_w);
  std::vector<double> out(n * out_w);
  if (!read_all(in)) return fail("short input");
  float* din = nullptr;
  double* dout = nullptr;
  cudaError_t e;
  if ((e = cudaMalloc(&din, in.size() * 4)) || (e = cudaMalloc(&dout, out.size() * 8))) return fail("cudaMalloc", e);
  cudaMemcpy(din, in.data(), in.size() * 4, cudaMemcpyHostToDevice);
  if (vertices) vertices_kernel<<<264, 256>>>(din, n, dout);
  else args_kernel<<<264, 256>>>(din, n, dout, dout + n);
  if ((e = cudaGetLastError()) || (e = cudaMemcpy(out.data(), dout, out.size() * 8, cudaMemcpyDeviceToHost)))
    return fail("kernel", e);
  fwrite(out.data(), 8, out.size(), stdout);
  cudaFree(din);
  cudaFree(dout);
  return 0;
}

}  // namespace

int main(int argc, char** argv) {
  if (argc == 5 && !strcmp(argv[1], "sweep"))
    return sweep(strtoull(argv[2], nullptr, 0), strtoull(argv[3], nullptr, 0), strtoull(argv[4], nullptr, 0));
  if (argc == 2 && !strcmp(argv[1], "args")) return args_or_vertices(false);
  if (argc == 2 && !strcmp(argv[1], "vertices")) return args_or_vertices(true);
  return fail("usage: sincos_probe sweep START STOP STRIDE | args | vertices");
}
