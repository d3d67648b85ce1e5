// Measures the FP8 tensor-core accumulation the e4m3 screen's bound assumes (screen_rel_err_fp8, sb_engine.cuh).
//
// One warpgroup computes D[64 x 128] = A[64 x K] B[128 x K]^T with wgmma_e4m3_m64n128 (sb_tc.cuh), chained over `steps`
// k32 steps exactly as the screen kernels advance it: operand tiles of 128 bytes (128 e4m3 values) per row in the
// 128-byte-swizzle K-major layout the screen's TMA maps produce, descriptors wgmma_desc(tile + 32 k) for k = 0..3 inside a
// tile.  The operands are written into shared memory with plain stores, not TMA, so the probe checks that layout too.
//
// stdin:  n_cases, then per case: int32 steps (1..16), A as 64 x 512 e4m3 bytes, B as 128 x 512 e4m3 bytes (row-major,
//         byte k of a row is feature k; features past 32 * steps are not read)
// stdout: per case, the 64 x 128 fp32 accumulators, row-major, as raw bytes
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "sb_tc.cuh"

namespace {

constexpr int kRowsA = 64, kRowsB = 128, kMaxK = 512, kTile = 128;   // kTile: bytes of a swizzle row
constexpr int kTiles = kMaxK / kTile;
constexpr int kSmem = kTiles * (kRowsA + kRowsB) * kTile + 1024;     // + alignment of the 1024-byte swizzle atoms

// byte offset of (row r, byte c) of a tile: 16-byte chunk c / 16 of row r lands in chunk (c / 16) ^ (r % 8)
__device__ __forceinline__ int swz(int r, int c) { return r * kTile + ((((c >> 4) ^ (r & 7)) << 4) | (c & 15)); }

__global__ void __launch_bounds__(128) probe_kernel(const unsigned char* A, const unsigned char* B, int steps, float* out) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char* sa = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  unsigned char* sb = sa + kTiles * kRowsA * kTile;
  for (int i = threadIdx.x; i < kRowsA * kMaxK; i += blockDim.x) {
    const int r = i / kMaxK, k = i % kMaxK;
    sa[(k / kTile) * kRowsA * kTile + swz(r, k % kTile)] = A[i];
  }
  for (int i = threadIdx.x; i < kRowsB * kMaxK; i += blockDim.x) {
    const int r = i / kMaxK, k = i % kMaxK;
    sb[(k / kTile) * kRowsB * kTile + swz(r, k % kTile)] = B[i];
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy stores -> visible to wgmma
  __syncthreads();

  float acc[128];   // wgmma_fence_acc covers 128 registers; the m64n128 MMA uses the first 64
#pragma unroll
  for (int i = 0; i < 128; ++i) acc[i] = 0.0f;
  sb::wgmma_fence();
  for (int s = 0; s < steps; ++s) {
    const int t = s / 4, k = s % 4;
    sb::wgmma_e4m3_m64n128(acc, sb::wgmma_desc(sb::smem_u32(sa + t * kRowsA * kTile) + k * 32),
                           sb::wgmma_desc(sb::smem_u32(sb + t * kRowsB * kTile) + k * 32), s != 0 ? 1u : 0u);
  }
  sb::wgmma_commit();
  sb::wgmma_wait<0>();
  sb::wgmma_fence_acc(acc);

  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
#pragma unroll
  for (int i = 0; i < 64; ++i) {
    const int row = warp * 16 + lane / 4 + 8 * ((i >> 1) & 1);
    const int col = 8 * (i >> 2) + 2 * (lane % 4) + (i & 1);
    out[row * kRowsB + col] = acc[i];
  }
}

int fail(const char* what, cudaError_t e = cudaSuccess) {
  fprintf(stderr, "fp8_wgmma_probe: %s %s\n", what, e == cudaSuccess ? "" : cudaGetErrorString(e));
  return 1;
}

}  // namespace

int main() {
  int n_cases = 0;
  if (fread(&n_cases, 4, 1, stdin) != 1 || n_cases <= 0) return fail("bad case count");
  unsigned char *dA = nullptr, *dB = nullptr;
  float* dOut = nullptr;
  cudaError_t e;
  if ((e = cudaMalloc(&dA, kRowsA * kMaxK)) || (e = cudaMalloc(&dB, kRowsB * kMaxK)) ||
      (e = cudaMalloc(&dOut, sizeof(float) * kRowsA * kRowsB)))
    return fail("cudaMalloc", e);
  if ((e = cudaFuncSetAttribute(probe_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem)))
    return fail("smem attribute", e);
  std::vector<unsigned char> a(kRowsA * kMaxK), b(kRowsB * kMaxK);
  std::vector<float> out(kRowsA * kRowsB);
  for (int c = 0; c < n_cases; ++c) {
    int steps = 0;
    if (fread(&steps, 4, 1, stdin) != 1 || steps < 1 || steps > kMaxK / 32) return fail("bad step count");
    if (fread(a.data(), 1, a.size(), stdin) != a.size() || fread(b.data(), 1, b.size(), stdin) != b.size())
      return fail("short operands");
    cudaMemcpy(dA, a.data(), a.size(), cudaMemcpyHostToDevice);
    cudaMemcpy(dB, b.data(), b.size(), cudaMemcpyHostToDevice);
    probe_kernel<<<1, 128, kSmem>>>(dA, dB, steps, dOut);
    if ((e = cudaGetLastError()) || (e = cudaMemcpy(out.data(), dOut, sizeof(float) * out.size(), cudaMemcpyDeviceToHost)))
      return fail("probe kernel", e);
    fwrite(out.data(), sizeof(float), out.size(), stdout);
  }
  cudaFree(dA);
  cudaFree(dB);
  cudaFree(dOut);
  return 0;
}
