// Shared helpers for libtwg.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <atomic>

#include "../../include/twg.h"

namespace twg {

extern thread_local char g_err[512];
extern std::atomic<int64_t> g_launches;

int fail(int code, const char* fmt, ...);
int check_launch(const char* what);

// Deterministic cross-block sums.  A kernel whose blocks would each add a partial sum into the same outputs instead stores
// block b's partial of output i at parts[b * n + i] (parts = partials(nb * n), zeroed when `zero`), and add_partials then
// adds them to out[i] in block order -- fp32 atomics would add them in whatever order the blocks finish, and the training
// step amplifies that last-bit noise into visibly different results from run to run.  The buffer is owned by the library
// (one per device), so kernels of this library must not run concurrently on two streams of one device.
float* partials(int64_t n, bool zero, cudaStream_t st);
int add_partials(float* out, const float* parts, int nb, int64_t n, cudaStream_t st);

inline cudaStream_t S(twg_stream_t s) { return reinterpret_cast<cudaStream_t>(s); }
inline int64_t cdiv(int64_t a, int64_t b) { return (a + b - 1) / b; }

constexpr float kLeak = 0.2f;        // util_misc.py:68
constexpr float kPixEps = 1e-6f;     // nets/pggan_utils.py:330
constexpr int kNumSMs = 132;         // H100 SXM: grid sizing (waves, split-K) only, never results

__device__ __forceinline__ float lrelu(float x) { return fmaxf(kLeak * x, x); }
__device__ __forceinline__ float lrelu_slope(float ref) { return ref > 0.f ? 1.f : kLeak; }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// sum across `g` consecutive lanes (g power of two <= 32)
__device__ __forceinline__ float group_sum(float v, int g) {
  for (int o = g >> 1; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// block-wide sum (blockDim.x multiple of 32, <= 1024); result valid in all threads
__device__ __forceinline__ float block_sum(float v, float* smem32) {
  v = warp_sum(v);
  int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) smem32[wid] = v;
  __syncthreads();
  int nw = (blockDim.x + 31) >> 5;
  float r = (threadIdx.x < nw) ? smem32[threadIdx.x] : 0.f;
  if (wid == 0) r = warp_sum(r);
  if (threadIdx.x == 0) smem32[0] = r;
  __syncthreads();
  r = smem32[0];
  return r;
}

#define TWG_LAUNCH_COUNT() (::twg::g_launches.fetch_add(1, std::memory_order_relaxed))

}  // namespace twg
