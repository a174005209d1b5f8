// Shared helpers for libtwg.so (sm_90a only).
#pragma once
#include <cuda_bf16.h>
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

// blocks of 256 threads for a grid-stride loop over n items, `per_thread` each, at most 16 blocks per SM
static inline int grid_for(int64_t n, int per_thread = 4) {
  int64_t b = cdiv(n, (int64_t)256 * per_thread);
  int64_t cap = (int64_t)kNumSMs * 16;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (int)b;
}

// Channel-vector geometry: a pixel's C channels are C/4 float4; G lanes cooperate on one pixel, each lane owning V float4
// (lane, lane+32, ...).
struct VecGeom {
  int G, V;
  bool ok;
};
static inline VecGeom vec_geom(int C) {
  VecGeom g{0, 0, false};
  if (C % 4) return g;
  int q = C / 4;
  if (q <= 32) {
    if (q & (q - 1)) return g;
    g.G = q;
    g.V = 1;
    g.ok = true;
  } else {
    if (q % 32 || q / 32 > 4 || (q / 32 == 3)) return g;
    g.G = 32;
    g.V = q / 32;
    g.ok = true;
  }
  return g;
}

__device__ __forceinline__ float lrelu(float x) { return fmaxf(kLeak * x, x); }
__device__ __forceinline__ float lrelu_slope(float ref) { return ref > 0.f ? 1.f : kLeak; }

__device__ __forceinline__ float4 ld4(const float* p, int64_t i4) { return reinterpret_cast<const float4*>(p)[i4]; }
__device__ __forceinline__ void st4(float* p, int64_t i4, float4 v) { reinterpret_cast<float4*>(p)[i4] = v; }

// ---- split-bf16 planes, the operand format of the tensor-core convs -------------------------------------------------
// x = hi + lo with hi = bf16_rn(x), lo = bf16_rn(x - hi).  A tensor of n elements is stored as the hi plane [n] followed
// by the lo plane [n] (bf16, the fp32 tensor's element order).  Two values per conversion instruction (cvt.rn.bf16x2.f32,
// the same round-to-nearest-even as the scalar conversion).
struct Split2 {
  __nv_bfloat162 hi, lo;
};
__device__ __forceinline__ Split2 split2(float a, float b) {
  Split2 s;
  s.hi = __floats2bfloat162_rn(a, b);
  const float2 f = __bfloat1622float2(s.hi);
  s.lo = __floats2bfloat162_rn(a - f.x, b - f.y);
  return s;
}
// element i of an n-element tensor
__device__ __forceinline__ void st_split1(void* planes, int64_t n, int64_t i, float x) {
  const Split2 s = split2(x, x);
  __nv_bfloat16* hi = reinterpret_cast<__nv_bfloat16*>(planes);
  hi[i] = s.hi.x;
  hi[n + i] = s.lo.x;
}
// elements e, e + 1 (e even)
__device__ __forceinline__ void st_planes2(void* planes, int64_t n, int64_t e, float a, float b) {
  const Split2 s = split2(a, b);
  __nv_bfloat16* hi = reinterpret_cast<__nv_bfloat16*>(planes);
  *reinterpret_cast<__nv_bfloat162*>(hi + e) = s.hi;
  *reinterpret_cast<__nv_bfloat162*>(hi + n + e) = s.lo;
}
// elements 4 i4 .. 4 i4 + 3: split2 of (x, y) and (z, w), with both hi conversions issued before the lo ones (the
// instruction order every memory-bound kernel that stores planes was tuned with)
__device__ __forceinline__ void st_split4(void* planes, int64_t n, int64_t i4, float4 v) {
  const __nv_bfloat162 h01 = __floats2bfloat162_rn(v.x, v.y), h23 = __floats2bfloat162_rn(v.z, v.w);
  const float2 f01 = __bfloat1622float2(h01), f23 = __bfloat1622float2(h23);
  const __nv_bfloat162 l01 = __floats2bfloat162_rn(v.x - f01.x, v.y - f01.y), l23 = __floats2bfloat162_rn(v.z - f23.x, v.w - f23.y);
  uint2 hv, lv;
  hv.x = *reinterpret_cast<const uint32_t*>(&h01); hv.y = *reinterpret_cast<const uint32_t*>(&h23);
  lv.x = *reinterpret_cast<const uint32_t*>(&l01); lv.y = *reinterpret_cast<const uint32_t*>(&l23);
  __nv_bfloat16* hi = reinterpret_cast<__nv_bfloat16*>(planes);
  reinterpret_cast<uint2*>(hi)[i4] = hv;
  reinterpret_cast<uint2*>(hi + n)[i4] = lv;
}

// ---- reductions -------------------------------------------------------------------------------------------------------
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
// Sum of v over the threads of a 256-thread block that share threadIdx.x % g (g a power of two <= 256): a tree over
// sm[256] from stride 128 down to g, so the order of the additions is fixed.  The result is valid in threads < g.
__device__ __forceinline__ float block_tree_sum(float v, int g, float* sm) {
  __syncthreads();
  sm[threadIdx.x] = v;
  __syncthreads();
  for (int s = 128; s >= g; s >>= 1) {
    if (threadIdx.x < s) sm[threadIdx.x] += sm[threadIdx.x + s];
    __syncthreads();
  }
  return sm[threadIdx.x];
}

}  // namespace twg
