// Memory-bound kernels of the TwinGAN step: normaliser + leaky-ReLU + pixel-norm (forward and both
// backward passes), resampling, UNet join, minibatch-stddev (incl. double backward), losses, DRAGAN
// helpers, Adam.  All NHWC fp32, vectorised float4 along C, coalesced; reductions are hierarchical
// (registers -> shared -> one atomic per (block, channel)).
#include <stdarg.h>
#include <string.h>

#include <cuda_bf16.h>
#include <cooperative_groups.h>

#include "twg_common.cuh"

namespace cg = cooperative_groups;

namespace twg {

thread_local char g_err[512] = {0};
std::atomic<int64_t> g_launches{0};

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

int check_launch(const char* what) {
  g_launches.fetch_add(1, std::memory_order_relaxed);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(TWG_ERR_CUDA, "%s: %s", what, cudaGetErrorString(e));
  return TWG_OK;
}

constexpr int64_t kPartialFloats = 8 << 20;        // 32 MB: the largest user is the tensor-core weight gradient (<= ~5 M)
__device__ float g_partials[kPartialFloats];

float* partials(int64_t n, bool zero, cudaStream_t st) {
  if (n > kPartialFloats) return nullptr;
  void* p = nullptr;
  if (cudaGetSymbolAddress(&p, g_partials) != cudaSuccess) return nullptr;
  if (zero) cudaMemsetAsync(p, 0, sizeof(float) * n, st);
  return static_cast<float*>(p);
}

__global__ void __launch_bounds__(256) k_add_partials(float* __restrict__ out, const float* __restrict__ parts, int nb,
                                                      int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int b = 0; b < nb; ++b) s += parts[(int64_t)b * n + i];
    out[i] += s;
  }
}

int add_partials(float* out, const float* parts, int nb, int64_t n, cudaStream_t st) {
  int64_t blocks = cdiv(n, 256);
  if (blocks > 4 * kNumSMs) blocks = 4 * kNumSMs;
  k_add_partials<<<(unsigned)blocks, 256, 0, st>>>(out, parts, nb, n);
  return check_launch("add_partials");
}

// ------------------------------------------------------------------------------------------------
// Channel-vector geometry: a pixel's C channels are C/4 float4; G lanes cooperate on one pixel,
// each lane owning V float4 (lane, lane+32, ...).
// ------------------------------------------------------------------------------------------------
struct VecGeom {
  int G, V;
  bool ok;
};
static VecGeom vec_geom(int C) {
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

__device__ __forceinline__ float4 ld4(const float* p, int64_t i4) { return reinterpret_cast<const float4*>(p)[i4]; }
// split-bf16 planes (x = hi + lo): hi plane [n] then lo plane [n] bf16; i4 indexes groups of 4 elements
__device__ __forceinline__ void st_split4(void* planes, int64_t n_total, int64_t i4, float4 v) {
  // hi = bf16(x), lo = bf16(x - hi), two values per conversion instruction (cvt.rn.bf16x2.f32); same rounding as the scalar form
  const __nv_bfloat162 h01 = __floats2bfloat162_rn(v.x, v.y), h23 = __floats2bfloat162_rn(v.z, v.w);
  const float2 f01 = __bfloat1622float2(h01), f23 = __bfloat1622float2(h23);
  const __nv_bfloat162 l01 = __floats2bfloat162_rn(v.x - f01.x, v.y - f01.y), l23 = __floats2bfloat162_rn(v.z - f23.x, v.w - f23.y);
  uint2 hv, lv;
  hv.x = *reinterpret_cast<const uint32_t*>(&h01); hv.y = *reinterpret_cast<const uint32_t*>(&h23);
  lv.x = *reinterpret_cast<const uint32_t*>(&l01); lv.y = *reinterpret_cast<const uint32_t*>(&l23);
  __nv_bfloat16* hi = reinterpret_cast<__nv_bfloat16*>(planes);
  reinterpret_cast<uint2*>(hi)[i4] = hv;
  reinterpret_cast<uint2*>(hi + n_total)[i4] = lv;
}
__device__ __forceinline__ void st4(float* p, int64_t i4, float4 v) { reinterpret_cast<float4*>(p)[i4] = v; }

// ------------------------------------------------------------------------------------------------
// moments: sums[n][c] = {sum y, sum y^2}
// ------------------------------------------------------------------------------------------------
// Shifted sums: sums[n][c] = {sum (y - p), sum (y - p)^2} with the pivot p = y[first sample of n's pivot group][pixel 0][c].
// tf.nn.moments is two-pass; a single pass over raw y, y^2 in fp32 cancels catastrophically once |mean| >> std
// (relative variance error ~ 6e-8 * mean^2 / var).  With a pivot drawn from the data the shifted mean is O(std).
template <int V>
__global__ void __launch_bounds__(256) k_moments_vec(const float* __restrict__ y, float* __restrict__ sums, int HW,
                                                     int C, int G, int chunk, int pivot_group) {
  __shared__ float sm[256];
  const int n = blockIdx.y, q = C / 4;
  const int gpb = 256 / G, grp = threadIdx.x / G, lg = threadIdx.x % G;
  const int p0 = blockIdx.x * chunk, p1 = min(HW, p0 + chunk);
  float4 pv[V];
#pragma unroll
  for (int v = 0; v < V; ++v) pv[v] = ld4(y, (int64_t)(n / pivot_group * pivot_group) * HW * q + lg + v * 32);
  float acc[8 * V];
#pragma unroll
  for (int i = 0; i < 8 * V; ++i) acc[i] = 0.f;
  constexpr int U = (V == 1) ? 4 : (V == 2 ? 2 : 1);     // pixels in flight per thread: enough bytes outstanding to cover HBM latency
  for (int pb = p0 + grp; pb < p1; pb += gpb * U) {
    float4 t[U][V];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int p = pb + u * gpb;
      const int64_t base = ((int64_t)n * HW + (p < p1 ? p : p0)) * q;
#pragma unroll
      for (int v = 0; v < V; ++v) t[u][v] = ld4(y, base + lg + v * 32);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (pb + u * gpb >= p1) continue;
#pragma unroll
      for (int v = 0; v < V; ++v) {
        float4 d = t[u][v];
        d.x -= pv[v].x; d.y -= pv[v].y; d.z -= pv[v].z; d.w -= pv[v].w;
        acc[8 * v + 0] += d.x; acc[8 * v + 1] += d.y; acc[8 * v + 2] += d.z; acc[8 * v + 3] += d.w;
        acc[8 * v + 4] += d.x * d.x; acc[8 * v + 5] += d.y * d.y; acc[8 * v + 6] += d.z * d.z; acc[8 * v + 7] += d.w * d.w;
      }
    }
  }
#pragma unroll
  for (int k = 0; k < 8 * V; ++k) {
    __syncthreads();
    sm[threadIdx.x] = acc[k];
    __syncthreads();
    for (int s = 128; s >= G; s >>= 1) {
      if (threadIdx.x < s) sm[threadIdx.x] += sm[threadIdx.x + s];
      __syncthreads();
    }
    if (threadIdx.x < G) {
      int v = k / 8, j = k % 8;
      int c = (lg + v * 32) * 4 + (j & 3);
      atomicAdd(&sums[((int64_t)n * C + c) * 2 + (j >> 2)], sm[threadIdx.x]);
    }
  }
}

__global__ void __launch_bounds__(256) k_moments_scalar(const float* __restrict__ y, float* __restrict__ sums, int HW,
                                                        int C, int chunk, int pivot_group) {
  __shared__ float sm[32];
  const int n = blockIdx.y;
  const int p0 = blockIdx.x * chunk, p1 = min(HW, p0 + chunk);
  for (int c = 0; c < C; ++c) {
    const float pv = y[(int64_t)(n / pivot_group * pivot_group) * HW * C + c];
    float a1 = 0.f, a2 = 0.f;
    for (int p = p0 + threadIdx.x; p < p1; p += blockDim.x) {
      float t = y[((int64_t)n * HW + p) * C + c] - pv;
      a1 += t;
      a2 += t * t;
    }
    a1 = block_sum(a1, sm);
    a2 = block_sum(a2, sm);
    if (threadIdx.x == 0) {
      atomicAdd(&sums[((int64_t)n * C + c) * 2 + 0], a1);
      atomicAdd(&sums[((int64_t)n * C + c) * 2 + 1], a2);
    }
  }
}

// One block per sample covers all HW pixels, so every per-(n, c) sum has exactly one writer and comes out the same on
// every run (several blocks per sample would add their partials in a varying order).
static int pick_chunk(int HW, int N, int pixels_per_pass) {
  (void)N; (void)pixels_per_pass;
  return HW;
}

// ------------------------------------------------------------------------------------------------
// finalize: sums -> per-(n,c) affine + saved mean/rstd
// ------------------------------------------------------------------------------------------------
// The batch is `N / gs` groups of `gs` samples (one group per original network pass when passes that share conv
// weights are batched); bit g of dom_mask selects the group's domain, i.e. which gamma/beta (and renorm state) it uses.
// Instance norm: statistics per (n, c).  Batch kinds: statistics over the group's samples.  `y` is only read for the
// pivots of the shifted sums (k_moments_*).  `clip` (device, nullable) = {rmin, rmax, dmax}.
__global__ void k_norm_finalize(const float* __restrict__ sums, const float* __restrict__ y,
                                const float* __restrict__ gamma0, const float* __restrict__ beta0,
                                const float* __restrict__ gamma1, const float* __restrict__ beta1, unsigned dom_mask, int gs,
                                const float* __restrict__ renorm0, const float* __restrict__ renorm1, int kind, float eps,
                                const float* __restrict__ clip, float* __restrict__ a, float* __restrict__ b,
                                float* __restrict__ mean_o, float* __restrict__ rstd_o, float* __restrict__ rd_out,
                                float* __restrict__ batch_stats, int N, int HW, int C) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float rmin = clip ? clip[0] : 1.f, rmax = clip ? clip[1] : 1.f, dmax = clip ? clip[2] : 0.f;
  const int groups = N / gs;
  for (int grp = 0; grp < groups; ++grp) {
    const int dom = (dom_mask >> grp) & 1u;
    const float* gamma = dom ? gamma1 : gamma0;
    const float* beta = dom ? beta1 : beta0;
    const float g = gamma ? gamma[c] : 1.f, be = beta ? beta[c] : 0.f;
    const int n0 = grp * gs, n1 = n0 + gs;
    if (kind == TWG_NORM_NONE) {
      for (int n = n0; n < n1; ++n) {
        a[n * C + c] = 1.f; b[n * C + c] = be; mean_o[n * C + c] = 0.f; rstd_o[n * C + c] = 1.f;
      }
      continue;
    }
    if (kind == TWG_NORM_INSTANCE) {
      const float inv = 1.f / (float)HW;
      for (int n = n0; n < n1; ++n) {
        const float pv = y[(int64_t)n * HW * C + c];
        float d1 = sums[(n * C + c) * 2] * inv;
        float var = fmaxf(sums[(n * C + c) * 2 + 1] * inv - d1 * d1, 0.f);
        float m = pv + d1;
        float rs = rsqrtf(var + eps);
        float aa = g * rs;
        a[n * C + c] = aa; b[n * C + c] = be - m * aa; mean_o[n * C + c] = m; rstd_o[n * C + c] = rs;
      }
      continue;
    }
    const float pv = y[(int64_t)n0 * HW * C + c];
    float s1 = 0.f, s2 = 0.f;
    for (int n = n0; n < n1; ++n) { s1 += sums[(n * C + c) * 2]; s2 += sums[(n * C + c) * 2 + 1]; }
    const float inv = 1.f / ((float)HW * (float)gs);
    const float d1 = s1 * inv;
    float m = pv + d1;
    float var = fmaxf(s2 * inv - d1 * d1, 0.f);
    float rs = rsqrtf(var + eps);
    float r = 1.f, d = 0.f;
    float second = var;
    if (kind == TWG_NORM_RENORM) {
      const float* renorm = dom ? renorm1 : renorm0;
      float stddev = sqrtf(var + eps);
      float rm = renorm[c], rsd = renorm[C + c], rmw = renorm[2 * C], rsw = renorm[2 * C + 1];
      float mixed_mean = rm + (1.f - rmw) * m;
      float mixed_std = rsd + (1.f - rsw) * stddev;
      r = fminf(fmaxf(stddev / mixed_std, rmin), rmax);
      d = fminf(fmaxf((m - mixed_mean) / mixed_std, -dmax), dmax);
      second = stddev;
    }
    float aa = g * r * rs;
    float bb = d * g + be - m * aa;
    for (int n = n0; n < n1; ++n) { a[n * C + c] = aa; b[n * C + c] = bb; mean_o[n * C + c] = m; rstd_o[n * C + c] = rs; }
    if (rd_out) { rd_out[grp * 2 * C + c] = r; rd_out[grp * 2 * C + C + c] = d; }
    if (batch_stats) { batch_stats[grp * 2 * C + c] = m; batch_stats[grp * 2 * C + C + c] = second; }
  }
}

// Instance norm: every (n, c) is independent, so one thread per (n, c) instead of one thread per channel looping over the
// batch (which made these two tiny kernels ~15 us of pure latency each at 64 samples, ~160 launches per step).
__global__ void __launch_bounds__(256) k_norm_finalize_inst(const float* __restrict__ sums, const float* __restrict__ y,
                                                            const float* __restrict__ gamma0, const float* __restrict__ beta0,
                                                            const float* __restrict__ gamma1, const float* __restrict__ beta1,
                                                            unsigned dom_mask, int gs, float eps, float* __restrict__ a,
                                                            float* __restrict__ b, float* __restrict__ mean_o,
                                                            float* __restrict__ rstd_o, int N, int HW, int C) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= N * C) return;
  const int n = idx / C, c = idx - n * C;
  const int dom = (dom_mask >> (n / gs)) & 1u;
  const float* gamma = dom ? gamma1 : gamma0;
  const float* beta = dom ? beta1 : beta0;
  const float g = gamma ? gamma[c] : 1.f, be = beta ? beta[c] : 0.f;
  const float inv = 1.f / (float)HW;
  const float pv = y[(int64_t)n * HW * C + c];
  const float d1 = sums[idx * 2] * inv;
  const float var = fmaxf(sums[idx * 2 + 1] * inv - d1 * d1, 0.f);
  const float m = pv + d1;
  const float rs = rsqrtf(var + eps);
  const float aa = g * rs;
  a[idx] = aa; b[idx] = be - m * aa; mean_o[idx] = m; rstd_o[idx] = rs;
}

// Instance norm from the conv epilogue's records (k_conv_halo_tc): stats[n][slot][c] = {count, pivot, sum (y - pivot),
// sum (y - pivot)^2} over the pixels one epilogue warp drained.  One warp per (n, c) re-bases every record to the first
// record's pivot p0 (sum (y - p0) = S1 + n d, sum (y - p0)^2 = S2 + 2 d S1 + n d^2 with d = pivot - p0) and takes
// var = E[(y - p0)^2] - E[y - p0]^2: all pivots are values of the data, so every term is O(std) and the |mean| >> std case
// keeps the accuracy of tf.nn.moments' two-pass form (same argument as k_moments_*).  One pass over the records, four
// loads in flight per lane.
__global__ void __launch_bounds__(256) k_norm_finalize_inst_partials(
    const float4* __restrict__ stats, int slots, const float* __restrict__ gamma0, const float* __restrict__ beta0,
    const float* __restrict__ gamma1, const float* __restrict__ beta1, unsigned dom_mask, int gs, float eps,
    float* __restrict__ a, float* __restrict__ b, float* __restrict__ mean_o, float* __restrict__ rstd_o, int N, int C) {
  const int idx = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (idx >= N * C) return;
  const int n = idx / C, c = idx - n * C;
  const float4* rec = stats + (int64_t)n * slots * C + c;
  const float p0 = rec[0].y;
  float cn = 0.f, sm = 0.f, q = 0.f;
  for (int s0 = lane; s0 < slots; s0 += 128) {
    float4 r[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int s = s0 + 32 * u;
      r[u] = s < slots ? rec[(int64_t)s * C] : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (r[u].x > 0.f) {
        const float d = r[u].y - p0;
        cn += r[u].x;
        sm += fmaf(d, r[u].x, r[u].z);
        q += r[u].w + d * fmaf(d, r[u].x, 2.f * r[u].z);
      }
    }
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    cn += __shfl_xor_sync(0xffffffffu, cn, off);
    sm += __shfl_xor_sync(0xffffffffu, sm, off);
    q += __shfl_xor_sync(0xffffffffu, q, off);
  }
  if (lane == 0) {
    const int dom = (dom_mask >> (n / gs)) & 1u;
    const float* gamma = dom ? gamma1 : gamma0;
    const float* beta = dom ? beta1 : beta0;
    const float g = gamma ? gamma[c] : 1.f, be = beta ? beta[c] : 0.f;
    const float inv = 1.f / cn;
    const float dm = sm * inv;                     // mean - p0
    const float m = p0 + dm;
    const float rs = rsqrtf(fmaxf(q * inv - dm * dm, 0.f) + eps);
    const float aa = g * rs;
    a[idx] = aa; b[idx] = be - m * aa; mean_o[idx] = m; rstd_o[idx] = rs;
  }
}

// red[n][c] -> {S1/HW, S2/HW}; parameter gradients += over the samples of each domain (outputs must be zeroed or be
// accumulation targets: the host clears fresh buffers first)
__global__ void __launch_bounds__(256) k_norm_bwd_coeffs_inst(float* __restrict__ red, float* __restrict__ ggamma0,
                                                              float* __restrict__ gbeta0, float* __restrict__ ggamma1,
                                                              float* __restrict__ gbeta1, unsigned dom_mask, int gs, int N,
                                                              int HW, int C) {
  // one thread per channel adds the samples in order (deterministic parameter gradients)
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float inv = 1.f / (float)HW;
  for (int n = 0; n < N; ++n) {
    const int idx = n * C + c;
    const int dom = (dom_mask >> (n / gs)) & 1u;
    const float t1 = red[idx * 2], t2 = red[idx * 2 + 1];
    float* gg = dom ? ggamma1 : ggamma0;
    float* gb = dom ? gbeta1 : gbeta0;
    if (gg) gg[c] += t2;
    if (gb) gb[c] += t1;
    red[idx * 2] = t1 * inv;
    red[idx * 2 + 1] = t2 * inv;
  }
}

__global__ void k_norm_eval_affine(const float* __restrict__ gamma, const float* __restrict__ beta,
                                   const float* __restrict__ mm, const float* __restrict__ mv, float eps,
                                   float* __restrict__ a, float* __restrict__ b, int N, int C) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float aa = gamma[c] * rsqrtf(mv[c] + eps);
  float bb = beta[c] - mm[c] * aa;
  for (int n = 0; n < N; ++n) { a[n * C + c] = aa; b[n * C + c] = bb; }
}

__global__ void k_norm_update_stats(float* __restrict__ st, const float* __restrict__ bs, int kind, float decay,
                                    float eps, int C) {
  // single block, blockDim.x >= C
  int c = threadIdx.x;
  float* mm = st; float* mv = st + C; float* rm = st + 2 * C; float* rs = st + 3 * C;
  float wm_old = st[4 * C], ws_old = st[4 * C + 1];
  __syncthreads();
  float om = 1.f - decay;
  if (c < C) {
    if (kind == TWG_NORM_RENORM) {
      float nrm = rm[c] * decay + bs[c] * om;
      float nrs = rs[c] * decay + bs[C + c] * om;
      float wm = wm_old * decay + om, ws = ws_old * decay + om;
      rm[c] = nrm; rs[c] = nrs;
      float new_mean = nrm / wm, new_std = nrs / ws;
      mm[c] = mm[c] * decay + new_mean * om;
      mv[c] = mv[c] * decay + (new_std * new_std - eps) * om;
    } else {
      mm[c] = mm[c] * decay + bs[c] * om;
      mv[c] = mv[c] * decay + bs[C + c] * om;
    }
  }
  if (c == 0 && kind == TWG_NORM_RENORM) { st[4 * C] = wm_old * decay + om; st[4 * C + 1] = ws_old * decay + om; }
}

// ------------------------------------------------------------------------------------------------
// forward apply
// ------------------------------------------------------------------------------------------------
template <int V>
__global__ void __launch_bounds__(256) k_norm_act_fwd_vec(const float* __restrict__ y, const float* __restrict__ a,
                                                          const float* __restrict__ b, float* __restrict__ z,
                                                          void* __restrict__ planes, int64_t total, int HW, int C, int G,
                                                          int flags) {
  const int q = C / 4, gpb = 256 / G, grp = threadIdx.x / G, lg = threadIdx.x % G;
  const bool act = flags & TWG_FLAG_LRELU, pix = flags & TWG_FLAG_PIXNORM;
  const float invC = 1.f / (float)C;
  for (int64_t base = (int64_t)blockIdx.x * gpb; base < total; base += (int64_t)gridDim.x * gpb) {
    const int64_t p = base + grp;
    const bool valid = p < total;
    const int n = valid ? (int)(p / HW) : 0;
    float4 u[V];
    float ss = 0.f;
#pragma unroll
    for (int v = 0; v < V; ++v) {
      const int cq = lg + v * 32;
      float4 yy = valid ? ld4(y, p * q + cq) : make_float4(0, 0, 0, 0);
      float4 aa = ld4(a, (int64_t)n * q + cq), bb = ld4(b, (int64_t)n * q + cq);
      float4 t = make_float4(fmaf(aa.x, yy.x, bb.x), fmaf(aa.y, yy.y, bb.y), fmaf(aa.z, yy.z, bb.z), fmaf(aa.w, yy.w, bb.w));
      if (act) { t.x = lrelu(t.x); t.y = lrelu(t.y); t.z = lrelu(t.z); t.w = lrelu(t.w); }
      ss += t.x * t.x + t.y * t.y + t.z * t.z + t.w * t.w;
      u[v] = t;
    }
    if (pix) {
      ss = group_sum(ss, G);
      const float rinv = rsqrtf(ss * invC + kPixEps);
#pragma unroll
      for (int v = 0; v < V; ++v) { u[v].x *= rinv; u[v].y *= rinv; u[v].z *= rinv; u[v].w *= rinv; }
    }
    if (valid) {
#pragma unroll
      for (int v = 0; v < V; ++v) {
        if (z) st4(z, p * q + lg + v * 32, u[v]);
        if (planes) st_split4(planes, total * C, p * q + lg + v * 32, u[v]);
      }
    }
  }
}

__global__ void __launch_bounds__(256) k_norm_act_fwd_scalar(const float* __restrict__ y, const float* __restrict__ a,
                                                             const float* __restrict__ b, float* __restrict__ z,
                                                             int64_t total, int HW, int C, int flags) {
  const bool act = flags & TWG_FLAG_LRELU, pix = flags & TWG_FLAG_PIXNORM;
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < total; p += (int64_t)gridDim.x * blockDim.x) {
    const int n = (int)(p / HW);
    float ss = 0.f;
    for (int c = 0; c < C; ++c) {
      float t = fmaf(a[n * C + c], y[p * C + c], b[n * C + c]);
      if (act) t = lrelu(t);
      ss += t * t;
    }
    const float rinv = pix ? rsqrtf(ss / (float)C + kPixEps) : 1.f;
    for (int c = 0; c < C; ++c) {
      float t = fmaf(a[n * C + c], y[p * C + c], b[n * C + c]);
      if (act) t = lrelu(t);
      z[p * C + c] = t * rinv;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// backward pass 1: gu and per-(n,c) {sum gu, sum gu*yhat}
// ------------------------------------------------------------------------------------------------
template <int V>
__global__ void __launch_bounds__(256) k_norm_act_bwd_reduce_vec(
    const float* __restrict__ y, const float* __restrict__ a, const float* __restrict__ b,
    const float* __restrict__ mean, const float* __restrict__ rstd, const float* __restrict__ gz,
    float* __restrict__ gu, float* __restrict__ red, int HW, int C, int G, int flags, int chunk,
    const float* __restrict__ gpool, int W) {
  // gz (may be null) is the gradient w.r.t. the layer output z at full resolution (e.g. from a UNet skip); gpool (may be
  // null) the gradient w.r.t. avg_pool2(z): its 2x2 broadcast * 1/4 is added on the fly instead of being materialised
  __shared__ float sm[256];
  const int n = blockIdx.y, q = C / 4;
  const int gpb = 256 / G, grp = threadIdx.x / G, lg = threadIdx.x % G;
  const bool act = flags & TWG_FLAG_LRELU, pix = flags & TWG_FLAG_PIXNORM;
  const float invC = 1.f / (float)C;
  const int p0 = blockIdx.x * chunk, p1 = min(HW, p0 + chunk);
  float4 aa[V], bb[V], mm[V], rr[V];
#pragma unroll
  for (int v = 0; v < V; ++v) {
    const int64_t i = (int64_t)n * q + lg + v * 32;
    aa[v] = ld4(a, i); bb[v] = ld4(b, i); mm[v] = ld4(mean, i); rr[v] = ld4(rstd, i);
  }
  float acc[8 * V];
#pragma unroll
  for (int i = 0; i < 8 * V; ++i) acc[i] = 0.f;
  constexpr int U = (V == 1) ? 2 : 1;      // pixels in flight per thread (all their loads are issued before the first use)
  for (int pb = p0; pb < p1; pb += gpb * U) {
    float4 yy[U][V], g[U][V];
    bool valid[U];
    int64_t base[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int p = pb + u * gpb + grp;
      valid[u] = p < p1;
      const int pp = valid[u] ? p : p0;
      base[u] = ((int64_t)n * HW + pp) * q;
#pragma unroll
      for (int v = 0; v < V; ++v) {
        yy[u][v] = ld4(y, base[u] + lg + v * 32);
        g[u][v] = gz ? ld4(gz, base[u] + lg + v * 32) : make_float4(0, 0, 0, 0);
        if (gpool) {
          const int h = pp / W, w = pp - h * W;
          const int64_t pq = (((int64_t)n * (HW / W / 2) + (h >> 1)) * (W >> 1) + (w >> 1)) * q;
          const float4 t = ld4(gpool, pq + lg + v * 32);
          g[u][v].x = fmaf(0.25f, t.x, g[u][v].x); g[u][v].y = fmaf(0.25f, t.y, g[u][v].y);
          g[u][v].z = fmaf(0.25f, t.z, g[u][v].z); g[u][v].w = fmaf(0.25f, t.w, g[u][v].w);
        }
        if (!valid[u]) g[u][v] = make_float4(0, 0, 0, 0);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      float4 uu[V], vv[V];
      float ss = 0.f;
#pragma unroll
      for (int v = 0; v < V; ++v) {
        uu[v] = make_float4(fmaf(aa[v].x, yy[u][v].x, bb[v].x), fmaf(aa[v].y, yy[u][v].y, bb[v].y),
                            fmaf(aa[v].z, yy[u][v].z, bb[v].z), fmaf(aa[v].w, yy[u][v].w, bb[v].w));
        vv[v] = uu[v];
        if (act) { vv[v].x = lrelu(uu[v].x); vv[v].y = lrelu(uu[v].y); vv[v].z = lrelu(uu[v].z); vv[v].w = lrelu(uu[v].w); }
        ss += vv[v].x * vv[v].x + vv[v].y * vv[v].y + vv[v].z * vv[v].z + vv[v].w * vv[v].w;
      }
      if (pix) {
        ss = group_sum(ss, G);
        const float rinv = rsqrtf(ss * invC + kPixEps);
        float dot = 0.f;
#pragma unroll
        for (int v = 0; v < V; ++v) {
          vv[v].x *= rinv; vv[v].y *= rinv; vv[v].z *= rinv; vv[v].w *= rinv;  // vv = z
          dot += g[u][v].x * vv[v].x + g[u][v].y * vv[v].y + g[u][v].z * vv[v].z + g[u][v].w * vv[v].w;
        }
        dot = group_sum(dot, G) * invC;
#pragma unroll
        for (int v = 0; v < V; ++v) {
          g[u][v].x = rinv * (g[u][v].x - vv[v].x * dot); g[u][v].y = rinv * (g[u][v].y - vv[v].y * dot);
          g[u][v].z = rinv * (g[u][v].z - vv[v].z * dot); g[u][v].w = rinv * (g[u][v].w - vv[v].w * dot);
        }
      }
      if (act) {
#pragma unroll
        for (int v = 0; v < V; ++v) {
          g[u][v].x *= lrelu_slope(uu[v].x); g[u][v].y *= lrelu_slope(uu[v].y);
          g[u][v].z *= lrelu_slope(uu[v].z); g[u][v].w *= lrelu_slope(uu[v].w);
        }
      }
      if (valid[u]) {
#pragma unroll
        for (int v = 0; v < V; ++v) {
          st4(gu, base[u] + lg + v * 32, g[u][v]);
          acc[8 * v + 0] += g[u][v].x; acc[8 * v + 1] += g[u][v].y; acc[8 * v + 2] += g[u][v].z; acc[8 * v + 3] += g[u][v].w;
          acc[8 * v + 4] += g[u][v].x * (yy[u][v].x - mm[v].x) * rr[v].x;
          acc[8 * v + 5] += g[u][v].y * (yy[u][v].y - mm[v].y) * rr[v].y;
          acc[8 * v + 6] += g[u][v].z * (yy[u][v].z - mm[v].z) * rr[v].z;
          acc[8 * v + 7] += g[u][v].w * (yy[u][v].w - mm[v].w) * rr[v].w;
        }
      }
    }
  }
#pragma unroll
  for (int k = 0; k < 8 * V; ++k) {
    __syncthreads();
    sm[threadIdx.x] = acc[k];
    __syncthreads();
    for (int s = 128; s >= G; s >>= 1) {
      if (threadIdx.x < s) sm[threadIdx.x] += sm[threadIdx.x + s];
      __syncthreads();
    }
    if (threadIdx.x < G) {
      int v = k / 8, j = k % 8;
      int c = (lg + v * 32) * 4 + (j & 3);
      atomicAdd(&red[((int64_t)n * C + c) * 2 + (j >> 2)], sm[threadIdx.x]);
    }
  }
}

__global__ void __launch_bounds__(256) k_norm_act_bwd_reduce_scalar(
    const float* __restrict__ y, const float* __restrict__ a, const float* __restrict__ b,
    const float* __restrict__ mean, const float* __restrict__ rstd, const float* __restrict__ gz,
    float* __restrict__ gu, float* __restrict__ red, int HW, int C, int flags, int chunk) {
  __shared__ float sm[32];
  const int n = blockIdx.y;
  const bool act = flags & TWG_FLAG_LRELU, pix = flags & TWG_FLAG_PIXNORM;
  const int p0 = blockIdx.x * chunk, p1 = min(HW, p0 + chunk);
  // pass A: gu
  for (int p = p0 + threadIdx.x; p < p1; p += blockDim.x) {
    const int64_t base = ((int64_t)n * HW + p) * C;
    float ss = 0.f, dot = 0.f;
    for (int c = 0; c < C; ++c) {
      float u = fmaf(a[n * C + c], y[base + c], b[n * C + c]);
      float v = act ? lrelu(u) : u;
      ss += v * v;
    }
    const float rinv = pix ? rsqrtf(ss / (float)C + kPixEps) : 1.f;
    if (pix) {
      for (int c = 0; c < C; ++c) {
        float u = fmaf(a[n * C + c], y[base + c], b[n * C + c]);
        float v = act ? lrelu(u) : u;
        dot += gz[base + c] * v * rinv;
      }
      dot /= (float)C;
    }
    for (int c = 0; c < C; ++c) {
      float u = fmaf(a[n * C + c], y[base + c], b[n * C + c]);
      float v = act ? lrelu(u) : u;
      float g = gz[base + c];
      if (pix) g = rinv * (g - v * rinv * dot);
      if (act) g *= lrelu_slope(u);
      gu[base + c] = g;
    }
  }
  __syncthreads();
  for (int c = 0; c < C; ++c) {
    float a1 = 0.f, a2 = 0.f;
    for (int p = p0 + threadIdx.x; p < p1; p += blockDim.x) {
      const int64_t i = ((int64_t)n * HW + p) * C + c;
      float g = gu[i];
      a1 += g;
      a2 += g * (y[i] - mean[n * C + c]) * rstd[n * C + c];
    }
    a1 = block_sum(a1, sm);
    a2 = block_sum(a2, sm);
    if (threadIdx.x == 0) {
      atomicAdd(&red[((int64_t)n * C + c) * 2], a1);
      atomicAdd(&red[((int64_t)n * C + c) * 2 + 1], a2);
    }
  }
}

// backward pass 2a: turn red into per-(n,c) k1=S1/M, k2=S2/M (in place) and the parameter gradients of each domain
// (groups / dom_mask as in k_norm_finalize; rd is [groups][2][C])
__global__ void k_norm_bwd_coeffs(float* __restrict__ red, const float* __restrict__ rd, float* __restrict__ ggamma0,
                                  float* __restrict__ gbeta0, float* __restrict__ ggamma1, float* __restrict__ gbeta1,
                                  unsigned dom_mask, int gs, int kind, int N, int HW, int C, int accumulate) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float gg[2] = {0.f, 0.f}, gb[2] = {0.f, 0.f};
  const int groups = N / gs;
  for (int grp = 0; grp < groups; ++grp) {
    const int dom = (dom_mask >> grp) & 1u;
    const int n0 = grp * gs, n1 = n0 + gs;
    float t1 = 0.f, t2 = 0.f;
    for (int n = n0; n < n1; ++n) { t1 += red[(n * C + c) * 2]; t2 += red[(n * C + c) * 2 + 1]; }
    const float r = rd ? rd[grp * 2 * C + c] : 1.f, d = rd ? rd[grp * 2 * C + C + c] : 0.f;
    gg[dom] += r * t2 + d * t1;
    gb[dom] += t1;
    if (kind == TWG_NORM_INSTANCE) {
      const float inv = 1.f / (float)HW;
      for (int n = n0; n < n1; ++n) { red[(n * C + c) * 2] *= inv; red[(n * C + c) * 2 + 1] *= inv; }
    } else if (kind == TWG_NORM_NONE) {
      for (int n = n0; n < n1; ++n) { red[(n * C + c) * 2] = 0.f; red[(n * C + c) * 2 + 1] = 0.f; }
    } else {
      const float inv = 1.f / ((float)HW * (float)gs);
      for (int n = n0; n < n1; ++n) { red[(n * C + c) * 2] = t1 * inv; red[(n * C + c) * 2 + 1] = t2 * inv; }
    }
  }
  // accumulate: the outputs are slices of the step's flat gradient buffer (several passes share one variable)
  if (ggamma0) ggamma0[c] = (accumulate ? ggamma0[c] : 0.f) + gg[0];
  if (gbeta0) gbeta0[c] = (accumulate ? gbeta0[c] : 0.f) + gb[0];
  if (ggamma1) ggamma1[c] = (accumulate ? ggamma1[c] : 0.f) + gg[1];
  if (gbeta1) gbeta1[c] = (accumulate ? gbeta1[c] : 0.f) + gb[1];
}

// backward pass 2b: gy = a*(gu - k1 - yhat*k2).  blockIdx.y = sample; when the block size is a multiple of the float4s per
// pixel (every channel count of the network), a thread always owns the same channels, so its five per-(n,c) coefficient
// vectors are loaded once and the loop streams y and gu only, two elements in flight.
template <int VEC>
__global__ void __launch_bounds__(256) k_norm_act_bwd_apply(const float* __restrict__ y, const float* __restrict__ a,
                                                            const float* __restrict__ mean,
                                                            const float* __restrict__ rstd,
                                                            const float* __restrict__ gu, const float* __restrict__ k,
                                                            float* __restrict__ gy, void* __restrict__ planes,
                                                            int64_t total_vec, int HW, int C) {
  const int q = C / VEC;
  const int n = blockIdx.y;
  const int per = HW * q;                               // vectors of this sample
  const int64_t base = (int64_t)n * per;
  const int stride = gridDim.x * blockDim.x;
  if (VEC == 4 && (256 % q) == 0) {
    const int cq = threadIdx.x % q;
    const int64_t j = (int64_t)n * q + cq;
    const float4 aa = ld4(a, j), mm = ld4(mean, j), rr = ld4(rstd, j);
    const float* kk = k + ((int64_t)n * C + cq * 4) * 2;
    const float4 k01 = reinterpret_cast<const float4*>(kk)[0], k23 = reinterpret_cast<const float4*>(kk)[1];
    for (int i0 = blockIdx.x * blockDim.x + threadIdx.x; i0 < per; i0 += 2 * stride) {
      const int i1 = i0 + stride;
      const bool two = i1 < per;
      const float4 y0 = ld4(y, base + i0), g0 = ld4(gu, base + i0);
      const float4 y1 = two ? ld4(y, base + i1) : y0, g1 = two ? ld4(gu, base + i1) : g0;
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        if (u == 1 && !two) break;
        const float4 yy = u ? y1 : y0, g = u ? g1 : g0;
        float4 o;
        o.x = aa.x * (g.x - k01.x - (yy.x - mm.x) * rr.x * k01.y);
        o.y = aa.y * (g.y - k01.z - (yy.y - mm.y) * rr.y * k01.w);
        o.z = aa.z * (g.z - k23.x - (yy.z - mm.z) * rr.z * k23.y);
        o.w = aa.w * (g.w - k23.z - (yy.w - mm.w) * rr.w * k23.w);
        const int64_t i = base + (u ? i1 : i0);
        if (gy) st4(gy, i, o);
        if (planes) st_split4(planes, total_vec * 4, i, o);
      }
    }
    return;
  }
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < per; idx += stride) {
    const int cq = idx % q;
    const int64_t i = base + idx;
    if (VEC == 4) {
      float4 yy = ld4(y, i), g = ld4(gu, i);
      const int64_t j = (int64_t)n * q + cq;
      float4 aa = ld4(a, j), mm = ld4(mean, j), rr = ld4(rstd, j);
      const float* kk = k + ((int64_t)n * C + cq * 4) * 2;
      float4 k01 = reinterpret_cast<const float4*>(kk)[0], k23 = reinterpret_cast<const float4*>(kk)[1];
      float4 o;
      o.x = aa.x * (g.x - k01.x - (yy.x - mm.x) * rr.x * k01.y);
      o.y = aa.y * (g.y - k01.z - (yy.y - mm.y) * rr.y * k01.w);
      o.z = aa.z * (g.z - k23.x - (yy.z - mm.z) * rr.z * k23.y);
      o.w = aa.w * (g.w - k23.z - (yy.w - mm.w) * rr.w * k23.w);
      if (gy) st4(gy, i, o);
      if (planes) st_split4(planes, total_vec * 4, i, o);
    } else {
      const int64_t j = (int64_t)n * C + cq;
      gy[i] = a[j] * (gu[i] - k[j * 2] - (y[i] - mean[j]) * rstd[j] * k[j * 2 + 1]);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// bias + lrelu, masks, column sums
// ------------------------------------------------------------------------------------------------
template <int VEC>
__global__ void __launch_bounds__(256) k_bias_lrelu(const float* __restrict__ y, const float* __restrict__ bias,
                                                    float* __restrict__ z, int64_t total_vec, int C, int act,
                                                    void* __restrict__ planes, uint8_t* __restrict__ mask) {
  // planes / mask (VEC = 4 only, may be null): z also as split-bf16 planes for the tensor-core conv that consumes it, and
  // its sign bits (one byte per float4) for the activation backward
  const int q = C / VEC;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total_vec; i += (int64_t)gridDim.x * blockDim.x) {
    const int cq = (int)(i % q);
    if (VEC == 4) {
      float4 t = ld4(y, i);
      if (bias) { float4 bb = ld4(bias, cq); t.x += bb.x; t.y += bb.y; t.z += bb.z; t.w += bb.w; }
      if (act) { t.x = lrelu(t.x); t.y = lrelu(t.y); t.z = lrelu(t.z); t.w = lrelu(t.w); }
      st4(z, i, t);
      if (planes) st_split4(planes, total_vec * 4, i, t);
      if (mask) mask[i] = (uint8_t)((t.x > 0.f ? 1 : 0) | (t.y > 0.f ? 2 : 0) | (t.z > 0.f ? 4 : 0) | (t.w > 0.f ? 8 : 0));
    } else {
      float t = y[i] + (bias ? bias[cq] : 0.f);
      z[i] = act ? lrelu(t) : t;
    }
  }
}

__global__ void __launch_bounds__(256) k_lrelu_bwd(const float* __restrict__ g, const float* __restrict__ ref,
                                                   float* __restrict__ out, int64_t n) {
  const int64_t n4 = n / 4;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    float4 a = ld4(g, i), r = ld4(ref, i);
    a.x *= lrelu_slope(r.x); a.y *= lrelu_slope(r.y); a.z *= lrelu_slope(r.z); a.w *= lrelu_slope(r.w);
    st4(out, i, a);
  }
  for (int64_t i = n4 * 4 + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = g[i] * lrelu_slope(ref[i]);
}

// out = g * slope(ref) and colsum[c] += sum_rows out[row][c] in one pass (bias gradient of the discriminator layers)
template <int V, bool MASK>
__global__ void __launch_bounds__(256) k_lrelu_bwd_colsum_vec(const float* __restrict__ g, const float* __restrict__ ref,
                                                              float* __restrict__ out, void* __restrict__ planes,
                                                              float* __restrict__ colsum, int64_t rows, int C, int G,
                                                              int64_t chunk, int act, int poolH, int poolW,
                                                              const uint8_t* __restrict__ mask) {
  // mask (may be null): sign bits of the activation, 4 per byte = one byte per float4, written by the conv epilogue; read
  // instead of `ref` (0.25 B instead of 4 B per element)
  // poolW > 0: `g` is the gradient w.r.t. avg_pool2(z) ([N, poolH/2, poolW/2, C]); the row's gradient is a quarter of
  // its pooled cell (the full-resolution gradient tensor is never written)
  __shared__ float sm[256];
  const int q = C / 4, gpb = 256 / G, grp = threadIdx.x / G, lg = threadIdx.x % G;
  const int64_t r0 = (int64_t)blockIdx.x * chunk, r1 = min(rows, r0 + chunk);
  float acc[4 * V];
#pragma unroll
  for (int i = 0; i < 4 * V; ++i) acc[i] = 0.f;
  // rows in flight per thread: with the sign mask a row is 16 B of loads per thread instead of 32, and at two rows in
  // flight the kernel ran latency-bound at 48 % of the HBM bandwidth (profiles/r02_ncu_summary_session2.md)
  constexpr int U = (V == 1) ? 4 : (V == 2 ? 2 : 1);
  const int hw = poolH * poolW;
  // 32-bit pixel arithmetic (64-bit divisions per row made this kernel instruction-bound): n0 = sample of the chunk's
  // first row, computed once; rows further on are located relative to it
  const int64_t n0 = poolW > 0 ? r0 / hw : 0;
  const int64_t row_of_n0 = n0 * hw;
  for (int64_t rb = r0 + grp; rb < r1; rb += (int64_t)gpb * U) {
    float4 a[U][V], rr[MASK ? 1 : U][V];
    unsigned mb[U][V];
    bool valid[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t r = rb + (int64_t)u * gpb;
      valid[u] = r < r1;
      const int64_t rv = valid[u] ? r : r0;
#pragma unroll
      for (int v = 0; v < V; ++v) {
        const int64_t i = rv * q + lg + v * 32;
        if (poolW > 0) {
          const unsigned rel = (unsigned)(rv - row_of_n0);          // < chunk + hw
          const unsigned dn = rel / (unsigned)hw, p = rel - dn * (unsigned)hw;
          const unsigned h = p / (unsigned)poolW, w = p - h * (unsigned)poolW;
          const int64_t nn = n0 + dn;
          a[u][v] = ld4(g, ((nn * (poolH >> 1) + (h >> 1)) * (poolW >> 1) + (w >> 1)) * q + lg + v * 32);
        } else {
          a[u][v] = ld4(g, i);
        }
        if (act) {
          if (MASK) mb[u][v] = mask[i];
          else rr[u][v] = ld4(ref, i);
        }
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (!valid[u]) continue;
      const int64_t r = rb + (int64_t)u * gpb;
#pragma unroll
      for (int v = 0; v < V; ++v) {
        const int64_t i = r * q + lg + v * 32;
        float4 t = a[u][v];
        if (poolW > 0) { t.x *= 0.25f; t.y *= 0.25f; t.z *= 0.25f; t.w *= 0.25f; }
        if (act) {
          if (MASK) {
            const unsigned m = mb[u][v];
            t.x *= (m & 1u) ? 1.f : kLeak; t.y *= (m & 2u) ? 1.f : kLeak;
            t.z *= (m & 4u) ? 1.f : kLeak; t.w *= (m & 8u) ? 1.f : kLeak;
          } else {
            t.x *= lrelu_slope(rr[MASK ? 0 : u][v].x); t.y *= lrelu_slope(rr[MASK ? 0 : u][v].y);
            t.z *= lrelu_slope(rr[MASK ? 0 : u][v].z); t.w *= lrelu_slope(rr[MASK ? 0 : u][v].w);
          }
          if (out) st4(out, i, t);
        }
        if (planes) st_split4(planes, rows * C, i, t);
        acc[4 * v + 0] += t.x; acc[4 * v + 1] += t.y; acc[4 * v + 2] += t.z; acc[4 * v + 3] += t.w;
      }
    }
  }
#pragma unroll
  for (int k = 0; k < 4 * V; ++k) {
    __syncthreads();
    sm[threadIdx.x] = acc[k];
    __syncthreads();
    for (int s = 128; s >= G; s >>= 1) {
      if (threadIdx.x < s) sm[threadIdx.x] += sm[threadIdx.x + s];
      __syncthreads();
    }
    if (threadIdx.x < G) colsum[(int64_t)blockIdx.x * C + (lg + (k / 4) * 32) * 4 + (k & 3)] = sm[threadIdx.x];
  }
}

// Pool-fed form of the kernel above, by IMAGE ROWS (C / 4 = q a power of two <= 32): `g` is the gradient w.r.t. avg_pool2(z),
// [N, H/2, W/2, C]; out = 0.25 * g[h/2][w/2] * slope.  The flat form spends three integer divisions per float4 on locating the
// pooled cell (ncu: issue slots 72 % busy at 55 % of the HBM bandwidth); here a block walks whole image rows, so the
// sample / row split is one division per row and the rest is shifts.
template <bool MASK>
__global__ void __launch_bounds__(256) k_lrelu_bwd_colsum_pool_rows(const float* __restrict__ g, const float* __restrict__ ref,
                                                                    void* __restrict__ planes, float* __restrict__ colsum,
                                                                    int img_rows, int H, int W, int lq, int rows_per_block,
                                                                    const uint8_t* __restrict__ mask, int64_t total_elems) {
  __shared__ float sm[256];
  const int q = 1 << lq, gpb = 256 >> lq, grp = threadIdx.x >> lq, lg = threadIdx.x & (q - 1);
  const int r0 = blockIdx.x * rows_per_block, r1 = min(img_rows, r0 + rows_per_block);
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  constexpr int U = 4;
  for (int r = r0; r < r1; ++r) {
    const int n = r / H, h = r - n * H;
    const float4* grow = reinterpret_cast<const float4*>(g) + (((int64_t)n * (H >> 1) + (h >> 1)) * (W >> 1) << lq);
    const int64_t zrow = ((int64_t)r * W) << lq;          // float4 index of this image row in z / mask / planes
    for (int w0 = grp; w0 < W; w0 += gpb * U) {
      float4 a[U], rr[MASK ? 1 : U];
      unsigned mb[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int w = w0 + u * gpb;
        const int wv = w < W ? w : w0;
        a[u] = grow[((wv >> 1) << lq) + lg];
        if (MASK) mb[u] = mask[zrow + (wv << lq) + lg];
        else rr[MASK ? 0 : u] = ld4(ref, zrow + (wv << lq) + lg);
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int w = w0 + u * gpb;
        if (w >= W) continue;
        float4 t = a[u];
        float sx, sy, sz, sw;
        if (MASK) {
          const unsigned m = mb[u];
          sx = (m & 1u) ? 0.25f : 0.25f * kLeak; sy = (m & 2u) ? 0.25f : 0.25f * kLeak;
          sz = (m & 4u) ? 0.25f : 0.25f * kLeak; sw = (m & 8u) ? 0.25f : 0.25f * kLeak;
        } else {
          const float4 z = rr[MASK ? 0 : u];
          sx = 0.25f * lrelu_slope(z.x); sy = 0.25f * lrelu_slope(z.y); sz = 0.25f * lrelu_slope(z.z); sw = 0.25f * lrelu_slope(z.w);
        }
        t.x *= sx; t.y *= sy; t.z *= sz; t.w *= sw;
        st_split4(planes, total_elems, zrow + (w << lq) + lg, t);
        acc[0] += t.x; acc[1] += t.y; acc[2] += t.z; acc[3] += t.w;
      }
    }
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    __syncthreads();
    sm[threadIdx.x] = acc[k];
    __syncthreads();
    for (int s_ = 128; s_ >= q; s_ >>= 1) {
      if (threadIdx.x < s_) sm[threadIdx.x] += sm[threadIdx.x + s_];
      __syncthreads();
    }
    if (threadIdx.x < q) colsum[((int64_t)blockIdx.x << (lq + 2)) + lg * 4 + k] = sm[threadIdx.x];
  }
}

// out[blockIdx.x * C + c] = sum over a chunk of rows (a partial, see add_partials); grid.x = row chunks, thread owns (c, row-lane)
__global__ void __launch_bounds__(256) k_colsum(const float* __restrict__ g, float* __restrict__ out, int64_t rows,
                                                int C, int64_t chunk) {
  __shared__ float sm[256];
  // threads laid out as [rl = tid / Cw][cl = tid % Cw] with Cw = min(C,256) rounded to pow2 <= 256
  int Cw = 1;
  while (Cw < C && Cw < 256) Cw <<= 1;
  const int rl = threadIdx.x / Cw, cl = threadIdx.x % Cw, RL = 256 / Cw;
  const int64_t r0 = (int64_t)blockIdx.x * chunk, r1 = min(rows, r0 + chunk);
  for (int c0 = 0; c0 < C; c0 += Cw) {
    const int c = c0 + cl;
    float acc = 0.f;
    if (c < C)
      for (int64_t r = r0 + rl; r < r1; r += RL) acc += g[r * C + c];
    __syncthreads();
    sm[threadIdx.x] = acc;
    __syncthreads();
    for (int s = 128; s >= Cw; s >>= 1) {
      if (threadIdx.x < s) sm[threadIdx.x] += sm[threadIdx.x + s];
      __syncthreads();
    }
    if (threadIdx.x < Cw && c < C) out[(int64_t)blockIdx.x * C + c] = sm[threadIdx.x];
  }
}

// ------------------------------------------------------------------------------------------------
// resampling
// ------------------------------------------------------------------------------------------------
// Row-decomposed float4 forms of the two heaviest resampling kernels: blockIdx.x = one OUTPUT row (n, ho), the threads walk
// its Wo * q float4 with 32-bit index arithmetic and four independent loads in flight.  The flat-index forms below spend
// four 64-bit divisions per float4 and keep one load in flight (they remain for the scalar / odd-width cases).
__global__ void __launch_bounds__(256) k_pool2_rows(const float* __restrict__ x, float* __restrict__ out,
                                                    void* __restrict__ planes, int H, int W, int q, float scale,
                                                    int64_t total_elems) {
  const int Ho = H >> 1, Wo = W >> 1;
  const int row = blockIdx.x;                        // n * Ho + ho
  const int n = row / Ho, ho = row - n * Ho;
  const float4* r0 = reinterpret_cast<const float4*>(x) + ((int64_t)n * H + 2 * ho) * W * q;
  const float4* r1 = r0 + (int64_t)W * q;
  const int64_t obase = (int64_t)row * Wo * q;
  const int per = Wo * q;
  for (int j0 = threadIdx.x; j0 < per; j0 += 256 * 2) {
    float4 a[2], b[2], c[2], d[2];
    int j[2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      j[u] = j0 + u * 256;
      const int jj = j[u] < per ? j[u] : j0;
      const int wo = jj / q, cq = jj - wo * q;
      const int i00 = 2 * wo * q + cq;
      a[u] = r0[i00]; b[u] = r0[i00 + q]; c[u] = r1[i00]; d[u] = r1[i00 + q];
    }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      if (j[u] >= per) continue;
      const float4 o = make_float4(scale * (a[u].x + b[u].x + c[u].x + d[u].x), scale * (a[u].y + b[u].y + c[u].y + d[u].y),
                                   scale * (a[u].z + b[u].z + c[u].z + d[u].z), scale * (a[u].w + b[u].w + c[u].w + d[u].w));
      if (out) st4(out, obase + j[u], o);
      if (planes) st_split4(planes, total_elems, obase + j[u], o);
    }
  }
}

__global__ void __launch_bounds__(256) k_upsample_concat_rows(const float* __restrict__ a, const float* __restrict__ b,
                                                              float* __restrict__ out, void* __restrict__ planes, int H, int W,
                                                              int qa, int qb, int Nb, int64_t total_elems) {
  const int q = qa + qb, Ho = 2 * H, Wo = 2 * W;
  const int row = blockIdx.x;                        // n * Ho + ho
  const int n = row / Ho, ho = row - n * Ho;
  const float4* ra = reinterpret_cast<const float4*>(a) + ((int64_t)n * H + (ho >> 1)) * W * qa;
  const float4* rb = reinterpret_cast<const float4*>(b) + ((int64_t)(n % Nb) * Ho + ho) * Wo * qb;
  const int64_t obase = (int64_t)row * Wo * q;
  const int per = Wo * q;
  for (int j0 = threadIdx.x; j0 < per; j0 += 256 * 4) {
    float4 v[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int j = j0 + u * 256;
      const int jj = j < per ? j : j0;
      const int wo = jj / q, cq = jj - wo * q;
      v[u] = (cq < qa) ? ra[(wo >> 1) * qa + cq] : rb[wo * qb + (cq - qa)];
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int j = j0 + u * 256;
      if (j >= per) continue;
      if (out) st4(out, obase + j, v[u]);
      if (planes) st_split4(planes, total_elems, obase + j, v[u]);
    }
  }
}

// Backward of the UNet join by rows (float4, 32-bit index arithmetic): blockIdx.x < Nb * Ho walks one row of the skip
// gradient gb[nb][ho] = sum over the N / Nb uses of that skip sample; the remaining N * H blocks each produce one row of
// ga[n][h] = sum of the 2x2 cells of the upsampled half.
__global__ void __launch_bounds__(256) k_upsample_concat_bwd_rows(const float* __restrict__ gout, float* __restrict__ ga,
                                                                  float* __restrict__ gb, int N, int H, int W, int qa, int qb,
                                                                  int Nb) {
  const int q = qa + qb, Ho = 2 * H, Wo = 2 * W;
  const float4* go = reinterpret_cast<const float4*>(gout);
  int row = blockIdx.x;
  if (row < Nb * Ho) {
    const int nb = row / Ho, ho = row - nb * Ho;
    const int reps = N / Nb;
    const int per = Wo * qb;
    float4* dst = reinterpret_cast<float4*>(gb) + (int64_t)row * per;
    for (int j = threadIdx.x; j < per; j += 256) {
      const int wo = j / qb, cq = j - wo * qb;
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int r = 0; r < reps; ++r) {
        const float4 t = go[(((int64_t)(nb + r * Nb) * Ho + ho) * Wo + wo) * q + qa + cq];
        acc.x += t.x; acc.y += t.y; acc.z += t.z; acc.w += t.w;
      }
      dst[j] = acc;
    }
    return;
  }
  row -= Nb * Ho;                                      // n * H + h
  const int n = row / H, h = row - n * H;
  const float4* r0 = go + ((int64_t)n * Ho + 2 * h) * Wo * q;
  const float4* r1 = r0 + (int64_t)Wo * q;
  const int per = W * qa;
  float4* dst = reinterpret_cast<float4*>(ga) + (int64_t)row * per;
  for (int j0 = threadIdx.x; j0 < per; j0 += 512) {
    float4 x0[2], x1[2], x2[2], x3[2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int j = j0 + u * 256 < per ? j0 + u * 256 : j0;
      const int w = j / qa, cq = j - w * qa;
      const int i00 = 2 * w * q + cq;
      x0[u] = r0[i00]; x1[u] = r0[i00 + q]; x2[u] = r1[i00]; x3[u] = r1[i00 + q];
    }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int j = j0 + u * 256;
      if (j >= per) continue;
      dst[j] = make_float4(x0[u].x + x1[u].x + x2[u].x + x3[u].x, x0[u].y + x1[u].y + x2[u].y + x3[u].y,
                           x0[u].z + x1[u].z + x2[u].z + x3[u].z, x0[u].w + x1[u].w + x2[u].w + x3[u].w);
    }
  }
}

template <int VEC>
__global__ void __launch_bounds__(256) k_pool2(const float* __restrict__ x, float* __restrict__ out,
                                               void* __restrict__ planes, int N, int H, int W, int C, float scale) {
  const int q = C / VEC, Ho = H / 2, Wo = W / 2;
  const int64_t total = (int64_t)N * Ho * Wo * q;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int cq = (int)(i % q);
    int64_t t = i / q;
    int wo = (int)(t % Wo); t /= Wo;
    int ho = (int)(t % Ho);
    int n = (int)(t / Ho);
    const int64_t b00 = (((int64_t)n * H + 2 * ho) * W + 2 * wo) * q + cq;
    if (VEC == 4) {
      float4 a = ld4(x, b00), b = ld4(x, b00 + q), c = ld4(x, b00 + (int64_t)W * q), d = ld4(x, b00 + (int64_t)W * q + q);
      const float4 o = make_float4(scale * (a.x + b.x + c.x + d.x), scale * (a.y + b.y + c.y + d.y),
                                   scale * (a.z + b.z + c.z + d.z), scale * (a.w + b.w + c.w + d.w));
      if (out) st4(out, i, o);
      if (planes) st_split4(planes, total * 4, i, o);
    } else {
      out[i] = scale * (x[b00] + x[b00 + q] + x[b00 + (int64_t)W * q] + x[b00 + (int64_t)W * q + q]);
    }
  }
}

template <int VEC>
__global__ void __launch_bounds__(256) k_upsample2(const float* __restrict__ x, float* __restrict__ out, int N, int H,
                                                   int W, int C, float scale) {
  const int q = C / VEC, Ho = 2 * H, Wo = 2 * W;
  const int64_t total = (int64_t)N * Ho * Wo * q;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int cq = (int)(i % q);
    int64_t t = i / q;
    int wo = (int)(t % Wo); t /= Wo;
    int ho = (int)(t % Ho);
    int n = (int)(t / Ho);
    const int64_t src = (((int64_t)n * H + ho / 2) * W + wo / 2) * q + cq;
    if (VEC == 4) {
      float4 a = ld4(x, src);
      st4(out, i, make_float4(scale * a.x, scale * a.y, scale * a.z, scale * a.w));
    } else {
      out[i] = scale * x[src];
    }
  }
}

template <int VEC>
// b (the UNet skip) may hold fewer samples than a: sample n of the output reads b[n % Nb] (batched generator passes that
// share one encoder pass)
__global__ void __launch_bounds__(256) k_upsample_concat(const float* __restrict__ a, const float* __restrict__ b,
                                                         float* __restrict__ out, void* __restrict__ planes, int N, int H,
                                                         int W, int Ca, int Cb, int Nb) {
  const int qa = Ca / VEC, qb = Cb / VEC, q = qa + qb, Ho = 2 * H, Wo = 2 * W;
  const int64_t total = (int64_t)N * Ho * Wo * q;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int cq = (int)(i % q);
    int64_t p = i / q;
    int wo = (int)(p % Wo);
    int64_t t = p / Wo;
    int ho = (int)(t % Ho);
    int n = (int)(t / Ho);
    if (VEC == 4) {
      const int64_t pb = p - (int64_t)(n - n % Nb) * Ho * Wo;     // the same pixel of sample n % Nb
      const float4 o = (cq < qa) ? ld4(a, (((int64_t)n * H + ho / 2) * W + wo / 2) * qa + cq) : ld4(b, pb * qb + (cq - qa));
      if (out) st4(out, i, o);
      if (planes) st_split4(planes, total * 4, i, o);
    } else if (cq < qa) {
      out[i] = a[(((int64_t)n * H + ho / 2) * W + wo / 2) * qa + cq];
    } else {
      out[i] = b[(p - (int64_t)(n - n % Nb) * Ho * Wo) * qb + (cq - qa)];
    }
  }
}

template <int VEC>
// gb has Nb <= N samples: gb[m] = sum_j gout[m + j*Nb][..., Ca:]  (the skip tensor fed N/Nb generator passes)
__global__ void __launch_bounds__(256) k_upsample_concat_bwd(const float* __restrict__ gout, float* __restrict__ ga,
                                                             float* __restrict__ gb, int N, int H, int W, int Ca, int Cb,
                                                             int Nb) {
  const int qa = Ca / VEC, qb = Cb / VEC, q = qa + qb, Ho = 2 * H, Wo = 2 * W;
  const int64_t total_b = (int64_t)Nb * Ho * Wo * qb;
  const int64_t total_a = (int64_t)N * H * W * qa;
  const int64_t rep_stride = (int64_t)Nb * Ho * Wo;        // pixels between two uses of the same skip sample
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total_a + total_b;
       i += (int64_t)gridDim.x * blockDim.x) {
    if (i < total_b) {
      int cq = (int)(i % qb);
      int64_t p = i / qb;
      if (VEC == 4) {
        float4 acc = ld4(gout, p * q + qa + cq);
        for (int j = 1; j < N / Nb; ++j) {
          const float4 t = ld4(gout, (p + j * rep_stride) * q + qa + cq);
          acc.x += t.x; acc.y += t.y; acc.z += t.z; acc.w += t.w;
        }
        st4(gb, i, acc);
      } else {
        float acc = gout[p * q + qa + cq];
        for (int j = 1; j < N / Nb; ++j) acc += gout[(p + j * rep_stride) * q + qa + cq];
        gb[i] = acc;
      }
    } else {
      int64_t j = i - total_b;
      int cq = (int)(j % qa);
      int64_t t = j / qa;
      int w = (int)(t % W); t /= W;
      int h = (int)(t % H);
      int n = (int)(t / H);
      const int64_t b00 = (((int64_t)n * Ho + 2 * h) * Wo + 2 * w) * q + cq;
      if (VEC == 4) {
        float4 x0 = ld4(gout, b00), x1 = ld4(gout, b00 + q), x2 = ld4(gout, b00 + (int64_t)Wo * q),
               x3 = ld4(gout, b00 + (int64_t)Wo * q + q);
        st4(ga, j, make_float4(x0.x + x1.x + x2.x + x3.x, x0.y + x1.y + x2.y + x3.y, x0.z + x1.z + x2.z + x3.z,
                               x0.w + x1.w + x2.w + x3.w));
      } else {
        ga[j] = gout[b00] + gout[b00 + q] + gout[b00 + (int64_t)Wo * q] + gout[b00 + (int64_t)Wo * q + q];
      }
    }
  }
}

__global__ void __launch_bounds__(256) k_axpby(const float* __restrict__ x, const float* __restrict__ y,
                                               float* __restrict__ out, float alpha, float beta, int64_t n) {
  const int64_t n4 = n / 4;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    float4 a = ld4(x, i);
    float4 o = make_float4(alpha * a.x, alpha * a.y, alpha * a.z, alpha * a.w);
    if (y) { float4 b = ld4(y, i); o.x += beta * b.x; o.y += beta * b.y; o.z += beta * b.z; o.w += beta * b.w; }
    st4(out, i, o);
  }
  for (int64_t i = n4 * 4 + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = alpha * x[i] + (y ? beta * y[i] : 0.f);
}

__global__ void __launch_bounds__(256) k_scale_by_dev(const float* __restrict__ x, const float* __restrict__ s,
                                                      float* __restrict__ out, float alpha, int64_t n) {
  const float f = alpha * s[0];
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = x[i] * f;
}

__global__ void __launch_bounds__(256) k_copy_cols(const float* __restrict__ src, float* __restrict__ dst, int64_t rows,
                                                   int Csrc, int so, int Cdst, int d_o, int ncols) {
  const int64_t total = rows * ncols;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t r = i / ncols;
    int c = (int)(i - r * ncols);
    dst[r * Cdst + d_o + c] = src[r * Csrc + so + c];
  }
}

// ------------------------------------------------------------------------------------------------
// minibatch stddev.  The tensor is tiny (N x 4 x 4 x C) and the op is one global reduction plus a broadcast, so a
// single block was latency-bound at ~35 us; one 8-CTA cluster splits the feature axis, exchanges its partial sums
// through distributed shared memory and stays a single launch.
// ------------------------------------------------------------------------------------------------
constexpr int kMbCluster = 8;

// sum of one value per CTA over the cluster; result valid in all threads of all CTAs
__device__ __forceinline__ float cluster_sum(float block_value, float* slot) {
  cg::cluster_group cl = cg::this_cluster();
  if (threadIdx.x == 0) *slot = block_value;
  cl.sync();
  float s = 0.f;
  for (unsigned r = 0; r < cl.num_blocks(); ++r) s += *cl.map_shared_rank(slot, r);
  cl.sync();                                   // nobody leaves (or reuses the slot) while peers still read it
  return s;
}

__global__ void __cluster_dims__(kMbCluster, 1, 1) __launch_bounds__(512)
k_mbstd_fwd(const float* __restrict__ x, float* __restrict__ out, float* __restrict__ s_out, int N, int P, int C, int Ct) {
  // out has Ct >= C+1 channels: [x | statistic | zeros] (the zero channels pad the next conv's GEMM-K to a
  // tensor-core channel count).  One cluster per group of N samples (blockIdx.x / kMbCluster = group: one original discriminator pass)
  __shared__ float sm[32];
  __shared__ float slot;
  const int F = P * C;
  const int grp = blockIdx.x / kMbCluster;
  x += (int64_t)grp * N * F;
  out += (int64_t)grp * N * P * Ct;
  const int gtid = (blockIdx.x % kMbCluster) * blockDim.x + threadIdx.x, gsz = kMbCluster * blockDim.x;
  float acc = 0.f;
  for (int f = gtid; f < F; f += gsz) {
    float m = 0.f;
    for (int n = 0; n < N; ++n) m += x[(int64_t)n * F + f];
    m /= (float)N;
    float v = 0.f;
    for (int n = 0; n < N; ++n) { float d = x[(int64_t)n * F + f] - m; v += d * d; }
    acc += sqrtf(v / (float)N + 1e-8f);
  }
  const float s = cluster_sum(block_sum(acc, sm), &slot) / (float)F;
  if (gtid == 0 && s_out) s_out[grp] = s;
  const int64_t total = (int64_t)N * P * Ct;
  for (int64_t i = gtid; i < total; i += gsz) {
    int64_t r = i / Ct;
    int c = (int)(i - r * Ct);
    out[i] = (c < C) ? x[r * C + c] : (c == C ? s : 0.f);
  }
}

__global__ void __cluster_dims__(kMbCluster, 1, 1) __launch_bounds__(512)
k_mbstd_bwd(const float* __restrict__ x, const float* __restrict__ gout, float* __restrict__ gx, int N, int P, int C, int Ct) {
  __shared__ float sm[32];
  const int F = P * C;
  const int grp = blockIdx.x / kMbCluster;
  x += (int64_t)grp * N * F;
  gx += (int64_t)grp * N * F;
  gout += (int64_t)grp * N * P * Ct;
  const int gtid = (blockIdx.x % kMbCluster) * blockDim.x + threadIdx.x, gsz = kMbCluster * blockDim.x;
  float acc = 0.f;       // G = sum of the statistic channel's gradient: N*P values, every CTA sums them itself
  for (int i = threadIdx.x; i < N * P; i += blockDim.x) acc += gout[(int64_t)i * Ct + C];
  const float G = block_sum(acc, sm);
  for (int f = gtid; f < F; f += gsz) {
    const int p = f / C, c = f - p * C;
    float m = 0.f;
    for (int n = 0; n < N; ++n) m += x[(int64_t)n * F + f];
    m /= (float)N;
    float v = 0.f;
    for (int n = 0; n < N; ++n) { float d = x[(int64_t)n * F + f] - m; v += d * d; }
    const float sig = sqrtf(v / (float)N + 1e-8f);
    const float coef = G / ((float)N * (float)F * sig);
    for (int n = 0; n < N; ++n)
      gx[(int64_t)n * F + f] = gout[((int64_t)n * P + p) * Ct + c] + coef * (x[(int64_t)n * F + f] - m);
  }
}

__global__ void __cluster_dims__(kMbCluster, 1, 1) __launch_bounds__(512)
k_mbstd_bwd2(const float* __restrict__ x, const float* __restrict__ gout, const float* __restrict__ ggx,
             float* __restrict__ dgout, float* __restrict__ dx, int N, int P, int C, int Ct) {
  __shared__ float sm[32];
  __shared__ float slot;
  const int F = P * C;
  const int grp = blockIdx.x / kMbCluster;
  x += (int64_t)grp * N * F;
  ggx += (int64_t)grp * N * F;
  dx += (int64_t)grp * N * F;
  gout += (int64_t)grp * N * P * Ct;
  dgout += (int64_t)grp * N * P * Ct;
  const int gtid = (blockIdx.x % kMbCluster) * blockDim.x + threadIdx.x, gsz = kMbCluster * blockDim.x;
  float acc = 0.f;
  for (int i = threadIdx.x; i < N * P; i += blockDim.x) acc += gout[(int64_t)i * Ct + C];
  const float G = block_sum(acc, sm);
  float dG = 0.f;
  for (int f = gtid; f < F; f += gsz) {
    float m = 0.f, gm = 0.f;
    for (int n = 0; n < N; ++n) { m += x[(int64_t)n * F + f]; gm += ggx[(int64_t)n * F + f]; }
    m /= (float)N; gm /= (float)N;
    float v = 0.f, gd = 0.f;
    for (int n = 0; n < N; ++n) {
      float d = x[(int64_t)n * F + f] - m;
      v += d * d;
      gd += ggx[(int64_t)n * F + f] * d;
    }
    const float var = v / (float)N + 1e-8f;
    const float sig = sqrtf(var);
    const float k = 1.f / ((float)N * (float)F * sig);
    dG += gd * k;
    for (int n = 0; n < N; ++n) {
      float d = x[(int64_t)n * F + f] - m;
      dx[(int64_t)n * F + f] = G * k * (ggx[(int64_t)n * F + f] - gm - d * gd / ((float)N * var));
    }
  }
  dG = cluster_sum(block_sum(dG, sm), &slot);
  const int64_t total = (int64_t)N * P * Ct;
  for (int64_t i = gtid; i < total; i += gsz) {
    int64_t r = i / Ct;
    int c = (int)(i - r * Ct);
    dgout[i] = (c < C) ? ggx[r * C + c] : (c == C ? dG : 0.f);
  }
}

// ------------------------------------------------------------------------------------------------
// losses
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_sigmoid_ce(const float* __restrict__ x, float label, float weight,
                                                    float* __restrict__ loss, float* __restrict__ grad, int64_t n,
                                                    int accumulate) {
  __shared__ float sm[32];
  float acc = 0.f;
  const float wn = weight / (float)n;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    float v = x[i];
    acc += fmaxf(v, 0.f) - v * label + log1pf(expf(-fabsf(v)));
    if (grad) grad[i] = wn * (1.f / (1.f + expf(-v)) - label);
  }
  acc = block_sum(acc, sm);
  if (threadIdx.x == 0) loss[0] = (accumulate ? loss[0] : 0.f) + acc * wn;
}

// weight * mean f(sign*x + margin), f: 0 identity, 1 relu, 2 square (WGAN / hinge terms, image_generation.py:330-389)
__global__ void __launch_bounds__(256) k_logit_mean(const float* __restrict__ x, float* __restrict__ loss, int64_t n,
                                                    float sign, float margin, int kind, float weight) {
  __shared__ float sm[32];
  float acc = 0.f;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    const float u = fmaf(sign, x[i], margin);
    acc += kind == 1 ? fmaxf(u, 0.f) : (kind == 2 ? u * u : u);
  }
  acc = block_sum(acc, sm);
  if (threadIdx.x == 0) loss[0] = acc * (weight / (float)n);
}

__global__ void __launch_bounds__(256) k_logit_mean_bwd(const float* __restrict__ x, const float* __restrict__ gl,
                                                        float* __restrict__ gx, int64_t n, float sign, float margin,
                                                        int kind, float weight) {
  const float s = gl[0] * weight / (float)n * sign;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float u = fmaf(sign, x[i], margin);
    gx[i] = s * (kind == 1 ? (u > 0.f ? 1.f : 0.f) : (kind == 2 ? 2.f * u : 1.f));
  }
}

__global__ void __launch_bounds__(256) k_l1(const float* __restrict__ a, const float* __restrict__ b, float wn,
                                            float* __restrict__ loss, float* __restrict__ grad, int64_t n) {
  __shared__ float sm[32];
  float acc = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float d = a[i] - b[i];
    acc += fabsf(d);
    if (grad) grad[i] = d > 0.f ? wn : (d < 0.f ? -wn : 0.f);
  }
  acc = block_sum(acc, sm);
  if (threadIdx.x == 0) loss[blockIdx.x] = acc * wn;     // partial of this block (add_partials)
}

__global__ void __launch_bounds__(256) k_sum_sq(const float* __restrict__ x, double* __restrict__ out2, int64_t n) {
  __shared__ float sm[32];
  float a1 = 0.f, a2 = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float v = x[i];
    a1 += v;
    a2 += v * v;
  }
  a1 = block_sum(a1, sm);
  a2 = block_sum(a2, sm);
  if (threadIdx.x == 0) { out2[0] = (double)a1; out2[1] = (double)a2; }     // launched as one block
}

__global__ void __launch_bounds__(256) k_dragan_xhat(const float* __restrict__ x, const float* __restrict__ alpha,
                                                     const float* __restrict__ noise, float* __restrict__ xhat,
                                                     const double* __restrict__ s2, int N, int64_t per) {
  const double cnt = (double)N * (double)per;
  const double m = s2[0] / cnt;
  const float var = (float)fmax(s2[1] / cnt - m * m, 0.0);
  const int64_t total = (int64_t)N * per;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int n = (int)(i / per);
    xhat[i] = x[i] + alpha[n] * (0.5f * var * noise[i]);
  }
}

__global__ void __launch_bounds__(256) k_row_sumsq(const float* __restrict__ g, float* __restrict__ ss, int64_t per,
                                                   int64_t chunk) {
  __shared__ float sm[32];
  const int n = blockIdx.y;
  const int64_t i0 = (int64_t)blockIdx.x * chunk, i1 = min(per, i0 + chunk);
  float acc = 0.f;
  for (int64_t i = i0 + threadIdx.x; i < i1; i += blockDim.x) { float v = g[(int64_t)n * per + i]; acc += v * v; }
  acc = block_sum(acc, sm);
  if (threadIdx.x == 0) ss[(int64_t)blockIdx.x * gridDim.y + n] = acc;     // partial of this block (add_partials)
}

__global__ void k_grad_penalty_finalize(float* __restrict__ coef, float lambda, float* __restrict__ loss, int N,
                                        int accumulate) {
  // single warp-block; coef holds sum of squares on entry
  __shared__ float sm[32];
  float acc = 0.f;
  for (int n = threadIdx.x; n < N; n += blockDim.x) {
    float s = sqrtf(coef[n]);
    acc += (s - 1.f) * (s - 1.f);
    coef[n] = lambda * 2.f * (s - 1.f) / ((float)N * fmaxf(s, 1e-20f));
  }
  acc = block_sum(acc, sm);
  if (threadIdx.x == 0) loss[0] = (accumulate ? loss[0] : 0.f) + lambda * acc / (float)N;
}

__global__ void __launch_bounds__(256) k_scale_rows(const float* __restrict__ x, const float* __restrict__ coef,
                                                    const float* __restrict__ s, float* __restrict__ out, int N,
                                                    int64_t per) {
  const float f = s ? s[0] : 1.f;
  const int64_t total = (int64_t)N * per;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = x[i] * coef[i / per] * f;
}

__global__ void __launch_bounds__(256) k_adam(float* __restrict__ p, const float* __restrict__ g,
                                              float* __restrict__ m, float* __restrict__ v, int64_t n,
                                              const float* __restrict__ lr_dev, float lr_host, float b1, float b2,
                                              float eps) {
  const float lr_t = lr_dev ? lr_dev[0] : lr_host;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float gi = g[i];
    const float mi = b1 * m[i] + (1.f - b1) * gi;
    const float vi = b2 * v[i] + (1.f - b2) * gi * gi;
    m[i] = mi;
    v[i] = vi;
    p[i] -= lr_t * mi / (sqrtf(vi) + eps);
  }
}

// ------------------------------------------------------------------------------------------------
// TwinGAN wiring kernels for the batched passes (twingan.py:196-284, 370-381, 451-505).  The four generator passes run
// as ONE batch ordered [s_cycle | t_cycle | t_prime | s_prime] (B samples each) and x = [sources | targets].
// ------------------------------------------------------------------------------------------------
// One pass over the generator output: assembles the two discriminator batches ds = [sources | s_cycle | s_prime],
// dt = [targets | t_cycle | t_prime], the second encoder batch
// e2 = [t_prime | s_prime] and the cycle losses l_cyc_{s,t} = w * mean|x - cycle| with their sign gradients.
__global__ void __launch_bounds__(256) k_fanout_fwd(const float* __restrict__ gout, const float* __restrict__ x,
                                                    float* __restrict__ ds, float* __restrict__ dt, float* __restrict__ e2,
                                                    float* __restrict__ sgn, float* __restrict__ loss, float wn,
                                                    int64_t per4) {
  __shared__ float sm[32];
  float acc0 = 0.f, acc1 = 0.f;
  const int64_t fake1 = per4, fake2 = 2 * per4;     // row blocks of the cycle / prime fakes in ds, dt
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < 4 * per4; i += (int64_t)gridDim.x * blockDim.x) {
    const int r = (int)(i / per4);
    const int64_t j = i - r * per4;
    const float4 v = ld4(gout, i);
    if (r < 2) {
      const float4 xv = ld4(x, i);                       // sources (r = 0) / targets (r = 1)
      float* dd = r == 0 ? ds : dt;
      st4(dd, j, xv);
      st4(dd, fake1 + j, v);
      const float d0 = v.x - xv.x, d1 = v.y - xv.y, d2 = v.z - xv.z, d3 = v.w - xv.w;
      const float a = fabsf(d0) + fabsf(d1) + fabsf(d2) + fabsf(d3);
      if (r == 0) acc0 += a; else acc1 += a;
      st4(sgn, i, make_float4(d0 > 0.f ? wn : (d0 < 0.f ? -wn : 0.f), d1 > 0.f ? wn : (d1 < 0.f ? -wn : 0.f),
                              d2 > 0.f ? wn : (d2 < 0.f ? -wn : 0.f), d3 > 0.f ? wn : (d3 < 0.f ? -wn : 0.f)));
    } else if (r == 2) {
      st4(dt, fake2 + j, v);
      st4(e2, j, v);
    } else {
      st4(ds, fake2 + j, v);
      st4(e2, per4 + j, v);
    }
  }
  acc0 = block_sum(acc0, sm);
  acc1 = block_sum(acc1, sm);
  if (threadIdx.x == 0) { loss[2 * blockIdx.x] = acc0 * wn; loss[2 * blockIdx.x + 1] = acc1 * wn; }   // partials
}

// gradient w.r.t. the generator output: sum of what the discriminator batches, the second encoder batch and the
// cycle losses send back (any of them may be absent)
__global__ void __launch_bounds__(256) k_fanout_bwd(const float* __restrict__ gds, const float* __restrict__ gdt,
                                                    const float* __restrict__ ge2, const float* __restrict__ sgn,
                                                    const float* __restrict__ gl_s, const float* __restrict__ gl_t,
                                                    float* __restrict__ gg, int64_t per4) {
  const int64_t fake1 = per4, fake2 = 2 * per4;
  const float ls = gl_s ? gl_s[0] : 0.f, lt = gl_t ? gl_t[0] : 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < 4 * per4; i += (int64_t)gridDim.x * blockDim.x) {
    const int r = (int)(i / per4);
    const int64_t j = i - r * per4;
    float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
    auto add = [&](const float* p, int64_t k, float f) {
      const float4 t = ld4(p, k);
      o.x = fmaf(f, t.x, o.x); o.y = fmaf(f, t.y, o.y); o.z = fmaf(f, t.z, o.z); o.w = fmaf(f, t.w, o.w);
    };
    if (r < 2) {
      const float* gd = r == 0 ? gds : gdt;
      if (gd) add(gd, fake1 + j, 1.f);
      const float l = r == 0 ? ls : lt;
      if (l != 0.f) add(sgn, i, l);
    } else if (r == 2) {
      if (gdt) add(gdt, fake2 + j, 1.f);
      if (ge2) add(ge2, j, 1.f);
    } else {
      if (gds) add(gds, fake2 + j, 1.f);
      if (ge2) add(ge2, per4 + j, 1.f);
    }
    st4(gg, i, o);
  }
}

// grouped L1: loss[g] = w * mean_g |a - b| over `groups` equal row blocks; grad = w/n_g * sign(a - b)
__global__ void __launch_bounds__(256) k_l1_groups(const float* __restrict__ a, const float* __restrict__ b, float wn,
                                                   float* __restrict__ loss, float* __restrict__ grad, int64_t per) {
  __shared__ float sm[32];
  const int g = blockIdx.y;
  float acc = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < per; i += (int64_t)gridDim.x * blockDim.x) {
    const float d = a[g * per + i] - b[g * per + i];
    acc += fabsf(d);
    grad[g * per + i] = d > 0.f ? wn : (d < 0.f ? -wn : 0.f);
  }
  acc = block_sum(acc, sm);
  if (threadIdx.x == 0) loss[(int64_t)blockIdx.x * gridDim.y + g] = acc * wn;     // partial of this block (add_partials)
}

// out[g*per + i] = grad[g*per + i] * sign * (gl_g ? *gl_g : 0)
__global__ void __launch_bounds__(256) k_scale_groups2(const float* __restrict__ grad, const float* __restrict__ gl0,
                                                       const float* __restrict__ gl1, float sign, float* __restrict__ out,
                                                       int64_t per) {
  const int g = blockIdx.y;
  const float* gl = g == 0 ? gl0 : gl1;
  const float f = gl ? sign * gl[0] : 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < per; i += (int64_t)gridDim.x * blockDim.x)
    out[g * per + i] = grad[g * per + i] * f;
}

// The sigmoid cross-entropy GAN losses of one discriminator batch [real | cycle | prime] (B logits each),
// image_generation.py:341-344, 392-401:
//   loss[0] = CE(1, cycle) generator_fool_cycle        loss[1] = CE(1, prime) generator_fool_prime
//   loss[2] = CE(0, cycle) discriminator_fake_cycle    loss[3] = CE(1, real)  discriminator_real (cycle term's copy)
//   loss[4] = CE(0, prime) discriminator_fake_prime    loss[5] = CE(1, real)  discriminator_real (prime term's copy)
// each = weight * mean over its B logits.  sig[i] = sigmoid(logit_i) is kept for the backward.
__device__ __forceinline__ float ce_term(float v, float label) { return fmaxf(v, 0.f) - v * label + log1pf(expf(-fabsf(v))); }
__global__ void __launch_bounds__(256) k_gan_losses(const float* __restrict__ x, float weight, float* __restrict__ loss,
                                                    float* __restrict__ sig, int B) {
  __shared__ float sm[32];
  float a[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
  for (int i = threadIdx.x; i < 3 * B; i += blockDim.x) {
    const float v = x[i];
    sig[i] = 1.f / (1.f + expf(-v));
    const int blk = i / B;
    if (blk == 0) a[3] += ce_term(v, 1.f);
    else if (blk == 1) { a[0] += ce_term(v, 1.f); a[2] += ce_term(v, 0.f); }
    else { a[1] += ce_term(v, 1.f); a[4] += ce_term(v, 0.f); }
  }
  const float wn = weight / (float)B;
  for (int k = 0; k < 5; ++k) {
    const float t = block_sum(a[k], sm);
    if (threadIdx.x == 0) { loss[k] = t * wn; if (k == 3) loss[5] = t * wn; }
    __syncthreads();
  }
}
// grad[i] = weight/B * sum_k g_k * (sig_i - label_k) over the losses that contain logit i (g_k device scalars, nullable)
__global__ void __launch_bounds__(256) k_gan_losses_bwd(const float* __restrict__ sig, float weight,
                                                        const float* __restrict__ g0, const float* __restrict__ g1,
                                                        const float* __restrict__ g2, const float* __restrict__ g3,
                                                        const float* __restrict__ g4, const float* __restrict__ g5,
                                                        float* __restrict__ grad, int B) {
  const float wn = weight / (float)B;
  const float u0 = g0 ? g0[0] : 0.f, u1 = g1 ? g1[0] : 0.f, u2 = g2 ? g2[0] : 0.f,
              u3 = (g3 ? g3[0] : 0.f) + (g5 ? g5[0] : 0.f), u4 = g4 ? g4[0] : 0.f;
  for (int i = threadIdx.x; i < 3 * B; i += blockDim.x) {
    const float s = sig[i];
    const int blk = i / B;
    float g;
    if (blk == 0) g = u3 * (s - 1.f);
    else if (blk == 1) g = u0 * (s - 1.f) + u2 * s;
    else g = u1 * (s - 1.f) + u4 * s;
    grad[i] = wn * g;
  }
}

// out[0] = scale * sum of n <= 16 device scalars (pointers passed by value)
struct ScalarPtrs { const float* p[16]; };
__global__ void k_sum_scalars(ScalarPtrs ptrs, int n, float scale, float* __restrict__ out) {
  float a = 0.f;
  for (int k = 0; k < n; ++k) a += ptrs.p[k][0];
  out[0] = a * scale;
}

// ------------------------------------------------------------------------------------------------
// Step counters on the device ({adam_t, global_step} int32): a captured CUDA graph of the step can be replayed while
// Adam's bias correction (model/model_inheritor.py:537-542, t shared by the generator and discriminator applies) and
// the batch-renorm clipping schedule (nets/pggan_utils.py:44-47, tf.train.piecewise_constant) keep advancing.
// ------------------------------------------------------------------------------------------------
__global__ void k_step_schedule(const int* __restrict__ counters, float lr, float b1, float b2, float* __restrict__ lr_out,
                                float* __restrict__ clip_out) {
  const int t = counters[0], gs = counters[1];
  for (int i = 0; i < 2; ++i) {       // the two applies of a mode-B step use t+1 and t+2
    const double tt = (double)(t + 1 + i);
    lr_out[i] = (float)((double)lr * sqrt(1.0 - pow((double)b2, tt)) / (1.0 - pow((double)b1, tt)));
  }
  const int idx = (gs > 10000) + (gs > 20000) + (gs > 30000);
  const float rmax[4] = {1.1f, 1.5f, 2.0f, 4.0f}, rmin[4] = {0.9f, 0.66f, 0.5f, 0.25f}, dmax[4] = {0.1f, 0.3f, 0.5f, 1.0f};
  clip_out[0] = rmin[idx]; clip_out[1] = rmax[idx]; clip_out[2] = dmax[idx];
}
__global__ void k_step_advance(int* __restrict__ counters, int d_adam_t, int d_global_step) {
  counters[0] += d_adam_t;
  counters[1] += d_global_step;
}

// all weight tensors of the model in one launch: table rows {src offset (floats), dst offset (bf16 elements of the hi
// plane), taps, Cin, Cout, dgrad}; blockIdx.y = table row.  dst holds hi at [off, off + n) and lo at [off + n, off + 2n).
struct SplitRow { long long src, dst; int taps, cin, cout, dgrad; };
__global__ void __launch_bounds__(256) k_split_weights_table(const float* __restrict__ flat, __nv_bfloat16* __restrict__ planes,
                                                             const SplitRow* __restrict__ table) {
  const SplitRow r = table[blockIdx.y];
  const float* w = flat + r.src;
  const int64_t total = (int64_t)r.taps * r.cin * r.cout;
  __nv_bfloat16* hi = planes + r.dst;
  __nv_bfloat16* lo = hi + total;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t t = i;
    float v;
    if (!r.dgrad) {
      const int ci = (int)(t % r.cin); t /= r.cin;
      const int co = (int)(t % r.cout);
      const int tap = (int)(t / r.cout);
      v = w[((int64_t)tap * r.cin + ci) * r.cout + co];
    } else {
      const int co = (int)(t % r.cout); t /= r.cout;
      const int ci = (int)(t % r.cin);
      const int tap = (int)(t / r.cin);
      v = w[((int64_t)(r.taps - 1 - tap) * r.cin + ci) * r.cout + co];
    }
    const __nv_bfloat16 h = __float2bfloat16_rn(v);
    hi[i] = h;
    lo[i] = __float2bfloat16_rn(v - __bfloat162float(h));
  }
}

static inline int grid_for(int64_t n, int per_thread = 4) {
  int64_t b = cdiv(n, (int64_t)256 * per_thread);
  int64_t cap = (int64_t)kNumSMs * 16;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (int)b;
}

}  // namespace twg

using namespace twg;

extern "C" {

int twg_version(void) { return 101; }
const char* twg_last_error(void) { return g_err; }
int64_t twg_launch_count(void) { return g_launches.load(); }

int twg_moments(const float* y, float* sums, int N, int HW, int C, int pivot_group, twg_stream_t stream) {
  if (!y || !sums || N <= 0 || HW <= 0 || C <= 0 || pivot_group <= 0 || N % pivot_group)
    return fail(TWG_ERR_INVALID, "twg_moments: bad args");
  cudaMemsetAsync(sums, 0, sizeof(float) * 2 * N * C, S(stream));
  VecGeom g = vec_geom(C);
  if (g.ok) {
    int gpb = 256 / g.G;
    int chunk = pick_chunk(HW, N, gpb);
    dim3 grid((unsigned)cdiv(HW, chunk), N);
    if (g.V == 1) k_moments_vec<1><<<grid, 256, 0, S(stream)>>>(y, sums, HW, C, g.G, chunk, pivot_group);
    else if (g.V == 2) k_moments_vec<2><<<grid, 256, 0, S(stream)>>>(y, sums, HW, C, g.G, chunk, pivot_group);
    else k_moments_vec<4><<<grid, 256, 0, S(stream)>>>(y, sums, HW, C, g.G, chunk, pivot_group);
  } else {
    if (C > 64) return fail(TWG_ERR_UNSUPPORTED, "twg_moments: C=%d unsupported", C);
    int chunk = pick_chunk(HW, N, 256);
    dim3 grid((unsigned)cdiv(HW, chunk), N);
    k_moments_scalar<<<grid, 256, 0, S(stream)>>>(y, sums, HW, C, chunk, pivot_group);
  }
  return check_launch("twg_moments");
}

int twg_norm_finalize(const float* sums, const float* y, const float* gamma0, const float* beta0, const float* gamma1,
                      const float* beta1, int dom_mask, int group_size, const float* renorm0, const float* renorm1,
                      int kind, float eps, const float* clip, float* a, float* b, float* mean, float* rstd, float* rd_out,
                      float* batch_stats, int N, int HW, int C, twg_stream_t stream) {
  if (!a || !b || !mean || !rstd) return fail(TWG_ERR_INVALID, "twg_norm_finalize: null output");
  if (group_size <= 0 || N % group_size || N / group_size > 32) return fail(TWG_ERR_INVALID, "twg_norm_finalize: bad group size");
  if (kind != TWG_NORM_NONE && (!sums || !y)) return fail(TWG_ERR_INVALID, "twg_norm_finalize: null sums / pivot source");
  if (kind == TWG_NORM_RENORM && (!renorm0 || (dom_mask && !renorm1)))
    return fail(TWG_ERR_INVALID, "twg_norm_finalize: renorm state missing");
  if (kind == TWG_NORM_INSTANCE)
    k_norm_finalize_inst<<<(unsigned)cdiv((int64_t)N * C, 256), 256, 0, S(stream)>>>(sums, y, gamma0, beta0, gamma1, beta1,
                                                                                      (unsigned)dom_mask, group_size, eps, a, b,
                                                                                      mean, rstd, N, HW, C);
  else
    k_norm_finalize<<<(unsigned)cdiv(C, 64), 64, 0, S(stream)>>>(sums, y, gamma0, beta0, gamma1, beta1, (unsigned)dom_mask,
                                                                  group_size, renorm0, renorm1, kind, eps, clip, a, b, mean,
                                                                  rstd, rd_out, batch_stats, N, HW, C);
  return check_launch("twg_norm_finalize");
}

int twg_norm_finalize_partials(const float* stats, int slots, const float* gamma0, const float* beta0, const float* gamma1,
                               const float* beta1, int dom_mask, int group_size, float eps, float* a, float* b, float* mean,
                               float* rstd, int N, int C, twg_stream_t stream) {
  if (!stats || slots <= 0 || !a || !b || !mean || !rstd || N <= 0 || C <= 0)
    return fail(TWG_ERR_INVALID, "twg_norm_finalize_partials: bad args");
  if (group_size <= 0 || N % group_size || N / group_size > 32) return fail(TWG_ERR_INVALID, "twg_norm_finalize_partials: bad group size");
  k_norm_finalize_inst_partials<<<(unsigned)cdiv((int64_t)N * C, 8), 256, 0, S(stream)>>>(
      reinterpret_cast<const float4*>(stats), slots, gamma0, beta0, gamma1, beta1, (unsigned)dom_mask, group_size, eps, a, b,
      mean, rstd, N, C);
  return check_launch("twg_norm_finalize_partials");
}

int twg_norm_eval_affine(const float* gamma, const float* beta, const float* moving_mean, const float* moving_var,
                         float eps, float* a, float* b, int N, int C, twg_stream_t stream) {
  if (!gamma || !beta || !moving_mean || !moving_var || !a || !b) return fail(TWG_ERR_INVALID, "twg_norm_eval_affine: null");
  k_norm_eval_affine<<<(unsigned)cdiv(C, 64), 64, 0, S(stream)>>>(gamma, beta, moving_mean, moving_var, eps, a, b, N, C);
  return check_launch("twg_norm_eval_affine");
}

int twg_norm_update_stats(float* state, const float* batch_stats, int kind, float decay, float eps, int C,
                          twg_stream_t stream) {
  if (!state || !batch_stats || C > 1024) return fail(TWG_ERR_INVALID, "twg_norm_update_stats: bad args");
  int threads = (int)cdiv(C, 32) * 32;
  k_norm_update_stats<<<1, threads, 0, S(stream)>>>(state, batch_stats, kind, decay, eps, C);
  return check_launch("twg_norm_update_stats");
}

int twg_norm_act_fwd(const float* y, const float* a, const float* b, float* z, void* planes, int N, int HW, int C,
                     int flags, twg_stream_t stream) {
  if (!y || !a || !b || (!z && !planes)) return fail(TWG_ERR_INVALID, "twg_norm_act_fwd: null");
  const int64_t total = (int64_t)N * HW;
  VecGeom g = vec_geom(C);
  if (g.ok) {
    int gpb = 256 / g.G;
    int64_t blocks = cdiv(total, (int64_t)gpb * 4);
    if (blocks > kNumSMs * 16) blocks = kNumSMs * 16;
    if (g.V == 1) k_norm_act_fwd_vec<1><<<(unsigned)blocks, 256, 0, S(stream)>>>(y, a, b, z, planes, total, HW, C, g.G, flags);
    else if (g.V == 2) k_norm_act_fwd_vec<2><<<(unsigned)blocks, 256, 0, S(stream)>>>(y, a, b, z, planes, total, HW, C, g.G, flags);
    else k_norm_act_fwd_vec<4><<<(unsigned)blocks, 256, 0, S(stream)>>>(y, a, b, z, planes, total, HW, C, g.G, flags);
  } else {
    if (planes || !z) return fail(TWG_ERR_UNSUPPORTED, "twg_norm_act_fwd: split-plane output needs a vectorisable channel count");
    k_norm_act_fwd_scalar<<<grid_for(total, 1), 256, 0, S(stream)>>>(y, a, b, z, total, HW, C, flags);
  }
  return check_launch("twg_norm_act_fwd");
}

int twg_norm_act_bwd_reduce(const float* y, const float* a, const float* b, const float* mean, const float* rstd,
                            const float* gz, const float* gpool, int W, float* gu, float* red, int N, int HW, int C,
                            int flags, twg_stream_t stream) {
  if (!y || !a || !b || !mean || !rstd || (!gz && !gpool) || !gu || !red) return fail(TWG_ERR_INVALID, "twg_norm_act_bwd_reduce: null");
  if (gpool && (W <= 0 || W % 2 || HW % W || (HW / W) % 2 || !vec_geom(C).ok))
    return fail(TWG_ERR_UNSUPPORTED, "twg_norm_act_bwd_reduce: the pool gradient needs even H, W and a vectorisable C");
  cudaMemsetAsync(red, 0, sizeof(float) * 2 * N * C, S(stream));
  VecGeom g = vec_geom(C);
  if (g.ok) {
    int gpb = 256 / g.G;
    int chunk = pick_chunk(HW, N, gpb);
    dim3 grid((unsigned)cdiv(HW, chunk), N);
    if (g.V == 1) k_norm_act_bwd_reduce_vec<1><<<grid, 256, 0, S(stream)>>>(y, a, b, mean, rstd, gz, gu, red, HW, C, g.G, flags, chunk, gpool, W);
    else if (g.V == 2) k_norm_act_bwd_reduce_vec<2><<<grid, 256, 0, S(stream)>>>(y, a, b, mean, rstd, gz, gu, red, HW, C, g.G, flags, chunk, gpool, W);
    else k_norm_act_bwd_reduce_vec<4><<<grid, 256, 0, S(stream)>>>(y, a, b, mean, rstd, gz, gu, red, HW, C, g.G, flags, chunk, gpool, W);
  } else {
    if (C > 64) return fail(TWG_ERR_UNSUPPORTED, "twg_norm_act_bwd_reduce: C=%d unsupported", C);
    int chunk = pick_chunk(HW, N, 256);
    dim3 grid((unsigned)cdiv(HW, chunk), N);
    k_norm_act_bwd_reduce_scalar<<<grid, 256, 0, S(stream)>>>(y, a, b, mean, rstd, gz, gu, red, HW, C, flags, chunk);
  }
  return check_launch("twg_norm_act_bwd_reduce");
}

int twg_norm_act_bwd_apply(const float* y, const float* a, const float* mean, const float* rstd, const float* gu,
                           const float* red, const float* rd, float* gy, void* gy_planes, float* ggamma0, float* gbeta0,
                           float* ggamma1, float* gbeta1, int accumulate, int dom_mask, int group_size, int kind, int N,
                           int HW, int C, twg_stream_t stream) {
  if (!y || !a || !mean || !rstd || !gu || !red || (!gy && !gy_planes)) return fail(TWG_ERR_INVALID, "twg_norm_act_bwd_apply: null");
  if (gy_planes && (C % 4)) return fail(TWG_ERR_UNSUPPORTED, "twg_norm_act_bwd_apply: split-plane output needs C % 4 == 0");
  if (group_size <= 0 || N % group_size || N / group_size > 32) return fail(TWG_ERR_INVALID, "twg_norm_act_bwd_apply: bad group size");
  if (kind == TWG_NORM_INSTANCE) {
    if (!accumulate) {
      float* outs[4] = {ggamma0, gbeta0, ggamma1, gbeta1};
      for (float* o : outs)
        if (o) cudaMemsetAsync(o, 0, sizeof(float) * C, S(stream));
    }
    k_norm_bwd_coeffs_inst<<<(unsigned)cdiv((int64_t)C, 256), 256, 0, S(stream)>>>(const_cast<float*>(red), ggamma0, gbeta0,
                                                                                        ggamma1, gbeta1, (unsigned)dom_mask,
                                                                                        group_size, N, HW, C);
  } else {
    k_norm_bwd_coeffs<<<(unsigned)cdiv(C, 64), 64, 0, S(stream)>>>(const_cast<float*>(red), rd, ggamma0, gbeta0, ggamma1, gbeta1,
                                                                    (unsigned)dom_mask, group_size, kind, N, HW, C, accumulate);
  }
  int rc = check_launch("twg_norm_bwd_coeffs");
  if (rc) return rc;
  const int64_t total = (int64_t)N * HW * C;
  const int vec = (C % 4 == 0) ? 4 : 1;
  const int64_t per = (int64_t)HW * C / vec;                       // vectors per sample
  if (per > (int64_t)1 << 30) return fail(TWG_ERR_UNSUPPORTED, "twg_norm_act_bwd_apply: sample too large");
  int64_t bx = cdiv(per, 256 * 4);                                 // >= 4 vectors per thread ...
  const int64_t want = cdiv(16 * kNumSMs, N);                      // ... and ~16 blocks per SM over the whole grid
  if (bx > want) bx = want;
  if (bx < 1) bx = 1;
  dim3 grid((unsigned)bx, (unsigned)N);
  if (vec == 4)
    k_norm_act_bwd_apply<4><<<grid, 256, 0, S(stream)>>>(y, a, mean, rstd, gu, red, gy, gy_planes, total / 4, HW, C);
  else
    k_norm_act_bwd_apply<1><<<grid, 256, 0, S(stream)>>>(y, a, mean, rstd, gu, red, gy, nullptr, total, HW, C);
  return check_launch("twg_norm_act_bwd_apply");
}

int twg_bias_lrelu_fwd(const float* y, const float* bias, float* z, void* planes, void* mask, int64_t rows, int C,
                       int lrelu_on, twg_stream_t stream) {
  if (!y || !z) return fail(TWG_ERR_INVALID, "twg_bias_lrelu_fwd: null");
  if ((planes || mask) && C % 4) return fail(TWG_ERR_UNSUPPORTED, "twg_bias_lrelu_fwd: planes / mask need C % 4 == 0");
  const int64_t total = rows * C;
  if (C % 4 == 0)
    k_bias_lrelu<4><<<grid_for(total / 4, 2), 256, 0, S(stream)>>>(y, bias, z, total / 4, C, lrelu_on, planes,
                                                                    reinterpret_cast<uint8_t*>(mask));
  else k_bias_lrelu<1><<<grid_for(total, 2), 256, 0, S(stream)>>>(y, bias, z, total, C, lrelu_on, nullptr, nullptr);
  return check_launch("twg_bias_lrelu_fwd");
}

int twg_lrelu_bwd(const float* g, const float* ref, float* out, int64_t n, twg_stream_t stream) {
  if (!g || !ref || !out) return fail(TWG_ERR_INVALID, "twg_lrelu_bwd: null");
  k_lrelu_bwd<<<grid_for(n / 4 + 1, 2), 256, 0, S(stream)>>>(g, ref, out, n);
  return check_launch("twg_lrelu_bwd");
}

int twg_colsum(const float* g, float* out, int64_t rows, int C, int accumulate, twg_stream_t stream) {
  if (!g || !out) return fail(TWG_ERR_INVALID, "twg_colsum: null");
  if (!accumulate) cudaMemsetAsync(out, 0, sizeof(float) * C, S(stream));
  int64_t blocks = cdiv(rows, 256);
  if (blocks > 4 * kNumSMs) blocks = 4 * kNumSMs;
  int64_t chunk = cdiv(rows, blocks);
  blocks = cdiv(rows, chunk);
  float* parts = partials(blocks * C, true, S(stream));
  if (!parts) return fail(TWG_ERR_UNSUPPORTED, "twg_colsum: C=%d too wide", C);
  k_colsum<<<(unsigned)blocks, 256, 0, S(stream)>>>(g, parts, rows, C, chunk);
  int rc = check_launch("twg_colsum");
  return rc ? rc : add_partials(out, parts, (int)blocks, C, S(stream));
}

int twg_lrelu_bwd_colsum(const float* g, const float* ref, const void* mask, float* out, void* planes, float* colsum,
                         int64_t rows, int C, int lrelu_on, int poolH, int poolW, int accumulate, twg_stream_t stream) {
  const uint8_t* mk = reinterpret_cast<const uint8_t*>(mask);
  if (mk && !vec_geom(C).ok) return fail(TWG_ERR_UNSUPPORTED, "twg_lrelu_bwd_colsum: the sign mask needs a vectorisable C");
  if (mk) ref = ref ? ref : reinterpret_cast<const float*>(mk);      // only tested for null below
  if (poolW > 0 && (poolH <= 0 || poolH % 2 || poolW % 2 || rows % ((int64_t)poolH * poolW) || !vec_geom(C).ok))
    return fail(TWG_ERR_UNSUPPORTED, "twg_lrelu_bwd_colsum: the pool gradient needs even H, W and a vectorisable C");
  if (!g || !colsum || (lrelu_on && (!ref || (!out && !planes)))) return fail(TWG_ERR_INVALID, "twg_lrelu_bwd_colsum: null");
  if (!accumulate) cudaMemsetAsync(colsum, 0, sizeof(float) * C, S(stream));
  VecGeom gm = vec_geom(C);
  if (!gm.ok) {   // odd widths (C=1 logits, C=257): two plain passes
    if (planes || (lrelu_on && !out)) return fail(TWG_ERR_UNSUPPORTED, "twg_lrelu_bwd_colsum: split-plane output needs a vectorisable C");
    if (lrelu_on) {
      k_lrelu_bwd<<<grid_for(rows * C / 4 + 1, 2), 256, 0, S(stream)>>>(g, ref, out, rows * C);
      int rc = check_launch("twg_lrelu_bwd_colsum/lrelu");
      if (rc) return rc;
    }
    return twg_colsum(lrelu_on ? out : g, colsum, rows, C, 1, stream);
  }
  if (poolW > 0 && lrelu_on && planes && !out && gm.V == 1 && poolW >= 2 * (256 / gm.G) && rows / poolW < (1ll << 31)) {
    // the first-order backward of a pooled discriminator layer (the common case): by image rows, no per-element divisions.
    // (0.25 * slope is applied as one factor: the products differ from the flat form's (0.25 g) * slope by at most an ulp)
    int lq = 0;
    while ((1 << lq) < gm.G) ++lq;
    const int img_rows = (int)(rows / poolW);
    int rpb = (int)cdiv(img_rows, (int64_t)8 * kNumSMs);
    if (rpb < 1) rpb = 1;
    const unsigned nb = (unsigned)cdiv(img_rows, rpb);
    float* parts = partials((int64_t)nb * C, true, S(stream));
    if (!parts) return fail(TWG_ERR_UNSUPPORTED, "twg_lrelu_bwd_colsum: C=%d too wide", C);
    if (mk) k_lrelu_bwd_colsum_pool_rows<true><<<nb, 256, 0, S(stream)>>>(g, ref, planes, parts, img_rows, poolH, poolW, lq, rpb, mk, rows * C);
    else k_lrelu_bwd_colsum_pool_rows<false><<<nb, 256, 0, S(stream)>>>(g, ref, planes, parts, img_rows, poolH, poolW, lq, rpb, mk, rows * C);
    int rc = check_launch("twg_lrelu_bwd_colsum");
    return rc ? rc : add_partials(colsum, parts, (int)nb, C, S(stream));
  }
  const int gpb = 256 / gm.G;
  int64_t blocks = cdiv(rows, (int64_t)gpb * 16);
  if (blocks > 8 * kNumSMs) blocks = 8 * kNumSMs;
  if (blocks < 1) blocks = 1;
  const int64_t chunk = cdiv(rows, blocks);
  blocks = cdiv(rows, chunk);
  float* parts = partials(blocks * C, true, S(stream));
  if (!parts) return fail(TWG_ERR_UNSUPPORTED, "twg_lrelu_bwd_colsum: C=%d too wide", C);
#define TWG_LBC(v, m) k_lrelu_bwd_colsum_vec<v, m><<<(unsigned)blocks, 256, 0, S(stream)>>>(g, ref, out, planes, parts, rows, C, gm.G, chunk, lrelu_on, poolH, poolW, mk)
  const bool use_mask = mk != nullptr && lrelu_on;
  if (gm.V == 1) { if (use_mask) TWG_LBC(1, true); else TWG_LBC(1, false); }
  else if (gm.V == 2) { if (use_mask) TWG_LBC(2, true); else TWG_LBC(2, false); }
  else { if (use_mask) TWG_LBC(4, true); else TWG_LBC(4, false); }
#undef TWG_LBC
  if (int rc = check_launch("twg_lrelu_bwd_colsum")) return rc;
  return add_partials(colsum, parts, (int)blocks, C, S(stream));
}

int twg_pool2(const float* x, float* out, void* planes, int N, int H, int W, int C, float scale, twg_stream_t stream) {
  if (!x || (!out && !planes) || (H & 1) || (W & 1)) return fail(TWG_ERR_INVALID, "twg_pool2: bad args");
  const int64_t total = (int64_t)N * (H / 2) * (W / 2) * C;
  if (C % 4 == 0 && (int64_t)N * (H / 2) < (1ll << 31) && (int64_t)(W / 2) * (C / 4) >= 64)
    k_pool2_rows<<<(unsigned)(N * (H / 2)), 256, 0, S(stream)>>>(x, out, planes, H, W, C / 4, scale, total);
  else if (C % 4 == 0) k_pool2<4><<<grid_for(total / 4, 2), 256, 0, S(stream)>>>(x, out, planes, N, H, W, C, scale);
  else {
    if (planes || !out) return fail(TWG_ERR_UNSUPPORTED, "twg_pool2: split-plane output needs C % 4 == 0");
    k_pool2<1><<<grid_for(total, 2), 256, 0, S(stream)>>>(x, out, nullptr, N, H, W, C, scale);
  }
  return check_launch("twg_pool2");
}

int twg_upsample2(const float* x, float* out, int N, int H, int W, int C, float scale, twg_stream_t stream) {
  if (!x || !out) return fail(TWG_ERR_INVALID, "twg_upsample2: null");
  const int64_t total = (int64_t)N * H * W * 4 * C;
  if (C % 4 == 0) k_upsample2<4><<<grid_for(total / 4, 2), 256, 0, S(stream)>>>(x, out, N, H, W, C, scale);
  else k_upsample2<1><<<grid_for(total, 2), 256, 0, S(stream)>>>(x, out, N, H, W, C, scale);
  return check_launch("twg_upsample2");
}

int twg_upsample_concat(const float* a, const float* b, float* out, void* planes, int N, int H, int W, int Ca, int Cb,
                        int Nb, twg_stream_t stream) {
  if (!a || !b || (!out && !planes)) return fail(TWG_ERR_INVALID, "twg_upsample_concat: null");
  if (Nb <= 0 || N % Nb) return fail(TWG_ERR_INVALID, "twg_upsample_concat: skip batch %d does not divide %d", Nb, N);
  const int64_t total = (int64_t)N * H * W * 4 * (Ca + Cb);
  if (Ca % 4 == 0 && Cb % 4 == 0) {
    if ((int64_t)N * 2 * H < (1ll << 31) && (int64_t)2 * W * ((Ca + Cb) / 4) >= 64)
      k_upsample_concat_rows<<<(unsigned)(N * 2 * H), 256, 0, S(stream)>>>(a, b, out, planes, H, W, Ca / 4, Cb / 4, Nb, total);
    else
      k_upsample_concat<4><<<grid_for(total / 4, 2), 256, 0, S(stream)>>>(a, b, out, planes, N, H, W, Ca, Cb, Nb);
  } else {
    if (planes || !out) return fail(TWG_ERR_UNSUPPORTED, "twg_upsample_concat: split-plane output needs C % 4 == 0");
    k_upsample_concat<1><<<grid_for(total, 2), 256, 0, S(stream)>>>(a, b, out, nullptr, N, H, W, Ca, Cb, Nb);
  }
  return check_launch("twg_upsample_concat");
}

int twg_upsample_concat_bwd(const float* gout, float* ga, float* gb, int N, int H, int W, int Ca, int Cb, int Nb,
                            twg_stream_t stream) {
  if (!gout || !ga || !gb) return fail(TWG_ERR_INVALID, "twg_upsample_concat_bwd: null");
  if (Nb <= 0 || N % Nb) return fail(TWG_ERR_INVALID, "twg_upsample_concat_bwd: skip batch %d does not divide %d", Nb, N);
  const int64_t total = (int64_t)H * W * ((int64_t)N * Ca + 4 * (int64_t)Nb * Cb);
  if (Ca % 4 == 0 && Cb % 4 == 0 && (int64_t)W * (Ca / 4) >= 64 && (int64_t)Nb * 2 * H + (int64_t)N * H < (1ll << 31))
    k_upsample_concat_bwd_rows<<<(unsigned)(Nb * 2 * H + N * H), 256, 0, S(stream)>>>(gout, ga, gb, N, H, W, Ca / 4, Cb / 4, Nb);
  else if (Ca % 4 == 0 && Cb % 4 == 0) k_upsample_concat_bwd<4><<<grid_for(total / 4, 2), 256, 0, S(stream)>>>(gout, ga, gb, N, H, W, Ca, Cb, Nb);
  else k_upsample_concat_bwd<1><<<grid_for(total, 2), 256, 0, S(stream)>>>(gout, ga, gb, N, H, W, Ca, Cb, Nb);
  return check_launch("twg_upsample_concat_bwd");
}

int twg_axpby(const float* x, const float* y, float* out, float alpha, float beta, int64_t n, twg_stream_t stream) {
  if (!x || !out) return fail(TWG_ERR_INVALID, "twg_axpby: null");
  k_axpby<<<grid_for(n / 4 + 1, 2), 256, 0, S(stream)>>>(x, y, out, alpha, beta, n);
  return check_launch("twg_axpby");
}

int twg_scale_by_dev(const float* x, const float* dev_scalar, float* out, float alpha, int64_t n, twg_stream_t stream) {
  if (!x || !dev_scalar || !out) return fail(TWG_ERR_INVALID, "twg_scale_by_dev: null");
  k_scale_by_dev<<<grid_for(n, 4), 256, 0, S(stream)>>>(x, dev_scalar, out, alpha, n);
  return check_launch("twg_scale_by_dev");
}

int twg_copy_cols(const float* src, float* dst, int64_t rows, int Csrc, int src_off, int Cdst, int dst_off, int ncols,
                  twg_stream_t stream) {
  if (!src || !dst || src_off + ncols > Csrc || dst_off + ncols > Cdst) return fail(TWG_ERR_INVALID, "twg_copy_cols: bad args");
  k_copy_cols<<<grid_for(rows * ncols, 4), 256, 0, S(stream)>>>(src, dst, rows, Csrc, src_off, Cdst, dst_off, ncols);
  return check_launch("twg_copy_cols");
}

int twg_mbstd_fwd(const float* x, float* out, float* s_out, int N, int P, int C, int Ct, int groups, twg_stream_t stream) {
  if (!x || !out) return fail(TWG_ERR_INVALID, "twg_mbstd_fwd: null");
  if (groups <= 0 || N % groups) return fail(TWG_ERR_INVALID, "twg_mbstd: %d groups do not divide %d samples", groups, N);
  if (Ct < C + 1) return fail(TWG_ERR_INVALID, "twg_mbstd: %d output channels < %d + 1", Ct, C);
  k_mbstd_fwd<<<kMbCluster * groups, 512, 0, S(stream)>>>(x, out, s_out, N / groups, P, C, Ct);
  return check_launch("twg_mbstd_fwd");
}
int twg_mbstd_bwd(const float* x, const float* gout, float* gx, int N, int P, int C, int Ct, int groups,
                  twg_stream_t stream) {
  if (!x || !gout || !gx) return fail(TWG_ERR_INVALID, "twg_mbstd_bwd: null");
  if (groups <= 0 || N % groups) return fail(TWG_ERR_INVALID, "twg_mbstd: %d groups do not divide %d samples", groups, N);
  if (Ct < C + 1) return fail(TWG_ERR_INVALID, "twg_mbstd: %d output channels < %d + 1", Ct, C);
  k_mbstd_bwd<<<kMbCluster * groups, 512, 0, S(stream)>>>(x, gout, gx, N / groups, P, C, Ct);
  return check_launch("twg_mbstd_bwd");
}
int twg_mbstd_bwd2(const float* x, const float* gout, const float* ggx, float* dgout, float* dx, int N, int P, int C,
                   int Ct, int groups, twg_stream_t stream) {
  if (!x || !gout || !ggx || !dgout || !dx) return fail(TWG_ERR_INVALID, "twg_mbstd_bwd2: null");
  if (groups <= 0 || N % groups) return fail(TWG_ERR_INVALID, "twg_mbstd: %d groups do not divide %d samples", groups, N);
  if (Ct < C + 1) return fail(TWG_ERR_INVALID, "twg_mbstd: %d output channels < %d + 1", Ct, C);
  k_mbstd_bwd2<<<kMbCluster * groups, 512, 0, S(stream)>>>(x, gout, ggx, dgout, dx, N / groups, P, C, Ct);
  return check_launch("twg_mbstd_bwd2");
}

int twg_sigmoid_ce(const float* logits, float label, float weight, float* loss_out, float* grad, int64_t n,
                   int accumulate, twg_stream_t stream) {
  if (!logits || !loss_out || n <= 0) return fail(TWG_ERR_INVALID, "twg_sigmoid_ce: bad args");
  k_sigmoid_ce<<<1, 256, 0, S(stream)>>>(logits, label, weight, loss_out, grad, n, accumulate);
  return check_launch("twg_sigmoid_ce");
}

int twg_logit_mean(const float* x, float* loss_out, int64_t n, float sign, float margin, int kind, float weight,
                   twg_stream_t stream) {
  if (!x || !loss_out || n <= 0 || kind < 0 || kind > 2) return fail(TWG_ERR_INVALID, "twg_logit_mean: bad args");
  k_logit_mean<<<1, 256, 0, S(stream)>>>(x, loss_out, n, sign, margin, kind, weight);
  return check_launch("twg_logit_mean");
}

int twg_logit_mean_bwd(const float* x, const float* gl, float* gx, int64_t n, float sign, float margin, int kind,
                       float weight, twg_stream_t stream) {
  if (!x || !gl || !gx || n <= 0 || kind < 0 || kind > 2) return fail(TWG_ERR_INVALID, "twg_logit_mean_bwd: bad args");
  k_logit_mean_bwd<<<grid_for(n, 1), 256, 0, S(stream)>>>(x, gl, gx, n, sign, margin, kind, weight);
  return check_launch("twg_logit_mean_bwd");
}

int twg_l1(const float* a, const float* b, float weight, float* loss_out, float* grad_a, int64_t n, int accumulate,
           twg_stream_t stream) {
  if (!a || !b || !loss_out || n <= 0) return fail(TWG_ERR_INVALID, "twg_l1: bad args");
  if (!accumulate) cudaMemsetAsync(loss_out, 0, sizeof(float), S(stream));
  const unsigned nb = grid_for(n, 8);
  float* parts = partials(nb, false, S(stream));
  if (!parts) return fail(TWG_ERR_UNSUPPORTED, "twg_l1: scratch");
  k_l1<<<nb, 256, 0, S(stream)>>>(a, b, weight / (float)n, parts, grad_a, n);
  if (int rc = check_launch("twg_l1")) return rc;
  return add_partials(loss_out, parts, (int)nb, 1, S(stream));
}

int twg_dragan_xhat(const float* x, const float* alpha, const float* noise, float* xhat, float* scratch2, int N,
                    int64_t per_sample, twg_stream_t stream) {
  if (!x || !alpha || !noise || !xhat || !scratch2) return fail(TWG_ERR_INVALID, "twg_dragan_xhat: null");
  double* s2 = reinterpret_cast<double*>(scratch2);  // caller provides >= 16 bytes, 8-byte aligned
  cudaMemsetAsync(s2, 0, 16, S(stream));
  const int64_t total = (int64_t)N * per_sample;
  k_sum_sq<<<1, 256, 0, S(stream)>>>(x, s2, total);     // one block: the sums come out the same on every run
  int rc = check_launch("twg_dragan_xhat/sum");
  if (rc) return rc;
  k_dragan_xhat<<<grid_for(total, 4), 256, 0, S(stream)>>>(x, alpha, noise, xhat, s2, N, per_sample);
  return check_launch("twg_dragan_xhat");
}

int twg_grad_penalty(const float* g, float lambda, float* loss_out, float* coef, int N, int64_t per_sample,
                     int accumulate, twg_stream_t stream) {
  if (!g || !loss_out || !coef) return fail(TWG_ERR_INVALID, "twg_grad_penalty: null");
  cudaMemsetAsync(coef, 0, sizeof(float) * N, S(stream));
  int64_t blocks = cdiv(per_sample, 256 * 8);
  if (blocks > 64) blocks = 64;
  int64_t chunk = cdiv(per_sample, blocks);
  dim3 grid((unsigned)cdiv(per_sample, chunk), N);
  float* parts = partials((int64_t)grid.x * N, false, S(stream));
  if (!parts) return fail(TWG_ERR_UNSUPPORTED, "twg_grad_penalty: scratch");
  k_row_sumsq<<<grid, 256, 0, S(stream)>>>(g, parts, per_sample, chunk);
  if (int rc = check_launch("twg_grad_penalty")) return rc;
  if (int rc = add_partials(coef, parts, (int)grid.x, N, S(stream))) return rc;
  k_grad_penalty_finalize<<<1, 64, 0, S(stream)>>>(coef, lambda, loss_out, N, accumulate);
  return check_launch("twg_grad_penalty");
}

int twg_scale_rows(const float* x, const float* coef, const float* dev_scalar, float* out, int N, int64_t per_sample,
                   twg_stream_t stream) {
  if (!x || !coef || !out) return fail(TWG_ERR_INVALID, "twg_scale_rows: null");
  k_scale_rows<<<grid_for((int64_t)N * per_sample, 4), 256, 0, S(stream)>>>(x, coef, dev_scalar, out, N, per_sample);
  return check_launch("twg_scale_rows");
}

int twg_adam(float* p, const float* g, float* m, float* v, int64_t n, float lr_t, float beta1, float beta2, float eps,
             twg_stream_t stream) {
  if (!p || !g || !m || !v) return fail(TWG_ERR_INVALID, "twg_adam: null");
  k_adam<<<grid_for(n, 4), 256, 0, S(stream)>>>(p, g, m, v, n, nullptr, lr_t, beta1, beta2, eps);
  return check_launch("twg_adam");
}

int twg_adam_dev_lr(float* p, const float* g, float* m, float* v, int64_t n, const float* lr_t_dev, float beta1,
                    float beta2, float eps, twg_stream_t stream) {
  if (!p || !g || !m || !v || !lr_t_dev) return fail(TWG_ERR_INVALID, "twg_adam_dev_lr: null");
  k_adam<<<grid_for(n, 4), 256, 0, S(stream)>>>(p, g, m, v, n, lr_t_dev, 0.f, beta1, beta2, eps);
  return check_launch("twg_adam_dev_lr");
}

int twg_fanout_fwd(const float* gout, const float* x, float* ds, float* dt, float* e2, float* sign_grad, float* loss2,
                   float weight, int B, int64_t per_sample, twg_stream_t stream) {
  if (!gout || !x || !ds || !dt || !e2 || !sign_grad || !loss2 || B <= 0 || per_sample <= 0 || (B * per_sample) % 4)
    return fail(TWG_ERR_INVALID, "twg_fanout_fwd: bad args");
  const int64_t per = (int64_t)B * per_sample;
  cudaMemsetAsync(loss2, 0, 2 * sizeof(float), S(stream));
  const unsigned nb = grid_for(per, 2);
  float* parts = partials(2 * (int64_t)nb, false, S(stream));
  if (!parts) return fail(TWG_ERR_UNSUPPORTED, "twg_fanout_fwd: scratch");
  k_fanout_fwd<<<nb, 256, 0, S(stream)>>>(gout, x, ds, dt, e2, sign_grad, parts, weight / (float)per, per / 4);
  if (int rc = check_launch("twg_fanout_fwd")) return rc;
  return add_partials(loss2, parts, (int)nb, 2, S(stream));
}

int twg_fanout_bwd(const float* gds, const float* gdt, const float* ge2, const float* sign_grad, const float* gl_s,
                   const float* gl_t, float* ggout, int B, int64_t per_sample, twg_stream_t stream) {
  if (!sign_grad || !ggout || B <= 0 || per_sample <= 0 || (B * per_sample) % 4) return fail(TWG_ERR_INVALID, "twg_fanout_bwd: bad args");
  const int64_t per = (int64_t)B * per_sample;
  k_fanout_bwd<<<grid_for(per, 2), 256, 0, S(stream)>>>(gds, gdt, ge2, sign_grad, gl_s, gl_t, ggout, per / 4);
  return check_launch("twg_fanout_bwd");
}

int twg_l1_groups(const float* a, const float* b, float weight, float* loss, float* grad_a, int groups, int64_t per_group,
                  twg_stream_t stream) {
  if (!a || !b || !loss || !grad_a || groups <= 0 || per_group <= 0) return fail(TWG_ERR_INVALID, "twg_l1_groups: bad args");
  cudaMemsetAsync(loss, 0, groups * sizeof(float), S(stream));
  dim3 grid((unsigned)grid_for(per_group, 8), (unsigned)groups);
  float* parts = partials((int64_t)grid.x * groups, false, S(stream));
  if (!parts) return fail(TWG_ERR_UNSUPPORTED, "twg_l1_groups: scratch");
  k_l1_groups<<<grid, 256, 0, S(stream)>>>(a, b, weight / (float)per_group, parts, grad_a, per_group);
  if (int rc = check_launch("twg_l1_groups")) return rc;
  return add_partials(loss, parts, (int)grid.x, groups, S(stream));
}

int twg_scale_groups2(const float* grad, const float* gl0, const float* gl1, float sign, float* out, int64_t per_group,
                      twg_stream_t stream) {
  if (!grad || !out || per_group <= 0) return fail(TWG_ERR_INVALID, "twg_scale_groups2: bad args");
  dim3 grid((unsigned)grid_for(per_group, 4), 2);
  k_scale_groups2<<<grid, 256, 0, S(stream)>>>(grad, gl0, gl1, sign, out, per_group);
  return check_launch("twg_scale_groups2");
}

int twg_gan_losses(const float* logits, float weight, float* loss6, float* sig, int B, twg_stream_t stream) {
  if (!logits || !loss6 || !sig || B <= 0) return fail(TWG_ERR_INVALID, "twg_gan_losses: bad args");
  k_gan_losses<<<1, 256, 0, S(stream)>>>(logits, weight, loss6, sig, B);
  return check_launch("twg_gan_losses");
}

int twg_gan_losses_bwd(const float* sig, float weight, const float* g0, const float* g1, const float* g2, const float* g3,
                       const float* g4, const float* g5, float* grad, int B, twg_stream_t stream) {
  if (!sig || !grad || B <= 0) return fail(TWG_ERR_INVALID, "twg_gan_losses_bwd: bad args");
  k_gan_losses_bwd<<<1, 256, 0, S(stream)>>>(sig, weight, g0, g1, g2, g3, g4, g5, grad, B);
  return check_launch("twg_gan_losses_bwd");
}

int twg_sum_scalars(const void* device_ptrs_host_array, int n, float scale, float* out, twg_stream_t stream) {
  if (!device_ptrs_host_array || !out || n <= 0 || n > 16) return fail(TWG_ERR_INVALID, "twg_sum_scalars: 1..16 scalars");
  ScalarPtrs ptrs{};
  const float* const* src = reinterpret_cast<const float* const*>(device_ptrs_host_array);
  for (int i = 0; i < n; ++i) {
    if (!src[i]) return fail(TWG_ERR_INVALID, "twg_sum_scalars: null scalar %d", i);
    ptrs.p[i] = src[i];
  }
  k_sum_scalars<<<1, 1, 0, S(stream)>>>(ptrs, n, scale, out);
  return check_launch("twg_sum_scalars");
}

int twg_step_schedule(const void* counters, float lr, float beta1, float beta2, float* lr_out2, float* clip_out3,
                      twg_stream_t stream) {
  if (!counters || !lr_out2 || !clip_out3) return fail(TWG_ERR_INVALID, "twg_step_schedule: null");
  k_step_schedule<<<1, 1, 0, S(stream)>>>(reinterpret_cast<const int*>(counters), lr, beta1, beta2, lr_out2, clip_out3);
  return check_launch("twg_step_schedule");
}

int twg_step_advance(void* counters, int d_adam_t, int d_global_step, twg_stream_t stream) {
  if (!counters) return fail(TWG_ERR_INVALID, "twg_step_advance: null");
  k_step_advance<<<1, 1, 0, S(stream)>>>(reinterpret_cast<int*>(counters), d_adam_t, d_global_step);
  return check_launch("twg_step_advance");
}

int twg_split_weights_table(const float* flat, void* planes, const void* table, int rows, int64_t max_elems,
                            twg_stream_t stream) {
  if (!flat || !planes || !table || rows <= 0) return fail(TWG_ERR_INVALID, "twg_split_weights_table: bad args");
  int64_t bx = cdiv(max_elems, 256 * 4);
  if (bx > 64) bx = 64;
  if (bx < 1) bx = 1;
  dim3 grid((unsigned)bx, (unsigned)rows);
  k_split_weights_table<<<grid, 256, 0, S(stream)>>>(flat, reinterpret_cast<__nv_bfloat16*>(planes),
                                                     reinterpret_cast<const SplitRow*>(table));
  return check_launch("twg_split_weights_table");
}

}  // extern "C"
