// Memory-bound kernels of the TwinGAN step besides the normaliser (twg_norm.cu): discriminator bias + leaky-ReLU and
// column sums, resampling, UNet join, minibatch-stddev (incl. double backward), losses, DRAGAN helpers, the wiring of
// the batched passes, Adam and the step counters.  All NHWC fp32, vectorised float4 along C, coalesced; cross-block
// sums go through per-block partials added in block order (add_partials), never fp32 atomics.
#include <cooperative_groups.h>

#include "twg_common.cuh"
#include "twg_stream.cuh"

namespace cg = cooperative_groups;

namespace twg {

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
    const float s = block_tree_sum(acc[k], G, sm);
    if (threadIdx.x < G) colsum[(int64_t)blockIdx.x * C + (lg + (k / 4) * 32) * 4 + (k & 3)] = s;
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
    const float s = block_tree_sum(acc[k], q, sm);
    if (threadIdx.x < q) colsum[((int64_t)blockIdx.x << (lq + 2)) + lg * 4 + k] = s;
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
    const float s = block_tree_sum(acc, Cw, sm);
    if (threadIdx.x < Cw && c < C) out[(int64_t)blockIdx.x * C + c] = s;
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

// k_sum_sq as one block with x arriving through a StreamRing (twelve stages of 16 KB): thread t adds x[t], x[t + 256],
// ... in that order, as in k_sum_sq launched as one block, so the two sums are the same bits.  One block of direct scalar
// loads walks the batch at the latency of one load per element per thread.
constexpr int kSumSqStages = 12;
__global__ void __launch_bounds__(256) k_sum_sq_stream(const float* __restrict__ x, double* __restrict__ out2, int64_t n) {
  extern __shared__ __align__(128) unsigned char ring_mem[];
  __shared__ float sm[32];
  constexpr int kPer = kStreamStage / 4 / 256;          // elements of a stage per thread
  StreamRing<1, kSumSqStages> ring;
  const void* const arrays[1] = {x};
  ring.start(ring_mem, arrays, n * 4);
  float a1 = 0.f, a2 = 0.f;
  for (int k = 0; k < ring.chunks; ++k) {
    ring.wait(k);
    const float* xs = reinterpret_cast<const float*>(ring.at(k, 0));
    const int64_t left = n - (int64_t)k * (kStreamStage / 4);
    float v[kPer];
#pragma unroll
    for (int j = 0; j < kPer; ++j) {
      const int i = j * 256 + threadIdx.x;
      v[j] = xs[i < left ? i : 0];
    }
    ring.release(k);
#pragma unroll
    for (int j = 0; j < kPer; ++j) {
      if (j * 256 + (int)threadIdx.x >= left) continue;
      a1 += v[j];
      a2 += v[j] * v[j];
    }
  }
  a1 = block_sum(a1, sm);
  a2 = block_sum(a2, sm);
  if (threadIdx.x == 0) { out2[0] = (double)a1; out2[1] = (double)a2; }
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

}  // namespace twg

using namespace twg;

extern "C" {

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
  // one block: the sums come out the same on every run.  The bulk copies of the streamed form move whole 16-byte units.
  if (stream_fills(total * 4) && total % 4 == 0 && reinterpret_cast<uintptr_t>(x) % 16 == 0) {
    constexpr int kBytes = StreamRing<1, kSumSqStages>::kBytes;
    static std::once_flag once;
    static cudaError_t attr_err = cudaSuccess;
    if (allow_ring(k_sum_sq_stream, kBytes, once, attr_err) != cudaSuccess)
      return fail(TWG_ERR_CUDA, "cudaFuncSetAttribute: %s", cudaGetErrorString(attr_err));
    k_sum_sq_stream<<<1, 256, kBytes, S(stream)>>>(x, s2, total);
  } else {
    k_sum_sq<<<1, 256, 0, S(stream)>>>(x, s2, total);
  }
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
}  // extern "C"
