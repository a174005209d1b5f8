// Normaliser (instance / batch / batch-renorm / none) + leaky-ReLU + pixel-norm: statistics, forward apply and both
// backward passes.  NHWC fp32, vectorised float4 along C; every per-(n, c) sum is added by one block in a fixed order.
#include "twg_common.cuh"

namespace twg {

// ------------------------------------------------------------------------------------------------
// moments: one block per sample (blockIdx.y = n) covers all HW pixels, so it is the only writer of its sums and adds
// them in the same order on every run
// ------------------------------------------------------------------------------------------------
// Shifted sums: sums[n][c] = {sum (y - p), sum (y - p)^2} with the pivot p = y[first sample of n's pivot group][pixel 0][c].
// tf.nn.moments is two-pass; a single pass over raw y, y^2 in fp32 cancels catastrophically once |mean| >> std
// (relative variance error ~ 6e-8 * mean^2 / var).  With a pivot drawn from the data the shifted mean is O(std).
template <int V>
__global__ void __launch_bounds__(256) k_moments_vec(const float* __restrict__ y, float* __restrict__ sums, int HW,
                                                     int C, int G, int pivot_group) {
  __shared__ float sm[256];
  const int n = blockIdx.y, q = C / 4;
  const int gpb = 256 / G, grp = threadIdx.x / G, lg = threadIdx.x % G;
  float4 pv[V];
#pragma unroll
  for (int v = 0; v < V; ++v) pv[v] = ld4(y, (int64_t)(n / pivot_group * pivot_group) * HW * q + lg + v * 32);
  float acc[8 * V];
#pragma unroll
  for (int i = 0; i < 8 * V; ++i) acc[i] = 0.f;
  constexpr int U = (V == 1) ? 4 : (V == 2 ? 2 : 1);     // pixels in flight per thread: enough bytes outstanding to cover HBM latency
  for (int pb = grp; pb < HW; pb += gpb * U) {
    float4 t[U][V];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int p = pb + u * gpb;
      const int64_t base = ((int64_t)n * HW + (p < HW ? p : 0)) * q;
#pragma unroll
      for (int v = 0; v < V; ++v) t[u][v] = ld4(y, base + lg + v * 32);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (pb + u * gpb >= HW) continue;
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
    const float s = block_tree_sum(acc[k], G, sm);
    if (threadIdx.x < G) {
      int v = k / 8, j = k % 8;
      int c = (lg + v * 32) * 4 + (j & 3);
      sums[((int64_t)n * C + c) * 2 + (j >> 2)] = s;
    }
  }
}

__global__ void __launch_bounds__(256) k_moments_scalar(const float* __restrict__ y, float* __restrict__ sums, int HW,
                                                        int C, int pivot_group) {
  __shared__ float sm[32];
  const int n = blockIdx.y;
  for (int c = 0; c < C; ++c) {
    const float pv = y[(int64_t)(n / pivot_group * pivot_group) * HW * C + c];
    float a1 = 0.f, a2 = 0.f;
    for (int p = threadIdx.x; p < HW; p += blockDim.x) {
      float t = y[((int64_t)n * HW + p) * C + c] - pv;
      a1 += t;
      a2 += t * t;
    }
    a1 = block_sum(a1, sm);
    a2 = block_sum(a2, sm);
    if (threadIdx.x == 0) {
      sums[((int64_t)n * C + c) * 2 + 0] = a1;
      sums[((int64_t)n * C + c) * 2 + 1] = a2;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// finalize: sums -> per-(n,c) affine + saved mean/rstd
// ------------------------------------------------------------------------------------------------
// The batch is `N / gs` groups of `gs` samples (one group per original network pass when passes that share conv
// weights are batched); bit g of dom_mask selects the group's domain, i.e. which gamma/beta (and renorm state) it uses.
// Batch kinds: statistics over the group's samples (instance norm is k_norm_finalize_inst).  `y` is only read for the
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

// Instance norm from the conv epilogue's records (k_conv_fwd_wgmma with `stats`): stats[n][slot][c] = {count, pivot, sum (y - pivot),
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
    float* __restrict__ gu, float* __restrict__ red, int HW, int C, int G, int flags,
    const float* __restrict__ gpool, int W) {
  // gz (may be null) is the gradient w.r.t. the layer output z at full resolution (e.g. from a UNet skip); gpool (may be
  // null) the gradient w.r.t. avg_pool2(z): its 2x2 broadcast * 1/4 is added on the fly instead of being materialised
  __shared__ float sm[256];
  const int n = blockIdx.y, q = C / 4;
  const int gpb = 256 / G, grp = threadIdx.x / G, lg = threadIdx.x % G;
  const bool act = flags & TWG_FLAG_LRELU, pix = flags & TWG_FLAG_PIXNORM;
  const float invC = 1.f / (float)C;
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
  for (int pb = 0; pb < HW; pb += gpb * U) {
    float4 yy[U][V], g[U][V];
    bool valid[U];
    int64_t base[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int p = pb + u * gpb + grp;
      valid[u] = p < HW;
      const int pp = valid[u] ? p : 0;
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
    const float s = block_tree_sum(acc[k], G, sm);
    if (threadIdx.x < G) {
      int v = k / 8, j = k % 8;
      int c = (lg + v * 32) * 4 + (j & 3);
      red[((int64_t)n * C + c) * 2 + (j >> 2)] = s;
    }
  }
}

__global__ void __launch_bounds__(256) k_norm_act_bwd_reduce_scalar(
    const float* __restrict__ y, const float* __restrict__ a, const float* __restrict__ b,
    const float* __restrict__ mean, const float* __restrict__ rstd, const float* __restrict__ gz,
    float* __restrict__ gu, float* __restrict__ red, int HW, int C, int flags) {
  __shared__ float sm[32];
  const int n = blockIdx.y;
  const bool act = flags & TWG_FLAG_LRELU, pix = flags & TWG_FLAG_PIXNORM;
  // pass A: gu
  for (int p = threadIdx.x; p < HW; p += blockDim.x) {
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
    for (int p = threadIdx.x; p < HW; p += blockDim.x) {
      const int64_t i = ((int64_t)n * HW + p) * C + c;
      float g = gu[i];
      a1 += g;
      a2 += g * (y[i] - mean[n * C + c]) * rstd[n * C + c];
    }
    a1 = block_sum(a1, sm);
    a2 = block_sum(a2, sm);
    if (threadIdx.x == 0) {
      red[((int64_t)n * C + c) * 2] = a1;
      red[((int64_t)n * C + c) * 2 + 1] = a2;
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
    if (kind == TWG_NORM_NONE) {
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

}  // namespace twg

using namespace twg;

extern "C" {

int twg_moments(const float* y, float* sums, int N, int HW, int C, int pivot_group, twg_stream_t stream) {
  if (!y || !sums || N <= 0 || HW <= 0 || C <= 0 || pivot_group <= 0 || N % pivot_group)
    return fail(TWG_ERR_INVALID, "twg_moments: bad args");
  const dim3 grid(1, N);                    // one block per sample writes all of its sums
  VecGeom g = vec_geom(C);
  if (g.ok) {
    if (g.V == 1) k_moments_vec<1><<<grid, 256, 0, S(stream)>>>(y, sums, HW, C, g.G, pivot_group);
    else if (g.V == 2) k_moments_vec<2><<<grid, 256, 0, S(stream)>>>(y, sums, HW, C, g.G, pivot_group);
    else k_moments_vec<4><<<grid, 256, 0, S(stream)>>>(y, sums, HW, C, g.G, pivot_group);
  } else {
    if (C > 64) return fail(TWG_ERR_UNSUPPORTED, "twg_moments: C=%d unsupported", C);
    k_moments_scalar<<<grid, 256, 0, S(stream)>>>(y, sums, HW, C, pivot_group);
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
  const dim3 grid(1, N);                    // one block per sample writes all of its sums
  VecGeom g = vec_geom(C);
  if (g.ok) {
    if (g.V == 1) k_norm_act_bwd_reduce_vec<1><<<grid, 256, 0, S(stream)>>>(y, a, b, mean, rstd, gz, gu, red, HW, C, g.G, flags, gpool, W);
    else if (g.V == 2) k_norm_act_bwd_reduce_vec<2><<<grid, 256, 0, S(stream)>>>(y, a, b, mean, rstd, gz, gu, red, HW, C, g.G, flags, gpool, W);
    else k_norm_act_bwd_reduce_vec<4><<<grid, 256, 0, S(stream)>>>(y, a, b, mean, rstd, gz, gu, red, HW, C, g.G, flags, gpool, W);
  } else {
    if (C > 64) return fail(TWG_ERR_UNSUPPORTED, "twg_norm_act_bwd_reduce: C=%d unsupported", C);
    k_norm_act_bwd_reduce_scalar<<<grid, 256, 0, S(stream)>>>(y, a, b, mean, rstd, gz, gu, red, HW, C, flags);
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

}  // extern "C"
