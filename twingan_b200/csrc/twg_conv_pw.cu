// Thin 1x1 convolutions: fromRGB (Cin = 3) and toRGB (Cout = 3) and their gradients (SURVEY K5).
// These layers carry ~0.15 % of the FLOPs but touch full-resolution tensors, so they are pure HBM
// streaming problems: one pass over the wide tensor, float4 along channels, the 3-channel side and the tiny
// weight matrix live in registers / shared memory.  Exact fp32 (CUDA cores); used for prec 0 and 1 alike.
#include "twg_common.cuh"

namespace twg {

constexpr int kMaxSmall = 4;

// ---- "expand": out[p][l] = sum_s small_in[p][s] * W(s,l)   (fromRGB forward, toRGB dgrad) ----------------
// W(s,l) = w[s*ws_s + l*ws_l]
__global__ void __launch_bounds__(256) k_pw_expand(const float* __restrict__ in, const float* __restrict__ w,
                                                   float* __restrict__ out, int64_t P, int S, int L, int ws_s, int ws_l) {
  extern __shared__ float sw[];   // [S][L]
  for (int i = threadIdx.x; i < S * L; i += blockDim.x) sw[i] = w[(i / L) * ws_s + (i % L) * ws_l];
  __syncthreads();
  const int q = L / 4;
  const int64_t total = P * q;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t p = i / q;
    const int lq = (int)(i - p * q);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int s = 0; s < S; ++s) {
      const float v = in[p * S + s];
      const float4 ww = *reinterpret_cast<const float4*>(&sw[s * L + lq * 4]);
      acc.x = fmaf(v, ww.x, acc.x); acc.y = fmaf(v, ww.y, acc.y); acc.z = fmaf(v, ww.z, acc.z); acc.w = fmaf(v, ww.w, acc.w);
    }
    reinterpret_cast<float4*>(out)[i] = acc;
  }
}

// ---- "reduce": out[p][s] = sum_l big_in[p][l] * W(s,l)    (toRGB forward, fromRGB dgrad) --------------------
template <int V>
__global__ void __launch_bounds__(256) k_pw_reduce(const float* __restrict__ in, const float* __restrict__ w,
                                                   float* __restrict__ out, int64_t P, int S, int L, int G, int ws_s,
                                                   int ws_l) {
  extern __shared__ float sw[];   // [S][L]
  for (int i = threadIdx.x; i < S * L; i += blockDim.x) sw[i] = w[(i / L) * ws_s + (i % L) * ws_l];
  __syncthreads();
  const int q = L / 4, gpb = 256 / G, grp = threadIdx.x / G, lg = threadIdx.x % G;
  // U pixels per group and iteration: all their loads are issued before the first use (one float4 in flight per thread left
  // this pure streaming kernel latency-bound at a fraction of the HBM bandwidth)
  constexpr int U = (V == 1) ? 4 : (V == 2 ? 2 : 1);
  for (int64_t base = (int64_t)blockIdx.x * gpb * U; base < P; base += (int64_t)gridDim.x * gpb * U) {
    float4 x[U][V];
    bool valid[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t p = base + (int64_t)u * gpb + grp;
      valid[u] = p < P;
#pragma unroll
      for (int v = 0; v < V; ++v)
        x[u][v] = valid[u] ? reinterpret_cast<const float4*>(in)[p * q + lg + v * 32] : make_float4(0, 0, 0, 0);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t p = base + (int64_t)u * gpb + grp;
      float acc[kMaxSmall] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int v = 0; v < V; ++v) {
        const int lq = lg + v * 32;
        for (int s = 0; s < S; ++s) {
          const float4 ww = *reinterpret_cast<const float4*>(&sw[s * L + lq * 4]);
          acc[s] += x[u][v].x * ww.x + x[u][v].y * ww.y + x[u][v].z * ww.z + x[u][v].w * ww.w;
        }
      }
      for (int s = 0; s < S; ++s) acc[s] = group_sum(acc[s], G);
      if (valid[u] && lg == 0)
        for (int s = 0; s < S; ++s) out[p * S + s] = acc[s];
    }
  }
}

// ---- "reduce" with ONE THREAD PER PIXEL (L = 16 or 32 wide channels): no cross-lane sums, the S x L weights broadcast
// from shared memory.  ncu on the lane-group form above (toRGB, 64 images at 256x256): issue slots 79 % busy at 33 % of the
// HBM bandwidth -- 35 instructions per float4 loaded (3 partial dots, 6 shuffles, 3 shared loads); this form needs ~17.
template <int L4>
__global__ void __launch_bounds__(256) k_pw_reduce_px(const float* __restrict__ in, const float* __restrict__ w,
                                                      float* __restrict__ out, int64_t P, int S, int ws_s, int ws_l) {
  constexpr int L = 4 * L4;
  __shared__ float4 sw[kMaxSmall * L4];   // [s][l4]
  for (int i = threadIdx.x; i < kMaxSmall * L; i += blockDim.x) {
    const int s_ = i / L, l = i - s_ * L;
    reinterpret_cast<float*>(sw)[i] = (s_ < S) ? w[s_ * ws_s + l * ws_l] : 0.f;
  }
  __syncthreads();
#pragma unroll 2
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < P; p += (int64_t)gridDim.x * blockDim.x) {
    float4 x[L4];
#pragma unroll
    for (int j = 0; j < L4; ++j) x[j] = reinterpret_cast<const float4*>(in)[p * L4 + j];
    float acc[kMaxSmall] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int s_ = 0; s_ < kMaxSmall; ++s_) {
#pragma unroll
      for (int j = 0; j < L4; ++j) {
        const float4 ww = sw[s_ * L4 + j];
        acc[s_] = fmaf(x[j].x, ww.x, acc[s_]); acc[s_] = fmaf(x[j].y, ww.y, acc[s_]);
        acc[s_] = fmaf(x[j].z, ww.z, acc[s_]); acc[s_] = fmaf(x[j].w, ww.w, acc[s_]);
      }
    }
    if (S == 3) { out[p * 3] = acc[0]; out[p * 3 + 1] = acc[1]; out[p * 3 + 2] = acc[2]; }
    else for (int s_ = 0; s_ < S; ++s_) out[p * S + s_] = acc[s_];
  }
}

static bool launch_reduce_px(const float* in, const float* w, float* out, int64_t P, int S, int L, int ws_s, int ws_l,
                             cudaStream_t st) {
  if (L != 16 && L != 32) return false;
  int64_t b = cdiv(P, 256);
  if (b > kNumSMs * 16) b = kNumSMs * 16;
  if (L == 16) k_pw_reduce_px<4><<<(unsigned)b, 256, 0, st>>>(in, w, out, P, S, ws_s, ws_l);
  else k_pw_reduce_px<8><<<(unsigned)b, 256, 0, st>>>(in, w, out, P, S, ws_s, ws_l);
  return true;
}

// ---- weight gradient: G(s,l) += sum_p small[p][s] * big[p][l] -----------------------------------------------
template <int V>
__global__ void __launch_bounds__(256) k_pw_wgrad(const float* __restrict__ small, const float* __restrict__ big,
                                                  float* __restrict__ gw, int64_t P, int S, int L, int G, int ws_s,
                                                  int ws_l, int64_t chunk) {
  __shared__ float sm[256];
  const int q = L / 4, gpb = 256 / G, grp = threadIdx.x / G, lg = threadIdx.x % G;
  const int64_t p0 = (int64_t)blockIdx.x * chunk, p1 = min(P, p0 + chunk);
  float acc[kMaxSmall][4 * V];
#pragma unroll
  for (int s = 0; s < kMaxSmall; ++s)
#pragma unroll
    for (int j = 0; j < 4 * V; ++j) acc[s][j] = 0.f;
  constexpr int U = (V == 1) ? 4 : (V == 2 ? 2 : 1);     // pixels in flight per thread (loads first, then the FMAs)
  for (int64_t pb = p0 + grp; pb < p1; pb += (int64_t)gpb * U) {
    float sv[U][kMaxSmall];
    float4 x[U][V];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t p = pb + (int64_t)u * gpb;
      const bool ok = p < p1;
#pragma unroll
      for (int s = 0; s < kMaxSmall; ++s) sv[u][s] = (ok && s < S) ? small[p * S + s] : 0.f;
#pragma unroll
      for (int v = 0; v < V; ++v)
        x[u][v] = ok ? reinterpret_cast<const float4*>(big)[p * q + lg + v * 32] : make_float4(0, 0, 0, 0);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
#pragma unroll
      for (int v = 0; v < V; ++v) {
#pragma unroll
        for (int s = 0; s < kMaxSmall; ++s) {
          acc[s][4 * v + 0] = fmaf(sv[u][s], x[u][v].x, acc[s][4 * v + 0]);
          acc[s][4 * v + 1] = fmaf(sv[u][s], x[u][v].y, acc[s][4 * v + 1]);
          acc[s][4 * v + 2] = fmaf(sv[u][s], x[u][v].z, acc[s][4 * v + 2]);
          acc[s][4 * v + 3] = fmaf(sv[u][s], x[u][v].w, acc[s][4 * v + 3]);
        }
      }
    }
  }
  for (int s = 0; s < S; ++s) {
#pragma unroll
    for (int j = 0; j < 4 * V; ++j) {
      const float sum = block_tree_sum(acc[s][j], G, sm);
      if (threadIdx.x < G) {
        const int l = (lg + (j / 4) * 32) * 4 + (j & 3);
        gw[(int64_t)blockIdx.x * S * L + s * ws_s + l * ws_l] = sum;   // this block's partial (add_partials)
      }
    }
  }
}

static bool geom_for(int L, int& G, int& V) {
  if (L % 4) return false;
  const int q = L / 4;
  if (q <= 32) {
    if (q & (q - 1)) return false;
    G = q; V = 1;
    return true;
  }
  if (q % 32 || (q / 32 != 2 && q / 32 != 4)) return false;
  G = 32; V = q / 32;
  return true;
}

bool pw_supported(int Cin, int Cout, int k, int pad) {
  if (k != 1 || pad != 0) return false;
  int G, V;
  if (Cin <= kMaxSmall && Cout > kMaxSmall) return geom_for(Cout, G, V);
  if (Cout <= kMaxSmall && Cin > kMaxSmall) return geom_for(Cin, G, V);
  return false;
}

static inline unsigned blocks_for(int64_t work_items) {
  int64_t b = cdiv(work_items, 256 * 4);
  if (b > kNumSMs * 16) b = kNumSMs * 16;
  if (b < 1) b = 1;
  return (unsigned)b;
}

// w: [Cin][Cout] (HWIO with k=1)
int pw_fwd(const float* x, const float* w, float* y, int64_t P, int Cin, int Cout, cudaStream_t st) {
  int G, V;
  if (Cin <= kMaxSmall) {   // expand: S=Cin, L=Cout, W(s,l) = w[s*Cout + l]
    k_pw_expand<<<blocks_for(P * Cout / 4), 256, sizeof(float) * Cin * Cout, st>>>(x, w, y, P, Cin, Cout, Cout, 1);
  } else {                  // reduce: S=Cout, L=Cin, W(s,l) = w[l*Cout + s]
    if (launch_reduce_px(x, w, y, P, Cout, Cin, 1, Cout, st)) return check_launch("twg_conv pointwise fwd");
    geom_for(Cin, G, V);
    const unsigned b = blocks_for(P * G);
    const size_t sh = sizeof(float) * Cin * Cout;
    if (V == 1) k_pw_reduce<1><<<b, 256, sh, st>>>(x, w, y, P, Cout, Cin, G, 1, Cout);
    else if (V == 2) k_pw_reduce<2><<<b, 256, sh, st>>>(x, w, y, P, Cout, Cin, G, 1, Cout);
    else k_pw_reduce<4><<<b, 256, sh, st>>>(x, w, y, P, Cout, Cin, G, 1, Cout);
  }
  return check_launch("twg_conv pointwise fwd");
}

int pw_dgrad(const float* gy, const float* w, float* gx, int64_t P, int Cin, int Cout, cudaStream_t st) {
  int G, V;
  if (Cin <= kMaxSmall) {   // gx[p][ci] = sum_co gy[p][co] w[ci][co]: reduce, S=Cin, L=Cout, W(s,l)=w[s*Cout+l]
    if (launch_reduce_px(gy, w, gx, P, Cin, Cout, Cout, 1, st)) return check_launch("twg_conv pointwise dgrad");
    geom_for(Cout, G, V);
    const unsigned b = blocks_for(P * G);
    const size_t sh = sizeof(float) * Cin * Cout;
    if (V == 1) k_pw_reduce<1><<<b, 256, sh, st>>>(gy, w, gx, P, Cin, Cout, G, Cout, 1);
    else if (V == 2) k_pw_reduce<2><<<b, 256, sh, st>>>(gy, w, gx, P, Cin, Cout, G, Cout, 1);
    else k_pw_reduce<4><<<b, 256, sh, st>>>(gy, w, gx, P, Cin, Cout, G, Cout, 1);
  } else {                  // gx[p][ci] = sum_j gy[p][j] w[ci][j]: expand, S=Cout, L=Cin, W(s,l)=w[l*Cout+s]
    k_pw_expand<<<blocks_for(P * Cin / 4), 256, sizeof(float) * Cin * Cout, st>>>(gy, w, gx, P, Cout, Cin, 1, Cout);
  }
  return check_launch("twg_conv pointwise dgrad");
}

int pw_wgrad(const float* x, const float* gy, float* gw, int64_t P, int Cin, int Cout, int accumulate, cudaStream_t st) {
  if (!accumulate) cudaMemsetAsync(gw, 0, sizeof(float) * Cin * Cout, st);
  int G, V;
  const float *small, *big;
  int S, L, ws_s, ws_l;
  if (Cin <= kMaxSmall) { small = x; big = gy; S = Cin; L = Cout; ws_s = Cout; ws_l = 1; }   // gw[ci][co]
  else { small = gy; big = x; S = Cout; L = Cin; ws_s = 1; ws_l = Cout; }                     // gw[ci][j]
  geom_for(L, G, V);
  const int gpb = 256 / G;
  int64_t blocks = cdiv(P, (int64_t)gpb * 16);
  if (blocks > 4 * kNumSMs) blocks = 4 * kNumSMs;
  const int64_t chunk = cdiv(P, blocks);
  blocks = cdiv(P, chunk);
  float* parts = partials(blocks * S * L, true, st);
  if (!parts) return fail(TWG_ERR_UNSUPPORTED, "twg_conv pointwise wgrad: %d x %d too wide", Cin, Cout);
  if (V == 1) k_pw_wgrad<1><<<(unsigned)blocks, 256, 0, st>>>(small, big, parts, P, S, L, G, ws_s, ws_l, chunk);
  else if (V == 2) k_pw_wgrad<2><<<(unsigned)blocks, 256, 0, st>>>(small, big, parts, P, S, L, G, ws_s, ws_l, chunk);
  else k_pw_wgrad<4><<<(unsigned)blocks, 256, 0, st>>>(small, big, parts, P, S, L, G, ws_s, ws_l, chunk);
  if (int rc = check_launch("twg_conv pointwise wgrad")) return rc;
  return add_partials(gw, parts, (int)blocks, (int64_t)S * L, st);
}

}  // namespace twg
