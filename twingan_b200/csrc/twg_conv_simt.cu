// fp32 CUDA-core (FFMA) implicit-GEMM convolution: forward, data-gradient, weight-gradient.
// This is the always-available exact-fp32 path (prec=0): it covers every shape of the TwinGAN graph
// (Cin=3 fromRGB, Cout=3 toRGB, the 257-channel minibatch-stddev conv, the 4x4 VALID head, the FC) and
// is the reference the tensor-core path (twg_conv_tc.cu) is checked against on the device.
//
// GEMM view (stride 1):  y[m, co] = sum_{tap, ci} x[pix(m) + tap, ci] * w[tap, ci, co],  m over N*Ho*Wo.
#include "twg_common.cuh"

namespace twg {

struct ConvGeom {
  int N, H, W, Cin, Cout, k, pad, Ho, Wo;
};

// ---- forward / dgrad -------------------------------------------------------------------------------
// TRANSPOSED=false: B[tap][ci][co] = w[tap][ci][co]                       (forward)
// TRANSPOSED=true : the kernel computes gx from gy: roles swapped, B[tap][co][ci] = w[flip(tap)][ci][co]
//                   (geometry passed in is that of the "forward conv" gy -> gx: Cin:=Cout_orig, Cout:=Cin_orig)
template <int BN, int TN, bool TRANSPOSED>
__global__ void __launch_bounds__(256) k_conv_fwd_simt(const float* __restrict__ x, const float* __restrict__ w,
                                                       float* __restrict__ y, ConvGeom g, int kb_per_split) {
  constexpr int BM = 128, BK = 8;
  constexpr int TX = BN / TN;        // threads along n
  constexpr int TY = 256 / TX;       // threads along m
  constexpr int TM = BM / TY;
  __shared__ float As[BK][BM + 4];
  __shared__ float Bs[BK][BN + 4];
  const int tid = threadIdx.x;
  const int tx = tid % TX, ty = tid / TX;
  const int64_t M = (int64_t)g.N * g.Ho * g.Wo;
  const int64_t m0 = (int64_t)blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;

  // A loader: thread -> (pixel row ar = tid/2, channel half ac = (tid%2)*4)
  const int ar = tid >> 1, ac = (tid & 1) * 4;
  const int64_t am = m0 + ar;
  const bool a_valid = am < M;
  int an = 0, aho = 0, awo = 0;
  if (a_valid) {
    int64_t t = am;
    awo = (int)(t % g.Wo); t /= g.Wo;
    aho = (int)(t % g.Ho);
    an = (int)(t / g.Ho);
  }
  // B loader: BK*BN floats by 256 threads
  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  const bool vec_a = (g.Cin % 4 == 0);
  // K loop over (tap, cin-chunk) blocks; blockIdx.z owns a contiguous range (split-K for tiny-M layers)
  const int cchunks = (g.Cin + BK - 1) / BK;
  const int num_kb = g.k * g.k * cchunks;
  const int kb0 = blockIdx.z * kb_per_split, kb1 = min(num_kb, kb0 + kb_per_split);
  {
    {
      for (int kb = kb0; kb < kb1; ++kb) {
        const int tap_lin = kb / cchunks, c0 = (kb - tap_lin * cchunks) * BK;
        const int kh = tap_lin / g.k, kw = tap_lin - kh * g.k;
        const int hi = aho + kh - g.pad, wi = awo + kw - g.pad;
        const bool in_ok = a_valid && hi >= 0 && hi < g.H && wi >= 0 && wi < g.W;
        const float* xp = x + (((int64_t)an * g.H + hi) * g.W + wi) * g.Cin;
        const int tap = TRANSPOSED ? ((g.k - 1 - kh) * g.k + (g.k - 1 - kw)) : (kh * g.k + kw);
        // ---- load A
        float4 av = make_float4(0.f, 0.f, 0.f, 0.f);
        if (in_ok) {
          const int c = c0 + ac;
          if (vec_a) {
            if (c < g.Cin) av = *reinterpret_cast<const float4*>(xp + c);
          } else {
            if (c + 0 < g.Cin) av.x = xp[c + 0];
            if (c + 1 < g.Cin) av.y = xp[c + 1];
            if (c + 2 < g.Cin) av.z = xp[c + 2];
            if (c + 3 < g.Cin) av.w = xp[c + 3];
          }
        }
        // ---- load B
        float bv[(BK * BN + 255) / 256];
#pragma unroll
        for (int i = 0; i < (BK * BN + 255) / 256; ++i) {
          const int e = tid + i * 256;
          float v = 0.f;
          if (e < BK * BN) {
            const int kk = e / BN, j = e % BN;
            const int ci = c0 + kk, co = n0 + j;
            if (ci < g.Cin && co < g.Cout) {
              // forward: w[tap][ci][co] with strides (Cin*Cout, Cout, 1)
              // transposed: logical B[ci=co_orig][co=ci_orig] = w[tap][ci_orig][co_orig]; here g.Cin = Cout_orig
              v = TRANSPOSED ? w[((int64_t)tap * g.Cout + co) * g.Cin + ci] : w[((int64_t)tap * g.Cin + ci) * g.Cout + co];
            }
          }
          bv[i] = v;
        }
        __syncthreads();
        As[ac + 0][ar] = av.x; As[ac + 1][ar] = av.y; As[ac + 2][ar] = av.z; As[ac + 3][ar] = av.w;
#pragma unroll
        for (int i = 0; i < (BK * BN + 255) / 256; ++i) {
          const int e = tid + i * 256;
          if (e < BK * BN) Bs[e / BN][e % BN] = bv[i];
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < BK; ++kk) {
          float a[TM], b[TN];
#pragma unroll
          for (int i = 0; i < TM; ++i) a[i] = As[kk][ty * TM + i];
#pragma unroll
          for (int j = 0; j < TN; ++j) b[j] = Bs[kk][tx * TN + j];
#pragma unroll
          for (int i = 0; i < TM; ++i)
#pragma unroll
            for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
      }
    }
  }
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int64_t m = m0 + ty * TM + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      const int co = n0 + tx * TN + j;
      if (co < g.Cout) {
        // split-K: y is the partial buffer, slice blockIdx.z (add_partials sums the slices in order)
        y[(int64_t)blockIdx.z * M * g.Cout + m * g.Cout + co] = acc[i][j];
      }
    }
  }
}

// ---- wgrad -------------------------------------------------------------------------------------------
// gw[tap][ci][co] += sum_{m in split} x[pix(m)+tap][ci] * gy[m][co]
template <int BMC, int BNC>
__global__ void __launch_bounds__(256) k_conv_wgrad_simt(const float* __restrict__ x, const float* __restrict__ gy,
                                                         float* __restrict__ gw, ConvGeom g, int64_t m_per_split) {
  constexpr int BK = 16;
  constexpr int TM = BMC / 16, TN = BNC / 16;
  __shared__ float As[BK][BMC + 1];
  __shared__ float Bs[BK][BNC + 1];
  const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
  const int ci_tiles = (g.Cin + BMC - 1) / BMC, co_tiles = (g.Cout + BNC - 1) / BNC;
  int b = blockIdx.x;
  const int co_t = b % co_tiles; b /= co_tiles;
  const int ci_t = b % ci_tiles; b /= ci_tiles;
  const int tap = b;
  const int kh = tap / g.k, kw = tap % g.k;
  const int ci0 = ci_t * BMC, co0 = co_t * BNC;
  const int64_t M = (int64_t)g.N * g.Ho * g.Wo;
  const int64_t ms = (int64_t)blockIdx.y * m_per_split, me = min(M, ms + m_per_split);
  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  for (int64_t mb = ms; mb < me; mb += BK) {
    __syncthreads();
    // A: BK x BMC elements
    for (int e = tid; e < BK * BMC; e += 256) {
      const int kk = e / BMC, i = e % BMC;
      const int64_t m = mb + kk;
      float v = 0.f;
      const int ci = ci0 + i;
      if (m < me && ci < g.Cin) {
        int64_t t = m;
        const int wo = (int)(t % g.Wo); t /= g.Wo;
        const int ho = (int)(t % g.Ho);
        const int n = (int)(t / g.Ho);
        const int hi = ho + kh - g.pad, wi = wo + kw - g.pad;
        if (hi >= 0 && hi < g.H && wi >= 0 && wi < g.W) v = x[(((int64_t)n * g.H + hi) * g.W + wi) * g.Cin + ci];
      }
      As[kk][i] = v;
    }
    for (int e = tid; e < BK * BNC; e += 256) {
      const int kk = e / BNC, j = e % BNC;
      const int64_t m = mb + kk;
      const int co = co0 + j;
      Bs[kk][j] = (m < me && co < g.Cout) ? gy[m * g.Cout + co] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float a[TM], bb[TN];
#pragma unroll
      for (int i = 0; i < TM; ++i) a[i] = As[kk][ty * TM + i];
#pragma unroll
      for (int j = 0; j < TN; ++j) bb[j] = Bs[kk][tx * TN + j];
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], bb[j], acc[i][j]);
    }
  }
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int ci = ci0 + ty * TM + i;
    if (ci >= g.Cin) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      const int co = co0 + tx * TN + j;
      if (co < g.Cout)   // this pixel split's partial (add_partials sums the splits in order)
        gw[(int64_t)blockIdx.y * g.k * g.k * g.Cin * g.Cout + ((int64_t)tap * g.Cin + ci) * g.Cout + co] = acc[i][j];
    }
  }
}

static int launch_fwd(const float* x, const float* w, float* y, ConvGeom g, bool transposed, cudaStream_t st) {
  const int64_t M = (int64_t)g.N * g.Ho * g.Wo;
  const int bn = g.Cout <= 16 ? 16 : 64;
  const int64_t ctas = cdiv(M, 128) * cdiv(g.Cout, bn);
  const int num_kb = g.k * g.k * (int)cdiv(g.Cin, 8);
  // split-K when the output tile grid cannot fill the GPU (4x4-resolution layers, the 4x4 VALID head, the FC); the
  // splits store partial tiles that add_partials sums in split order, so the result is the same on every run
  int64_t splits = 1;
  if (ctas < kNumSMs) splits = cdiv(2 * kNumSMs, ctas);
  if (splits > num_kb / 4) splits = num_kb / 4 > 0 ? num_kb / 4 : 1;
  const int kbps = (int)cdiv(num_kb, splits);
  splits = cdiv(num_kb, kbps);
  float* out = y;
  if (splits > 1) {
    out = partials(splits * M * g.Cout, false, st);
    if (!out) return fail(TWG_ERR_UNSUPPORTED, "twg_conv simt: output too large for the split buffer");
    cudaMemsetAsync(y, 0, sizeof(float) * M * g.Cout, st);
  }
  dim3 grid((unsigned)cdiv(M, 128), (unsigned)cdiv(g.Cout, bn), (unsigned)splits);
  if (bn == 16) {
    if (transposed) k_conv_fwd_simt<16, 2, true><<<grid, 256, 0, st>>>(x, w, out, g, kbps);
    else k_conv_fwd_simt<16, 2, false><<<grid, 256, 0, st>>>(x, w, out, g, kbps);
  } else {
    if (transposed) k_conv_fwd_simt<64, 4, true><<<grid, 256, 0, st>>>(x, w, out, g, kbps);
    else k_conv_fwd_simt<64, 4, false><<<grid, 256, 0, st>>>(x, w, out, g, kbps);
  }
  if (int rc = check_launch("twg_conv simt")) return rc;
  return splits > 1 ? add_partials(y, out, (int)splits, M * g.Cout, st) : TWG_OK;
}

int conv_fwd_simt(const float* x, const float* w, float* y, int N, int H, int W, int Cin, int Cout, int k, int pad,
                  cudaStream_t st) {
  ConvGeom g{N, H, W, Cin, Cout, k, pad, H + 2 * pad - k + 1, W + 2 * pad - k + 1};
  if (g.Ho <= 0 || g.Wo <= 0) return fail(TWG_ERR_INVALID, "twg_conv_fwd: empty output");
  return launch_fwd(x, w, y, g, false, st);
}

int conv_dgrad_simt(const float* gy, const float* w, float* gx, int N, int H, int W, int Cin, int Cout, int k, int pad,
                    cudaStream_t st) {
  // gx = conv(gy, flip/transpose(w)) with pad' = k-1-pad; "input" is gy [N,Ho,Wo,Cout], "output" gx [N,H,W,Cin]
  const int Ho = H + 2 * pad - k + 1, Wo = W + 2 * pad - k + 1;
  ConvGeom g{N, Ho, Wo, Cout, Cin, k, k - 1 - pad, H, W};
  return launch_fwd(gy, w, gx, g, true, st);
}

int conv_wgrad_simt(const float* x, const float* gy, float* gw, int N, int H, int W, int Cin, int Cout, int k, int pad,
                    int accumulate, cudaStream_t st) {
  ConvGeom g{N, H, W, Cin, Cout, k, pad, H + 2 * pad - k + 1, W + 2 * pad - k + 1};
  if (!accumulate) cudaMemsetAsync(gw, 0, sizeof(float) * k * k * Cin * Cout, st);
  const int64_t M = (int64_t)g.N * g.Ho * g.Wo;
  const int bmc = Cin <= 16 ? 16 : 64, bnc = Cout <= 16 ? 16 : 64;
  const int tiles = k * k * (int)cdiv(Cin, bmc) * (int)cdiv(Cout, bnc);
  int64_t splits = cdiv(4 * kNumSMs, tiles);
  int64_t max_splits = cdiv(M, 64);
  if (splits > max_splits) splits = max_splits;
  if (splits < 1) splits = 1;
  int64_t mps = cdiv(cdiv(M, splits), 16) * 16;
  splits = cdiv(M, mps);
  dim3 grid((unsigned)tiles, (unsigned)splits);
  const int64_t gw_elems = (int64_t)k * k * Cin * Cout;
  float* parts = partials(splits * gw_elems, true, st);
  if (!parts) return fail(TWG_ERR_UNSUPPORTED, "twg_conv_wgrad simt: weight too large for the split buffer");
  if (bmc == 16 && bnc == 16) k_conv_wgrad_simt<16, 16><<<grid, 256, 0, st>>>(x, gy, parts, g, mps);
  else if (bmc == 16) k_conv_wgrad_simt<16, 64><<<grid, 256, 0, st>>>(x, gy, parts, g, mps);
  else if (bnc == 16) k_conv_wgrad_simt<64, 16><<<grid, 256, 0, st>>>(x, gy, parts, g, mps);
  else k_conv_wgrad_simt<64, 64><<<grid, 256, 0, st>>>(x, gy, parts, g, mps);
  if (int rc = check_launch("twg_conv_wgrad simt")) return rc;
  return add_partials(gw, parts, (int)splits, gw_elems, st);
}

}  // namespace twg
