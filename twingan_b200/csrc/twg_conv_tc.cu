// wgmma tensor-core convolution for sm_90a: implicit-GEMM forward / data-gradient and weight-gradient with
// split-bf16 operands ("bf16x3": x = hi + lo, three MMAs per product -- lo.hi, hi.lo, hi.hi -- fp32 register
// accumulation), so results match an fp32 convolution to ~1e-5 relative while running on the tensor cores.
//
// Both kernels are warp-specialised around an mbarrier ring (288 threads per CTA):
//   warps 0-7 : two consumer warpgroups; each issues wgmma.mma_async m64nNk16 on its 64-row half of the M = 128 tile
//               straight from the swizzled shared-memory tiles and runs the epilogue from its accumulator registers
//   warp 8    : TMA producer -- cp.async.bulk.tensor 4D boxes {C, TW, TH, TN} of the NHWC bf16 hi/lo planes (signed
//               start coordinates + hardware zero fill == SAME padding) and 2D boxes of the K-major weight planes,
//               landing in 128B/64B/32B-swizzled shared memory (the swizzle width is the channel chunk's row length)
// The forward reads pixels as the K-major A operand; the weight gradient reads the same NHWC tiles as MN-major operands
// (pixels are its GEMM K dimension), so no operand is ever transposed in memory.
#include <cuda.h>
#include <cuda_bf16.h>

#include <mutex>

#include "twg_common.cuh"

namespace twg {

// ----------------------------------------------------------------------------------------------------
// PTX wrappers
// ----------------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_load_4d(const CUtensorMap* tm, uint64_t* bar, void* dst, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(dst)), "l"(tm), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d(const CUtensorMap* tm, uint64_t* bar, void* dst, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(dst)), "l"(tm), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* tm) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(tm) : "memory");
}

// warpgroup MMA: D[64 x N] (+)= A[64 x 16] * B[16 x N], A and B described by shared-memory matrix descriptors.
// TA / TB = 1: the operand is MN-major (M or N contiguous in shared memory) instead of K-major.
template <int N>
struct Wgmma;
template <>
struct Wgmma<16> {
  template <int TA, int TB>
  __device__ __forceinline__ static void mma(float (&d)[8], uint64_t a, uint64_t b) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, 1, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, %10, %11;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(a), "l"(b), "n"(TA), "n"(TB));
  }
};
template <>
struct Wgmma<32> {
  template <int TA, int TB>
  __device__ __forceinline__ static void mma(float (&d)[16], uint64_t a, uint64_t b) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, 1, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %18, %19;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(a), "l"(b), "n"(TA), "n"(TB));
  }
};
template <>
struct Wgmma<64> {
  template <int TA, int TB>
  __device__ __forceinline__ static void mma(float (&d)[32], uint64_t a, uint64_t b) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, 1, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %34, %35;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a), "l"(b), "n"(TA), "n"(TB));
  }
};
template <>
struct Wgmma<128> {
  template <int TA, int TB>
  __device__ __forceinline__ static void mma(float (&d)[64], uint64_t a, uint64_t b) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, 1, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %66, %67;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(a), "l"(b), "n"(TA), "n"(TB));
  }
};
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs
template <int R>
__device__ __forceinline__ void fence_acc(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// ---- sm_90 shared-memory matrix descriptor ------------------------------------------------------------
// start>>4 [0,14) | LBO>>4 [16,30) | SBO>>4 [32,46) | base offset [49,52) = 0 | layout [62,64): 1 = 128B, 2 = 64B, 3 = 32B swizzle.
// K-major swizzled operand: SBO = stride between 8-row groups, LBO unused; a K step of 16 bf16 inside the swizzle atom
// advances the start address by 32 bytes.  MN-major swizzled operand: LBO = stride between MN atoms (one atom = one
// swizzle row of channels), SBO = stride between groups of 8 K rows.
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes, uint32_t layout) {
  uint64_t d = (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)layout << 62;
  return d;
}
// advance a descriptor's start address by a byte offset (multiple of 16)
__device__ __forceinline__ uint64_t desc_add(uint64_t d, uint32_t byte_off) { return d + (uint64_t)(byte_off >> 4); }
__host__ __device__ constexpr uint32_t swizzle_layout_for(int cc) { return cc == 64 ? 1u : (cc == 32 ? 2u : 3u); }

// ----------------------------------------------------------------------------------------------------
// split kernels: fp32 -> bf16 hi/lo planes
// ----------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_split_act(const float* __restrict__ x, void* __restrict__ planes, int64_t n4) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x)
    st_split4(planes, n4 * 4, i, reinterpret_cast<const float4*>(x)[i]);
}

// One conv weight w[taps][Cin][Cout] (HWIO, at flat + src) -> planes at planes + dst, in the layout the weight TMA maps read:
// forward: out[tap][co][ci] = w[tap][ci][co]           (K = Cin contiguous)
// dgrad  : out[tap][ci][co] = w[flip(tap)][ci][co]     (K = Cout contiguous)
struct SplitRow { long long src, dst; int taps, cin, cout, dgrad; };
__device__ __forceinline__ void split_weight_row(const float* __restrict__ flat, __nv_bfloat16* __restrict__ planes,
                                                 const SplitRow& r) {
  const float* w = flat + r.src;
  const int64_t total = (int64_t)r.taps * r.cin * r.cout;
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
    st_split1(planes + r.dst, total, i, v);
  }
}
__global__ void __launch_bounds__(256) k_split_weights(const float* __restrict__ w, __nv_bfloat16* __restrict__ planes,
                                                       SplitRow r) {
  split_weight_row(w, planes, r);
}
// every conv weight of the model in one launch: blockIdx.y = table row
__global__ void __launch_bounds__(256) k_split_weights_table(const float* __restrict__ flat, __nv_bfloat16* __restrict__ planes,
                                                             const SplitRow* __restrict__ table) {
  split_weight_row(flat, planes, table[blockIdx.y]);
}

// ----------------------------------------------------------------------------------------------------
// forward / dgrad kernel
// ----------------------------------------------------------------------------------------------------
struct TcGeom {
  int N, H, W;        // activation (input == output spatial size; SAME 3x3 or 1x1)
  int Cin, Cout;      // GEMM K channels, GEMM N channels
  int k, pad;
  int TW, TH, TN;     // pixel tile: TW*TH*TN == 128
  int tiles_w, tiles_h, tiles_n;
};

constexpr int kConsumerWarps = 8;                       // two warpgroups
constexpr int kThreads = (kConsumerWarps + 1) * 32;     // + the TMA producer warp
// Registers are allocated in units of four warps, so a CTA of kThreads gets at most 168 a thread: every tile's
// accumulators (BN / 2, or groups * BNW / 2 for the weight gradient) must fit well below that.

template <int CC, int BN>
struct FwdSmem {
  static constexpr int kATile = 128 * CC * 2;                       // bytes, one plane
  static constexpr int kBTileRaw = BN * CC * 2;
  static constexpr int kBTile = (kBTileRaw + 1023) / 1024 * 1024;
  static constexpr int kStage = 2 * kATile + 2 * kBTile;
  // enough stages to keep ~100+ KB of TMA traffic in flight per CTA, within the 227 KB an H100 block may use
  static constexpr int kStagesRaw = (200 * 1024) / kStage;
  static constexpr int kStages = kStagesRaw > 8 ? 8 : (kStagesRaw < 2 ? 2 : kStagesRaw);
  static constexpr int kBytes = kStages * kStage + 1024 /*align*/ + 256 /*barriers*/;
  static_assert(kBytes <= 227 * 1024, "forward conv exceeds shared memory");
};

// Forward epilogue of one 128-pixel tile from a consumer warp's accumulator fragment.  Options (all null / 0 = plain fp32
// store):
//   bias, act & 1      : + bias[c], leaky-ReLU                       (discriminator layers)
//   z_planes           : also store the result as split-bf16 planes  (input of the next conv)
//   act_mask           : sign of the (activated) result, 4 bits per 4 channels (the activation backward reads these)
//   stats              : {count, pivot, S1, S2} per (image, tile, consumer warp, channel) for the instance-norm statistics
//   aff_a              : z = pixel_norm?(lrelu?(aff_a[c] * conv + bias[c])), act bit 1 = pixel norm (Cout == BN: a row of
//                        the accumulator fragment is spread over 4 lanes, so the pixel's mean square is a 4-lane sum)
// The thread holds rows r0 = 16 (warp % 4) + lane / 4 (+ 8) of warpgroup warp / 4's half and columns 8 j + 2 (lane % 4) (+ 1).
template <int BN>
__device__ __forceinline__ void fwd_epilogue(float (&acc)[BN / 2], float* __restrict__ y, const TcGeom& g, int tw_i,
                                             int th_i, int n0, int co0, int warp, int lane, const float* __restrict__ bias,
                                             int act, void* __restrict__ z_planes, float4* __restrict__ stats,
                                             uint8_t* __restrict__ act_mask, const float* __restrict__ aff_a) {
  // the statistics, sign-mask and pixel-norm epilogues exist for the single-block shapes only (Cout <= 64; the host
  // never asks for them otherwise), which keeps the BN = 128 instantiations within their registers
  constexpr bool kFused = BN <= 64;
  const int wg = warp >> 2;
  const int w0 = tw_i * g.TW, h0 = th_i * g.TH;
  const int quad = lane & 3;
  int64_t e_row[2];
  bool ok[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    int t = wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * i;
    const int tw = t % g.TW; t /= g.TW;
    const int th = t % g.TH;
    const int tn = t / g.TH;
    const int n = n0 + tn, h = h0 + th, w = w0 + tw;
    ok[i] = n < g.N && h < g.H && w < g.W;
    e_row[i] = (((int64_t)n * g.H + h) * g.W + w) * g.Cout + co0;
  }
  if (bias) {
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int c = co0 + 8 * j + 2 * quad;
      const float b0 = __ldg(bias + c), b1 = __ldg(bias + c + 1);
      float a0 = 1.f, a1 = 1.f;
      if (aff_a) { a0 = __ldg(aff_a + c); a1 = __ldg(aff_a + c + 1); }
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        float v0 = fmaf(a0, acc[4 * j + 2 * i], b0), v1 = fmaf(a1, acc[4 * j + 2 * i + 1], b1);
        if (act & 1) { v0 = lrelu(v0); v1 = lrelu(v1); }
        acc[4 * j + 2 * i] = v0; acc[4 * j + 2 * i + 1] = v1;
      }
    }
  }
  if (kFused && aff_a && (act & 2)) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      float ss = 0.f;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) ss = fmaf(acc[4 * j + 2 * i], acc[4 * j + 2 * i], fmaf(acc[4 * j + 2 * i + 1], acc[4 * j + 2 * i + 1], ss));
      ss += __shfl_xor_sync(0xffffffffu, ss, 1);
      ss += __shfl_xor_sync(0xffffffffu, ss, 2);
      const float rinv = rsqrtf(ss * (1.f / (float)BN) + kPixEps);
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) { acc[4 * j + 2 * i] *= rinv; acc[4 * j + 2 * i + 1] *= rinv; }
    }
  }
  const int64_t n_total = (int64_t)g.N * g.H * g.W * g.Cout;
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int c = 8 * j + 2 * quad;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const float v0 = acc[4 * j + 2 * i], v1 = acc[4 * j + 2 * i + 1];
      uint32_t m = 0;
      if (kFused && act_mask) {   // lanes 2q and 2q+1 hold channels 4q' .. 4q'+3 of the row: one mask byte per float4 of z
        m = (v0 > 0.f ? 1u : 0u) | (v1 > 0.f ? 2u : 0u);
        m |= __shfl_xor_sync(0xffffffffu, m, 1) << 2;
      }
      if (!ok[i]) continue;
      const int64_t e = e_row[i] + c;
      if (y) *reinterpret_cast<float2*>(y + e) = make_float2(v0, v1);
      if (z_planes) st_planes2(z_planes, n_total, e, v0, v1);
      if (kFused && act_mask && (quad & 1) == 0) act_mask[e >> 2] = (uint8_t)m;
    }
  }
  if (kFused && stats) {
    // One record per (consumer warp, channel) over the warp's 16 pixel rows, around the pivot p = the value of the warp's
    // first row (lanes 0..3); twg_norm_finalize_partials merges the records.  Tiles never span images (TN == 1 here).
    float cnt = (ok[0] ? 1.f : 0.f) + (ok[1] ? 1.f : 0.f);
#pragma unroll
    for (int off = 4; off < 32; off <<= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, off);
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const float p = __shfl_sync(0xffffffffu, acc[4 * j + e], quad);
        float s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          if (ok[i]) {
            const float d = acc[4 * j + 2 * i + e] - p;
            s1 += d;
            s2 = fmaf(d, d, s2);
          }
        }
#pragma unroll
        for (int off = 4; off < 32; off <<= 1) {
          s1 += __shfl_xor_sync(0xffffffffu, s1, off);
          s2 += __shfl_xor_sync(0xffffffffu, s2, off);
        }
        if (lane < 4) {
          const int slots = g.tiles_h * g.tiles_w * kConsumerWarps;
          const int slot = (th_i * g.tiles_w + tw_i) * kConsumerWarps + warp;
          stats[((int64_t)n0 * slots + slot) * g.Cout + co0 + 8 * j + 2 * quad + e] = make_float4(cnt, p, s1, s2);
        }
      }
    }
  }
}

// One accumulation chain of the forward / dgrad consumer.  The MMAs of NST consecutive pipeline stages go into a fresh
// fragment `part`, which is then added to `acc` with fp32 adds and cleared: one tensor-core accumulation chain over the whole
// K = 9 * Cin (up to ~14 k products) would lose ~1e-5 relative.  NST is a compile-time constant and the loop is fully
// unrolled, so no data-dependent branch touches `part` between a wgmma's issue and its wait; with one, ptxas serialises every
// wgmma of the kernel (warning C7518) and the commit / wait_group pipelining below does nothing.
// The ring `full` / `empty` has KST stages.  A stage goes back to the producer once the next stage's MMAs are issued and its
// own have completed (wait_group 1); the chain's last stage once all of its MMAs have completed.
// operands(J0 + j, stage, dah, dal, dbh, dbl) gives the A hi / lo and B hi / lo descriptors of the chain's stage j.
template <int BN, int CC, int KST, int J0, int NST, class Operands>
__device__ __forceinline__ void mma_chain(float (&acc)[BN / 2], float (&part)[BN / 2], uint64_t* full, uint64_t* empty,
                                          int& stage, uint32_t& phase, int lane, const Operands& operands) {
  int prev = 0;
#pragma unroll
  for (int j = 0; j < NST; ++j) {
    mbar_wait(&full[stage], phase);
    uint64_t dah, dal, dbh, dbl;
    operands(J0 + j, stage, dah, dal, dbh, dbl);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < CC / 16; ++ks) {
      const uint32_t off = ks * 32;   // 16 bf16 along K inside the swizzle atom
      Wgmma<BN>::template mma<0, 0>(part, desc_add(dal, off), desc_add(dbh, off));
      Wgmma<BN>::template mma<0, 0>(part, desc_add(dah, off), desc_add(dbl, off));
      Wgmma<BN>::template mma<0, 0>(part, desc_add(dah, off), desc_add(dbh, off));
    }
    wgmma_commit();
    wgmma_wait<1>();                  // the previous stage's MMAs have read their operands: hand that stage back
    if (j > 0) { __syncwarp(); mbar_arrive_lane0(&empty[prev], lane); }
    prev = stage;
    if (++stage == KST) { stage = 0; phase ^= 1; }
  }
  wgmma_wait<0>();
  __syncwarp();
  mbar_arrive_lane0(&empty[prev], lane);
  fence_acc(part);
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) { acc[i] += part[i]; part[i] = 0.f; }
  fence_acc(part);
}

// General forward / dgrad: one CTA per (128-pixel tile, output-channel block), one pipeline stage per (tap, channel chunk)
// holding that tap's shifted A tile and its weight tile.  Epilogue options: fwd_epilogue.
template <int CC, int BN>
__global__ void __launch_bounds__(kThreads, 1) k_conv_fwd_wgmma(const __grid_constant__ CUtensorMap tm_a_hi,
                                                                const __grid_constant__ CUtensorMap tm_a_lo,
                                                                const __grid_constant__ CUtensorMap tm_b_hi,
                                                                const __grid_constant__ CUtensorMap tm_b_lo,
                                                                float* __restrict__ y, TcGeom g,
                                                                const float* __restrict__ bias, int act,
                                                                void* __restrict__ z_planes, float4* __restrict__ stats,
                                                                uint8_t* __restrict__ act_mask, const float* __restrict__ aff_a) {
  using SM = FwdSmem<CC, BN>;
  constexpr int kStages = SM::kStages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + kStages * SM::kStage);   // [kStages]
  uint64_t* empty = full + kStages;                                           // [kStages]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int mt = blockIdx.x;
  const int tw_i = mt % g.tiles_w; mt /= g.tiles_w;
  const int th_i = mt % g.tiles_h;
  const int tn_i = mt / g.tiles_h;
  const int w0 = tw_i * g.TW, h0 = th_i * g.TH, n0 = tn_i * g.TN;
  const int co0 = blockIdx.y * BN;
  const int cchunks = g.Cin / CC;
  const int kb_begin = 0, kb_end = g.k * g.k * cchunks;

  if (warp == kConsumerWarps && lane == 0) {
    prefetch_tmap(&tm_a_hi); prefetch_tmap(&tm_a_lo); prefetch_tmap(&tm_b_hi); prefetch_tmap(&tm_b_lo);
    for (int s = 0; s < kStages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], kConsumerWarps); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == kConsumerWarps) {
    if (lane == 0) {
      int stage = 0; uint32_t phase = 0;
      for (int kb = kb_begin; kb < kb_end; ++kb) {
        mbar_wait(&empty[stage], phase ^ 1);
        const int tap = kb / cchunks, cc = kb - tap * cchunks;
        const int kh = tap / g.k, kw = tap - kh * g.k;
        uint8_t* sa = smem + stage * SM::kStage;
        mbar_expect_tx(&full[stage], 2 * SM::kATile + 2 * SM::kBTileRaw);
        tma_load_4d(&tm_a_hi, &full[stage], sa, cc * CC, w0 + kw - g.pad, h0 + kh - g.pad, n0);
        tma_load_4d(&tm_a_lo, &full[stage], sa + SM::kATile, cc * CC, w0 + kw - g.pad, h0 + kh - g.pad, n0);
        tma_load_2d(&tm_b_hi, &full[stage], sa + 2 * SM::kATile, cc * CC, tap * g.Cout + co0);
        tma_load_2d(&tm_b_lo, &full[stage], sa + 2 * SM::kATile + SM::kBTile, cc * CC, tap * g.Cout + co0);
        if (++stage == kStages) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }

  // ---- consumers: warpgroup wg owns accumulator rows [64 wg, 64 wg + 64) of the 128-pixel tile ----
  const int wg = warp >> 2;
  constexpr int kFlush = 4;   // stages per accumulation chain (mma_chain)
  float acc[BN / 2], part[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) { acc[i] = 0.f; part[i] = 0.f; }
  {
    constexpr uint32_t layout = swizzle_layout_for(CC);
    constexpr uint32_t sbo = 8 * CC * 2;   // 8 rows of CC bf16
    // stage 0's descriptors; stage s is SM::kStage * s bytes further
    const uint32_t a_hi = smem_u32(smem) + wg * (64 * CC * 2), b_hi = smem_u32(smem) + 2 * SM::kATile;
    const uint64_t dah0 = make_desc(a_hi, 16, sbo, layout), dbh0 = make_desc(b_hi, 16, sbo, layout);
    const auto operands = [&](int, int s, uint64_t& dah, uint64_t& dal, uint64_t& dbh, uint64_t& dbl) {
      dah = desc_add(dah0, s * SM::kStage); dal = desc_add(dah, SM::kATile);
      dbh = desc_add(dbh0, s * SM::kStage); dbl = desc_add(dbh, SM::kBTile);
    };
    int stage = 0; uint32_t phase = 0;
    int kb = kb_begin;
#pragma unroll 1
    for (; kb + kFlush <= kb_end; kb += kFlush)
      mma_chain<BN, CC, kStages, 0, kFlush>(acc, part, full, empty, stage, phase, lane, operands);
    switch (kb_end - kb) {   // the last, shorter chain
      case 1: mma_chain<BN, CC, kStages, 0, 1>(acc, part, full, empty, stage, phase, lane, operands); break;
      case 2: mma_chain<BN, CC, kStages, 0, 2>(acc, part, full, empty, stage, phase, lane, operands); break;
      case 3: mma_chain<BN, CC, kStages, 0, 3>(acc, part, full, empty, stage, phase, lane, operands); break;
      default: break;
    }
    static_assert(kFlush == 4, "the tail chains above cover 1 .. kFlush - 1 stages");
  }

  fwd_epilogue<BN>(acc, y, g, tw_i, th_i, n0, co0, warp, lane, bias, act, z_planes, stats, act_mask, aff_a);
}

// ---- column-box forward / dgrad: 3x3 SAME, one channel chunk (GEMM K == CC <= 64), 16 x 8 pixel tiles inside one image.
// Per tile the A operand is three boxes {CC, 16, 10, 1} per plane, one per kw, loaded at (w0 + kw - 1, h0 - 1): box kw's
// pixel row r holds input pixel (w0 + kw - 1 + r % 16, h0 - 1 + r / 16), so tap (kh, kw)'s 128-pixel A tile is box kw from
// pixel row 16 kh on, and warpgroup wg's 64-row half starts at row 16 (kh + 4 wg).  16 rows are a whole number of swizzle
// atoms, so each tap view is an ordinary swizzled K-major operand at a different start address.  Every input pixel crosses
// into shared memory 3 times instead of 9, with the same hardware zero fill at the borders; the consumer issues the same MMAs
// in the same order (tap-major, lo.hi, hi.lo, hi.hi, in chains of taps 0-3, 4-7 and 8) as k_conv_fwd_wgmma on the same
// operand values, so the results are bit-identical to it.
// The CTAs are persistent: CTA b computes work items b, b + gridDim.x, ... (item = tile + tiles * output-channel block),
// each exactly once; the A boxes are double-buffered where they fit (CC <= 32), so the next tile's boxes load while the
// current one computes, and weight tiles stream through their own per-tap ring.  The keys with a small single weight block
// keep it in shared memory instead (cols_resident, conv_cols_resident below).
template <int CC, int BN>
struct ColSmem {
  static constexpr int kBox = 160 * CC * 2;                         // one box, one plane
  static constexpr int kABuf = 6 * kBox;                            // [hi: kw 0, 1, 2][lo: kw 0, 1, 2]
  static constexpr int kABufs = CC == 64 ? 1 : 2;                   // 2 x 120 KB would not fit at CC = 64
  static constexpr int kBTileRaw = BN * CC * 2;
  static constexpr int kBTile = (kBTileRaw + 1023) / 1024 * 1024;
  static constexpr int kWStage = 2 * kBTile;
  static constexpr int kWStagesRaw = (220 * 1024 - kABufs * kABuf) / kWStage;
  static constexpr int kWStages = kWStagesRaw > 9 ? 9 : kWStagesRaw;
  static constexpr int kBytes = kABufs * kABuf + kWStages * kWStage + 1024 /*align*/ + 256 /*barriers*/;
  static_assert(kWStages >= 2, "column-box conv: weight ring too short");
  static_assert(kBytes <= 227 * 1024, "column-box conv exceeds shared memory");
};

// The keys with one output-channel block (BN == Cout <= 64) and a chunk of CC <= 32 keep all 9 hi / lo weight tiles (at
// most 72 KB) in shared memory for the CTA's lifetime instead of streaming them through the per-tap ring for every tile,
// and still fit two or more A buffers beside them.  (At CC = 64 one A buffer is 120 KB: with resident weights it stays a
// single buffer, and on an H100 that measured no faster than the streaming kernel, so CC = 64 keeps that.)  Where two
// 128-row accumulators fit in registers (BN <= 32; at BN = 64 ptxas spills) each consumer warpgroup also takes a tile
// stream of its own.
__host__ __device__ constexpr bool cols_resident(int cc, int bn) { return cc <= 32 && bn <= 64; }
__host__ __device__ constexpr bool cols_dual(int cc, int bn) { return cols_resident(cc, bn) && bn <= 32; }

template <int CC, int BN>
struct ColResSmem {
  static constexpr int kBox = 160 * CC * 2;                         // one box, one plane
  static constexpr int kABuf = 6 * kBox;                            // [hi: kw 0, 1, 2][lo: kw 0, 1, 2]
  static constexpr int kBTileRaw = BN * CC * 2;
  static constexpr int kBTile = (kBTileRaw + 1023) / 1024 * 1024;
  static constexpr int kW = 9 * 2 * kBTile;                         // [tap][hi, lo]
  static constexpr int kABufsRaw = (220 * 1024 - kW) / kABuf;
  static constexpr int kABufs = kABufsRaw > 4 ? 4 : kABufsRaw;
  static constexpr int kBytes = kW + kABufs * kABuf + 1024 /*align*/ + 256 /*barriers*/;
  static_assert(kABufs >= 2, "column-box conv: too few A buffers beside the weights");
  static_assert(kBytes <= 227 * 1024, "column-box conv exceeds shared memory");
};

template <int CC, int BN>
constexpr int col_smem_bytes() {
  if constexpr (cols_resident(CC, BN)) return ColResSmem<CC, BN>::kBytes;
  else return ColSmem<CC, BN>::kBytes;
}

// One accumulation chain of the resident-weight consumer: taps J0 .. J0 + NST - 1 of the warpgroup's KB m64 blocks, all
// issued before one wait, each block into its own fragment part[b] that is then added to acc[b] (mma_chain's chains and
// per-block MMA order, without its per-stage handshakes: weights and A boxes are resident for the whole tile).
// operands(tap, b, dah, dal, dbh, dbl) gives block b's A hi / lo and the tap's B hi / lo descriptors.
template <int BN, int CC, int KB, int J0, int NST, class Operands>
__device__ __forceinline__ void mma_chain_resident(float (&acc)[KB][BN / 2], float (&part)[KB][BN / 2],
                                                   const Operands& operands) {
  wgmma_fence();
#pragma unroll
  for (int j = 0; j < NST; ++j) {
#pragma unroll
    for (int b = 0; b < KB; ++b) {
      uint64_t dah, dal, dbh, dbl;
      operands(J0 + j, b, dah, dal, dbh, dbl);
      asm volatile("" : "+l"(dah), "+l"(dal), "+l"(dbh), "+l"(dbl));
#pragma unroll
      for (int ks = 0; ks < CC / 16; ++ks) {
        const uint32_t off = ks * 32;   // 16 bf16 along K inside the swizzle atom
        Wgmma<BN>::template mma<0, 0>(part[b], desc_add(dal, off), desc_add(dbh, off));
        Wgmma<BN>::template mma<0, 0>(part[b], desc_add(dah, off), desc_add(dbl, off));
        Wgmma<BN>::template mma<0, 0>(part[b], desc_add(dah, off), desc_add(dbh, off));
      }
    }
  }
  wgmma_commit();
  wgmma_wait<0>();
#pragma unroll
  for (int b = 0; b < KB; ++b) {
    fence_acc(part[b]);
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) { acc[b][i] += part[b][i]; part[b][i] = 0.f; }
    fence_acc(part[b]);
  }
}

// Column-box forward / dgrad with resident weights (cols_resident keys).  The producer loads the 9 hi / lo weight tiles
// once, under one mbarrier, then the CTA's tiles' A boxes in order through a ring of kABufs buffers.
//   dual (BN <= 32): warpgroup wg takes every other work item of the CTA (items wg, wg + 2, ...) and computes all 128 rows
//     of it as two m64 blocks with two accumulators, so one warpgroup's epilogue overlaps the other's MMAs.
//   otherwise (BN = 64): both warpgroups share every item, 64 rows each, as in the streaming kernel.
// Block r (rows 64 r .. 64 r + 63) is computed and stored exactly as consumer warpgroup r of the streaming kernel does it --
// same MMAs in the same order on the same operands, same statistics slots (warp 4 r + warp % 4) -- so every output is
// bit-identical to it.
template <int CC, int BN>
__device__ __forceinline__ void conv_cols_resident(uint8_t* smem, const CUtensorMap* tm_a_hi, const CUtensorMap* tm_a_lo,
                                                   const CUtensorMap* tm_b_hi, const CUtensorMap* tm_b_lo,
                                                   float* __restrict__ y, const TcGeom& g, const float* __restrict__ bias,
                                                   int act, void* __restrict__ z_planes, float4* __restrict__ stats,
                                                   uint8_t* __restrict__ act_mask, const float* __restrict__ aff_a) {
  using SM = ColResSmem<CC, BN>;
  constexpr int kABufs = SM::kABufs;
  constexpr bool kDual = cols_dual(CC, BN);
  constexpr int KB = kDual ? 2 : 1;                                      // m64 blocks per warpgroup and item
  uint8_t* sw = smem + kABufs * SM::kABuf;                                 // weights [tap][hi, lo]
  uint64_t* afull = reinterpret_cast<uint64_t*>(sw + SM::kW);              // [kABufs]
  uint64_t* aempty = afull + kABufs;                                       // [kABufs]
  uint64_t* wfull = aempty + kABufs;                                       // [1]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles = g.tiles_w * g.tiles_h * g.tiles_n;   // == work items: one output-channel block

  if (warp == kConsumerWarps && lane == 0) {
    prefetch_tmap(tm_a_hi); prefetch_tmap(tm_a_lo); prefetch_tmap(tm_b_hi); prefetch_tmap(tm_b_lo);
    for (int s = 0; s < kABufs; ++s) { mbar_init(&afull[s], 1); mbar_init(&aempty[s], kDual ? 4 : kConsumerWarps); }
    mbar_init(wfull, 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == kConsumerWarps) {
    if (lane == 0) {
      mbar_expect_tx(wfull, 18 * SM::kBTileRaw);
      for (int tap = 0; tap < 9; ++tap) {
        tma_load_2d(tm_b_hi, wfull, sw + (2 * tap) * SM::kBTile, 0, tap * BN);
        tma_load_2d(tm_b_lo, wfull, sw + (2 * tap + 1) * SM::kBTile, 0, tap * BN);
      }
      int ab = 0; uint32_t aph = 0;
      for (int u = blockIdx.x; u < tiles; u += gridDim.x) {
        const int tw_i = u % g.tiles_w, th_i = (u / g.tiles_w) % g.tiles_h, n0 = u / (g.tiles_w * g.tiles_h);
        const int w0 = tw_i * 16, h0 = th_i * 8;
        mbar_wait(&aempty[ab], aph ^ 1);
        mbar_expect_tx(&afull[ab], SM::kABuf);
        uint8_t* sa = smem + ab * SM::kABuf;
        for (int kw = 0; kw < 3; ++kw) {
          tma_load_4d(tm_a_hi, &afull[ab], sa + kw * SM::kBox, 0, w0 + kw - 1, h0 - 1, n0);
          tma_load_4d(tm_a_lo, &afull[ab], sa + (3 + kw) * SM::kBox, 0, w0 + kw - 1, h0 - 1, n0);
        }
        if (++ab == kABufs) { ab = 0; aph ^= 1; }
      }
    }
    return;
  }

  const int wg = warp >> 2;
  constexpr uint32_t layout = swizzle_layout_for(CC);
  constexpr uint32_t sbo = 8 * CC * 2;     // 8 rows of CC bf16
  // tap 0's hi weight tile; tap t's hi / lo tiles are 2 t / 2 t + 1 tiles further
  const uint64_t dbh0 = make_desc(smem_u32(sw), 16, sbo, layout);
  // item i of the CTA (work item blockIdx.x + i gridDim.x) sits in A buffer i % kABufs, phase (i / kABufs) & 1.  A
  // warpgroup waits for its items in order, and the producer loads all items in order, so by the time it waits for item i
  // item i - kABufs (<= its previous item when kABufs >= 2) has been loaded and the parity names the right phase.
  const int i0 = kDual ? wg : 0, di = kDual ? 2 : 1;
  bool weights_ready = false;
  for (int i = i0, u = blockIdx.x + i0 * gridDim.x; u < tiles; i += di, u += di * gridDim.x) {
    const int tw_i = u % g.tiles_w, th_i = (u / g.tiles_w) % g.tiles_h, n0 = u / (g.tiles_w * g.tiles_h);
    const int ab = i % kABufs;
    if (!weights_ready) { mbar_wait(wfull, 0); weights_ready = true; }
    float acc[KB][BN / 2], part[KB][BN / 2];
#pragma unroll
    for (int b = 0; b < KB; ++b)
#pragma unroll
      for (int j = 0; j < BN / 2; ++j) { acc[b][j] = 0.f; part[b][j] = 0.f; }
    mbar_wait(&afull[ab], (uint32_t)(i / kABufs) & 1u);
    // hi box 0 from pixel row 0; block r's tap (kh, kw) view starts kw boxes and 16 (kh + 4 r) pixel rows further
    const uint64_t dah0 = make_desc(smem_u32(smem + ab * SM::kABuf), 16, sbo, layout);
    // the weight descriptors are the same for every item: hidden from the compiler per item, so that it does not hoist
    // them out of the loop into registers the accumulators need (mma_chain_resident does the same per tap)
    uint64_t dbt = dbh0;
    asm volatile("" : "+l"(dbt));
    const auto operands = [&](int tap, int b, uint64_t& dah, uint64_t& dal, uint64_t& dbh, uint64_t& dbl) {
      const int kh = tap / 3, kw = tap - kh * 3;
      const int r = kDual ? b : wg;
      dah = desc_add(dah0, kw * SM::kBox + (kh + 4 * r) * (16 * CC * 2)); dal = desc_add(dah, 3 * SM::kBox);
      dbh = desc_add(dbt, 2 * tap * SM::kBTile); dbl = desc_add(dbh, SM::kBTile);
    };
    // taps 0-3, 4-7 and 8: the chains of k_conv_fwd_wgmma
    mma_chain_resident<BN, CC, KB, 0, 4>(acc, part, operands);
    mma_chain_resident<BN, CC, KB, 4, 4>(acc, part, operands);
    mma_chain_resident<BN, CC, KB, 8, 1>(acc, part, operands);
    // every MMA of the item has completed: its A buffer goes back to the producer
    __syncwarp();
    mbar_arrive_lane0(&aempty[ab], lane);
#pragma unroll
    for (int b = 0; b < KB; ++b) {
      const int r = kDual ? b : wg;
      fwd_epilogue<BN>(acc[b], y, g, tw_i, th_i, n0, 0, 4 * r + (warp & 3), lane, bias, act, z_planes, stats, act_mask,
                       aff_a);
    }
  }
}

template <int CC, int BN>
__global__ void __launch_bounds__(kThreads, 1) k_conv_fwd_cols_wgmma(const __grid_constant__ CUtensorMap tm_a_hi,
                                                                     const __grid_constant__ CUtensorMap tm_a_lo,
                                                                     const __grid_constant__ CUtensorMap tm_b_hi,
                                                                     const __grid_constant__ CUtensorMap tm_b_lo,
                                                                     float* __restrict__ y, TcGeom g,
                                                                     const float* __restrict__ bias, int act,
                                                                     void* __restrict__ z_planes, float4* __restrict__ stats,
                                                                     uint8_t* __restrict__ act_mask,
                                                                     const float* __restrict__ aff_a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  if constexpr (cols_resident(CC, BN)) {
    conv_cols_resident<CC, BN>(smem, &tm_a_hi, &tm_a_lo, &tm_b_hi, &tm_b_lo, y, g, bias, act, z_planes, stats, act_mask,
                               aff_a);
    return;
  }
  using SM = ColSmem<CC, BN>;
  constexpr int kABufs = SM::kABufs, kWStages = SM::kWStages;
  uint8_t* sw = smem + kABufs * SM::kABuf;                                     // weight ring [kWStages][hi][lo]
  uint64_t* afull = reinterpret_cast<uint64_t*>(sw + kWStages * SM::kWStage);  // [kABufs]
  uint64_t* aempty = afull + kABufs;                                           // [kABufs]
  uint64_t* wfull = aempty + kABufs;                                           // [kWStages]
  uint64_t* wempty = wfull + kWStages;                                         // [kWStages]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles = g.tiles_w * g.tiles_h * g.tiles_n;
  const int work = tiles * (g.Cout / BN);

  if (warp == kConsumerWarps && lane == 0) {
    prefetch_tmap(&tm_a_hi); prefetch_tmap(&tm_a_lo); prefetch_tmap(&tm_b_hi); prefetch_tmap(&tm_b_lo);
    for (int s = 0; s < kABufs; ++s) { mbar_init(&afull[s], 1); mbar_init(&aempty[s], kConsumerWarps); }
    for (int s = 0; s < kWStages; ++s) { mbar_init(&wfull[s], 1); mbar_init(&wempty[s], kConsumerWarps); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == kConsumerWarps) {
    if (lane == 0) {
      int ab = 0, ws = 0; uint32_t aph = 0, wph = 0;
      for (int u = blockIdx.x; u < work; u += gridDim.x) {
        const int mt = u % tiles, co0 = (u / tiles) * BN;
        const int tw_i = mt % g.tiles_w, th_i = (mt / g.tiles_w) % g.tiles_h, n0 = mt / (g.tiles_w * g.tiles_h);
        const int w0 = tw_i * 16, h0 = th_i * 8;
        mbar_wait(&aempty[ab], aph ^ 1);
        mbar_expect_tx(&afull[ab], SM::kABuf);
        uint8_t* sa = smem + ab * SM::kABuf;
        for (int kw = 0; kw < 3; ++kw) {
          tma_load_4d(&tm_a_hi, &afull[ab], sa + kw * SM::kBox, 0, w0 + kw - 1, h0 - 1, n0);
          tma_load_4d(&tm_a_lo, &afull[ab], sa + (3 + kw) * SM::kBox, 0, w0 + kw - 1, h0 - 1, n0);
        }
        if (++ab == kABufs) { ab = 0; aph ^= 1; }
        for (int tap = 0; tap < 9; ++tap) {
          mbar_wait(&wempty[ws], wph ^ 1);
          uint8_t* sb = sw + ws * SM::kWStage;
          mbar_expect_tx(&wfull[ws], 2 * SM::kBTileRaw);
          tma_load_2d(&tm_b_hi, &wfull[ws], sb, 0, tap * g.Cout + co0);
          tma_load_2d(&tm_b_lo, &wfull[ws], sb + SM::kBTile, 0, tap * g.Cout + co0);
          if (++ws == kWStages) { ws = 0; wph ^= 1; }
        }
      }
    }
    return;
  }

  const int wg = warp >> 2;
  constexpr uint32_t layout = swizzle_layout_for(CC);
  constexpr uint32_t sbo = 8 * CC * 2;     // 8 rows of CC bf16
  // weight stage 0's descriptor; stage s is SM::kWStage * s bytes further
  const uint64_t dbh0 = make_desc(smem_u32(sw), 16, sbo, layout);
  int ab = 0, ws = 0; uint32_t aph = 0, wph = 0;
  for (int u = blockIdx.x; u < work; u += gridDim.x) {
    const int mt = u % tiles, co0 = (u / tiles) * BN;
    const int tw_i = mt % g.tiles_w, th_i = (mt / g.tiles_w) % g.tiles_h, n0 = mt / (g.tiles_w * g.tiles_h);
    float acc[BN / 2], part[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) { acc[i] = 0.f; part[i] = 0.f; }
    mbar_wait(&afull[ab], aph);
    // hi box 0 from warpgroup wg's first pixel row; tap (kh, kw) starts kw boxes and 16 kh pixel rows further
    const uint64_t dah0 = make_desc(smem_u32(smem + ab * SM::kABuf) + 4 * wg * (16 * CC * 2), 16, sbo, layout);
    const auto operands = [&](int tap, int s, uint64_t& dah, uint64_t& dal, uint64_t& dbh, uint64_t& dbl) {
      const int kh = tap / 3, kw = tap - kh * 3;
      dah = desc_add(dah0, kw * SM::kBox + kh * (16 * CC * 2)); dal = desc_add(dah, 3 * SM::kBox);
      dbh = desc_add(dbh0, s * SM::kWStage); dbl = desc_add(dbh, SM::kBTile);
    };
    // taps 0-3, 4-7 and 8: the chains of k_conv_fwd_wgmma (one stage there == one tap here)
    mma_chain<BN, CC, kWStages, 0, 4>(acc, part, wfull, wempty, ws, wph, lane, operands);
    mma_chain<BN, CC, kWStages, 4, 4>(acc, part, wfull, wempty, ws, wph, lane, operands);
    mma_chain<BN, CC, kWStages, 8, 1>(acc, part, wfull, wempty, ws, wph, lane, operands);
    // every MMA of the tile has completed: the A buffer goes back to the producer, which loads the next tile's boxes while
    // this one runs its epilogue
    __syncwarp();
    mbar_arrive_lane0(&aempty[ab], lane);
    if (++ab == kABufs) { ab = 0; aph ^= 1; }
    fwd_epilogue<BN>(acc, y, g, tw_i, th_i, n0, co0, warp, lane, bias, act, z_planes, stats, act_mask, aff_a);
  }
}

// ----------------------------------------------------------------------------------------------------
// weight-gradient kernel ("tap-stacked"):  gw[tap][ci][co] += sum_pix x[pix + tap][ci] * gy[pix][co]
//   D[M = (tap, ci) stacked: TG = 128/CN taps x CN channels][N = BNW output channels], K = pixels.
//   A = TG shifted x tap tiles back to back in shared memory, read MN-major with LBO = one tap tile, so one M = 128 tile
//   covers TG taps (warpgroup wg takes taps [TG/2 wg, TG/2 wg + TG/2)); B = the gy tile, MN-major.  The ceil(9/TG)
//   accumulators of all tap groups stay in registers over the CTA's pixel tiles and are added to gw once.
//   Pipeline unit = one tap group (TG*2 tiles = 64 KB), two stages; gy tiles have their own 2-stage ring.
// ----------------------------------------------------------------------------------------------------
template <int CN, int BNW>
struct WgCfg {
  static constexpr int TG = 128 / CN;                       // taps per M = 128 group
  static constexpr int kXTile = 128 * CN * 2;               // one tap tile, one plane
  static constexpr int kAStage = 2 * TG * kXTile;           // hi group + lo group = 64 KB
  static constexpr int kGTile = 128 * BNW * 2;              // gy tile, one plane
  static constexpr int kGStage = 2 * kGTile;
  static constexpr int kAStages = 2, kGStages = 2;
  static constexpr int kBytes = kAStages * kAStage + kGStages * kGStage + 1024 + 256;
  static constexpr int kMaxGroups = (9 + TG - 1) / TG;
  static_assert(kBytes <= 227 * 1024, "weight-gradient conv exceeds shared memory");
};

template <int CN, int BNW>
__global__ void __launch_bounds__(kThreads, 1) k_conv_wgrad_wgmma(const __grid_constant__ CUtensorMap tm_g_hi,
                                                                  const __grid_constant__ CUtensorMap tm_g_lo,
                                                                  const __grid_constant__ CUtensorMap tm_x_hi,
                                                                  const __grid_constant__ CUtensorMap tm_x_lo,
                                                                  float* __restrict__ gw, TcGeom g, int tiles_per_cta) {
  using C = WgCfg<CN, BNW>;
  constexpr int TG = C::TG;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sa = smem;                                     // [kAStages][hi: TG tiles][lo: TG tiles]
  uint8_t* sg = smem + C::kAStages * C::kAStage;          // [kGStages][hi][lo]
  uint64_t* afull = reinterpret_cast<uint64_t*>(sg + C::kGStages * C::kGStage);
  uint64_t* aempty = afull + C::kAStages;
  uint64_t* gfull = aempty + C::kAStages;
  uint64_t* gempty = gfull + C::kGStages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int taps = g.k * g.k;
  const int groups = (taps + TG - 1) / TG;
  const int co0 = blockIdx.y * BNW;
  const int ci0 = blockIdx.z * CN;
  const int total_tiles = g.tiles_w * g.tiles_h * g.tiles_n;
  const int t_begin = blockIdx.x * tiles_per_cta;
  const int t_end = min(total_tiles, t_begin + tiles_per_cta);

  if (warp == kConsumerWarps && lane == 0) {
    prefetch_tmap(&tm_g_hi); prefetch_tmap(&tm_g_lo); prefetch_tmap(&tm_x_hi); prefetch_tmap(&tm_x_lo);
    for (int s = 0; s < C::kAStages; ++s) { mbar_init(&afull[s], 1); mbar_init(&aempty[s], kConsumerWarps); }
    for (int s = 0; s < C::kGStages; ++s) { mbar_init(&gfull[s], 1); mbar_init(&gempty[s], kConsumerWarps); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == kConsumerWarps) {
    if (lane == 0) {
      int as = 0, gs = 0; uint32_t aph = 0, gph = 0;
      for (int t = t_begin; t < t_end; ++t) {
        int mt = t;
        const int tw_i = mt % g.tiles_w; mt /= g.tiles_w;
        const int th_i = mt % g.tiles_h;
        const int tn_i = mt / g.tiles_h;
        const int w0 = tw_i * g.TW, h0 = th_i * g.TH, n0 = tn_i * g.TN;
        mbar_wait(&gempty[gs], gph ^ 1);
        mbar_expect_tx(&gfull[gs], C::kGStage);
        tma_load_4d(&tm_g_hi, &gfull[gs], sg + gs * C::kGStage, co0, w0, h0, n0);
        tma_load_4d(&tm_g_lo, &gfull[gs], sg + gs * C::kGStage + C::kGTile, co0, w0, h0, n0);
        if (++gs == C::kGStages) { gs = 0; gph ^= 1; }
        for (int grp = 0; grp < groups; ++grp) {
          const int tap0 = grp * TG, ntap = min(TG, taps - tap0);
          mbar_wait(&aempty[as], aph ^ 1);
          mbar_expect_tx(&afull[as], 2 * ntap * C::kXTile);
          uint8_t* base = sa + as * C::kAStage;
          for (int j = 0; j < ntap; ++j) {
            const int tap = tap0 + j;
            const int kh = tap / g.k, kw = tap - kh * g.k;
            tma_load_4d(&tm_x_hi, &afull[as], base + j * C::kXTile, ci0, w0 + kw - g.pad, h0 + kh - g.pad, n0);
            tma_load_4d(&tm_x_lo, &afull[as], base + (TG + j) * C::kXTile, ci0, w0 + kw - g.pad, h0 + kh - g.pad, n0);
          }
          if (++as == C::kAStages) { as = 0; aph ^= 1; }
        }
      }
    }
    return;
  }

  const int wg = warp >> 2;
  float acc[C::kMaxGroups][BNW / 2];
#pragma unroll
  for (int a = 0; a < C::kMaxGroups; ++a)
#pragma unroll
    for (int i = 0; i < BNW / 2; ++i) acc[a][i] = 0.f;
  {
    constexpr uint32_t la = swizzle_layout_for(CN), lb = swizzle_layout_for(BNW);
    constexpr uint32_t sbo_a = 8 * CN * 2, sbo_b = 8 * BNW * 2;        // stride between 8-pixel groups (K)
    int as = 0, gs = 0; uint32_t aph = 0, gph = 0;
    for (int t = t_begin; t < t_end; ++t) {
      mbar_wait(&gfull[gs], gph);
      const uint32_t gb_hi = smem_u32(sg + gs * C::kGStage), gb_lo = gb_hi + C::kGTile;
      const uint64_t dbh = make_desc(gb_hi, C::kGTile, sbo_b, lb), dbl = make_desc(gb_lo, C::kGTile, sbo_b, lb);
#pragma unroll
      for (int grp = 0; grp < C::kMaxGroups; ++grp) {
        if (grp >= groups) break;
        mbar_wait(&afull[as], aph);
        if (grp * TG + wg * (TG / 2) < taps) {         // warpgroup-uniform: skip a half tile that holds no tap
          const uint32_t xa_hi = smem_u32(sa + as * C::kAStage) + wg * (TG / 2) * C::kXTile, xa_lo = xa_hi + TG * C::kXTile;
          const uint64_t dah = make_desc(xa_hi, C::kXTile, sbo_a, la), dal = make_desc(xa_lo, C::kXTile, sbo_a, la);
          // one tile's 128 pixels go to a fresh fragment that is then added to the running sum with fp32 adds: a CTA
          // covers up to ~10^4 pixels, and one tensor-core accumulation chain that long loses ~1e-4 relative
          float part[BNW / 2];
#pragma unroll
          for (int i = 0; i < BNW / 2; ++i) part[i] = 0.f;
          fence_acc(part);
          wgmma_fence();
#pragma unroll
          for (int ks = 0; ks < 128 / 16; ++ks) {          // 16 pixels per MMA
            const uint32_t offa = ks * 2 * sbo_a, offb = ks * 2 * sbo_b;
            Wgmma<BNW>::template mma<1, 1>(part, desc_add(dal, offa), desc_add(dbh, offb));
            Wgmma<BNW>::template mma<1, 1>(part, desc_add(dah, offa), desc_add(dbl, offb));
            Wgmma<BNW>::template mma<1, 1>(part, desc_add(dah, offa), desc_add(dbh, offb));
          }
          wgmma_commit();
          wgmma_wait<0>();
          fence_acc(part);
#pragma unroll
          for (int i = 0; i < BNW / 2; ++i) acc[grp][i] += part[i];
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&aempty[as]);
        if (++as == C::kAStages) { as = 0; aph ^= 1; }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&gempty[gs]);
      if (++gs == C::kGStages) { gs = 0; gph ^= 1; }
    }
  }
  if (t_begin >= t_end) return;
  // accumulator row m = (tap within group) * CN + ci, column = output channel
  const int quad = lane & 3;
#pragma unroll
  for (int grp = 0; grp < C::kMaxGroups; ++grp) {
    if (grp >= groups) break;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int m = wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * i;
      const int tap = grp * TG + m / CN, ci = ci0 + (m % CN);
      if (tap >= taps || ci >= g.Cin) continue;
      // gw here is the pixel-split partial buffer: slice blockIdx.x, summed over the splits in order by add_partials
      float* dst = gw + (int64_t)blockIdx.x * taps * g.Cin * g.Cout + ((int64_t)tap * g.Cin + ci) * g.Cout + co0 + 2 * quad;
#pragma unroll
      for (int j = 0; j < BNW / 8; ++j)
        *reinterpret_cast<float2*>(dst + 8 * j) = make_float2(acc[grp][4 * j + 2 * i], acc[grp][4 * j + 2 * i + 1]);
    }
  }
}

// ---- column-box weight gradient: 3x3 SAME, 16 x 8 pixel tiles inside one image.  Same grid, pixel split and partial slices
// as k_conv_wgrad_wgmma, but per tile and plane x arrives as the forward's three boxes {CN, 16, 10, 1}, one per kw, at
// (w0 + kw - 1, h0 - 1): tap (kh, kw)'s 128-pixel tile is box kw from pixel row 16 kh on.  Every x pixel crosses into shared
// memory 3 times instead of 9.
// The MN-major A operand stacks CN-channel tap slots in M at the descriptor's LBO, which must be one uniform stride: taps
// (kh, kw), (kh + 1, kw), ... are 16 pixel rows apart (whole swizzle atoms at 32, 64 and 128 B), taps (kh, kw), (kh, kw + 1)
// one box apart.  A warpgroup's units of M = 64 rows (WgUnit) are
//   CN = 16: one kw column per unit, 3 taps and a padding slot   -- warpgroup 0: kw 0, 1;  warpgroup 1: kw 2
//   CN = 32: two taps per unit                                    -- 0: (0-1, 0), (2, 0-1), (0-1, 1);  1: (0-1, 2), (2, 2) + pad
//   CN = 64: one tap per unit, in kw-major order t = 3 kw + kh    -- 0: even t;  1: odd t
// A padding slot's accumulator rows are discarded; its A rows reach at most 16 pixel rows past its box, which is still this
// CTA's shared memory (the next box, x stage or the gy ring).
// Every element gw[tap][ci][co] sees the same arithmetic as in k_conv_wgrad_wgmma -- per tile a fresh fragment of the MMAs
// ks = 0..7 x (lo.hi, hi.lo, hi.hi) on the same operand values, added to the running sum in fp32, tiles in order -- so the
// results are bit-identical to it.
// Pipeline: an x stage holds the boxes of the whole tile where two or more fit (CN <= 32), else of one kw column (CN = 64: the
// next tile's kw = 0 boxes load while kw = 2 computes); gy tiles have their own ring.  Each warpgroup issues its units as
// fully unrolled MMA sequences, one commit group per unit, and keeps one group in flight (two fragments) where registers allow;
// an x stage goes back to the producer once its units' MMAs have completed.
struct WgUnit { int kw, kh, along_kw, n; };   // taps (kh + q, kw) or, along_kw, (kh, kw + q), q < n; box kw from row 16 kh

__host__ __device__ constexpr int wg_units(int cn, int wg) {
  return cn == 16 ? (wg == 0 ? 2 : 1) : (cn == 32 ? (wg == 0 ? 3 : 2) : (wg == 0 ? 5 : 4));
}
__host__ __device__ constexpr WgUnit wg_unit(int cn, int wg, int j) {
  if (cn == 16) return WgUnit{wg == 0 ? j : 2, 0, 0, 3};
  if (cn == 32) {
    if (wg == 0) return j == 0 ? WgUnit{0, 0, 0, 2} : (j == 1 ? WgUnit{0, 2, 1, 2} : WgUnit{1, 0, 0, 2});
    return j == 0 ? WgUnit{2, 0, 0, 2} : WgUnit{2, 2, 0, 1};
  }
  return WgUnit{(2 * j + wg) / 3, (2 * j + wg) % 3, 0, 1};
}
// every tap in exactly one slot, each warpgroup's units in non-decreasing kw (the order the CN = 64 stages arrive in), and no
// slot beyond the box's 10 rows / the tile's 3 boxes other than one trailing padding slot
__host__ __device__ constexpr bool wg_units_ok(int cn) {
  int seen[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  for (int wg = 0; wg < 2; ++wg)
    for (int j = 0; j < wg_units(cn, wg); ++j) {
      const WgUnit u = wg_unit(cn, wg, j);
      if (j > 0 && u.kw < wg_unit(cn, wg, j - 1).kw) return false;
      if (u.n < 1 || u.n > 64 / cn || (u.n < 64 / cn && u.n + 1 < 64 / cn)) return false;
      for (int q = 0; q < u.n; ++q) {
        const int kh = u.kh + (u.along_kw ? 0 : q), kw = u.kw + (u.along_kw ? q : 0);
        if (kh > 2 || kw > 2) return false;
        ++seen[3 * kh + kw];
      }
    }
  for (int t = 0; t < 9; ++t)
    if (seen[t] != 1) return false;
  return true;
}
static_assert(wg_units_ok(16) && wg_units_ok(32) && wg_units_ok(64), "column-box wgrad: tap units");

// Registers: a warpgroup keeps two fragments (one commit group in flight while the previous one is added) where they fit in
// ~96 floats beside its accumulators, and at most ~96 floats of fragments and accumulators in all: the rest of the 168 go to
// descriptors and ring state (above that, ptxas spills).  Accumulators beyond the budget live in shared memory.
__host__ __device__ constexpr int wg_fragments(int cn, int bnw, int wg) { return (wg_units(cn, wg) + 2) * (bnw / 2) <= 96 ? 2 : 1; }
__host__ __device__ constexpr int wg_reg_units(int cn, int bnw, int wg) {
  return (96 / (bnw / 2) - wg_fragments(cn, bnw, wg)) < wg_units(cn, wg) ? (96 / (bnw / 2) - wg_fragments(cn, bnw, wg))
                                                                          : wg_units(cn, wg);
}

template <int CN, int BNW>
struct WgColCfg {
  static constexpr int kBox = 160 * CN * 2;                 // one {CN, 16, 10, 1} box, one plane
  static constexpr int kKws = CN == 64 ? 1 : 3;             // kw columns per x stage
  static constexpr int kXStage = 2 * kKws * kBox;           // [hi: kKws boxes][lo: kKws boxes]
  static constexpr int kGTile = 128 * BNW * 2;              // gy tile, one plane
  static constexpr int kGStage = 2 * kGTile;
  static constexpr int kGStages = 2;
  static constexpr int kXStagesRaw = (200 * 1024 - kGStages * kGStage) / kXStage;
  static constexpr int kXStages = kXStagesRaw > 4 ? 4 : kXStagesRaw;
  // accumulators in shared memory, [warpgroup 0's][warpgroup 1's], each [unit][BNW / 2][128 threads]
  static constexpr int kSmemAcc0 = wg_units(CN, 0) - wg_reg_units(CN, BNW, 0);
  static constexpr int kSmemAcc1 = wg_units(CN, 1) - wg_reg_units(CN, BNW, 1);
  static constexpr int kAccBytes = (kSmemAcc0 + kSmemAcc1) * (BNW / 2) * 128 * 4;
  static constexpr int kBytes = kXStages * kXStage + kGStages * kGStage + kAccBytes + 1024 /*align*/ + 256 /*barriers*/;
  static_assert(wg_reg_units(CN, BNW, 0) >= 1 && wg_reg_units(CN, BNW, 1) >= 1, "column-box wgrad: register budget");
  static_assert(kXStages * kKws >= 4, "column-box wgrad: the x ring must hold more than one tile's boxes");
  static_assert(kBytes <= 227 * 1024, "column-box wgrad exceeds shared memory");
};

__device__ __forceinline__ void ring_next(int& s, uint32_t& ph, int stages) {
  if (++s == stages) { s = 0; ph ^= 1; }
}

template <int R>
__device__ __forceinline__ void add_fragment(float (&acc)[R], float (&part)[R]) {
  fence_acc(part);
#pragma unroll
  for (int i = 0; i < R; ++i) { acc[i] += part[i]; part[i] = 0.f; }
  fence_acc(part);
}
// the same fp32 adds into an accumulator in shared memory (element i at sacc[128 i])
template <int R>
__device__ __forceinline__ void add_fragment_smem(float* sacc, float (&part)[R]) {
  fence_acc(part);
#pragma unroll
  for (int i = 0; i < R; ++i) { sacc[128 * i] += part[i]; part[i] = 0.f; }
  fence_acc(part);
}

// consumer warpgroup WG: its units over the CTA's tiles, then its slice of the partial gw
template <int CN, int BNW, int WG>
__device__ __forceinline__ void wgrad_cols_consumer(uint8_t* smem, uint64_t* xfull, uint64_t* xempty, uint64_t* gfull,
                                                    uint64_t* gempty, float* __restrict__ gw, const TcGeom& g, int t_begin,
                                                    int t_end, int ci0, int co0, int warp, int lane) {
  using C = WgColCfg<CN, BNW>;
  constexpr int NU = wg_units(CN, WG), NP = wg_fragments(CN, BNW, WG), NR = wg_reg_units(CN, BNW, WG);
  constexpr uint32_t la = swizzle_layout_for(CN), lb = swizzle_layout_for(BNW);
  constexpr uint32_t sbo_a = 8 * CN * 2, sbo_b = 8 * BNW * 2;   // stride between 8-pixel groups (K)
  constexpr uint32_t rows16 = 16 * CN * 2;                      // 16 pixel rows of x
  const uint8_t* sg = smem + C::kXStages * C::kXStage;
  // units NR .. NU - 1 accumulate in shared memory: this thread's element i of unit j at sacc[128 ((j - NR) BNW / 2 + i)]
  float* sacc = reinterpret_cast<float*>(smem + C::kXStages * C::kXStage + C::kGStages * C::kGStage) +
                (WG == 0 ? 0 : C::kSmemAcc0 * (BNW / 2) * 128) + (threadIdx.x & 127);
  float acc[NR][BNW / 2], part[NP][BNW / 2];
#pragma unroll
  for (int u = 0; u < NR; ++u)
#pragma unroll
    for (int i = 0; i < BNW / 2; ++i) acc[u][i] = 0.f;
#pragma unroll
  for (int i = 0; i < (NU - NR) * (BNW / 2); ++i) sacc[128 * i] = 0.f;
  // unit j's fragment goes into its accumulator, in registers or in shared memory
  const auto add_unit = [&](int j, float (&p)[BNW / 2]) {
    if (j < NR) add_fragment(acc[j < NR ? j : 0], p);
    else add_fragment_smem(sacc + 128 * (j - NR) * (BNW / 2), p);
  };
  const auto acc_at = [&](int j, int i) { return j < NR ? acc[j < NR ? j : 0][i] : sacc[128 * ((j - NR) * (BNW / 2) + i)]; };
#pragma unroll
  for (int p = 0; p < NP; ++p)
#pragma unroll
    for (int i = 0; i < BNW / 2; ++i) part[p][i] = 0.f;
  int xs = 0, gs = 0; uint32_t xph = 0, gph = 0;
  for (int t = t_begin; t < t_end; ++t) {
    mbar_wait(&gfull[gs], gph);
    const uint32_t gb_hi = smem_u32(sg + gs * C::kGStage);
    int prev_x = 0;
#pragma unroll
    for (int j = 0; j < NU; ++j) {
      const WgUnit u = wg_unit(CN, WG, j);
      const bool new_stage = j == 0 || u.kw / C::kKws != wg_unit(CN, WG, j - 1).kw / C::kKws;
      if (new_stage && j > 0) {
        if (NP == 1) { __syncwarp(); mbar_arrive_lane0(&xempty[xs], lane); }   // its MMAs completed at the last wait
        prev_x = xs;
        ring_next(xs, xph, C::kXStages);
      }
      if (new_stage) mbar_wait(&xfull[xs], xph);
      uint32_t xa_hi = smem_u32(smem + xs * C::kXStage) + (u.kw % C::kKws) * C::kBox + u.kh * rows16, gb = gb_hi;
      // per-unit descriptors: without this ptxas keeps every unit's 64-bit descriptors live over the tile and spills
      asm volatile("" : "+r"(xa_hi), "+r"(gb));
      const uint32_t lbo = u.along_kw ? (uint32_t)C::kBox : rows16;
      const uint64_t dah = make_desc(xa_hi, lbo, sbo_a, la), dal = make_desc(xa_hi + C::kKws * C::kBox, lbo, sbo_a, la);
      const uint64_t dbh = make_desc(gb, C::kGTile, sbo_b, lb), dbl = make_desc(gb + C::kGTile, C::kGTile, sbo_b, lb);
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 128 / 16; ++ks) {          // 16 pixels per MMA
        const uint32_t offa = ks * 2 * sbo_a, offb = ks * 2 * sbo_b;
        Wgmma<BNW>::template mma<1, 1>(part[j % NP], desc_add(dal, offa), desc_add(dbh, offb));
        Wgmma<BNW>::template mma<1, 1>(part[j % NP], desc_add(dah, offa), desc_add(dbl, offb));
        Wgmma<BNW>::template mma<1, 1>(part[j % NP], desc_add(dah, offa), desc_add(dbh, offb));
      }
      wgmma_commit();
      if (NP == 2) {
        wgmma_wait<1>();                                // unit j - 1 has completed
        if (j > 0) {
          add_unit(j - 1, part[(j - 1) % NP]);
          if (new_stage) { __syncwarp(); mbar_arrive_lane0(&xempty[prev_x], lane); }
        }
      } else {
        wgmma_wait<0>();
        add_unit(j, part[0]);
      }
    }
    if (NP == 2) {
      wgmma_wait<0>();
      add_unit(NU - 1, part[(NU - 1) % NP]);
    }
    __syncwarp();
    mbar_arrive_lane0(&xempty[xs], lane);
    ring_next(xs, xph, C::kXStages);
    mbar_arrive_lane0(&gempty[gs], lane);
    ring_next(gs, gph, C::kGStages);
  }
  if (t_begin >= t_end) return;
  // accumulator row m of unit u = slot m / CN (a tap or padding), input channel m % CN; column = output channel
  const int quad = lane & 3;
#pragma unroll
  for (int j = 0; j < NU; ++j) {
    const WgUnit u = wg_unit(CN, WG, j);
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int m = (warp & 3) * 16 + (lane >> 2) + 8 * i;
      const int q = m / CN, ci = ci0 + m % CN;
      if (q >= u.n) continue;
      const int tap = 3 * (u.kh + (u.along_kw ? 0 : q)) + u.kw + (u.along_kw ? q : 0);
      // the pixel-split partial buffer: slice blockIdx.x, summed over the splits in order by add_partials
      float* dst = gw + (int64_t)blockIdx.x * 9 * g.Cin * g.Cout + ((int64_t)tap * g.Cin + ci) * g.Cout + co0 + 2 * quad;
#pragma unroll
      for (int k = 0; k < BNW / 8; ++k)
        *reinterpret_cast<float2*>(dst + 8 * k) = make_float2(acc_at(j, 4 * k + 2 * i), acc_at(j, 4 * k + 2 * i + 1));
    }
  }
}

template <int CN, int BNW>
__global__ void __launch_bounds__(kThreads, 1) k_conv_wgrad_cols_wgmma(const __grid_constant__ CUtensorMap tm_g_hi,
                                                                       const __grid_constant__ CUtensorMap tm_g_lo,
                                                                       const __grid_constant__ CUtensorMap tm_x_hi,
                                                                       const __grid_constant__ CUtensorMap tm_x_lo,
                                                                       float* __restrict__ gw, TcGeom g, int tiles_per_cta) {
  using C = WgColCfg<CN, BNW>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  // x ring, gy ring [hi][lo], accumulators in shared memory, barriers
  uint8_t* sg = smem + C::kXStages * C::kXStage;
  uint64_t* xfull = reinterpret_cast<uint64_t*>(sg + C::kGStages * C::kGStage + C::kAccBytes);   // [kXStages]
  uint64_t* xempty = xfull + C::kXStages;                                         // [kXStages]
  uint64_t* gfull = xempty + C::kXStages;                                         // [kGStages]
  uint64_t* gempty = gfull + C::kGStages;                                         // [kGStages]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int co0 = blockIdx.y * BNW;
  const int ci0 = blockIdx.z * CN;
  const int total_tiles = g.tiles_w * g.tiles_h * g.tiles_n;
  const int t_begin = blockIdx.x * tiles_per_cta;
  const int t_end = min(total_tiles, t_begin + tiles_per_cta);

  if (warp == kConsumerWarps && lane == 0) {
    prefetch_tmap(&tm_g_hi); prefetch_tmap(&tm_g_lo); prefetch_tmap(&tm_x_hi); prefetch_tmap(&tm_x_lo);
    for (int s = 0; s < C::kXStages; ++s) { mbar_init(&xfull[s], 1); mbar_init(&xempty[s], kConsumerWarps); }
    for (int s = 0; s < C::kGStages; ++s) { mbar_init(&gfull[s], 1); mbar_init(&gempty[s], kConsumerWarps); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == kConsumerWarps) {
    if (lane == 0) {
      int xs = 0, gs = 0; uint32_t xph = 0, gph = 0;
      for (int t = t_begin; t < t_end; ++t) {
        const int tw_i = t % g.tiles_w, th_i = (t / g.tiles_w) % g.tiles_h, n0 = t / (g.tiles_w * g.tiles_h);
        const int w0 = tw_i * 16, h0 = th_i * 8;
        mbar_wait(&gempty[gs], gph ^ 1);
        mbar_expect_tx(&gfull[gs], C::kGStage);
        tma_load_4d(&tm_g_hi, &gfull[gs], sg + gs * C::kGStage, co0, w0, h0, n0);
        tma_load_4d(&tm_g_lo, &gfull[gs], sg + gs * C::kGStage + C::kGTile, co0, w0, h0, n0);
        ring_next(gs, gph, C::kGStages);
        for (int kw0 = 0; kw0 < 3; kw0 += C::kKws) {
          mbar_wait(&xempty[xs], xph ^ 1);
          mbar_expect_tx(&xfull[xs], C::kXStage);
          uint8_t* sx = smem + xs * C::kXStage;
          for (int b = 0; b < C::kKws; ++b) {
            const int kw = kw0 + b;
            tma_load_4d(&tm_x_hi, &xfull[xs], sx + b * C::kBox, ci0, w0 + kw - 1, h0 - 1, n0);
            tma_load_4d(&tm_x_lo, &xfull[xs], sx + (C::kKws + b) * C::kBox, ci0, w0 + kw - 1, h0 - 1, n0);
          }
          ring_next(xs, xph, C::kXStages);
        }
      }
    }
    return;
  }
  if (warp < 4)
    wgrad_cols_consumer<CN, BNW, 0>(smem, xfull, xempty, gfull, gempty, gw, g, t_begin, t_end, ci0, co0, warp, lane);
  else
    wgrad_cols_consumer<CN, BNW, 1>(smem, xfull, xempty, gfull, gempty, gw, g, t_begin, t_end, ci0, co0, warp, lane);
}

// ----------------------------------------------------------------------------------------------------
// host side
// ----------------------------------------------------------------------------------------------------
typedef CUresult (*PFN_tmapEncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                        const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                        CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_tmapEncodeTiled get_encode() {
  static PFN_tmapEncodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_tmapEncodeTiled>(p);
  }
  return fn;
}

static CUtensorMapSwizzle swz_for(int cc) {
  return cc == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : (cc == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
}

// NHWC bf16 activation plane: dims {C, W, H, N}, box {cc, TW, TH, TN}
static int make_act_map(CUtensorMap* tm, const void* base, int N, int H, int W, int C, int cc, int TW, int TH, int TN) {
  PFN_tmapEncodeTiled enc = get_encode();
  if (!enc) return fail(TWG_ERR_CUDA, "cuTensorMapEncodeTiled unavailable");
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
  cuuint32_t box[4] = {(cuuint32_t)cc, (cuuint32_t)TW, (cuuint32_t)TH, (cuuint32_t)TN};
  cuuint32_t es[4] = {1, 1, 1, 1};
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), dims, strides, box, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, swz_for(cc), CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(TWG_ERR_CUDA, "cuTensorMapEncodeTiled(act) failed: %d", (int)r);
  return TWG_OK;
}

// weight plane [rows][K] bf16 (K contiguous): dims {K, rows}, box {cc, bn}
static int make_w_map(CUtensorMap* tm, const void* base, int rows, int K, int cc, int bn) {
  PFN_tmapEncodeTiled enc = get_encode();
  if (!enc) return fail(TWG_ERR_CUDA, "cuTensorMapEncodeTiled unavailable");
  cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)K * 2};
  cuuint32_t box[2] = {(cuuint32_t)cc, (cuuint32_t)bn};
  cuuint32_t es[2] = {1, 1};
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, swz_for(cc), CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(TWG_ERR_CUDA, "cuTensorMapEncodeTiled(w) failed: %d", (int)r);
  return TWG_OK;
}

// Shapes whose forward epilogue also offers the instance-norm statistics, the activation sign mask and the evaluation-mode
// affine: the small-channel high-resolution layers (one output-channel block, 16 x 8 pixel tiles inside one image).
// They never split K, so every epilogue variant computes bit-identical outputs.
static bool epi_shape_ok(int H, int W, int K, int Nc, int k, int pad) {
  auto small = [](int c) { return c == 16 || c == 32 || c == 64; };
  return k == 3 && pad == 1 && small(K) && small(Nc) && K * Nc <= 2048 && H >= 16 && W >= 16;
}

static int pow2_le(int v) {
  int p = 1;
  while (p * 2 <= v) p *= 2;
  return p;
}

static bool pick_tile(TcGeom& g) {
  g.TW = pow2_le(g.W < 16 ? g.W : 16);
  int th_cap = 128 / g.TW;
  g.TH = pow2_le(g.H < th_cap ? g.H : th_cap);
  g.TN = 128 / (g.TW * g.TH);
  if (g.TN > 256) return false;
  g.tiles_w = (int)cdiv(g.W, g.TW);
  g.tiles_h = (int)cdiv(g.H, g.TH);
  g.tiles_n = (int)cdiv(g.N, g.TN);
  return true;
}

static int chunk_for(int c) { return (c % 64 == 0) ? 64 : ((c % 32 == 0) ? 32 : ((c % 16 == 0) ? 16 : 0)); }

static bool tc_shape_ok(int N, int H, int W, int Cin, int Cout, int k, int pad) {
  if (!((k == 3 && pad == 1) || (k == 1 && pad == 0))) return false;
  // channel counts of the PGGAN schedule: 16, 32, 64 or a multiple of 128 (tile/box shapes are built for these)
  auto ok = [](int c) { return c == 16 || c == 32 || c == 64 || (c >= 128 && c % 128 == 0); };
  if (!ok(Cin) || !ok(Cout)) return false;
  (void)N; (void)H; (void)W;
  return true;
}

template <int CC, int BN>
static int launch_fwd(const CUtensorMap& ah, const CUtensorMap& al, const CUtensorMap& bh, const CUtensorMap& bl, float* y,
                      const TcGeom& g, const float* bias, int act, void* z_planes, float4* stats, uint8_t* act_mask,
                      const float* aff_a, cudaStream_t st) {
  using SM = FwdSmem<CC, BN>;
  auto kern = k_conv_fwd_wgmma<CC, BN>;
  static std::once_flag once;                 // one-time attribute set-up, safe from several host threads
  static cudaError_t attr_err = cudaSuccess;
  std::call_once(once, [&] { attr_err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SM::kBytes); });
  if (attr_err != cudaSuccess) return fail(TWG_ERR_CUDA, "cudaFuncSetAttribute: %s", cudaGetErrorString(attr_err));
  const int tiles = g.tiles_w * g.tiles_h * g.tiles_n, nblk = g.Cout / BN;
  dim3 grid((unsigned)tiles, (unsigned)nblk);
  kern<<<grid, kThreads, SM::kBytes, st>>>(ah, al, bh, bl, y, g, bias, act, z_planes, stats, act_mask, aff_a);
  return check_launch("twg_conv tc");
}

// ah / al: activation maps with the column box {CC, 16, 10, 1}
template <int CC, int BN>
static int launch_fwd_cols(const CUtensorMap& ah, const CUtensorMap& al, const CUtensorMap& bh, const CUtensorMap& bl,
                           float* y, const TcGeom& g, const float* bias, int act, void* z_planes, float4* stats,
                           uint8_t* act_mask, const float* aff_a, cudaStream_t st) {
  constexpr int kBytes = col_smem_bytes<CC, BN>();
  // the resident-weight kernel holds one output-channel block, at weight rows tap * BN
  if (cols_resident(CC, BN) && g.Cout != BN) return fail(TWG_ERR_UNSUPPORTED, "tensor-core conv: column-box Cout != BN");
  auto kern = k_conv_fwd_cols_wgmma<CC, BN>;
  static std::once_flag once;                 // one-time attribute set-up, safe from several host threads
  static cudaError_t attr_err = cudaSuccess;
  static int per_sm = 1;
  std::call_once(once, [&] {
    attr_err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kBytes);
    if (attr_err == cudaSuccess)
      attr_err = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kThreads, kBytes);
    if (per_sm < 1) per_sm = 1;
  });
  if (attr_err != cudaSuccess) return fail(TWG_ERR_CUDA, "cudaFuncSetAttribute: %s", cudaGetErrorString(attr_err));
  const int64_t work = (int64_t)g.tiles_w * g.tiles_h * g.tiles_n * (g.Cout / BN);
  const int64_t ctas = work < (int64_t)kNumSMs * per_sm ? work : (int64_t)kNumSMs * per_sm;
  kern<<<(unsigned)ctas, kThreads, kBytes, st>>>(ah, al, bh, bl, y, g, bias, act, z_planes, stats, act_mask, aff_a);
  return check_launch("twg_conv tc cols");
}

static unsigned split_blocks(int64_t n4) {
  int64_t blocks = cdiv(n4, 256 * 4);
  if (blocks > kNumSMs * 16) blocks = kNumSMs * 16;
  if (blocks < 1) blocks = 1;
  return (unsigned)blocks;
}

int split_act_planes(const float* x, void* planes, int64_t n, cudaStream_t st) {
  if (n % 4) return fail(TWG_ERR_INVALID, "twg_split_act: element count must be a multiple of 4");
  k_split_act<<<split_blocks(n / 4), 256, 0, st>>>(x, planes, n / 4);
  return check_launch("twg_split_act");
}

int split_weight_planes(const float* w, void* planes, int k, int Cin, int Cout, int dgrad, cudaStream_t st) {
  const SplitRow r{0, 0, k * k, Cin, Cout, dgrad ? 1 : 0};
  k_split_weights<<<(unsigned)cdiv((int64_t)r.taps * Cin * Cout, 256), 256, 0, st>>>(
      w, reinterpret_cast<__nv_bfloat16*>(planes), r);
  return check_launch("twg_split_weights");
}

int split_weight_table(const float* flat, void* planes, const void* table, int rows, int64_t max_elems, cudaStream_t st) {
  int64_t bx = cdiv(max_elems, 256 * 4);
  if (bx > 64) bx = 64;
  if (bx < 1) bx = 1;
  dim3 grid((unsigned)bx, (unsigned)rows);
  k_split_weights_table<<<grid, 256, 0, st>>>(flat, reinterpret_cast<__nv_bfloat16*>(planes),
                                              reinterpret_cast<const SplitRow*>(table));
  return check_launch("twg_split_weights_table");
}

bool conv_tc_supported(int N, int H, int W, int Cin, int Cout, int k, int pad) {
  if (!tc_shape_ok(N, H, W, Cin, Cout, k, pad)) return false;
  TcGeom g{};
  g.N = N; g.H = H; g.W = W;
  return pick_tile(g);
}

// Records per image the forward kernel writes when asked for epilogue statistics: one {count, pivot, S1, S2} per
// (16 x 8 tile, consumer warp, channel).  0: the shape has no fused epilogue (no statistics, sign mask or affine).
int conv_fwd_epilogue_slots(int N, int H, int W, int Cin, int Cout, int k, int pad) {
  if (!tc_shape_ok(N, H, W, Cin, Cout, k, pad) || !epi_shape_ok(H, W, Cin, Cout, k, pad)) return 0;
  return (int)(cdiv(H, 8) * cdiv(W, 16) * kConsumerWarps);
}

// core: activation planes [2][N,H,W,Kc] (Kc = Cin for forward, Cout for dgrad), weight planes from split_weight_planes
int conv_fwd_tc_planes(const void* a_planes, const void* w_planes, float* y, int N, int H, int W, int Cin, int Cout,
                       int k, int pad, bool dgrad, cudaStream_t st, const float* bias = nullptr, int act = 0,
                       void* z_planes = nullptr, float4* stats = nullptr, uint8_t* act_mask = nullptr,
                       const float* aff_a = nullptr) {
  if (!tc_shape_ok(N, H, W, Cin, Cout, k, pad)) return fail(TWG_ERR_UNSUPPORTED, "tensor-core conv: shape not covered");
  const bool fused = conv_fwd_epilogue_slots(N, H, W, Cin, Cout, k, pad) > 0;
  if (aff_a && (dgrad || !bias || stats || act_mask || !fused))
    return fail(TWG_ERR_UNSUPPORTED, "tensor-core conv: no affine epilogue for this call");
  if (!y && !(aff_a && z_planes)) return fail(TWG_ERR_INVALID, "tensor-core conv: null output");
  if (act_mask && (dgrad || !bias || !act || !fused))
    return fail(TWG_ERR_UNSUPPORTED, "tensor-core conv: no activation mask for this call");
  if (stats && (dgrad || bias || z_planes || !fused))
    return fail(TWG_ERR_UNSUPPORTED, "tensor-core conv: no epilogue statistics for this call");
  TcGeom g{};
  g.N = N; g.H = H; g.W = W; g.k = k; g.pad = pad;
  g.Cin = dgrad ? Cout : Cin;     // GEMM K channels
  g.Cout = dgrad ? Cin : Cout;    // GEMM N channels
  if (!pick_tile(g)) return fail(TWG_ERR_UNSUPPORTED, "tensor-core conv: tile");
  const int64_t px = (int64_t)N * H * W;
  const int taps = k * k;
  const __nv_bfloat16* a_hi = reinterpret_cast<const __nv_bfloat16*>(a_planes);
  const __nv_bfloat16* a_lo = a_hi + px * g.Cin;
  const __nv_bfloat16* w_hi = reinterpret_cast<const __nv_bfloat16*>(w_planes);
  const __nv_bfloat16* w_lo = w_hi + (int64_t)taps * Cin * Cout;
  const int CC = chunk_for(g.Cin);
  // No split-K: its fp32 atomics would add the partial tiles in a different order on every run.  The tile shape depends on
  // the layer only, never on the batch, so a sample's output is the same whichever batch it is computed in.
  const int BN = g.Cout >= 128 ? 128 : g.Cout;
  // 3x3 SAME convs with one channel chunk on 16 x 8 tiles take the column-box kernel (same results, a third of the A traffic)
  const bool cols = k == 3 && pad == 1 && g.Cin == CC && g.TW == 16 && g.TH == 8 && g.TN == 1 && H >= 10;
  CUtensorMap ah, al, bh, bl;
  int rc;
  if ((rc = make_act_map(&ah, a_hi, N, H, W, g.Cin, CC, g.TW, cols ? 10 : g.TH, g.TN))) return rc;
  if ((rc = make_act_map(&al, a_lo, N, H, W, g.Cin, CC, g.TW, cols ? 10 : g.TH, g.TN))) return rc;
  if ((rc = make_w_map(&bh, w_hi, taps * g.Cout, g.Cin, CC, BN))) return rc;
  if ((rc = make_w_map(&bl, w_lo, taps * g.Cout, g.Cin, CC, BN))) return rc;
#define TWG_COLS_CASE(cc, bn) \
  if (CC == cc && BN == bn)   \
    return launch_fwd_cols<cc, bn>(ah, al, bh, bl, y, g, bias, act, z_planes, stats, act_mask, aff_a, st);
  if (cols) {
    TWG_COLS_CASE(16, 16) TWG_COLS_CASE(16, 32) TWG_COLS_CASE(16, 64) TWG_COLS_CASE(16, 128)
    TWG_COLS_CASE(32, 16) TWG_COLS_CASE(32, 32) TWG_COLS_CASE(32, 64) TWG_COLS_CASE(32, 128)
    TWG_COLS_CASE(64, 16) TWG_COLS_CASE(64, 32) TWG_COLS_CASE(64, 64) TWG_COLS_CASE(64, 128)
    return fail(TWG_ERR_UNSUPPORTED, "tensor-core conv: no column-box kernel for CC=%d BN=%d", CC, BN);
  }
#undef TWG_COLS_CASE
#define TWG_FWD_CASE(cc, bn) \
  if (CC == cc && BN == bn)  \
    return launch_fwd<cc, bn>(ah, al, bh, bl, y, g, bias, act, z_planes, stats, act_mask, aff_a, st);
  TWG_FWD_CASE(16, 16) TWG_FWD_CASE(16, 32) TWG_FWD_CASE(16, 64) TWG_FWD_CASE(16, 128)
  TWG_FWD_CASE(32, 16) TWG_FWD_CASE(32, 32) TWG_FWD_CASE(32, 64) TWG_FWD_CASE(32, 128)
  TWG_FWD_CASE(64, 16) TWG_FWD_CASE(64, 32) TWG_FWD_CASE(64, 64) TWG_FWD_CASE(64, 128)
#undef TWG_FWD_CASE
  return fail(TWG_ERR_UNSUPPORTED, "tensor-core conv: no kernel for CC=%d BN=%d", CC, BN);
}

// kCols: the column-box kernel (xh / xl with the box {CN, 16, 10, 1}); both kernels take the same grid and pixel split
template <int CN, int BNW, bool kCols>
static int launch_wgrad(const CUtensorMap& gh, const CUtensorMap& gl, const CUtensorMap& xh, const CUtensorMap& xl,
                        float* gw, const TcGeom& g, cudaStream_t st) {
  constexpr int kBytes = kCols ? WgColCfg<CN, BNW>::kBytes : WgCfg<CN, BNW>::kBytes;
  auto kern = kCols ? k_conv_wgrad_cols_wgmma<CN, BNW> : k_conv_wgrad_wgmma<CN, BNW>;
  static std::once_flag once;                 // one-time attribute set-up, safe from several host threads
  static cudaError_t attr_err = cudaSuccess;
  std::call_once(once, [&] { attr_err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kBytes); });
  if (attr_err != cudaSuccess) return fail(TWG_ERR_CUDA, "cudaFuncSetAttribute: %s", cudaGetErrorString(attr_err));
  const int total_tiles = g.tiles_w * g.tiles_h * g.tiles_n;
  const int yb = g.Cout / BNW, zb = g.Cin / CN;
  // one CTA per SM (~200 KB of stages): the grid must fit in one wave, or the channel-block-heavy layers run two
  int64_t want = kNumSMs / ((int64_t)yb * zb);
  if (want > total_tiles) want = total_tiles;
  if (want < 1) want = 1;
  const int tiles_per_cta = (int)cdiv(total_tiles, want);
  const int xb = (int)cdiv(total_tiles, tiles_per_cta);
  dim3 grid((unsigned)xb, (unsigned)yb, (unsigned)zb);
  const int64_t gw_elems = (int64_t)g.k * g.k * g.Cin * g.Cout;
  float* parts = partials(xb * gw_elems, true, st);
  if (!parts) return fail(TWG_ERR_UNSUPPORTED, "tensor-core wgrad: weight too large for the split buffer");
  kern<<<grid, kThreads, kBytes, st>>>(gh, gl, xh, xl, parts, g, tiles_per_cta);
  if (int rc = check_launch(kCols ? "twg_conv_wgrad tc cols" : "twg_conv_wgrad tc")) return rc;
  return add_partials(gw, parts, xb, gw_elems, st);
}

// The weight gradient always forms all three split-bf16 partial products: although gw sums over 10^4..10^6 pixels, the
// real gradients of this step have too little signal above the rounding residue to drop x_lo.gy.
int conv_wgrad_tc_planes(const void* x_planes, const void* g_planes, float* gw, int N, int H, int W, int Cin, int Cout,
                         int k, int pad, int accumulate, cudaStream_t st) {
  if (!tc_shape_ok(N, H, W, Cin, Cout, k, pad)) return fail(TWG_ERR_UNSUPPORTED, "tensor-core wgrad: shape not covered");
  TcGeom g{};
  g.N = N; g.H = H; g.W = W; g.k = k; g.pad = pad; g.Cin = Cin; g.Cout = Cout;
  if (!pick_tile(g)) return fail(TWG_ERR_UNSUPPORTED, "tensor-core wgrad: tile");
  const int64_t px = (int64_t)N * H * W;
  const __nv_bfloat16* x_hi = reinterpret_cast<const __nv_bfloat16*>(x_planes);
  const __nv_bfloat16* x_lo = x_hi + px * Cin;
  const __nv_bfloat16* g_hi = reinterpret_cast<const __nv_bfloat16*>(g_planes);
  const __nv_bfloat16* g_lo = g_hi + px * Cout;
  if (!accumulate) cudaMemsetAsync(gw, 0, sizeof(float) * k * k * Cin * Cout, st);
  const int CN = chunk_for(Cin);                      // channels per tap in the stacked A operand
  // output-channel block (N of the MMA): 64 channels, 32 for 64-channel chunks, whose five tap groups of accumulators
  // would not fit in registers at 64
  const int BNW = (Cout >= 64 && CN < 64) ? 64 : (Cout >= 32 ? 32 : Cout);
  // 3x3 SAME on 16 x 8 tiles inside one image takes the column-box kernel (same results, a third of the x traffic)
  const bool cols = k == 3 && pad == 1 && g.TW == 16 && g.TH == 8 && g.TN == 1 && H >= 10;
  CUtensorMap gh, gl, xh, xl;
  int rc;
  if ((rc = make_act_map(&gh, g_hi, N, H, W, Cout, BNW, g.TW, g.TH, g.TN))) return rc;
  if ((rc = make_act_map(&gl, g_lo, N, H, W, Cout, BNW, g.TW, g.TH, g.TN))) return rc;
  if ((rc = make_act_map(&xh, x_hi, N, H, W, Cin, CN, g.TW, cols ? 10 : g.TH, g.TN))) return rc;
  if ((rc = make_act_map(&xl, x_lo, N, H, W, Cin, CN, g.TW, cols ? 10 : g.TH, g.TN))) return rc;
#define TWG_WG_CASE(cn, bn)                                                                     \
  if (CN == cn && BNW == bn)                                                                    \
    return cols ? launch_wgrad<cn, bn, true>(gh, gl, xh, xl, gw, g, st)                         \
                : launch_wgrad<cn, bn, false>(gh, gl, xh, xl, gw, g, st);
  TWG_WG_CASE(16, 16) TWG_WG_CASE(16, 32) TWG_WG_CASE(16, 64)
  TWG_WG_CASE(32, 16) TWG_WG_CASE(32, 32) TWG_WG_CASE(32, 64)
  TWG_WG_CASE(64, 16) TWG_WG_CASE(64, 32)
#undef TWG_WG_CASE
  return fail(TWG_ERR_UNSUPPORTED, "tensor-core wgrad: no kernel for CN=%d BNW=%d", CN, BNW);
}

}  // namespace twg
