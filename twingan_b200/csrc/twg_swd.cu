// Sliced Wasserstein distance of PGGAN (Karras et al., ICLR 2018, section 5 and appendix D): Laplacian pyramid, 7x7
// neighbourhood descriptors, per-channel normalisation, projection onto random unit directions, a sort of every
// projection column and the mean absolute difference of the sorted columns.  An evaluation, not part of the step.
//
// Reproducibility: every cross-block sum goes through g_swd_parts in block order (no atomics on floating-point values;
// the sort counts with integer shared-memory atomics, whose result does not depend on their order), so two evaluations of
// the same inputs give bit-identical results.  Finite inputs are a precondition: with a NaN or an infinity the statistics,
// the sort order and the distance are undefined.
#include "twg_common.cuh"

namespace twg {

constexpr int kSwdParts = 8192;          // fp64 partial sums of the statistics (6 per block) and of the L1 (1 per block)
constexpr int kSwdMaxBlocks = 1024;
__device__ double g_swd_parts[kSwdParts];

static double* swd_parts() {
  void* p = nullptr;
  if (cudaGetSymbolAddress(&p, g_swd_parts) != cudaSuccess) return nullptr;
  return static_cast<double*>(p);
}

static int reduce_blocks(int64_t n) {
  int64_t b = cdiv(n, 256 * 16);
  if (b > kSwdMaxBlocks) b = kSwdMaxBlocks;
  return b < 1 ? 1 : (int)b;
}

// fixed-order block sum of a double over 256 threads; valid in thread 0
__device__ __forceinline__ double block_sum_f64(double v, double* sm) {
  __syncthreads();
  sm[threadIdx.x] = v;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) sm[threadIdx.x] += sm[threadIdx.x + s];
    __syncthreads();
  }
  return sm[0];
}

// ---- Laplacian pyramid ------------------------------------------------------------------------------------------------
// g = [1,4,6,4,1]^T [1,4,6,4,1] / 256 with mirror borders (reflection about the edge pixel's centre, d c b | a b c d | c b a:
// scipy.ndimage.convolve(mode='mirror'), cv2.pyrDown / pyrUp).  The integer taps are exact in fp32; the 1/256 and 1/64
// scales are powers of two.
__device__ __forceinline__ int mirror(int i, int n) {
  i = i < 0 ? -i : i;
  return i >= n ? 2 * (n - 1) - i : i;
}
__device__ __forceinline__ float tap5(int i) { return i == 2 ? 6.f : (i & 1) ? 4.f : 1.f; }

// dst[N, Rs/2, Rs/2, 3] = conv(src, g)[::2, ::2]
__global__ void __launch_bounds__(256) k_pyr_down(const float* __restrict__ src, float* __restrict__ dst, int N, int Rs) {
  const int Rd = Rs >> 1;
  const int64_t total = (int64_t)N * Rd * Rd;
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < total; p += (int64_t)gridDim.x * blockDim.x) {
    const int x = (int)(p % Rd), y = (int)((p / Rd) % Rd);
    const int64_t n = p / ((int64_t)Rd * Rd);
    float acc[3] = {0.f, 0.f, 0.f};
    for (int dy = 0; dy < 5; ++dy) {
      const int sy = mirror(2 * y + dy - 2, Rs);
      const float* row = src + (n * Rs + sy) * Rs * 3;
      float r[3] = {0.f, 0.f, 0.f};
#pragma unroll
      for (int dx = 0; dx < 5; ++dx) {
        const float* q = row + mirror(2 * x + dx - 2, Rs) * 3;
#pragma unroll
        for (int c = 0; c < 3; ++c) r[c] = fmaf(tap5(dx), q[c], r[c]);
      }
#pragma unroll
      for (int c = 0; c < 3; ++c) acc[c] = fmaf(tap5(dy), r[c], acc[c]);
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) dst[p * 3 + c] = acc[c] * (1.f / 256.f);
  }
}

// out[N, Rf, Rf, 3] = fine - pyr_up(coarse): pyr_up inserts zeros (values at the even indices) and convolves with 4 g.
// `out` may be `fine` (each element is read and written by the same thread).
__global__ void __launch_bounds__(256) k_pyr_up_sub(const float* fine, const float* __restrict__ coarse, float* out, int N,
                                                    int Rf) {
  const int Rc = Rf >> 1;
  const int64_t total = (int64_t)N * Rf * Rf;
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < total; p += (int64_t)gridDim.x * blockDim.x) {
    const int x = (int)(p % Rf), y = (int)((p / Rf) % Rf);
    const int64_t n = p / ((int64_t)Rf * Rf);
    float acc[3] = {0.f, 0.f, 0.f};
    for (int dy = 0; dy < 5; ++dy) {
      const int sy = mirror(y + dy - 2, Rf);
      if (sy & 1) continue;
      const float* row = coarse + (n * Rc + (sy >> 1)) * Rc * 3;
      float r[3] = {0.f, 0.f, 0.f};
#pragma unroll
      for (int dx = 0; dx < 5; ++dx) {
        const int sx = mirror(x + dx - 2, Rf);
        if (sx & 1) continue;
#pragma unroll
        for (int c = 0; c < 3; ++c) r[c] = fmaf(tap5(dx), row[(sx >> 1) * 3 + c], r[c]);
      }
#pragma unroll
      for (int c = 0; c < 3; ++c) acc[c] = fmaf(tap5(dy), r[c], acc[c]);
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) out[p * 3 + c] = fine[p * 3 + c] - acc[c] * (1.f / 64.f);
  }
}

// ---- descriptors --------------------------------------------------------------------------------------------------
// desc[(n*nhoods + k)][c*s*s + dy*s + dx] = level[n][cy - h + dy][cx - h + dx][c], h = s/2: the NCHW component order of
// PGGAN's descriptors, gathered from the NHWC level.  Centres outside [h, Rl - 1 - h] are clamped into it.
__global__ void __launch_bounds__(256) k_swd_gather(const float* __restrict__ level, const int* __restrict__ centres,
                                                    float* __restrict__ desc, int64_t rows, int nhoods, int Rl, int s) {
  const int ss = s * s, D = 3 * ss, h = s >> 1;
  const int64_t total = rows * D;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = e / D;
    const int k = (int)(e - row * D);
    const int c = k / ss, r = k - c * ss, dy = r / s, dx = r - dy * s;
    const int cy = min(max(centres[2 * row], h), Rl - 1 - h), cx = min(max(centres[2 * row + 1], h), Rl - 1 - h);
    const int64_t n = row / nhoods;
    desc[e] = level[((n * Rl + cy - h + dy) * Rl + cx - h + dx) * 3 + c];
  }
}

// ---- per-channel statistics (PGGAN finalize_descriptors): fp64 sums per block, combined in block order -----------------
__global__ void __launch_bounds__(256) k_swd_stats_part(const float* __restrict__ desc, double* __restrict__ parts,
                                                        int64_t total, int D, int ss) {
  __shared__ double sm[256];
  double s[3] = {0., 0., 0.}, q[3] = {0., 0., 0.};
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(e % D) / ss;
    const double v = desc[e];
    // c is 0, 1 or 2: selects without a local-memory index
    s[0] += c == 0 ? v : 0.; s[1] += c == 1 ? v : 0.; s[2] += c == 2 ? v : 0.;
    q[0] += c == 0 ? v * v : 0.; q[1] += c == 1 ? v * v : 0.; q[2] += c == 2 ? v * v : 0.;
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const double a = block_sum_f64(s[c], sm);
    const double b = block_sum_f64(q[c], sm);
    if (threadIdx.x == 0) {
      parts[blockIdx.x * 6 + c] = a;
      parts[blockIdx.x * 6 + 3 + c] = b;
    }
  }
}

// stats = {mean[3], rstd[3]}: population (ddof 0) std over rows x s*s values per channel; rstd = 0 where the std is 0
__global__ void k_swd_stats_final(const double* __restrict__ parts, int nb, double count, float* __restrict__ stats) {
  const int c = threadIdx.x;
  if (c >= 3) return;
  double s = 0., q = 0.;
  for (int b = 0; b < nb; ++b) {
    s += parts[b * 6 + c];
    q += parts[b * 6 + 3 + c];
  }
  const double mean = s / count;
  const double var = fmax(q / count - mean * mean, 0.);
  const double sd = sqrt(var);
  stats[c] = (float)mean;
  stats[3 + c] = sd > 0. ? (float)(1. / sd) : 0.f;
}

// ---- projection: proj[j][i] = sum_k ((desc[i][k] - mean[c(k)]) * rstd[c(k)]) * dirs[k][j] -----------------------------
// Exact fp32 FMA on the CUDA cores, k ascending in one accumulator.  Chosen over split-bf16 tensor cores because the
// sort of the same columns bounds the evaluation: at 8192 images of 256^2 (2.4 TFLOP of projections with the floor) this
// kernel took 135 ms against 485 ms of sorting (tools/swd_bench.py, H100 80GB HBM3 at a 400 W power limit), so three bf16
// MMAs per product would buy little and give up the exactness of fp32.
// 128 x 128 output tile per 256-thread block, 8 x 8 per thread (rows tx + 16 i, columns ty + 16 j: a warp stores 16
// consecutive rows of two columns of the column-major output).
constexpr int PM = 128, PN = 128, PK = 16;
__global__ void __launch_bounds__(256) k_swd_project(const float* __restrict__ A, const float* __restrict__ stats,
                                                     const float* __restrict__ B, float* __restrict__ out, int64_t M,
                                                     int K, int ss, int ndirs) {
  __shared__ float As[PK][PM + 1];
  __shared__ float Bs[PK][PN];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int64_t m0 = (int64_t)blockIdx.x * PM;
  const int n0 = blockIdx.y * PN;
  const float mean[3] = {stats[0], stats[1], stats[2]}, rstd[3] = {stats[3], stats[4], stats[5]};
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
  for (int k0 = 0; k0 < K; k0 += PK) {
#pragma unroll
    for (int q = 0; q < PM * PK / 256; ++q) {
      const int e = tid + 256 * q, r = e >> 4, kk = e & 15, k = k0 + kk;
      const int64_t m = m0 + r;
      float v = 0.f;
      if (m < M && k < K) {
        const int c = k / ss;
        v = (A[m * K + k] - (c == 0 ? mean[0] : c == 1 ? mean[1] : mean[2])) *
            (c == 0 ? rstd[0] : c == 1 ? rstd[1] : rstd[2]);
      }
      As[kk][r] = v;
    }
#pragma unroll
    for (int q = 0; q < PN * PK / 256; ++q) {
      const int e = tid + 256 * q, kk = e >> 7, j = e & 127, k = k0 + kk;
      Bs[kk][j] = k < K ? B[(int64_t)k * ndirs + n0 + j] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < PK; ++kk) {
      float a[8], b[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) a[i] = As[kk][tx + 16 * i];
#pragma unroll
      for (int j = 0; j < 8; ++j) b[j] = Bs[kk][ty + 16 * j];
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    float* col = out + (int64_t)(n0 + ty + 16 * j) * M;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int64_t m = m0 + tx + 16 * i;
      if (m < M) col[m] = acc[i][j];
    }
  }
}

// ---- segmented LSD radix sort of fp32 keys: 4 passes of 8 bits over order-preserving uint32 keys ----------------------
// Per pass: k_sort_hist counts each tile's digits, k_sort_scan turns the counts into every tile's first output slot per
// digit, and k_sort_scatter moves the keys there.  Within a tile, warp w owns keys [256 w, 256 w + 256) in rounds of 32
// consecutive keys, ranked among equal digits with __match_any_sync, so keys with equal digits keep their order (stable)
// and the result of the four passes is the sorted column.
constexpr int kSortThreads = 256, kSortTile = 2048, kRadix = 256;

__device__ __forceinline__ uint32_t f2key(float f) {
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key2f(uint32_t k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k); }

template <bool IN_F>
__device__ __forceinline__ uint32_t load_key(const uint32_t* p) {
  const uint32_t v = *p;
  return IN_F ? f2key(__uint_as_float(v)) : v;
}

// counts[seg][tile][digit]
template <bool IN_F>
__global__ void __launch_bounds__(kSortThreads) k_sort_hist(const uint32_t* __restrict__ in, uint32_t* __restrict__ counts,
                                                            int64_t seg_len, int tiles, int shift) {
  __shared__ uint32_t h[kRadix];
  h[threadIdx.x] = 0;
  __syncthreads();
  const int64_t seg = blockIdx.y, t0 = (int64_t)blockIdx.x * kSortTile;
  const uint32_t* src = in + seg * seg_len;
  for (int i = threadIdx.x; i < kSortTile; i += kSortThreads) {
    const int64_t p = t0 + i;
    if (p < seg_len) atomicAdd(&h[(load_key<IN_F>(src + p) >> shift) & 0xFF], 1u);
  }
  __syncthreads();
  counts[(seg * tiles + blockIdx.x) * kRadix + threadIdx.x] = h[threadIdx.x];
}

// counts -> exclusive prefix over the tiles per digit (in place); digit_base[seg][d] = number of keys with a smaller digit
__global__ void __launch_bounds__(kRadix) k_sort_scan(uint32_t* __restrict__ counts, uint32_t* __restrict__ digit_base,
                                                      int tiles) {
  __shared__ uint32_t tot[kRadix];
  const int d = threadIdx.x;
  uint32_t* c = counts + (int64_t)blockIdx.x * tiles * kRadix;
  uint32_t run = 0;
  for (int t = 0; t < tiles; ++t) {
    const uint32_t v = c[(int64_t)t * kRadix + d];
    c[(int64_t)t * kRadix + d] = run;
    run += v;
  }
  tot[d] = run;
  __syncthreads();
  for (int o = 1; o < kRadix; o <<= 1) {          // inclusive Hillis-Steele scan of the digit totals
    const uint32_t v = d >= o ? tot[d - o] : 0u;
    __syncthreads();
    tot[d] += v;
    __syncthreads();
  }
  digit_base[blockIdx.x * kRadix + d] = tot[d] - run;
}

template <bool IN_F, bool OUT_F>
__global__ void __launch_bounds__(kSortThreads) k_sort_scatter(const uint32_t* __restrict__ in, uint32_t* __restrict__ out,
                                                               const uint32_t* __restrict__ counts,
                                                               const uint32_t* __restrict__ digit_base, int64_t seg_len,
                                                               int tiles, int shift) {
  constexpr int kWarps = kSortThreads / 32, kRounds = kSortTile / kSortThreads;
  __shared__ uint32_t wcnt[kWarps][kRadix];
  __shared__ uint32_t base[kRadix];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t seg = blockIdx.y, t0 = (int64_t)blockIdx.x * kSortTile;
  for (int i = threadIdx.x; i < kWarps * kRadix; i += kSortThreads) (&wcnt[0][0])[i] = 0;
  base[threadIdx.x] = digit_base[seg * kRadix + threadIdx.x] + counts[(seg * tiles + blockIdx.x) * kRadix + threadIdx.x];
  __syncthreads();
  const uint32_t* src = in + seg * seg_len;
  const uint32_t lt = (1u << lane) - 1u;
  uint32_t key[kRounds], loc[kRounds];
#pragma unroll
  for (int r = 0; r < kRounds; ++r) {
    const int64_t p = t0 + w * (kSortTile / kWarps) + r * 32 + lane;
    const bool valid = p < seg_len;
    key[r] = valid ? load_key<IN_F>(src + p) : 0u;
    const uint32_t d = valid ? (key[r] >> shift) & 0xFF : kRadix;     // invalid lanes form their own group
    const uint32_t peers = __match_any_sync(0xffffffffu, d);
    const uint32_t before = valid ? wcnt[w][d] : 0u;
    __syncwarp();
    if (valid && lane == __ffs(peers) - 1) wcnt[w][d] = before + __popc(peers);
    __syncwarp();
    loc[r] = before + __popc(peers & lt);
  }
  __syncthreads();
  {                                               // exclusive prefix over the warps, per digit
    uint32_t run = 0;
    for (int v = 0; v < kWarps; ++v) {
      const uint32_t c = wcnt[v][threadIdx.x];
      wcnt[v][threadIdx.x] = run;
      run += c;
    }
  }
  __syncthreads();
  uint32_t* dst = out + seg * seg_len;
#pragma unroll
  for (int r = 0; r < kRounds; ++r) {
    const int64_t p = t0 + w * (kSortTile / kWarps) + r * 32 + lane;
    if (p < seg_len) {
      const uint32_t d = (key[r] >> shift) & 0xFF;
      const uint32_t o = base[d] + wcnt[w][d] + loc[r];
      dst[o] = OUT_F ? __float_as_uint(key2f(key[r])) : key[r];
    }
  }
}

// ---- sum |a - b| in fp64 ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_swd_l1_part(const float* __restrict__ a, const float* __restrict__ b,
                                                     double* __restrict__ parts, int64_t n) {
  __shared__ double sm[256];
  double s = 0.;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    s += fabs((double)a[i] - (double)b[i]);
  s = block_sum_f64(s, sm);
  if (threadIdx.x == 0) parts[blockIdx.x] = s;
}

__global__ void k_swd_l1_final(const double* __restrict__ parts, int nb, double* __restrict__ out) {
  if (threadIdx.x) return;
  double s = 0.;
  for (int b = 0; b < nb; ++b) s += parts[b];
  out[0] = s;
}

struct SortWs {
  uint32_t *alt, *counts, *digit_base;
  int tiles;
};
static SortWs sort_ws(void* ws, int segments, int64_t seg_len) {
  SortWs w;
  w.tiles = (int)cdiv(seg_len, kSortTile);
  w.alt = static_cast<uint32_t*>(ws);
  w.counts = w.alt + (int64_t)segments * seg_len;
  w.digit_base = w.counts + (int64_t)segments * w.tiles * kRadix;
  return w;
}

}  // namespace twg

using namespace twg;

extern "C" {

int twg_swd_pyramid(const float* x, float* pyr, int N, int R, int levels, twg_stream_t stream) {
  if (!x || !pyr) return fail(TWG_ERR_INVALID, "twg_swd_pyramid: null");
  if (N < 1 || R < 4 || (R & (R - 1)) || levels < 1 || levels > 30 || (R >> (levels - 1)) < 4)
    return fail(TWG_ERR_INVALID, "twg_swd_pyramid: N=%d R=%d levels=%d (R a power of two, R >> (levels-1) >= 4)", N, R,
                levels);
  cudaStream_t st = S(stream);
  float* lv[32];
  int64_t off = 0;
  for (int l = 0; l < levels; ++l) {
    lv[l] = pyr + off;
    off += (int64_t)N * (R >> l) * (R >> l) * 3;
  }
  if (levels == 1) {
    if (cudaMemcpyAsync(pyr, x, sizeof(float) * (int64_t)N * R * R * 3, cudaMemcpyDeviceToDevice, st) != cudaSuccess)
      return fail(TWG_ERR_CUDA, "twg_swd_pyramid: copy failed");
    return TWG_OK;
  }
  for (int l = 1; l < levels; ++l) {              // Gaussian levels 1 .. levels-1
    const int Rs = R >> (l - 1);
    k_pyr_down<<<grid_for((int64_t)N * (Rs / 2) * (Rs / 2), 1), 256, 0, st>>>(l == 1 ? x : lv[l - 1], lv[l], N, Rs);
    const int rc = check_launch("twg_swd_pyramid");
    if (rc) return rc;
  }
  for (int l = 0; l + 1 < levels; ++l) {          // level l -= pyr_up(Gaussian level l + 1), finest first
    const int Rf = R >> l;
    k_pyr_up_sub<<<grid_for((int64_t)N * Rf * Rf, 1), 256, 0, st>>>(l == 0 ? x : lv[l], lv[l + 1], lv[l], N, Rf);
    const int rc = check_launch("twg_swd_pyramid");
    if (rc) return rc;
  }
  return TWG_OK;
}

int twg_swd_gather(const float* level, const void* centres, float* desc, int N, int Rl, int nhoods, int nhood_size,
                   twg_stream_t stream) {
  if (!level || !centres || !desc) return fail(TWG_ERR_INVALID, "twg_swd_gather: null");
  if (N < 1 || nhoods < 1 || nhood_size < 1 || !(nhood_size & 1) || Rl < nhood_size)
    return fail(TWG_ERR_INVALID, "twg_swd_gather: N=%d Rl=%d nhoods=%d nhood_size=%d (odd, <= Rl)", N, Rl, nhoods,
                nhood_size);
  const int64_t rows = (int64_t)N * nhoods;
  k_swd_gather<<<grid_for(rows * 3 * nhood_size * nhood_size, 4), 256, 0, S(stream)>>>(
      level, static_cast<const int*>(centres), desc, rows, nhoods, Rl, nhood_size);
  return check_launch("twg_swd_gather");
}

int twg_swd_stats(const float* desc, float* stats, int64_t rows, int nhood_size, twg_stream_t stream) {
  if (!desc || !stats) return fail(TWG_ERR_INVALID, "twg_swd_stats: null");
  if (rows < 1 || nhood_size < 1) return fail(TWG_ERR_INVALID, "twg_swd_stats: rows=%lld nhood_size=%d",
                                               (long long)rows, nhood_size);
  double* parts = swd_parts();
  if (!parts) return fail(TWG_ERR_CUDA, "twg_swd_stats: no partial-sum buffer");
  const int ss = nhood_size * nhood_size;
  const int64_t total = rows * 3 * ss;
  const int nb = reduce_blocks(total);
  cudaStream_t st = S(stream);
  k_swd_stats_part<<<nb, 256, 0, st>>>(desc, parts, total, 3 * ss, ss);
  int rc = check_launch("twg_swd_stats");
  if (rc) return rc;
  k_swd_stats_final<<<1, 32, 0, st>>>(parts, nb, (double)rows * ss, stats);
  return check_launch("twg_swd_stats");
}

int twg_swd_project(const float* desc, const float* stats, const float* dirs, float* proj, int64_t rows, int nhood_size,
                    int ndirs, twg_stream_t stream) {
  if (!desc || !stats || !dirs || !proj) return fail(TWG_ERR_INVALID, "twg_swd_project: null");
  if (rows < 1 || nhood_size < 1 || ndirs < 1 || ndirs % PN || ndirs / PN > 65535 || cdiv(rows, PM) > 0x7FFFFFFF)
    return fail(TWG_ERR_INVALID, "twg_swd_project: rows=%lld nhood_size=%d ndirs=%d (a multiple of %d)", (long long)rows,
                nhood_size, ndirs, PN);
  const int ss = nhood_size * nhood_size;
  dim3 grid((unsigned)cdiv(rows, PM), (unsigned)(ndirs / PN));
  k_swd_project<<<grid, 256, 0, S(stream)>>>(desc, stats, dirs, proj, rows, 3 * ss, ss, ndirs);
  return check_launch("twg_swd_project");
}

int64_t twg_swd_sort_workspace(int segments, int64_t seg_len) {
  if (segments < 1 || segments > 65535 || seg_len < 1 || seg_len >= (1ll << 31))
    return fail(TWG_ERR_INVALID, "twg_swd_sort_workspace: segments=%d seg_len=%lld", segments, (long long)seg_len);
  const int64_t tiles = cdiv(seg_len, kSortTile);
  return 4 * ((int64_t)segments * seg_len + (int64_t)segments * tiles * kRadix + (int64_t)segments * kRadix);
}

int twg_swd_sort(float* keys, void* workspace, int segments, int64_t seg_len, twg_stream_t stream) {
  if (!keys || !workspace) return fail(TWG_ERR_INVALID, "twg_swd_sort: null");
  if (twg_swd_sort_workspace(segments, seg_len) < 0) return TWG_ERR_INVALID;
  const SortWs w = sort_ws(workspace, segments, seg_len);
  cudaStream_t st = S(stream);
  uint32_t* k = reinterpret_cast<uint32_t*>(keys);
  const dim3 grid((unsigned)w.tiles, (unsigned)segments);
  // keys -> alt -> keys -> alt -> keys; floats become keys on the first read and floats again on the last write
  for (int pass = 0; pass < 4; ++pass) {
    const uint32_t* in = (pass & 1) ? w.alt : k;
    uint32_t* out = (pass & 1) ? k : w.alt;
    const int shift = 8 * pass;
    if (pass == 0) k_sort_hist<true><<<grid, kSortThreads, 0, st>>>(in, w.counts, seg_len, w.tiles, shift);
    else k_sort_hist<false><<<grid, kSortThreads, 0, st>>>(in, w.counts, seg_len, w.tiles, shift);
    int rc = check_launch("twg_swd_sort");
    if (rc) return rc;
    k_sort_scan<<<segments, kRadix, 0, st>>>(w.counts, w.digit_base, w.tiles);
    if ((rc = check_launch("twg_swd_sort"))) return rc;
    if (pass == 0)
      k_sort_scatter<true, false><<<grid, kSortThreads, 0, st>>>(in, out, w.counts, w.digit_base, seg_len, w.tiles, shift);
    else if (pass == 3)
      k_sort_scatter<false, true><<<grid, kSortThreads, 0, st>>>(in, out, w.counts, w.digit_base, seg_len, w.tiles, shift);
    else
      k_sort_scatter<false, false><<<grid, kSortThreads, 0, st>>>(in, out, w.counts, w.digit_base, seg_len, w.tiles,
                                                                  shift);
    if ((rc = check_launch("twg_swd_sort"))) return rc;
  }
  return TWG_OK;
}

int twg_swd_sorted_l1(const float* a, const float* b, void* out_f64, int64_t n, twg_stream_t stream) {
  if (!a || !b || !out_f64) return fail(TWG_ERR_INVALID, "twg_swd_sorted_l1: null");
  if (n < 1) return fail(TWG_ERR_INVALID, "twg_swd_sorted_l1: n=%lld", (long long)n);
  double* parts = swd_parts();
  if (!parts) return fail(TWG_ERR_CUDA, "twg_swd_sorted_l1: no partial-sum buffer");
  const int nb = reduce_blocks(n);
  cudaStream_t st = S(stream);
  k_swd_l1_part<<<nb, 256, 0, st>>>(a, b, parts, n);
  const int rc = check_launch("twg_swd_sorted_l1");
  if (rc) return rc;
  k_swd_l1_final<<<1, 32, 0, st>>>(parts, nb, static_cast<double*>(out_f64));
  return check_launch("twg_swd_sorted_l1");
}

}  // extern "C"
