// Baseline JPEG decoding for image translation (twingan_b200/jpeg.py picks the files and packs the descriptors): Huffman
// entropy decoding, the integer "islow" inverse DCT and fancy chroma upsampling + YCbCr -> RGB, each stage a kernel, the
// result bit for bit what libjpeg-turbo (PIL's decoder) returns with its defaults.  Written from ITU-T T.81 and the
// published integer algorithms; oracle/jpeg_oracle.py restates every stage in numpy.
//
// A stream the kernels do not restate exactly is flagged in its image's status word (bits TWG_JPEG_*), never decoded
// differently: the caller decodes a flagged image on the host.
#include <assert.h>
#include <limits.h>

#include "../../include/twgjpeg.h"
#include "twg_common.cuh"
#include "twg_jpeg_bits.cuh"

namespace twg {

// One thread per segment; `spw` segments per warp (lanes >= spw idle), so that a few long segments get a warp each.
__global__ void __launch_bounds__(128) k_jpeg_entropy(const uint8_t* __restrict__ data, const int64_t* __restrict__ segs,
                                                      int nseg, int spw, const int64_t* __restrict__ images,
                                                      const int64_t* __restrict__ comps, const int32_t* __restrict__ huff,
                                                      int16_t* __restrict__ coef, int* __restrict__ status) {
  const int gid = blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = gid & 31;
  const int s = (gid >> 5) * spw + lane;
  if (lane >= spw || s >= nseg) return;
  const int64_t* sg = segs + (int64_t)s * SEG_FIELDS;
  const int img = (int)sg[SEG_IMAGE];
  const int64_t* im = images + (int64_t)img * IMAGE_FIELDS;
  const int nc = (int)im[I_NCOMP], mcux = (int)im[I_MCUX], index = (int)sg[SEG_INDEX];
  Bits b{data + sg[SEG_START], data + sg[SEG_END], 0ull, 0, 0, 0};
  // the marker after the segment: RSTn in sequence, EOI after the image's last segment (the packed scan keeps its EOI)
  const uint8_t* term = data + sg[SEG_END];
  const uint32_t want = index == (int)im[I_NSEG] - 1 ? 0xD9u : 0xD0u + (index & 7);
  int err = (__ldg(term) != 0xFF || __ldg(term + 1) != want) ? TWG_JPEG_RESTART : 0;
  int64_t block0[3], bw[3];
  int h[3], v[3];
  const int32_t* dct[3];
  const int32_t* act[3];
  int pred[3] = {0, 0, 0};
  for (int c = 0; c < 3; ++c) {
    const int64_t* cp = comps + (im[I_COMP0] + min(c, nc - 1)) * COMP_FIELDS;
    block0[c] = cp[C_BLOCK0];
    bw[c] = cp[C_BW];
    h[c] = (int)cp[C_H];
    v[c] = (int)cp[C_V];
    dct[c] = huff + cp[C_DC] * kHuffWords;
    act[c] = huff + cp[C_AC] * kHuffWords;
  }
  const int64_t m0 = sg[SEG_MCU0], m1 = m0 + sg[SEG_MCUS];
  for (int64_t m = m0; m < m1 && !err; ++m) {
    const int64_t my = m / mcux, mx = m - my * mcux;
    for (int c = 0; c < nc && !err; ++c) {
      for (int by = 0; by < v[c] && !err; ++by) {
        for (int bx = 0; bx < h[c] && !err; ++bx) {
          int16_t* blk = coef + (block0[c] + (my * v[c] + by) * bw[c] + mx * h[c] + bx) * 64;
          uint4* z = reinterpret_cast<uint4*>(blk);
#pragma unroll
          for (int q = 0; q < 8; ++q) z[q] = make_uint4(0, 0, 0, 0);
          b.fill();
          const int t = b.symbol(dct[c]);
          pred[c] += extend(b.take(t), t);
          if (pred[c] < -32768 || pred[c] > 32767) b.err |= TWG_JPEG_COEF_RANGE;
          blk[0] = (int16_t)pred[c];
          int k = 1;
          while (k < 64 && !b.err) {
            b.fill();
            const int rs = b.symbol(act[c]);
            const int r = rs >> 4, sz = rs & 15;
            if (sz == 0) {
              if (r != 15) break;         // EOB
              k += 16;                    // ZRL
              continue;
            }
            k += r;
            if (k > 63) {
              b.err |= TWG_JPEG_COEF_RANGE;
              break;
            }
            blk[k] = (int16_t)extend(b.take(sz), sz);
            ++k;
          }
          if (k > 64) b.err |= TWG_JPEG_COEF_RANGE;
          err |= b.err;
        }
      }
    }
  }
  if (err) atomicOr(status + img, err);
}

// ---- inverse DCT ---------------------------------------------------------------------------------------------------

// jidctint.c's constants, FIX(x) = round(x * 2^13)
constexpr int F0298 = 2446, F0390 = 3196, F0541 = 4433, F0765 = 6270, F0899 = 7373, F1175 = 9633, F1501 = 12299,
              F1847 = 15137, F1961 = 16069, F2053 = 16819, F2562 = 20995, F3072 = 25172;
constexpr int kConstBits = 13, kPass1Bits = 2;

// one islow pass over the eight values x[0], x[st], ..., x[7 st], in place, descaled by `shift` with rounding; 64-bit
// arithmetic as libjpeg's C path (JLONG), so no input in int16 overflows
template <int shift>
__device__ __forceinline__ void idct_1d(int* x, int st) {
  typedef long long L;
  const L z1e = ((L)x[2 * st] + x[6 * st]) * F0541;
  const L t2e = z1e - (L)x[6 * st] * F1847;
  const L t3e = z1e + (L)x[2 * st] * F0765;
  const L t0e = ((L)x[0] + x[4 * st]) * (1 << kConstBits);
  const L t1e = ((L)x[0] - x[4 * st]) * (1 << kConstBits);
  const L t10 = t0e + t3e, t13 = t0e - t3e, t11 = t1e + t2e, t12 = t1e - t2e;
  L o0 = x[7 * st], o1 = x[5 * st], o2 = x[3 * st], o3 = x[st];
  const L z1 = o0 + o3, z2 = o1 + o2, z3 = o0 + o2, z4 = o1 + o3;
  const L z5 = (z3 + z4) * F1175;
  const L y1 = -z1 * F0899, y2 = -z2 * F2562, y3 = -z3 * F1961 + z5, y4 = -z4 * F0390 + z5;
  o0 = o0 * F0298 + y1 + y3;
  o1 = o1 * F2053 + y2 + y4;
  o2 = o2 * F3072 + y2 + y3;
  o3 = o3 * F1501 + y1 + y4;
  constexpr L r = 1ll << (shift - 1);
  const L lo = INT_MIN, hi = INT_MAX;     // a flagged block's values only need to stay flagged
  x[0] = (int)max(lo, min(hi, (t10 + o3 + r) >> shift));
  x[7 * st] = (int)max(lo, min(hi, (t10 - o3 + r) >> shift));
  x[st] = (int)max(lo, min(hi, (t11 + o2 + r) >> shift));
  x[6 * st] = (int)max(lo, min(hi, (t11 - o2 + r) >> shift));
  x[2 * st] = (int)max(lo, min(hi, (t12 + o1 + r) >> shift));
  x[5 * st] = (int)max(lo, min(hi, (t12 - o1 + r) >> shift));
  x[3 * st] = (int)max(lo, min(hi, (t13 + o0 + r) >> shift));
  x[4 * st] = (int)max(lo, min(hi, (t13 - o0 + r) >> shift));
}

// One thread per 8x8 block of the batch: dequantise, columns then rows, +128 into the component's sample plane.  A block
// whose dequantised coefficients or first-pass values leave int16, or whose result leaves [-512, 511] before the +128, is
// flagged: there libjpeg's C path (wrap-around range limit) and its SIMD paths (16-bit saturation) part ways.
__global__ void __launch_bounds__(256) k_jpeg_idct(const int16_t* __restrict__ coef, const int64_t* __restrict__ comps,
                                                   int ncomps, int64_t nblocks, const int32_t* __restrict__ qt,
                                                   uint8_t* __restrict__ planes, int* __restrict__ status) {
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < nblocks; g += (int64_t)gridDim.x * blockDim.x) {
    int lo = 0, hi = ncomps - 1;             // the component holding block g: last row with block0 <= g
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (__ldg(comps + (int64_t)mid * COMP_FIELDS + C_BLOCK0) <= g) lo = mid; else hi = mid - 1;
    }
    const int64_t* cp = comps + (int64_t)lo * COMP_FIELDS;
    const int64_t local = g - __ldg(cp + C_BLOCK0), bwc = __ldg(cp + C_BW);
    const int64_t by = local / bwc, bx = local - by * bwc;
    const int4* q4 = reinterpret_cast<const int4*>(qt + __ldg(cp + C_QT) * 64);
    const uint4* c4 = reinterpret_cast<const uint4*>(coef + g * 64);
    int x[64];
    bool bad = false;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const uint4 w = __ldg(c4 + i);
      const int4 qa = __ldg(q4 + 2 * i), qb = __ldg(q4 + 2 * i + 1);
      const uint32_t ws[4] = {w.x, w.y, w.z, w.w};
      const int qs[8] = {qa.x, qa.y, qa.z, qa.w, qb.x, qb.y, qb.z, qb.w};
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int c = (int)(int16_t)(ws[j >> 1] >> (16 * (j & 1)));
        const int d = c * qs[j];
        bad |= d < -32768 || d > 32767;
        x[natural_of(8 * i + j)] = d;
      }
    }
#pragma unroll
    for (int col = 0; col < 8; ++col) idct_1d<kConstBits - kPass1Bits>(x + col, 8);
#pragma unroll
    for (int i = 0; i < 64; ++i) bad |= x[i] < -32768 || x[i] > 32767;
    uint8_t* out = planes + __ldg(cp + C_PLANE) + (by * 8) * (bwc * 8) + bx * 8;
#pragma unroll
    for (int row = 0; row < 8; ++row) {
      int* r = x + 8 * row;
      idct_1d<kConstBits + kPass1Bits + 3>(r, 1);
      uint32_t w[2] = {0, 0};
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        bad |= r[j] < -512 || r[j] > 511;
        w[j >> 2] |= (uint32_t)min(max(r[j] + 128, 0), 255) << (8 * (j & 3));
      }
      *reinterpret_cast<uint2*>(out + row * bwc * 8) = make_uint2(w[0], w[1]);
    }
    if (bad) atomicOr(status + __ldg(cp + C_IMAGE), TWG_JPEG_IDCT_RANGE);
  }
}

// ---- upsampling and colour conversion ------------------------------------------------------------------------------

// libjpeg's fancy upsampling of a chroma plane (cw x ch real samples, row stride `st`) at output pixel (y, x): h2v1
// (3 c[j] + c[j -/+ 1] + 1 / 2) >> 2 and h2v2 (3 s[j] + s[j -/+ 1] + 8 / 7) >> 4 over column sums s = 3 c[i] + c[i -/+ 1],
// the last real column / row replicated.  Planes of at most two columns are replicated (jdsample.c h2v1/h2v2_upsample).
__device__ __forceinline__ int chroma_at(const uint8_t* __restrict__ p, int64_t st, int cw, int ch, bool v2, int y, int x) {
  const int j = x >> 1;
  const int i = v2 ? y >> 1 : y;
  if (cw <= 2) return __ldg(p + i * st + j);
  const int jn = (x & 1) ? min(j + 1, cw - 1) : max(j - 1, 0);
  if (!v2) {
    const uint8_t* r = p + i * st;
    return (3 * __ldg(r + j) + __ldg(r + jn) + ((x & 1) ? 2 : 1)) >> 2;
  }
  const int in = (y & 1) ? min(i + 1, ch - 1) : max(i - 1, 0);
  const uint8_t* r0 = p + i * st;
  const uint8_t* r1 = p + in * st;
  const int s = 3 * __ldg(r0 + j) + __ldg(r1 + j);
  const int sn = 3 * __ldg(r0 + jn) + __ldg(r1 + jn);
  return (3 * s + sn + ((x & 1) ? 7 : 8)) >> 4;
}

__device__ __forceinline__ uint32_t clamp255(int v) { return (uint32_t)min(max(v, 0), 255); }

// One thread per output pixel of the batch's JPEG images: Y (and Cb, Cr upsampled) -> RGB at the image's payload offset.
// jdcolor.c's fixed point: R = y + ((91881 cr' + 2^15) >> 16), G = y + ((-22554 cb' + 2^15 - 46802 cr') >> 16), B = y +
// ((116130 cb' + 2^15) >> 16), c' = c - 128, clamped; a grey image repeats Y in the three channels.
__global__ void __launch_bounds__(256) k_jpeg_color(const uint8_t* __restrict__ planes,
                                                    const int64_t* __restrict__ images, int nimages,
                                                    const int64_t* __restrict__ comps, int64_t npix,
                                                    uint8_t* __restrict__ payload) {
  for (int64_t P = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; P < npix; P += (int64_t)gridDim.x * blockDim.x) {
    int lo = 0, hi = nimages - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (__ldg(images + (int64_t)mid * IMAGE_FIELDS + I_PIX0) <= P) lo = mid; else hi = mid - 1;
    }
    const int64_t* im = images + (int64_t)lo * IMAGE_FIELDS;
    const int H = (int)__ldg(im + I_H), W = (int)__ldg(im + I_W);
    const int64_t r = P - __ldg(im + I_PIX0);
    const int y = (int)(r / W), x = (int)(r - (int64_t)y * W);
    const int64_t* c0 = comps + __ldg(im + I_COMP0) * COMP_FIELDS;
    const int64_t st0 = __ldg(c0 + C_BW) * 8;
    const int Y = __ldg(planes + __ldg(c0 + C_PLANE) + y * st0 + x);
    uint8_t* o = payload + __ldg(im + I_OUT) + r * 3;
    if (__ldg(im + I_NCOMP) == 1) {
      o[0] = o[1] = o[2] = (uint8_t)Y;
      continue;
    }
    const bool h2 = __ldg(im + I_HMAX) == 2, v2 = __ldg(im + I_VMAX) == 2;
    const int cw = h2 ? (W + 1) >> 1 : W, ch = v2 ? (H + 1) >> 1 : H;
    int cc[2];
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const int64_t* cp = c0 + (k + 1) * COMP_FIELDS;
      const uint8_t* p = planes + __ldg(cp + C_PLANE);
      const int64_t st = __ldg(cp + C_BW) * 8;
      cc[k] = h2 ? chroma_at(p, st, cw, ch, v2, y, x) : __ldg(p + y * st + x);
    }
    const int cb = cc[0] - 128, cr = cc[1] - 128;
    o[0] = (uint8_t)clamp255(Y + ((91881 * cr + 32768) >> 16));
    o[1] = (uint8_t)clamp255(Y + ((-22554 * cb + 32768 - 46802 * cr) >> 16));
    o[2] = (uint8_t)clamp255(Y + ((116130 * cb + 32768) >> 16));
  }
}

}  // namespace twg

using namespace twg;

extern "C" {

int twgjpeg_entropy(const void* data, const int64_t* segs, int nseg, const int64_t* images, int nimages,
                     const int64_t* comps, const void* huff, void* coefs, void* status, twg_stream_t stream) {
  if (!data || !segs || !images || !comps || !huff || !coefs || !status)
    return fail(TWG_ERR_INVALID, "twgjpeg_entropy: null");
  if (nseg < 1 || nimages < 1) return fail(TWG_ERR_INVALID, "twgjpeg_entropy: nseg=%d nimages=%d", nseg, nimages);
  if (reinterpret_cast<uintptr_t>(coefs) & 15) return fail(TWG_ERR_INVALID, "twgjpeg_entropy: coefs not 16-byte aligned");
  if (cudaMemsetAsync(status, 0, sizeof(int) * (size_t)nimages, S(stream)) != cudaSuccess)
    return check_launch("twgjpeg_entropy: status reset");
  // few segments: one per warp, so that each runs alone; many: up to 32 per warp
  int spw = 1;
  while (spw < 32 && cdiv(nseg, spw) > (int64_t)kNumSMs * 32) spw *= 2;
  const int64_t threads = cdiv(nseg, spw) * 32;
  k_jpeg_entropy<<<(unsigned)cdiv(threads, 128), 128, 0, S(stream)>>>(
      static_cast<const uint8_t*>(data), segs, nseg, spw, images, comps, static_cast<const int32_t*>(huff),
      static_cast<int16_t*>(coefs), static_cast<int*>(status));
  return check_launch("twgjpeg_entropy");
}

int twgjpeg_idct(const void* coefs, const int64_t* comps, int ncomps, int64_t nblocks, const void* qt, void* planes,
                  void* status, twg_stream_t stream) {
  if (!coefs || !comps || !qt || !planes || !status) return fail(TWG_ERR_INVALID, "twgjpeg_idct: null");
  if (ncomps < 1 || nblocks < 1) return fail(TWG_ERR_INVALID, "twgjpeg_idct: ncomps=%d nblocks=%lld", ncomps,
                                             (long long)nblocks);
  if ((reinterpret_cast<uintptr_t>(coefs) | reinterpret_cast<uintptr_t>(qt) | reinterpret_cast<uintptr_t>(planes)) & 15)
    return fail(TWG_ERR_INVALID, "twgjpeg_idct: coefs, qt and planes must be 16-byte aligned");
  k_jpeg_idct<<<grid_for(nblocks, 1), 256, 0, S(stream)>>>(static_cast<const int16_t*>(coefs), comps, ncomps, nblocks,
                                                           static_cast<const int32_t*>(qt), static_cast<uint8_t*>(planes),
                                                           static_cast<int*>(status));
  return check_launch("twgjpeg_idct");
}

int twgjpeg_color(const void* planes, const int64_t* images, int nimages, const int64_t* comps, int64_t npixels,
                   void* payload, twg_stream_t stream) {
  if (!planes || !images || !comps || !payload) return fail(TWG_ERR_INVALID, "twgjpeg_color: null");
  if (nimages < 1 || npixels < 1)
    return fail(TWG_ERR_INVALID, "twgjpeg_color: nimages=%d npixels=%lld", nimages, (long long)npixels);
  k_jpeg_color<<<grid_for(npixels, 4), 256, 0, S(stream)>>>(static_cast<const uint8_t*>(planes), images, nimages, comps,
                                                            npixels, static_cast<uint8_t*>(payload));
  return check_launch("twgjpeg_color");
}

}  // extern "C"
