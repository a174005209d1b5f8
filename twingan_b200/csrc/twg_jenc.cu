// Baseline JPEG encoding for image translation (twingan_b200/jpeg.py writes the header): the entropy-coded scan of each
// uint8 RGB image, byte for byte what libjpeg-turbo writes for PIL's Image.save(f, 'JPEG') at its defaults.  Written from
// ITU-T T.81 and libjpeg's published integer algorithms; tests/jenc_oracle.py restates every stage in numpy.
//
// Stages: colour conversion, edge expansion, downsampling, forward DCT and quantisation, one thread per block; the code
// length of every block and its prefix sum, one CTA per image; the codes written at their bit positions with 32-bit
// atomicOr into a zeroed buffer (OR does not depend on order), then 0xFF stuffing and packing.  Integer throughout, and
// no result depends on scheduling.
#include "../../include/twgjenc.h"
#include "twg_common.cuh"

namespace twg {
namespace {

constexpr int kBlocksPerMcu = 6;          // Y00 Y01 Y10 Y11 Cb Cr
// bits of one block's codes at most: DC code 11 + 11 value bits, 63 AC codes of 16 + 10 value bits (8-bit samples)
constexpr int kMaxBlockBytes = 208;
constexpr int kScanThreads = 256;

__host__ __device__ constexpr int natural_of(int k) {
  constexpr int t[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                         41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                         30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
  return t[k];
}

// ---- Annex K Huffman tables (T.81 K.3): (code length << 16) | code, per symbol ------------------------------------------
constexpr uint8_t kHuffBits[4][16] = {{0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0},           // DC luma
                                      {0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7D},        // AC luma
                                      {0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0},           // DC chroma
                                      {0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77}};       // AC chroma
constexpr uint8_t kHuffVals[4][162] = {
    {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11},
    {0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14,
     0x32, 0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09,
     0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a,
     0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65,
     0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88,
     0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9,
     0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca,
     0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea,
     0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa},
    {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11},
    {0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32,
     0x81, 0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16,
     0x24, 0x34, 0xe1, 0x25, 0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39,
     0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64,
     0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86,
     0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7,
     0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8,
     0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9,
     0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa}};

struct HuffEnc {
  uint32_t e[4][256];
};

// canonical codes (T.81 C.2): lengths in order, each code one more than the last, shifted left at each new length
constexpr HuffEnc make_huff() {
  HuffEnc h{};
  for (int t = 0; t < 4; ++t) {
    int code = 0, k = 0;
    for (int l = 1; l <= 16; ++l) {
      for (int i = 0; i < kHuffBits[t][l - 1]; ++i) h.e[t][kHuffVals[t][k++]] = ((uint32_t)l << 16) | (uint32_t)code++;
      code <<= 1;
    }
  }
  return h;
}

__device__ constexpr HuffEnc kHuff = make_huff();

struct Geometry {
  int h, w, mx, my;
  int64_t mcus, blocks;       // per image
};

__host__ __device__ inline Geometry geometry(int h, int w) {
  Geometry g{h, w, (w + 15) >> 4, (h + 15) >> 4, 0, 0};
  g.mcus = (int64_t)g.mx * g.my;
  g.blocks = g.mcus * kBlocksPerMcu;
  return g;
}

// ---- colour conversion, downsampling, forward DCT, quantisation ----------------------------------------------------

// jccolor.c rgb_ycc_convert, SCALEBITS 16: FIX(0.299) 19595, FIX(0.587) 38470, FIX(0.114) 7471, FIX(0.16874) 11059,
// FIX(0.33126) 21709, FIX(0.5) 32768, FIX(0.41869) 27439, FIX(0.08131) 5329; ONE_HALF on Y, ONE_HALF - 1 on Cb and Cr
__device__ __forceinline__ int ycc_of(const uint8_t* __restrict__ p, int k) {
  const int r = __ldg(p), g = __ldg(p + 1), b = __ldg(p + 2);
  if (k == 0) return (19595 * r + 38470 * g + 7471 * b + 32768) >> 16;
  if (k == 1) return (-11059 * r - 21709 * g + 32768 * b + (128 << 16) + 32767) >> 16;
  return (32768 * r - 27439 * g - 5329 * b + (128 << 16) + 32767) >> 16;
}

// One jfdctint.c islow pass over x[0], x[st], ..., x[7 st], in place.  Pass 1 (rows) keeps PASS1_BITS extra bits, pass 2
// (columns) removes them; the result is the DCT scaled up by 8.  The samples are 8-bit, so every product fits 32 bits.
template <bool pass1>
__device__ __forceinline__ void fdct_1d(int* x, int st) {
  constexpr int kConst = 13, kPass1 = 2;
  constexpr int sh = pass1 ? kConst - kPass1 : kConst + kPass1;
  const int t0 = x[0] + x[7 * st], t7 = x[0] - x[7 * st];
  const int t1 = x[st] + x[6 * st], t6 = x[st] - x[6 * st];
  const int t2 = x[2 * st] + x[5 * st], t5 = x[2 * st] - x[5 * st];
  const int t3 = x[3 * st] + x[4 * st], t4 = x[3 * st] - x[4 * st];
  const int t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
  if (pass1) {
    x[0] = (t10 + t11) * (1 << kPass1);
    x[4 * st] = (t10 - t11) * (1 << kPass1);
  } else {
    x[0] = (t10 + t11 + (1 << (kPass1 - 1))) >> kPass1;
    x[4 * st] = (t10 - t11 + (1 << (kPass1 - 1))) >> kPass1;
  }
  constexpr int r = 1 << (sh - 1);
  const int z1 = (t12 + t13) * 4433;                               // FIX(0.541196100)
  x[2 * st] = (z1 + t13 * 6270 + r) >> sh;                         // FIX(0.765366865)
  x[6 * st] = (z1 - t12 * 15137 + r) >> sh;                        // FIX(1.847759065)
  const int z5 = (t4 + t5 + t6 + t7) * 9633;                       // FIX(1.175875602)
  const int y1 = -(t4 + t7) * 7373, y2 = -(t5 + t6) * 20995;       // FIX(0.899976223), FIX(2.562915447)
  const int y3 = -(t4 + t6) * 16069 + z5, y4 = -(t5 + t7) * 3196 + z5;   // FIX(1.961570560), FIX(0.390180644)
  x[7 * st] = (t4 * 2446 + y1 + y3 + r) >> sh;                     // FIX(0.298631336)
  x[5 * st] = (t5 * 16819 + y2 + y4 + r) >> sh;                    // FIX(2.053119869)
  x[3 * st] = (t6 * 25172 + y2 + y3 + r) >> sh;                    // FIX(3.072711026)
  x[st] = (t7 * 12299 + y1 + y4 + r) >> sh;                        // FIX(1.501321110)
}

// libjpeg-turbo jcdctmgr.c compute_reciprocal for a 16-bit DCTELEM: q = ((|c| + corr) * recip) >> shift, sign restored
struct Recip {
  uint32_t recip, corr, shift;
};

__device__ inline Recip reciprocal(uint32_t divisor) {
  const int b = 31 - __clz(divisor);
  int r = 16 + b;
  uint32_t fq = (1u << r) / divisor;
  const uint32_t fr = (1u << r) % divisor;
  uint32_t c = divisor / 2;
  if (fr == 0) {
    fq >>= 1;
    --r;
  } else if (fr <= divisor / 2) {
    ++c;
  } else {
    ++fq;
  }
  return {fq, c, (uint32_t)r};
}

// One thread per coded block, numbered so that a warp holds one block kind (Y00 .. Cr) of consecutive MCUs.  A Y block
// right of or below the image is a jccoefct.c dummy: its AC is zero and its DC is that of the block it copies (the one
// to its left; below the image, the MCU's block 1, itself block 0's copy when it lies right of the image).
__global__ void __launch_bounds__(256) k_jenc_dct(const uint8_t* __restrict__ rgb, int n, Geometry geo,
                                                  const int32_t* __restrict__ qt, int16_t* __restrict__ coefs) {
  __shared__ Recip q[2][64];
  if (threadIdx.x < 128) {
    const int t = threadIdx.x >> 6, z = threadIdx.x & 63;
    q[t][z] = reciprocal((uint32_t)__ldg(qt + threadIdx.x) << 3);
  }
  __syncthreads();
  const int64_t total = (int64_t)n * geo.blocks;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (int64_t)gridDim.x * blockDim.x) {
    const int64_t img = g / geo.blocks, rest = g - img * geo.blocks;
    const int kind = (int)(rest / geo.mcus);
    const int64_t m = rest - kind * geo.mcus;
    const int my = (int)(m / geo.mx), mx = (int)(m - (int64_t)my * geo.mx);
    const uint8_t* im = rgb + img * geo.h * geo.w * 3;
    int x[64];
    bool dummy = false;
    if (kind < 4) {
      const int ybw = (geo.w + 7) >> 3, ybh = (geo.h + 7) >> 3;
      int bx = 2 * mx + (kind & 1), by = 2 * my + (kind >> 1);
      if (by >= ybh) {
        by = 2 * my;
        bx = 2 * mx + 1;
        dummy = true;
      }
      if (bx >= ybw) {
        bx = 2 * mx;
        dummy = true;
      }
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        const uint8_t* row = im + (int64_t)min(by * 8 + r, geo.h - 1) * geo.w * 3;
#pragma unroll
        for (int c = 0; c < 8; ++c) x[8 * r + c] = ycc_of(row + min(bx * 8 + c, geo.w - 1) * 3, 0) - 128;
      }
    } else {
      // h2v2_downsample on rows padded to a row pair and columns replicated to the MCU width; the last chroma row is
      // replicated below (jcprepct.c)
      const int k = kind - 3, ch = (geo.h + 1) >> 1;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int cy = min(my * 8 + i, ch - 1);
        const uint8_t* r0 = im + (int64_t)(2 * cy) * geo.w * 3;
        const uint8_t* r1 = im + (int64_t)min(2 * cy + 1, geo.h - 1) * geo.w * 3;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int c0 = min(2 * (mx * 8 + j), geo.w - 1) * 3, c1 = min(2 * (mx * 8 + j) + 1, geo.w - 1) * 3;
          const int s = ycc_of(r0 + c0, k) + ycc_of(r0 + c1, k) + ycc_of(r1 + c0, k) + ycc_of(r1 + c1, k);
          x[8 * i + j] = ((s + 1 + (j & 1)) >> 2) - 128;
        }
      }
    }
#pragma unroll
    for (int r = 0; r < 8; ++r) fdct_1d<true>(x + 8 * r, 1);
#pragma unroll
    for (int c = 0; c < 8; ++c) fdct_1d<false>(x + c, 8);
    const Recip* qq = q[kind < 4 ? 0 : 1];
    uint32_t out[32];
#pragma unroll
    for (int z = 0; z < 64; ++z) {
      const int v = x[natural_of(z)];
      const Recip d = qq[z];
      const int a = (int)(((uint32_t)abs(v) + d.corr) * d.recip >> d.shift);
      const int c = (dummy && z) ? 0 : (v < 0 ? -a : a);
      if (z & 1) out[z >> 1] |= (uint32_t)(uint16_t)c << 16;
      else out[z >> 1] = (uint16_t)c;
    }
    uint4* dst = reinterpret_cast<uint4*>(coefs + ((img * geo.mcus + m) * kBlocksPerMcu + kind) * 64);
#pragma unroll
    for (int i = 0; i < 8; ++i) dst[i] = make_uint4(out[4 * i], out[4 * i + 1], out[4 * i + 2], out[4 * i + 3]);
  }
}

// ---- Huffman coding ------------------------------------------------------------------------------------------------

// jchuff.c encode_one_block for block `b` (in MCU order) of one image's coefficients: the DC difference from the previous
// block of its component (0 before the first), then the AC run/size symbols with ZRL for runs of 16 and EOB after the
// last non-zero coefficient.  sink.put(code, length) receives every code and value in order.
template <class Sink>
__device__ __forceinline__ void code_block(const int16_t* __restrict__ blocks, int64_t b, const uint32_t* huff,
                                           Sink& sink) {
  const int kind = (int)(b % kBlocksPerMcu);
  const int16_t* blk = blocks + b * 64;
  int64_t prev = -1;
  if (kind >= 1 && kind <= 3) prev = b - 1;
  else if (b >= kBlocksPerMcu) prev = kind == 0 ? b - 3 : b - kBlocksPerMcu;
  const uint4* v4 = reinterpret_cast<const uint4*>(blk);
  uint64_t nz = 0;
  int dc = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const uint4 w = __ldg(v4 + i);
    const uint32_t ws[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (ws[j] & 0xFFFFu) nz |= 1ull << (8 * i + 2 * j);
      if (ws[j] >> 16) nz |= 1ull << (8 * i + 2 * j + 1);
    }
    if (i == 0) dc = (int16_t)(w.x & 0xFFFFu);
  }
  const uint32_t* dct = huff + (kind < 4 ? 0 : 2) * 256;
  const uint32_t* act = dct + 256;
  const int diff = dc - (prev >= 0 ? (int)__ldg(blocks + prev * 64) : 0);
  int nb = diff ? 32 - __clz(abs(diff)) : 0;
  uint32_t e = dct[nb];
  sink.put(e & 0xFFFFu, e >> 16);
  sink.put((uint32_t)(diff < 0 ? diff - 1 : diff) & ((1u << nb) - 1), nb);
  int last = 0;
  for (uint64_t rest = nz & ~1ull; rest; rest &= rest - 1) {
    const int k = __ffsll((long long)rest) - 1;
    int run = k - last - 1;
    for (; run > 15; run -= 16) {
      e = act[0xF0];
      sink.put(e & 0xFFFFu, e >> 16);
    }
    const int v = __ldg(blk + k);
    nb = 32 - __clz(abs(v));
    e = act[(run << 4) | nb];
    sink.put(e & 0xFFFFu, e >> 16);
    sink.put((uint32_t)(v < 0 ? v - 1 : v) & ((1u << nb) - 1), nb);
    last = k;
  }
  if (last < 63) {
    e = act[0x00];
    sink.put(e & 0xFFFFu, e >> 16);
  }
}

struct CountBits {
  int n = 0;
  __device__ __forceinline__ void put(uint32_t, int len) { n += len; }
};

// Bits MSB first from bit position `pos` of the stream, flushed as 32-bit words OR-ed into a zeroed buffer.  Stream bytes
// lie in memory order, so each big-endian word is byte-swapped before the OR.
struct WriteBits {
  uint32_t* words;
  int64_t word;
  uint64_t acc;
  int n;
  __device__ __forceinline__ WriteBits(uint32_t* w, int64_t pos) : words(w), word(pos >> 5), acc(0), n((int)(pos & 31)) {}
  __device__ __forceinline__ void put(uint32_t bits, int len) {
    if (!len) return;
    acc |= (uint64_t)bits << (64 - n - len);
    n += len;
    if (n >= 32) {
      const uint32_t hi = (uint32_t)(acc >> 32);
      if (hi) atomicOr(words + word, __byte_perm(hi, 0, 0x0123));
      acc <<= 32;
      n -= 32;
      ++word;
    }
  }
  __device__ __forceinline__ void flush() {
    const uint32_t hi = (uint32_t)(acc >> 32);
    if (n && hi) atomicOr(words + word, __byte_perm(hi, 0, 0x0123));
  }
};

__device__ __forceinline__ void load_huff(uint32_t* s) {
  const uint32_t* src = &kHuff.e[0][0];
  for (int i = threadIdx.x; i < 4 * 256; i += blockDim.x) s[i] = src[i];
  __syncthreads();
}

// Exclusive prefix sum over the CTA (blockDim.x a multiple of 32, at most 1024); *total gets the sum.  sh holds 33 ints.
__device__ __forceinline__ int64_t block_exclusive_scan(int64_t v, int64_t* sh, int64_t* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  int64_t incl = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int64_t t = __shfl_up_sync(0xFFFFFFFFu, incl, o);
    if (lane >= o) incl += t;
  }
  if (lane == 31) sh[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    int64_t s = lane < nw ? sh[lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int64_t t = __shfl_up_sync(0xFFFFFFFFu, s, o);
      if (lane >= o) s += t;
    }
    if (lane < nw) sh[lane] = s;
  }
  __syncthreads();
  const int64_t out = (warp ? sh[warp - 1] : 0) + incl - v;
  *total = sh[nw - 1];
  __syncthreads();
  return out;
}

// One CTA per image: every block's code length, and bitpos = their exclusive prefix sum (+ the total at the end).
__global__ void __launch_bounds__(kScanThreads) k_jenc_bits(const int16_t* __restrict__ coefs, Geometry geo,
                                                            int32_t* __restrict__ bitpos) {
  __shared__ uint32_t huff[4 * 256];
  __shared__ int64_t sh[33];
  load_huff(huff);
  const int64_t img = blockIdx.x;
  const int16_t* blocks = coefs + img * geo.blocks * 64;
  int32_t* pos = bitpos + img * (geo.blocks + 1);
  int64_t carry = 0;
  for (int64_t b0 = 0; b0 < geo.blocks; b0 += blockDim.x) {
    const int64_t b = b0 + threadIdx.x;
    CountBits c;
    if (b < geo.blocks) code_block(blocks, b, huff, c);
    int64_t total;
    const int64_t at = block_exclusive_scan(c.n, sh, &total);
    if (b < geo.blocks) pos[b] = (int32_t)(carry + at);
    carry += total;
  }
  if (threadIdx.x == 0) pos[geo.blocks] = (int32_t)carry;
}

// One thread per block: its codes at its bit position of its image's region (capw words each); the last block of an image
// also writes the padding, 1 bits to the end of the byte.
__global__ void __launch_bounds__(256) k_jenc_emit(const int16_t* __restrict__ coefs, const int32_t* __restrict__ bitpos,
                                                   int n, Geometry geo, int64_t capw, uint32_t* __restrict__ words) {
  __shared__ uint32_t huff[4 * 256];
  load_huff(huff);
  const int64_t total = (int64_t)n * geo.blocks;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (int64_t)gridDim.x * blockDim.x) {
    const int64_t img = g / geo.blocks, b = g - img * geo.blocks;
    const int32_t* pos = bitpos + img * (geo.blocks + 1);
    WriteBits wb(words + img * capw, __ldg(pos + b));
    code_block(coefs + img * geo.blocks * 64, b, huff, wb);
    if (b == geo.blocks - 1) {
      const int pad = -__ldg(pos + geo.blocks) & 7;
      wb.put((1u << pad) - 1, pad);
    }
    wb.flush();
  }
}

__device__ __forceinline__ int ff_bytes(uint32_t w) { return __popc(__vcmpeq4(w, 0xFFFFFFFFu)) >> 3; }

// One CTA per image: the scan's length after stuffing, its bytes plus one per 0xFF byte.
__global__ void __launch_bounds__(kScanThreads) k_jenc_count(const int32_t* __restrict__ bitpos, Geometry geo,
                                                             int64_t capw, const uint32_t* __restrict__ words,
                                                             int64_t* __restrict__ lens) {
  __shared__ int64_t sh[33];
  const int64_t img = blockIdx.x;
  const int64_t nbytes = ((int64_t)__ldg(bitpos + img * (geo.blocks + 1) + geo.blocks) + 7) >> 3;
  const uint32_t* w = words + img * capw;
  int64_t ff = 0;
  for (int64_t i = threadIdx.x; i < (nbytes + 3) >> 2; i += blockDim.x) ff += ff_bytes(__ldg(w + i));
  int64_t total;
  block_exclusive_scan(ff, sh, &total);
  if (threadIdx.x == 0) lens[img] = nbytes + total;
}

// One CTA per image: the scan's bytes at its offset (the stuffed lengths of the images before it), a 0x00 after every
// 0xFF; offsets[img] and, for the last image, offsets[n].
__global__ void __launch_bounds__(kScanThreads) k_jenc_pack(const int32_t* __restrict__ bitpos, int n, Geometry geo,
                                                            int64_t capw, const uint32_t* __restrict__ words,
                                                            const int64_t* __restrict__ lens, uint8_t* __restrict__ out,
                                                            int64_t* __restrict__ offsets) {
  __shared__ int64_t sh[33];
  const int64_t img = blockIdx.x;
  int64_t before = 0, start;
  for (int64_t j = threadIdx.x; j < img; j += blockDim.x) before += __ldg(lens + j);
  block_exclusive_scan(before, sh, &start);
  if (threadIdx.x == 0) {
    offsets[img] = start;
    if (img == n - 1) offsets[n] = start + __ldg(lens + img);
  }
  const int64_t nbytes = ((int64_t)__ldg(bitpos + img * (geo.blocks + 1) + geo.blocks) + 7) >> 3;
  const int64_t nwords = (nbytes + 3) >> 2;
  const uint32_t* w = words + img * capw;
  int64_t carry = start;
  for (int64_t w0 = 0; w0 < nwords; w0 += blockDim.x) {
    const int64_t i = w0 + threadIdx.x;
    const uint32_t v = i < nwords ? __ldg(w + i) : 0u;      // bytes past the scan are zero, never 0xFF
    int64_t total;
    int64_t at = carry + 4 * i + block_exclusive_scan(ff_bytes(v), sh, &total);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (i >= nwords || 4 * i + k >= nbytes) break;
      const uint8_t byte = (uint8_t)(v >> (8 * k));
      out[at + k] = byte;
      if (byte == 0xFF) out[++at + k] = 0;
    }
    carry += total;
  }
}

// the unstuffed scan of one image, in 32-bit words: every block at its worst case, and slack; even, so that the int64
// lengths after the n regions stay 8-byte aligned
int64_t image_words(const Geometry& g) { return g.blocks * (kMaxBlockBytes / 4) + 2; }

bool bad_shape(const char* who, int n, int h, int w) {
  if (n < 1 || h < 1 || w < 1 || h > 65535 || w > 65535 || (int64_t)h * w > (1ll << 25)) {
    fail(TWG_ERR_INVALID, "%s: n=%d h=%d w=%d (1 <= h, w <= 65535, h * w <= 2^25)", who, n, h, w);
    return true;
  }
  return false;
}

}  // namespace
}  // namespace twg

using namespace twg;

extern "C" {

int64_t twgjenc_workspace_bytes(int n, int h, int w) {
  if (bad_shape("twgjenc_workspace_bytes", n, h, w)) return TWG_ERR_INVALID;
  return (int64_t)n * image_words(geometry(h, w)) * 4 + (int64_t)n * 8;
}

int64_t twgjenc_scan_capacity(int n, int h, int w) {
  if (bad_shape("twgjenc_scan_capacity", n, h, w)) return TWG_ERR_INVALID;
  return (int64_t)n * image_words(geometry(h, w)) * 4 * 2;
}

int twgjenc_dct(const void* rgb, int n, int h, int w, const void* qt, void* coefs, twg_stream_t stream) {
  if (!rgb || !qt || !coefs) return fail(TWG_ERR_INVALID, "twgjenc_dct: null");
  if (bad_shape("twgjenc_dct", n, h, w)) return TWG_ERR_INVALID;
  if (reinterpret_cast<uintptr_t>(coefs) & 15) return fail(TWG_ERR_INVALID, "twgjenc_dct: coefs not 16-byte aligned");
  const Geometry g = geometry(h, w);
  k_jenc_dct<<<grid_for(n * g.blocks, 1), 256, 0, S(stream)>>>(static_cast<const uint8_t*>(rgb), n, g,
                                                                static_cast<const int32_t*>(qt),
                                                                static_cast<int16_t*>(coefs));
  return check_launch("twgjenc_dct");
}

int twgjenc_bits(const void* coefs, int n, int h, int w, void* bitpos, twg_stream_t stream) {
  if (!coefs || !bitpos) return fail(TWG_ERR_INVALID, "twgjenc_bits: null");
  if (bad_shape("twgjenc_bits", n, h, w)) return TWG_ERR_INVALID;
  if (reinterpret_cast<uintptr_t>(coefs) & 15) return fail(TWG_ERR_INVALID, "twgjenc_bits: coefs not 16-byte aligned");
  k_jenc_bits<<<n, kScanThreads, 0, S(stream)>>>(static_cast<const int16_t*>(coefs), geometry(h, w),
                                                 static_cast<int32_t*>(bitpos));
  return check_launch("twgjenc_bits");
}

int twgjenc_pack(const void* coefs, const void* bitpos, int n, int h, int w, void* workspace, void* out, void* offsets,
                 twg_stream_t stream) {
  if (!coefs || !bitpos || !workspace || !out || !offsets) return fail(TWG_ERR_INVALID, "twgjenc_pack: null");
  if (bad_shape("twgjenc_pack", n, h, w)) return TWG_ERR_INVALID;
  if ((reinterpret_cast<uintptr_t>(coefs) | reinterpret_cast<uintptr_t>(workspace)) & 15)
    return fail(TWG_ERR_INVALID, "twgjenc_pack: coefs and workspace must be 16-byte aligned");
  const Geometry g = geometry(h, w);
  const int64_t capw = image_words(g);
  uint32_t* words = static_cast<uint32_t*>(workspace);
  int64_t* lens = reinterpret_cast<int64_t*>(words + n * capw);
  if (cudaMemsetAsync(words, 0, sizeof(uint32_t) * (size_t)(n * capw), S(stream)) != cudaSuccess)
    return check_launch("twgjenc_pack: zeroing");
  const int16_t* c = static_cast<const int16_t*>(coefs);
  const int32_t* pos = static_cast<const int32_t*>(bitpos);
  k_jenc_emit<<<grid_for(n * g.blocks, 1), 256, 0, S(stream)>>>(c, pos, n, g, capw, words);
  k_jenc_count<<<n, kScanThreads, 0, S(stream)>>>(pos, g, capw, words, lens);
  k_jenc_pack<<<n, kScanThreads, 0, S(stream)>>>(pos, n, g, capw, words, lens, static_cast<uint8_t*>(out),
                                                 static_cast<int64_t*>(offsets));
  return check_launch("twgjenc_pack");
}

}  // extern "C"
