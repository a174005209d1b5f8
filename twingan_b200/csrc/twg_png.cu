// PNG decoding for image translation (twingan_b200/png.py picks the files and packs the descriptors): inflate (RFC 1950 /
// 1951) with the Adler-32 check, unfiltering (PNG 1.2 section 6) and PIL's convert('RGB') of each colour type and bit
// depth, each a kernel.  PNG is lossless, so the result is PIL's pixels exactly; tests/png_oracle.py restates the three
// stages in Python and numpy.
//
// A stream the kernels cannot decode exactly as zlib would (a corrupt or truncated one, one that inflates to the wrong
// size, one with trailing bytes) is flagged in its image's status word (bits TWG_PNG_*), never decoded differently: the
// caller decodes a flagged image on the host, where PIL decides.
#include "../../include/twgpng.h"
#include "twg_common.cuh"

namespace twg {

// descriptor row, int64 (twingan_b200/png.py IMAGE_FIELDS)
enum { P_START, P_END, P_RAW, P_RAW_BYTES, P_OUT, P_H, P_W, P_CTYPE, P_DEPTH, P_ROW_BYTES, P_PALETTE, P_PIX0, PNG_FIELDS };

// ---- inflate -------------------------------------------------------------------------------------------------------
//
// One warp per image.  Huffman decoding is serial, so every lane runs the same decoder on the same bits (the loads are
// broadcasts and the branches uniform); the lanes part only to build a block's tables and to copy: a back-reference
// is written by all 32 lanes at once, a literal by lane 0.

constexpr int kLut = 11;                     // primary table: every code of <= 11 bits, indexed by the next 11 bits
constexpr int kMaxBits = 15;
constexpr unsigned kFull = 0xffffffffu;

__constant__ uint16_t kLenBase[29] = {3,  4,  5,  6,  7,  8,  9,  10, 11,  13,  15,  17,  19,  23, 27,
                                      31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
__constant__ uint8_t kLenExtra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ uint16_t kDistBase[30] = {1,   2,   3,   4,   5,   7,    9,    13,   17,   25,   33,   49,   65,    97,    129,
                                       193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
__constant__ uint8_t kDistExtra[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
__constant__ uint8_t kClOrder[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

// One canonical Huffman code in shared memory: lut[bits] = length << 9 | symbol for codes of <= kLut bits (0: a longer
// code, or none), and the symbols sorted by (length, value) with the count of each length for longer codes (puff's
// decode, RFC 1951 3.2.2).
struct Huff {
  uint16_t lut[1 << kLut];
  uint16_t count[kMaxBits + 1];
  uint16_t first[kMaxBits + 1];            // first canonical code of each length
  uint16_t index[kMaxBits + 1];            // position in sym of the first symbol of each length
  uint16_t next[kMaxBits + 1];             // build's cursor into sym
  uint16_t sym[288];
};

// The bits of [p, end), least significant first.  Past the end the reader feeds zero bytes and counts their bits in
// `pad`; consuming one of them is a truncated stream.  Every byte read lies in [p, end).
struct Bits {
  const uint8_t* p;
  const uint8_t* end;
  uint64_t acc;
  int n, pad;
  bool trunc;

  // at least 33 bits in acc afterwards: four independent loads while the stream lasts, so one latency per 4 bytes
  __device__ __forceinline__ void fill() {
    if (n > 32) return;
    if (end - p >= 4) {
      const uint32_t w = __ldg(p) | __ldg(p + 1) << 8 | __ldg(p + 2) << 16 | (uint32_t)__ldg(p + 3) << 24;
      acc |= (uint64_t)w << n;
      p += 4;
      n += 32;
      return;
    }
    while (n <= 32) {
      uint64_t b = 0;
      if (p < end) {
        b = __ldg(p++);
      } else {
        pad += 8;
      }
      acc |= b << n;
      n += 8;
    }
  }
  // at least 57 bits in acc afterwards, a byte at a time (block headers only)
  __device__ __forceinline__ void fill_all() {
    while (n <= 56) {
      uint64_t b = 0;
      if (p < end) {
        b = __ldg(p++);
      } else {
        pad += 8;
      }
      acc |= b << n;
      n += 8;
    }
  }
  __device__ __forceinline__ void skip(int k) {
    acc >>= k;
    n -= k;
    if (n < pad) trunc = true;
  }
  __device__ __forceinline__ uint32_t take(int k) {     // k <= 32
    if (n < k) fill();
    const uint32_t v = (uint32_t)(acc & ((1ull << k) - 1));
    skip(k);
    return v;
  }
  // real bits left in acc
  __device__ __forceinline__ int real() const { return n - pad; }
};

// Builds `h` from the code lengths len[0..nsym).  Returns nonzero for a set zlib refuses: over-subscribed, or incomplete
// unless (outside the code-length code) it is a single code of length 1 or no code at all (inftrees.c); decoding with
// an empty set finds no symbol.
__device__ int build(Huff& h, const uint8_t* len, int nsym, bool code_lengths, int lane) {
  for (int i = lane; i < (1 << kLut); i += 32) h.lut[i] = 0;
  int bad = 0;
  if (lane == 0) {
    for (int l = 0; l <= kMaxBits; ++l) h.count[l] = 0;
    for (int s = 0; s < nsym; ++s) h.count[len[s]]++;
    int left = 1, maxl = 0, code = 0, idx = 0;
    for (int l = 1; l <= kMaxBits; ++l) {
      left = (left << 1) - h.count[l];
      if (left < 0) bad = 1;
      if (h.count[l]) maxl = l;
      h.first[l] = (uint16_t)code;
      h.index[l] = (uint16_t)idx;
      code = (code + h.count[l]) << 1;
      idx += h.count[l];
    }
    if (!bad && left > 0 && (code_lengths || maxl > 1)) bad = 1;
    for (int l = 1; l <= kMaxBits; ++l) h.next[l] = h.index[l];
    for (int s = 0; s < nsym; ++s)
      if (len[s]) h.sym[h.next[len[s]]++] = (uint16_t)s;
  }
  bad = __shfl_sync(kFull, bad, 0);
  __syncwarp();
  if (bad) return bad;
  const int ncoded = nsym - h.count[0];
  for (int k = lane; k < ncoded; k += 32) {
    const int s = h.sym[k];
    const int l = len[s];
    if (l > kLut) continue;
    const uint32_t code = h.first[l] + (k - h.index[l]);
    const uint32_t rev = __brev(code) >> (32 - l);
    for (uint32_t j = rev; j < (1u << kLut); j += 1u << l) h.lut[j] = (uint16_t)(l << 9 | s);
  }
  __syncwarp();
  return 0;
}

// the next symbol of `h` (b.acc holds >= kMaxBits bits); -1 when the bits are no code of it
__device__ __forceinline__ int decode(const Huff& h, Bits& b) {
  const int e = h.lut[b.acc & ((1u << kLut) - 1)];
  if (e) {
    b.skip(e >> 9);
    return e & 511;
  }
  // a longer code, or none: the l-bit code is the next l bits reversed (RFC 1951 3.1.1); it is a code of length l
  // when it falls among that length's count[l] consecutive codes from first[l]
  const uint32_t rev = __brev((uint32_t)b.acc);
#pragma unroll
  for (int l = kLut + 1; l <= kMaxBits; ++l) {
    const int code = (int)(rev >> (32 - l)) - h.first[l];
    if (code >= 0 && code < h.count[l]) {
      b.skip(l);
      return h.sym[h.index[l] + code];
    }
  }
  return -1;
}

// a code of no symbol: truncated when fewer than kMaxBits real bits remained to read it, else a bad code
__device__ __forceinline__ int no_code(const Bits& b) { return b.real() < kMaxBits ? TWG_PNG_TRUNCATED : TWG_PNG_SYMBOL; }

__device__ int inflate_stream(const uint8_t* __restrict__ src, const uint8_t* __restrict__ src_end,
                              uint8_t* __restrict__ out, int64_t size, int64_t& pos, uint32_t& trailer, Huff& lit,
                              Huff& dist, uint8_t* lens, int lane) {
  Bits b{src, src_end, 0ull, 0, 0, false};
  b.fill();
  const uint32_t cmf = b.take(8), flg = b.take(8);
  if (b.trunc) return TWG_PNG_TRUNCATED;
  if ((cmf & 15) != 8 || (cmf >> 4) > 7 || (cmf * 256 + flg) % 31 || (flg & 0x20)) return TWG_PNG_HEADER;
  const int64_t window = 1ll << ((cmf >> 4) + 8);
  pos = 0;
  bool last = false;
  while (!last) {
    b.fill();
    last = b.take(1);
    const int type = b.take(2);
    if (b.trunc) return TWG_PNG_TRUNCATED;
    if (type == 3) return TWG_PNG_BLOCK;
    if (type == 0) {                                  // stored
      b.skip(b.n & 7);
      const uint32_t len = b.take(16), nlen = b.take(16);
      if (b.trunc) return TWG_PNG_TRUNCATED;
      if (len != (~nlen & 0xffff)) return TWG_PNG_BLOCK;
      const uint8_t* q = b.p - (b.real() >> 3);       // the next byte of the stream
      if (len > src_end - q) return TWG_PNG_TRUNCATED;
      if (pos + len > size) return TWG_PNG_LONG;
      for (uint32_t i = lane; i < len; i += 32) out[pos + i] = __ldg(q + i);
      __syncwarp();
      pos += len;
      b = Bits{q + len, src_end, 0ull, 0, 0, false};
      continue;
    }
    if (type == 1) {                                  // fixed codes
      for (int s = lane; s < 288 + 32; s += 32)
        lens[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : s < 288 ? 8 : 5;
      __syncwarp();
      build(lit, lens, 288, false, lane);
      build(dist, lens + 288, 32, false, lane);
    } else {                                          // dynamic codes: the code-length code, then the two sets
      const int nlit = b.take(5) + 257, ndist = b.take(5) + 1, ncl = b.take(4) + 4;
      if (b.trunc) return TWG_PNG_TRUNCATED;
      if (nlit > 286 || ndist > 30) return TWG_PNG_CODES;
      b.fill_all();                                   // 3 * 19 <= 57 bits: lane i takes code length i
      if (lane < 19) lens[kClOrder[lane]] = lane < ncl ? (uint8_t)((b.acc >> (3 * lane)) & 7) : 0;
      b.skip(3 * ncl);
      if (b.trunc) return TWG_PNG_TRUNCATED;
      __syncwarp();
      if (build(lit, lens, 19, true, lane)) return TWG_PNG_CODES;
      int k = 0;
      uint8_t prev = 0;
      while (k < nlit + ndist) {
        b.fill();
        const int s = decode(lit, b);
        if (s < 0) return no_code(b);
        if (b.trunc) return TWG_PNG_TRUNCATED;
        int rep = 1;
        uint8_t v = (uint8_t)s;
        if (s == 16) {
          if (k == 0) return TWG_PNG_CODES;
          rep = 3 + b.take(2);
          v = prev;
        } else if (s == 17) {
          rep = 3 + b.take(3);
          v = 0;
        } else if (s == 18) {
          rep = 11 + b.take(7);
          v = 0;
        }
        if (b.trunc) return TWG_PNG_TRUNCATED;
        if (k + rep > nlit + ndist) return TWG_PNG_CODES;
        if (lane < rep) lens[k + lane] = v;            // rep <= 138: five rounds at most
        if (lane + 32 < rep) lens[k + lane + 32] = v;
        if (lane + 64 < rep) lens[k + lane + 64] = v;
        if (lane + 96 < rep) lens[k + lane + 96] = v;
        if (lane + 128 < rep) lens[k + lane + 128] = v;
        k += rep;
        prev = v;
      }
      __syncwarp();
      if (lens[256] == 0) return TWG_PNG_CODES;
      if (build(lit, lens, nlit, false, lane)) return TWG_PNG_CODES;
      if (build(dist, lens + nlit, ndist, false, lane)) return TWG_PNG_CODES;
    }
    for (;;) {                                        // the block's symbols
      b.fill();
      const int s = decode(lit, b);
      if (s < 0) return no_code(b);
      if (b.trunc) return TWG_PNG_TRUNCATED;
      if (s < 256) {
        if (pos >= size) return TWG_PNG_LONG;
        if (lane == 0) out[pos] = (uint8_t)s;
        ++pos;
        continue;
      }
      if (s == 256) break;
      if (s > 285) return TWG_PNG_SYMBOL;
      const int len = kLenBase[s - 257] + b.take(kLenExtra[s - 257]);
      b.fill();
      const int d = decode(dist, b);
      if (d < 0) return no_code(b);
      if (b.trunc) return TWG_PNG_TRUNCATED;
      if (d > 29) return TWG_PNG_SYMBOL;
      const int64_t off = kDistBase[d] + b.take(kDistExtra[d]);
      if (b.trunc) return TWG_PNG_TRUNCATED;
      if (off > pos || off > window) return TWG_PNG_DISTANCE;
      if (pos + len > size) return TWG_PNG_LONG;
      __syncwarp();                                   // the bytes copied were written by other lanes
      // out[pos + i] = out[pos + i - off] = ... = from[i % off]: every byte read was written before the copy
      const uint8_t* from = out + pos - off;
      if (off >= len) {
        for (int i = lane; i < len; i += 32) out[pos + i] = from[i];
      } else {                                        // a repeating pattern: off < len <= 258
        const int period = (int)off, step = 32 % period;
        int j = lane % period;
        for (int i = lane; i < len; i += 32) {
          out[pos + i] = from[j];
          j += step;
          if (j >= period) j -= period;
        }
      }
      pos += len;
    }
  }
  b.skip(b.n & 7);                                    // the Adler-32 trailer, big-endian, on a byte boundary
  trailer = 0;
  for (int i = 0; i < 4; ++i) trailer = trailer << 8 | b.take(8);
  if (b.trunc) return TWG_PNG_TRUNCATED;
  int st = 0;
  if (pos < size) st |= TWG_PNG_SHORT;
  if (b.p < src_end || b.real() > 0) st |= TWG_PNG_TRAILING;
  return st;
}

// Adler-32 of out[0, n): s1 = 1 + sum d_i, s2 = n + sum (n - i) d_i (mod 65521).  Lane j adds the bytes j, j + 32, ...
// with the weight (n - i) mod 65521 carried down by 32 per step, into 64-bit sums that cannot overflow (each term is
// < 2^24, at most 2^26 terms per lane between reductions); the lanes' sums are combined by a fixed shuffle tree.
__device__ uint32_t adler32(const uint8_t* out, int64_t n, int lane) {
  constexpr uint32_t M = 65521;
  uint64_t s1 = 0, s2 = 0;
  int64_t w = (n - lane) % M;
  int64_t steps = 0;
  for (int64_t i = lane; i < n; i += 32) {
    const uint32_t d = out[i];
    s1 += d;
    s2 += (uint64_t)w * d;
    w -= 32;
    if (w < 0) w += M;
    if (++steps == (1 << 26)) {
      s1 %= M;
      s2 %= M;
      steps = 0;
    }
  }
  s1 %= M;
  s2 %= M;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s1 += __shfl_xor_sync(kFull, s1, o);
    s2 += __shfl_xor_sync(kFull, s2, o);
  }
  s1 = (1 + s1) % M;
  s2 = (n % M + s2) % M;
  return (uint32_t)(s2 << 16 | s1);
}

__global__ void __launch_bounds__(32) k_png_inflate(const uint8_t* __restrict__ data, const int64_t* __restrict__ images,
                                                    uint8_t* __restrict__ raw, int* __restrict__ status) {
  __shared__ Huff lit, dist;
  __shared__ uint8_t lens[288 + 32];
  const int lane = threadIdx.x;
  const int64_t* im = images + (int64_t)blockIdx.x * PNG_FIELDS;
  const int64_t size = im[P_RAW_BYTES];
  uint8_t* out = raw + im[P_RAW];
  int64_t pos = 0;
  uint32_t trailer = 0;
  int st = inflate_stream(data + im[P_START], data + im[P_END], out, size, pos, trailer, lit, dist, lens, lane);
  if (!(st & ~(TWG_PNG_SHORT | TWG_PNG_TRAILING))) {     // the stream ended where it should: check its sum
    __syncwarp();
    if (adler32(out, pos, lane) != trailer) st |= TWG_PNG_ADLER;
  }
  if (lane == 0 && st) status[blockIdx.x] = st;
}

// ---- unfiltering ---------------------------------------------------------------------------------------------------

__device__ __forceinline__ int paeth(int a, int b, int c) {
  const int p = a + b - c, pa = abs(p - a), pb = abs(p - b), pc = abs(p - c);
  return (pa <= pb && pa <= pc) ? a : pb <= pc ? b : c;
}

// One CTA per image, rows in order, in place.  None and Up are parallel across the row; Sub, Average and Paeth run
// along the row in `bpp` lanes, one per byte of a pixel.
__global__ void __launch_bounds__(128) k_png_unfilter(uint8_t* __restrict__ raw, const int64_t* __restrict__ images,
                                                      int* __restrict__ status) {
  const int64_t* im = images + (int64_t)blockIdx.x * PNG_FIELDS;
  if (status[blockIdx.x]) return;
  const int64_t H = im[P_H], rb = im[P_ROW_BYTES];
  const int ct = (int)im[P_CTYPE], depth = (int)im[P_DEPTH];
  const int chans = ct == 0 || ct == 3 ? 1 : ct == 2 ? 3 : ct == 4 ? 2 : 4;
  const int bpp = max(1, chans * depth / 8);
  const int t = threadIdx.x;
  uint8_t* row = raw + im[P_RAW];
  const uint8_t* up = nullptr;                       // the row above, unfiltered (none above the first)
  for (int64_t y = 0; y < H; ++y) {
    const int f = row[0];
    if (f > 4) {
      if (t == 0) status[blockIdx.x] = TWG_PNG_FILTER;
      return;
    }
    uint8_t* x = row + 1;
    if (f == 2 && up) {
      for (int64_t i = t; i < rb; i += blockDim.x) x[i] = (uint8_t)(x[i] + up[i]);
    } else if ((f == 1 || f == 3 || f == 4) && t < bpp) {
      int a = 0, c = 0;
      int64_t i = t;
      // eight pixels' loads issued before their chain, which then runs in registers
      for (; i + 7 * bpp < rb; i += 8 * bpp) {
        int xs[8], bs[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          xs[k] = x[i + k * bpp];
          bs[k] = up ? up[i + k * bpp] : 0;
        }
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const int pred = f == 1 ? a : f == 3 ? (a + bs[k]) >> 1 : paeth(a, bs[k], c);
          a = (uint8_t)(xs[k] + pred);
          x[i + k * bpp] = (uint8_t)a;
          c = bs[k];
        }
      }
      for (; i < rb; i += bpp) {
        const int b = up ? up[i] : 0;
        const int pred = f == 1 ? a : f == 3 ? (a + b) >> 1 : paeth(a, b, c);
        a = (uint8_t)(x[i] + pred);
        x[i] = (uint8_t)a;
        c = b;
      }
    }
    __syncthreads();
    up = x;
    row += rb + 1;
  }
}

// ---- convert('RGB') ------------------------------------------------------------------------------------------------

// sample k of a row of `depth`-bit samples (most significant first within a byte; 16-bit: big-endian)
__device__ __forceinline__ uint32_t sample(const uint8_t* r, int64_t k, int depth) {
  if (depth == 8) return __ldg(r + k);
  if (depth == 16) return (uint32_t)__ldg(r + 2 * k) << 8 | __ldg(r + 2 * k + 1);
  const int64_t bit = k * depth;
  return (__ldg(r + (bit >> 3)) >> (8 - depth - (int)(bit & 7))) & ((1u << depth) - 1);
}

// One thread per output pixel of the batch's PNG images, uint8 RGB at the image's payload offset.
__global__ void __launch_bounds__(256) k_png_rgb(const uint8_t* __restrict__ raw, const int64_t* __restrict__ images,
                                                 int nimages, const uint8_t* __restrict__ palettes, int64_t npix,
                                                 const int* __restrict__ status, uint8_t* __restrict__ payload) {
  for (int64_t P = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; P < npix; P += (int64_t)gridDim.x * blockDim.x) {
    int lo = 0, hi = nimages - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (__ldg(images + (int64_t)mid * PNG_FIELDS + P_PIX0) <= P) lo = mid; else hi = mid - 1;
    }
    if (__ldg(status + lo)) continue;
    const int64_t* im = images + (int64_t)lo * PNG_FIELDS;
    const int64_t W = __ldg(im + P_W), rb = __ldg(im + P_ROW_BYTES);
    const int ct = (int)__ldg(im + P_CTYPE), depth = (int)__ldg(im + P_DEPTH);
    const int64_t r = P - __ldg(im + P_PIX0);
    const int64_t y = r / W, x = r - y * W;
    const uint8_t* row = raw + __ldg(im + P_RAW) + y * (rb + 1) + 1;
    uint32_t R, G, B;
    if (ct == 0) {                                     // grey: L;1 L;2 L;4 scale to 0..255, I;16 clamps to 255
      const uint32_t v = sample(row, x, depth);
      R = depth == 16 ? min(v, 255u) : depth == 8 ? v : v * (255u / ((1u << depth) - 1));
      G = B = R;
    } else if (ct == 3) {
      const uint8_t* p = palettes + __ldg(im + P_PALETTE) * 768 + 3 * sample(row, x, depth);
      R = __ldg(p);
      G = __ldg(p + 1);
      B = __ldg(p + 2);
    } else {                                           // RGB, LA, RGBA: channel 0 (grey) or 0..2, high byte of 16 bits
      const int chans = ct == 2 ? 3 : ct == 4 ? 2 : 4, step = depth / 8;
      const uint8_t* px = row + x * chans * step;
      R = __ldg(px);
      G = ct == 4 ? R : __ldg(px + step);
      B = ct == 4 ? R : __ldg(px + 2 * step);
    }
    uint8_t* o = payload + __ldg(im + P_OUT) + r * 3;
    o[0] = (uint8_t)R;
    o[1] = (uint8_t)G;
    o[2] = (uint8_t)B;
  }
}

}  // namespace twg

using namespace twg;

extern "C" {

int twgpng_inflate(const void* data, const int64_t* images, int nimages, void* raw, void* status, twg_stream_t stream) {
  if (!data || !images || !raw || !status) return fail(TWG_ERR_INVALID, "twgpng_inflate: null");
  if (nimages < 1) return fail(TWG_ERR_INVALID, "twgpng_inflate: nimages=%d", nimages);
  if (cudaMemsetAsync(status, 0, sizeof(int) * (size_t)nimages, S(stream)) != cudaSuccess)
    return check_launch("twgpng_inflate: status reset");
  k_png_inflate<<<nimages, 32, 0, S(stream)>>>(static_cast<const uint8_t*>(data), images, static_cast<uint8_t*>(raw),
                                               static_cast<int*>(status));
  return check_launch("twgpng_inflate");
}

int twgpng_unfilter(void* raw, const int64_t* images, int nimages, void* status, twg_stream_t stream) {
  if (!raw || !images || !status) return fail(TWG_ERR_INVALID, "twgpng_unfilter: null");
  if (nimages < 1) return fail(TWG_ERR_INVALID, "twgpng_unfilter: nimages=%d", nimages);
  k_png_unfilter<<<nimages, 128, 0, S(stream)>>>(static_cast<uint8_t*>(raw), images, static_cast<int*>(status));
  return check_launch("twgpng_unfilter");
}

int twgpng_rgb(const void* raw, const int64_t* images, int nimages, const void* palettes, int64_t npixels,
               const void* status, void* payload, twg_stream_t stream) {
  if (!raw || !images || !palettes || !status || !payload) return fail(TWG_ERR_INVALID, "twgpng_rgb: null");
  if (nimages < 1 || npixels < 1)
    return fail(TWG_ERR_INVALID, "twgpng_rgb: nimages=%d npixels=%lld", nimages, (long long)npixels);
  k_png_rgb<<<grid_for(npixels, 4), 256, 0, S(stream)>>>(static_cast<const uint8_t*>(raw), images, nimages,
                                                         static_cast<const uint8_t*>(palettes), npixels,
                                                         static_cast<const int*>(status),
                                                         static_cast<uint8_t*>(payload));
  return check_launch("twgpng_rgb");
}

}  // extern "C"
