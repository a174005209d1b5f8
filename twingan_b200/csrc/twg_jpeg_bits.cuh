// Device pieces shared by the baseline (twg_jpeg.cu) and progressive (twg_jpegp.cu) JPEG decoders: the descriptor row
// layouts of twingan_b200/jpeg.py, the zig-zag order, the bit reader of an entropy-coded segment and Huffman decoding.
#pragma once
#include <assert.h>
#include <stdint.h>

#include "../../include/twgjpeg.h"

namespace twg {

// descriptor rows, int64 (twingan_b200/jpeg.py SEG_FIELDS / COMP_FIELDS / IMAGE_FIELDS)
enum { SEG_START, SEG_END, SEG_IMAGE, SEG_MCU0, SEG_MCUS, SEG_INDEX, SEG_FIELDS };
enum { C_BLOCK0, C_BW, C_BH, C_PLANE, C_QT, C_DC, C_AC, C_H, C_V, C_IMAGE, COMP_FIELDS };
enum { I_COMP0, I_NCOMP, I_MCUX, I_H, I_W, I_OUT, I_PIX0, I_NSEG, I_HMAX, I_VMAX, I_PAD0, I_PAD1, IMAGE_FIELDS };
// one Huffman table, int32: lut[512] | maxcode[18] | valoff[18] | vals[256] (jpeg.huff_table)
constexpr int kLutBits = 9, kMaxcode = 512, kValoff = 530, kVals = 548, kHuffWords = 1024;

// natural (row-major) position of the k-th coefficient in zig-zag order; called with constant k only
__host__ __device__ constexpr int natural_of(int k) {
  constexpr int t[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                         41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                         30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
  return t[k];
}

// ---- entropy decoding ----------------------------------------------------------------------------------------------

// The bits of one segment [p, end), MSB first in `acc`, FF 00 unstuffed.  Past the end the reader feeds zero bytes and
// counts them in `pad`; consuming one of them is a truncated segment.  Every byte read lies in [p, end).
struct Bits {
  const uint8_t* p;
  const uint8_t* end;
  uint64_t acc;
  int n, pad, err;

  __device__ __forceinline__ uint32_t byte_at(const uint8_t* q) const {
    assert(q < end);
    return __ldg(q);
  }

  // at least 57 bits in acc afterwards
  __device__ __forceinline__ void fill() {
    while (n <= 56) {
      uint32_t b = 0;
      bool real = false;
      if (p < end) {
        b = byte_at(p++);
        real = true;
        if (b == 0xFF) {
          if (p < end && byte_at(p) == 0) {
            ++p;
          } else {                      // a marker inside the segment
            err |= TWG_JPEG_MARKER;
            b = 0;
            real = false;
            p = end;
          }
        }
      }
      if (!real) pad += 8;
      acc |= (uint64_t)b << (56 - n);
      n += 8;
    }
  }

  __device__ __forceinline__ void skip(int len) {
    acc <<= len;
    n -= len;
    if (n < pad) err |= TWG_JPEG_TRUNCATED;
  }

  __device__ __forceinline__ int take(int s) {
    const int v = s ? (int)(acc >> (64 - s)) : 0;
    skip(s);
    return v;
  }

  // one Huffman symbol (acc holds >= 16 bits): the 9-bit table, else the canonical code lengths 10..16 (T.81 F.2.2.3)
  __device__ __forceinline__ int symbol(const int32_t* __restrict__ t) {
    const int e = __ldg(t + (int)(acc >> (64 - kLutBits)));
    if (e) {
      skip(e >> 8);
      return e & 255;
    }
    for (int l = kLutBits + 1; l <= 16; ++l) {
      const int code = (int)(acc >> (64 - l));
      if (code <= __ldg(t + kMaxcode + l)) {
        skip(l);
        return __ldg(t + kVals + code + __ldg(t + kValoff + l));
      }
    }
    err |= TWG_JPEG_BAD_CODE;
    return 0;
  }
};

// HUFF_EXTEND of T.81 F.2.2.1: the s-bit value v as a signed coefficient
__device__ __forceinline__ int extend(int v, int s) { return (s && v < (1 << (s - 1))) ? v - (1 << s) + 1 : v; }

}  // namespace twg
