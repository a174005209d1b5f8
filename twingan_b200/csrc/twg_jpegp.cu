// Progressive JPEG entropy decoding for image translation (twingan_b200/jpeg_progressive.py picks the files, orders the
// scans in levels and packs the descriptors): the four scan kinds of ITU-T T.81 G.1.2 with Huffman coding, into the
// zig-zag int16 coefficient blocks the baseline inverse DCT and colour kernels (twg_jpeg.cu) read.  The decoding of each
// kind is that of T.81 G.2 as libjpeg-turbo's jdphuff.c (PIL's decoder) carries it out; tests/jpegp_oracle.py restates it
// bit by bit.
//
// A stream the kernel does not restate exactly is flagged in its image's status word (TWG_JPEG_* / TWG_JPEGP_* bits),
// never decoded differently: the caller decodes a flagged image on the host.
#include "../../include/twgjpegp.h"
#include "twg_common.cuh"
#include "twg_jpeg_bits.cuh"

namespace twg {

// scan rows, int64 (twingan_b200/jpeg_progressive.py SCAN_FIELDS); a segment row's SEG_INDEX field holds its scan row
// and the field after SEG_MCUS the marker that must follow it
enum { S_IMAGE, S_SS, S_SE, S_AH, S_AL, S_NCOMP, S_COMP0, S_TBL0 = S_COMP0 + 3, S_GRIDW = S_TBL0 + 3, S_RI, S_LEVEL,
       S_PAD, SCAN_FIELDS };
enum { SEG_SCAN = SEG_IMAGE, SEG_MARKER = SEG_INDEX };

__device__ __forceinline__ bool outside_int16(int v) { return v < -32768 || v > 32767; }

// decode_mcu_DC_first / decode_mcu_DC_refine of one block: the difference from the component's prediction, << Al; or
// one raw bit of precision Al
__device__ __forceinline__ void dc_block(Bits& b, const int32_t* __restrict__ t, int16_t* blk, int ah, int al,
                                         int& pred) {
  b.fill();
  if (ah) {
    if (b.take(1)) blk[0] = (int16_t)(blk[0] | (1 << al));
    return;
  }
  const int s = b.symbol(t);
  pred += extend(b.take(s), s);
  const int val = pred * (1 << al);
  if (outside_int16(pred) || outside_int16(val)) b.err |= TWG_JPEGP_VALUE_RANGE;
  blk[0] = (int16_t)val;
}

// decode_mcu_AC_first of one block: the band Ss..Se at precision Al, or one block of a pending end-of-band run
__device__ __forceinline__ void ac_first(Bits& b, const int32_t* __restrict__ t, int16_t* blk, int ss, int se, int al,
                                         int& eobrun) {
  if (eobrun > 0) {
    --eobrun;
    return;
  }
  for (int k = ss; k <= se && !b.err; ++k) {
    b.fill();
    const int rs = b.symbol(t);
    const int r = rs >> 4, sz = rs & 15;
    if (sz) {
      k += r;
      if (k > se) {
        b.err |= TWG_JPEGP_BAND;
        return;
      }
      const int v = extend(b.take(sz), sz) * (1 << al);
      if (outside_int16(v)) {
        b.err |= TWG_JPEGP_VALUE_RANGE;
        return;
      }
      blk[k] = (int16_t)v;
    } else if (r == 15) {
      k += 15;                          // ZRL: sixteen zeros
    } else {
      eobrun = (1 << r) + b.take(r) - 1;  // EOBr: this block and 2^r + bits - 1 more end here
      return;
    }
  }
}

// one correction bit of a coefficient already nonzero: its magnitude gains 1 << Al when the bit is set
__device__ __forceinline__ void correct(Bits& b, int16_t* c, int p1) {
  b.fill();
  if (b.take(1) && (*c & p1) == 0) {
    const int v = *c >= 0 ? *c + p1 : *c - p1;
    if (outside_int16(v)) b.err |= TWG_JPEGP_VALUE_RANGE;
    *c = (int16_t)v;
  }
}

// decode_mcu_AC_refine of one block: new coefficients of +-(1 << Al), correction bits of the nonzero ones
__device__ __forceinline__ void ac_refine(Bits& b, const int32_t* __restrict__ t, int16_t* blk, int ss, int se, int al,
                                          int& eobrun) {
  const int p1 = 1 << al;
  int k = ss;
  if (eobrun == 0) {
    for (; k <= se && !b.err; ++k) {
      b.fill();
      const int rs = b.symbol(t);
      int r = rs >> 4, s = rs & 15;
      if (s) {
        if (s != 1) {
          b.err |= TWG_JPEGP_REFINE_SIZE;
          return;
        }
        b.fill();
        s = b.take(1) ? p1 : -p1;
      } else if (r != 15) {
        eobrun = (1 << r) + b.take(r);
        break;
      }
      do {                              // skip r zero coefficients (stop at the next), correcting the nonzero ones
        if (blk[k] != 0) {
          correct(b, blk + k, p1);
        } else if (--r < 0) {
          break;
        }
        ++k;
      } while (k <= se && !b.err);
      if (s) {
        if (k > se) {
          b.err |= TWG_JPEGP_BAND;
          return;
        }
        blk[k] = (int16_t)s;
      }
    }
  }
  if (eobrun > 0) {                     // the rest of the band lies in an end-of-band run: corrections only
    for (; k <= se && !b.err; ++k)
      if (blk[k] != 0) correct(b, blk + k, p1);
    --eobrun;
  }
}

enum { kDC, kFirst, kRefine };

// the blocks [m0, m1) of a one-component scan's grid, `gridw` blocks wide (m0 at row by, column bx), in a plane `bw`
// blocks wide from c0; returns the segment's status bits
template <int kind>
__device__ __forceinline__ int one_component(Bits& b, const int32_t* __restrict__ t, int16_t* c0, int64_t bw,
                                             int64_t gridw, int64_t m0, int64_t m1, int64_t by,
                                             int64_t bx, int ss, int se, int ah, int al) {
  int pred = 0, eobrun = 0;
  for (int64_t m = m0; m < m1 && !b.err; ++m, bx = bx + 1 == gridw ? 0 : bx + 1, by += bx == 0) {
    int16_t* blk = c0 + (by * bw + bx) * 64;
    if (kind == kDC)
      dc_block(b, t, blk, ah, al, pred);
    else if (kind == kFirst)
      ac_first(b, t, blk, ss, se, al, eobrun);
    else
      ac_refine(b, t, blk, ss, se, al, eobrun);
  }
  return b.err;
}

// One thread per segment of one level; `spw` segments per warp (lanes >= spw idle), as k_jpeg_entropy.
__global__ void __launch_bounds__(128, 1) k_jpegp_entropy(const uint8_t* __restrict__ data,
                                                       const int64_t* __restrict__ segs, int nseg, int spw,
                                                       const int64_t* __restrict__ scans,
                                                       const int64_t* __restrict__ comps,
                                                       const int32_t* __restrict__ huff, int16_t* __restrict__ coef,
                                                       int* __restrict__ status) {
  const int gid = blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = gid & 31;
  const int s = (gid >> 5) * spw + lane;
  if (lane >= spw || s >= nseg) return;
  const int64_t* sg = segs + (int64_t)s * SEG_FIELDS;
  const int64_t* sc = scans + sg[SEG_SCAN] * SCAN_FIELDS;
  const int img = (int)sc[S_IMAGE];
  const int ss = (int)sc[S_SS], se = (int)sc[S_SE], ah = (int)sc[S_AH], al = (int)sc[S_AL];
  const int ns = (int)sc[S_NCOMP];
  const int64_t gridw = sc[S_GRIDW];
  Bits b{data + sg[SEG_START], data + sg[SEG_END], 0ull, 0, 0, 0};
  const uint8_t* term = data + sg[SEG_END];
  int err = (__ldg(term) != 0xFF || __ldg(term + 1) != (uint32_t)sg[SEG_MARKER]) ? TWG_JPEG_RESTART : 0;
  const int64_t m0 = sg[SEG_MCU0], m1 = m0 + sg[SEG_MCUS];
  // the segment's first MCU (or block) in its grid; a component has fewer than 2^26 blocks
  const int64_t y0 = (int)m0 / (int)gridw, x0 = m0 - y0 * gridw;
  if (ns == 1) {                          // one component: one block per MCU, in its own grid (T.81 A.2.2)
    const int64_t* cp = comps + sc[S_COMP0] * COMP_FIELDS;
    int16_t* c0 = coef + cp[C_BLOCK0] * 64;
    const int32_t* t = huff + max(sc[S_TBL0], (int64_t)0) * kHuffWords;
    if (ss == 0)
      err |= one_component<kDC>(b, t, c0, cp[C_BW], gridw, m0, m1, y0, x0, ss, se, ah, al);
    else if (ah == 0)
      err |= one_component<kFirst>(b, t, c0, cp[C_BW], gridw, m0, m1, y0, x0, ss, se, ah, al);
    else
      err |= one_component<kRefine>(b, t, c0, cp[C_BW], gridw, m0, m1, y0, x0, ss, se, ah, al);
  } else {                                // interleaved (DC scans only): each component's h x v blocks of every MCU
    int pred0 = 0, pred1 = 0, pred2 = 0;
    int64_t my = y0, mx = x0;
    for (int64_t m = m0; m < m1 && !err; ++m, mx = mx + 1 == gridw ? 0 : mx + 1, my += mx == 0) {
      for (int c = 0; c < ns && !err; ++c) {
        const int64_t* cp = comps + __ldg(sc + S_COMP0 + c) * COMP_FIELDS;
        const int64_t bw = __ldg(cp + C_BW);
        const int h = (int)__ldg(cp + C_H), v = (int)__ldg(cp + C_V);
        int16_t* c0 = coef + (__ldg(cp + C_BLOCK0) + my * v * bw + mx * h) * 64;
        const int32_t* t = huff + max((int64_t)__ldg(sc + S_TBL0 + c), (int64_t)0) * kHuffWords;
        int pred = c == 0 ? pred0 : c == 1 ? pred1 : pred2;
        for (int by = 0; by < v && !b.err; ++by)
          for (int bx = 0; bx < h && !b.err; ++bx) dc_block(b, t, c0 + (by * bw + bx) * 64, ah, al, pred);
        if (c == 0) pred0 = pred; else if (c == 1) pred1 = pred; else pred2 = pred;
        err |= b.err;
      }
    }
  }
  if (err) atomicOr(status + img, err);
}

}  // namespace twg

using namespace twg;

extern "C" {

int twgjpegp_reset(void* coefs, int64_t nblocks, void* status, int nimages, twg_stream_t stream) {
  if (!coefs || !status) return fail(TWG_ERR_INVALID, "twgjpegp_reset: null");
  if (nblocks < 1 || nimages < 1)
    return fail(TWG_ERR_INVALID, "twgjpegp_reset: nblocks=%lld nimages=%d", (long long)nblocks, nimages);
  if (reinterpret_cast<uintptr_t>(coefs) & 15) return fail(TWG_ERR_INVALID, "twgjpegp_reset: coefs not 16-byte aligned");
  if (cudaMemsetAsync(coefs, 0, sizeof(int16_t) * 64 * (size_t)nblocks, S(stream)) != cudaSuccess ||
      cudaMemsetAsync(status, 0, sizeof(int) * (size_t)nimages, S(stream)) != cudaSuccess)
    return check_launch("twgjpegp_reset");
  return 0;
}

int twgjpegp_entropy(const void* data, const int64_t* segs, int nseg, const int64_t* scans, const int64_t* comps,
                     const void* huff, void* coefs, void* status, twg_stream_t stream) {
  if (!data || !segs || !scans || !comps || !huff || !coefs || !status)
    return fail(TWG_ERR_INVALID, "twgjpegp_entropy: null");
  if (nseg < 1) return fail(TWG_ERR_INVALID, "twgjpegp_entropy: nseg=%d", nseg);
  // few segments: one per warp, so that each runs alone; many: up to 32 per warp
  int spw = 1;
  while (spw < 32 && cdiv(nseg, spw) > (int64_t)kNumSMs * 32) spw *= 2;
  const int64_t threads = cdiv(nseg, spw) * 32;
  k_jpegp_entropy<<<(unsigned)cdiv(threads, 128), 128, 0, S(stream)>>>(
      static_cast<const uint8_t*>(data), segs, nseg, spw, scans, comps, static_cast<const int32_t*>(huff),
      static_cast<int16_t*>(coefs), static_cast<int*>(status));
  return check_launch("twgjpegp_entropy");
}

}  // extern "C"
