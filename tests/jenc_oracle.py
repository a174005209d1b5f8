"""Integer restatement of the device JPEG encoder (twingan_b200/csrc/twg_jenc.cu), stage by stage, in numpy.

The target is the file PIL writes for `Image.fromarray(rgb).save(f, 'JPEG')`: libjpeg-turbo at its defaults (baseline,
quality 75, 4:2:0, Annex K Huffman tables, islow forward DCT).  Written from ITU-T T.81 and libjpeg's published integer
algorithms:
  * `rgb_to_ycc`: jccolor.c rgb_ycc_convert, 16-bit fixed point, ONE_HALF - 1 on Cb and Cr;
  * `expand`: the last column replicated to the MCU width before downsampling (jcsample.c expand_right_edge); below
    the image, jcprepct.c replicates the last row to a whole row group (2 rows) before downsampling and the last
    downsampled row to the iMCU height after it;
  * `downsample`: jcsample.c h2v2_downsample, bias 1, 2, 1, 2, ... along each output row;
  * `fdct`: jfdctint.c's islow forward DCT on samples - 128 (output scaled up by 8);
  * `quantise`: rounded division by quantval << 3, held to libjpeg-turbo's reciprocal method (`quantise_reciprocal`)
    over the whole range by tests/test_cpu_jenc.py;
  * `blocks`: the coded blocks in MCU order (Y00 Y01 Y10 Y11 Cb Cr), dummy blocks of jccoefct.c compress_data filling a
    partial MCU (AC zero, DC copied);
  * `huffman_bits` / `stuff`: jchuff.c's symbols with DC predicted per component from 0, ZRL, EOB, 1-bit padding and a
    0x00 after every 0xFF.
Test infrastructure only: the package never imports it.  It sits beside the suites that use it rather than in
oracle/jpeg_oracle.py, so that the decoder's restatement, which the decoder's suites hold to PIL, stays exactly as those
suites were written against; the two share nothing but twingan_b200.jpeg's constants, which the byte-for-byte checks of
whole files against PIL pin as well.
"""
from __future__ import annotations

import numpy as np

from twingan_b200 import jpeg as J

ZZ = np.asarray(J.ZIGZAG)


def rgb_to_ycc(rgb: np.ndarray) -> np.ndarray:
  """uint8 [..., 3] RGB -> int64 [..., 3] YCbCr."""
  r, g, b = [rgb[..., k].astype(np.int64) for k in range(3)]
  y = (19595 * r + 38470 * g + 7471 * b + 32768) >> 16
  cb = (-11059 * r - 21709 * g + 32768 * b + (128 << 16) + 32767) >> 16
  cr = (32768 * r - 27439 * g - 5329 * b + (128 << 16) + 32767) >> 16
  return np.stack([y, cb, cr], -1)


def expand(plane: np.ndarray, rows: int, cols: int) -> np.ndarray:
  """[H, W, ...] -> [rows, cols, ...], the last row and column replicated."""
  H, W = plane.shape[:2]
  return plane[np.minimum(np.arange(rows), H - 1)][:, np.minimum(np.arange(cols), W - 1)]


def downsample(p: np.ndarray) -> np.ndarray:
  """[2h, 2w] -> [h, w]: (sum of each 2x2 + bias) >> 2, bias 1 at even and 2 at odd output columns."""
  s = p[0::2, 0::2] + p[0::2, 1::2] + p[1::2, 0::2] + p[1::2, 1::2]
  bias = np.where(np.arange(s.shape[1]) % 2 == 0, 1, 2)
  return (s + bias[None, :]) >> 2


# jfdctint.c constants: FIX(x) = round(x * 2^13)
F0298, F0390, F0541, F0765, F0899, F1175 = 2446, 3196, 4433, 6270, 7373, 9633
F1501, F1847, F1961, F2053, F2562, F3072 = 12299, 15137, 16069, 16819, 20995, 25172
CONST_BITS, PASS1_BITS = 13, 2


def _descale(x, n):
  return (x + (1 << (n - 1))) >> n


def _fdct_1d(d, pass1):
  """One islow pass over the last axis of int64 [..., 8]."""
  t0, t7 = d[..., 0] + d[..., 7], d[..., 0] - d[..., 7]
  t1, t6 = d[..., 1] + d[..., 6], d[..., 1] - d[..., 6]
  t2, t5 = d[..., 2] + d[..., 5], d[..., 2] - d[..., 5]
  t3, t4 = d[..., 3] + d[..., 4], d[..., 3] - d[..., 4]
  t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
  out = [None] * 8
  if pass1:
    out[0], out[4] = (t10 + t11) << PASS1_BITS, (t10 - t11) << PASS1_BITS
    sh = CONST_BITS - PASS1_BITS
  else:
    out[0], out[4] = _descale(t10 + t11, PASS1_BITS), _descale(t10 - t11, PASS1_BITS)
    sh = CONST_BITS + PASS1_BITS
  z1 = (t12 + t13) * F0541
  out[2] = _descale(z1 + t13 * F0765, sh)
  out[6] = _descale(z1 - t12 * F1847, sh)
  z1, z2, z3, z4 = t4 + t7, t5 + t6, t4 + t6, t5 + t7
  z5 = (z3 + z4) * F1175
  t4, t5, t6, t7 = t4 * F0298, t5 * F2053, t6 * F3072, t7 * F1501
  z1, z2, z3, z4 = -z1 * F0899, -z2 * F2562, -z3 * F1961 + z5, -z4 * F0390 + z5
  out[7] = _descale(t4 + z1 + z3, sh)
  out[5] = _descale(t5 + z2 + z4, sh)
  out[3] = _descale(t6 + z2 + z3, sh)
  out[1] = _descale(t7 + z1 + z4, sh)
  return np.stack(out, -1)


def fdct(samples: np.ndarray) -> np.ndarray:
  """int [..., 8, 8] samples (0..255) -> int64 [..., 8, 8] islow DCT of samples - 128, natural order."""
  x = samples.astype(np.int64) - 128
  rows = _fdct_1d(x, True)
  return np.swapaxes(_fdct_1d(np.swapaxes(rows, -1, -2), False), -1, -2)


def quantise(coef: np.ndarray, divisor) -> np.ndarray:
  """Rounded division, half away from zero: sign(c) * ((|c| + d // 2) // d)."""
  d = np.asarray(divisor, np.int64)
  return np.sign(coef) * ((np.abs(coef) + d // 2) // d)


def reciprocal(divisor: int):
  """libjpeg-turbo jcdctmgr.c compute_reciprocal with 16-bit DCTELEM: (reciprocal, correction, total shift)."""
  b = int(divisor).bit_length() - 1
  r = 16 + b
  fq, fr = divmod(1 << r, divisor)
  c = divisor // 2
  if fr == 0:
    fq >>= 1
    r -= 1
  elif fr <= divisor // 2:
    c += 1
  else:
    fq += 1
  return fq, c, r


def quantise_reciprocal(coef: np.ndarray, divisor: int) -> np.ndarray:
  """jcdctmgr.c quantize: |c| + correction, times the reciprocal, shifted right; the sign restored."""
  fq, c, r = reciprocal(divisor)
  a = np.abs(coef.astype(np.int64))
  return np.sign(coef) * (((a + c) * fq) >> r)


def blocks(rgb: np.ndarray) -> np.ndarray:
  """uint8 [H, W, 3] -> int64 [MCUs, 6, 64] quantised coefficients in zig-zag order, MCU order, dummy blocks
  included."""
  H, W = rgb.shape[:2]
  mx, my = -(-W // 16), -(-H // 16)
  ycc = rgb_to_ycc(rgb)
  even = expand(ycc, H + H % 2, 16 * mx)
  qt = J.encoder_qt().astype(np.int64)
  div = [np.empty(64, np.int64), np.empty(64, np.int64)]
  for t in (0, 1):
    div[t][ZZ] = qt[t] << 3                                    # natural order
  y = expand(ycc[..., 0], 16 * my, 16 * mx).reshape(2 * my, 8, 2 * mx, 8).transpose(0, 2, 1, 3)
  chroma = [expand(downsample(even[..., k]), 8 * my, 8 * mx).reshape(my, 8, mx, 8).transpose(0, 2, 1, 3)
            for k in (1, 2)]
  qy = quantise(fdct(y), div[0].reshape(8, 8)).reshape(2 * my, 2 * mx, 64)[..., ZZ]
  qc = [quantise(fdct(c), div[1].reshape(8, 8)).reshape(my, mx, 64)[..., ZZ] for c in chroma]
  bw, bh = -(-W // 8), -(-H // 8)                            # Y blocks holding image samples
  out = np.zeros((my, mx, 6, 64), np.int64)
  for b in range(4):
    out[:, :, b] = qy[b >> 1::2, b & 1::2]
  out[:, :, 4], out[:, :, 5] = qc
  for j in range(my):
    for i in range(mx):
      right = 2 * i + 1 >= bw
      bottom = 2 * j + 1 >= bh
      blk = out[j, i]
      if right:                                              # jccoefct.c: dummy blocks right of the image ...
        blk[1] = 0
        blk[1, 0] = blk[0, 0]
        blk[3] = 0
        blk[3, 0] = blk[2, 0]
      if bottom:                                             # ... and a dummy row below it: DC of the row above's last
        blk[2:4] = 0
        blk[2:4, 0] = blk[1, 0]
  return out.reshape(my * mx, 6, 64)


def _codes(bits, vals):
  """{symbol: (code, length)} of a canonical Huffman table."""
  out, code, k = {}, 0, 0
  for l in range(1, 17):
    for _ in range(bits[l - 1]):
      out[vals[k]] = (code, l)
      code += 1
      k += 1
    code <<= 1
  return out


_TABLES = [_codes(*t) for t in J.STD_HUFF]     # DC0, AC0, DC1, AC1


def _nbits(v):
  return int(abs(int(v))).bit_length()


def huffman_bits(coefs: np.ndarray):
  """int [MCUs, 6, 64] zig-zag blocks -> (per block the bit string of its codes, in MCU order).  DC predicted per
  component from 0 across the whole scan."""
  out = []
  pred = [0, 0, 0]
  for mcu in coefs:
    for b, blk in enumerate(mcu):
      c = 0 if b < 4 else b - 3
      dc, ac = _TABLES[0 if c == 0 else 2], _TABLES[1 if c == 0 else 3]
      s = []

      def put(code, n):
        if n:
          s.append(format(code, '0%db' % n))

      diff = int(blk[0]) - pred[c]
      pred[c] = int(blk[0])
      n = _nbits(diff)
      put(*dc[n])
      put(diff if diff >= 0 else diff - 1 + (1 << n), n)
      run = 0
      for k in range(1, 64):
        v = int(blk[k])
        if v == 0:
          run += 1
          continue
        while run > 15:
          put(*ac[0xF0])
          run -= 16
        n = _nbits(v)
        put(*ac[(run << 4) | n])
        put(v if v >= 0 else v - 1 + (1 << n), n)
        run = 0
      if run:
        put(*ac[0x00])
      out.append(''.join(s))
  return out


def stuff(bits: str) -> bytes:
  """The scan bytes: padded with 1 bits to a whole byte, 0x00 after every 0xFF."""
  bits += '1' * (-len(bits) % 8)
  raw = int(bits, 2).to_bytes(len(bits) // 8, 'big') if bits else b''
  return raw.replace(b'\xff', b'\xff\x00')


def encode(rgb: np.ndarray):
  """Every stage of one image: {'coef', 'lengths', 'scan', 'file'}."""
  coef = blocks(rgb)
  bits = huffman_bits(coef)
  scan = stuff(''.join(bits))
  return {'coef': coef, 'lengths': np.asarray([len(b) for b in bits], np.int64), 'scan': scan,
          'file': J.encoder_header(*rgb.shape[:2]) + scan + J.EOI}
