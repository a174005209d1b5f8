"""Integer restatement of the device JPEG decoder (twingan_b200/csrc/twg_jpeg.cu), stage by stage, in numpy.

The target is what PIL returns for `Image.open(f).convert('RGB')` of a baseline file: libjpeg-turbo with its defaults.
Written from ITU-T T.81 (Huffman decoding, F.2.2; restart intervals, F.2.2.5 / B.2.5) and the published integer
algorithms libjpeg uses by default:
  * `idct`: the "islow" inverse DCT (Loeffler, Ligtenberg & Moschytz, ICASSP 1989, as scaled in libjpeg's jidctint.c):
    13-bit constants, 2 extra bits between the passes, descale by rounding right shifts, +128 and a range limit;
  * `upsample`: "fancy" triangle-filter chroma upsampling, 3/4 nearer + 1/4 further sample, with the rounding bias
    alternating between the two output pixels of an input pixel (+1 / +2 across, +8 / +7 for h2v2), the last real
    column and row of the chroma plane replicated past the edge, and plain replication for planes of at most 2 columns;
  * `ycc_to_rgb`: JFIF YCbCr -> RGB with 16-bit fixed-point constants, each term rounded as libjpeg's tables are.
Every stage is exact integer arithmetic.  The status bits are those of the device (twingan_b200.jpeg.STATUS_*): a stream
the decoder does not restate exactly is flagged, not decoded differently.
"""
from __future__ import annotations

import numpy as np

from twingan_b200 import jpeg as J

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,
                   7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31,
                   39, 46, 53, 60, 61, 54, 47, 55, 62, 63])    # natural index of the k-th coefficient in zig-zag order


def _codes(bits, vals):
  out, code, k = {}, 0, 0
  for l in range(1, 17):
    for _ in range(bits[l - 1]):
      out[format(code, '0%db' % l)] = vals[k]
      code += 1
      k += 1
    code <<= 1
  return out


class _Bits(object):
  """The bits of one entropy-coded segment, unstuffed; reading past the end is an error."""

  def __init__(self, seg: bytes):
    self.err = 0
    i = seg.find(b'\xff')
    while i >= 0:
      if i + 1 >= len(seg) or seg[i + 1] != 0:
        self.err |= J.STATUS_MARKER
        seg = seg[:i]
        break
      i = seg.find(b'\xff', i + 2)
    seg = seg.replace(b'\xff\x00', b'\xff')
    self.s = ''.join(format(x, '08b') for x in seg)
    self.p = 0

  def symbol(self, codes):
    for l in range(1, 17):
      c = self.s[self.p:self.p + l]
      if len(c) < l:
        raise _Stop(J.STATUS_TRUNCATED)
      if c in codes:
        self.p += l
        return codes[c]
    raise _Stop(J.STATUS_BAD_CODE)

  def take(self, n):
    if self.p + n > len(self.s):
      raise _Stop(J.STATUS_TRUNCATED)
    v = int(self.s[self.p:self.p + n], 2) if n else 0
    self.p += n
    return v


class _Stop(Exception):
  pass


def _extend(v, s):
  return v - (1 << s) + 1 if s and v < (1 << (s - 1)) else v


def coefficients(data: bytes, info: 'J.JpegInfo'):
  """(per component int32 [blocks high, blocks wide, 64] quantised coefficients in zig-zag order, status bits)."""
  dims = info.block_dims()
  coef = [np.zeros((bh, bw, 64), np.int32) for bw, bh in dims]
  dc = [_codes(*t) for t in info.dc]
  ac = [_codes(*t) for t in info.ac]
  per = info.mcus if info.restart_interval == 0 else info.restart_interval
  nseg = -(-info.mcus // per)
  status = 0
  for s in range(nseg):
    a, e = info.segments[s] if s < len(info.segments) else (info.eoi, info.eoi)
    want = b'\xff\xd9' if s == nseg - 1 else bytes([0xFF, 0xD0 + s % 8])
    if data[e:e + 2] != want:
      status |= J.STATUS_RESTART
    r = _Bits(bytes(data[a:e]))
    pred = [0] * len(info.comps)
    try:
      for m in range(s * per, min((s + 1) * per, info.mcus)):
        my, mx = divmod(m, info.mcux)
        for c, comp in enumerate(info.comps):
          for by in range(comp.v):
            for bx in range(comp.h):
              blk = coef[c][my * comp.v + by, mx * comp.h + bx]
              t = r.symbol(dc[c])
              pred[c] += _extend(r.take(t), t)
              if not -32768 <= pred[c] <= 32767:
                raise _Stop(J.STATUS_COEF_RANGE)
              blk[0] = pred[c]
              k = 1
              while k < 64:
                rs = r.symbol(ac[c])
                run, size = rs >> 4, rs & 15
                if size == 0:
                  if run != 15:
                    break
                  k += 16
                  continue
                k += run
                if k > 63:
                  raise _Stop(J.STATUS_COEF_RANGE)
                blk[k] = _extend(r.take(size), size)
                k += 1
              if k > 64:
                raise _Stop(J.STATUS_COEF_RANGE)
    except _Stop as e:
      status |= e.args[0]
    status |= r.err
  return coef, status


# jidctint.c constants: FIX(x) = round(x * 2^13)
F0298, F0390, F0541, F0765, F0899, F1175 = 2446, 3196, 4433, 6270, 7373, 9633
F1501, F1847, F1961, F2053, F2562, F3072 = 12299, 15137, 16069, 16819, 20995, 25172
CONST_BITS, PASS1_BITS = 13, 2


def _idct_1d(d0, d1, d2, d3, d4, d5, d6, d7, shift):
  """One islow pass over int64 arrays (the eight inputs of a column or row); returns the eight descaled outputs."""
  z1 = (d2 + d6) * F0541
  t2 = z1 - d6 * F1847
  t3 = z1 + d2 * F0765
  t0 = (d0 + d4) << CONST_BITS
  t1 = (d0 - d4) << CONST_BITS
  t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
  o0, o1, o2, o3 = d7, d5, d3, d1
  z1, z2, z3, z4 = o0 + o3, o1 + o2, o0 + o2, o1 + o3
  z5 = (z3 + z4) * F1175
  o0, o1, o2, o3 = o0 * F0298, o1 * F2053, o2 * F3072, o3 * F1501
  z1, z2, z3, z4 = -z1 * F0899, -z2 * F2562, -z3 * F1961 + z5, -z4 * F0390 + z5
  o0, o1, o2, o3 = o0 + z1 + z3, o1 + z2 + z4, o2 + z2 + z3, o3 + z1 + z4
  r = 1 << (shift - 1)
  return [(t10 + o3 + r) >> shift, (t11 + o2 + r) >> shift, (t12 + o1 + r) >> shift, (t13 + o0 + r) >> shift,
          (t13 - o0 + r) >> shift, (t12 - o1 + r) >> shift, (t11 - o2 + r) >> shift, (t10 - o3 + r) >> shift]


def idct(coef: np.ndarray, qt: np.ndarray):
  """Zig-zag coefficients [..., 64] and their quantisation table (zig-zag) -> (uint8 [..., 8, 8] samples, status bits).
  Flags a block whose dequantised coefficients or first-pass outputs leave int16, or whose output leaves [-512, 511]
  before the +128: outside those ranges libjpeg's C and SIMD paths disagree."""
  shape = coef.shape[:-1]
  c = coef.reshape(-1, 64).astype(np.int64)
  deq = np.zeros_like(c)
  deq[:, ZIGZAG] = c * qt.astype(np.int64)[None, :]
  bad = (np.abs(deq + 0.5) > 32767.5).any(1)
  blk = deq.reshape(-1, 8, 8)                       # [n][row][col]
  cols = _idct_1d(*[blk[:, k, :] for k in range(8)], shift=CONST_BITS - PASS1_BITS)
  ws = np.stack(cols, 1)                            # [n][row][col]
  bad |= ((ws < -32768) | (ws > 32767)).reshape(len(ws), -1).any(1)
  rows = _idct_1d(*[ws[:, :, k] for k in range(8)], shift=CONST_BITS + PASS1_BITS + 3)
  out = np.stack(rows, 2)
  bad |= ((out < -512) | (out > 511)).reshape(len(out), -1).any(1)
  samples = np.clip(out + 128, 0, 255).astype(np.uint8)
  return samples.reshape(shape + (8, 8)), (J.STATUS_IDCT_RANGE if bad.any() else 0)


def planes(blocks: np.ndarray) -> np.ndarray:
  """uint8 [bh, bw, 8, 8] -> the component's sample plane [bh * 8, bw * 8]."""
  bh, bw = blocks.shape[:2]
  return blocks.transpose(0, 2, 1, 3).reshape(bh * 8, bw * 8)


def upsample(plane: np.ndarray, h2: bool, v2: bool, H: int, W: int) -> np.ndarray:
  """A chroma plane -> [H, W] (libjpeg's fancy upsampling, h2v1 or h2v2; a 1x1 plane is cropped)."""
  if not h2:
    return plane[:H, :W].astype(np.int32)
  cw, ch = -(-W // 2), -(-H // (2 if v2 else 1))
  p = plane[:ch, :cw].astype(np.int32)
  if cw <= 2:                                       # jdsample.c: plain replication
    p = np.repeat(p, 2, 1)
    return (np.repeat(p, 2, 0) if v2 else p)[:H, :W]
  j = np.arange(cw)
  left, right = np.maximum(j - 1, 0), np.minimum(j + 1, cw - 1)
  out = np.empty((p.shape[0] * (2 if v2 else 1), 2 * cw), np.int32)
  if not v2:
    out[:, 0::2] = (3 * p + p[:, left] + 1) >> 2
    out[:, 1::2] = (3 * p + p[:, right] + 2) >> 2
    return out[:H, :W]
  i = np.arange(ch)
  for parity, nb in ((0, np.maximum(i - 1, 0)), (1, np.minimum(i + 1, ch - 1))):
    cs = 3 * p + p[nb]
    out[parity::2, 0::2] = (3 * cs + cs[:, left] + 8) >> 4
    out[parity::2, 1::2] = (3 * cs + cs[:, right] + 7) >> 4
  return out[:H, :W]


def ycc_to_rgb(y, cb, cr) -> np.ndarray:
  """jdcolor.c ycc_rgb_convert: R = y + round(1.402 cr'), G = y + ((-0.34414 cb' - 0.71414 cr' + 1/2) >> 16 in 2^-16
  units), B = y + round(1.772 cb'), c' = c - 128, clamped to [0, 255]."""
  cb = cb.astype(np.int64) - 128
  cr = cr.astype(np.int64) - 128
  y = y.astype(np.int64)
  r = y + ((91881 * cr + 32768) >> 16)
  g = y + ((-22554 * cb + 32768 - 46802 * cr) >> 16)
  b = y + ((116130 * cb + 32768) >> 16)
  return np.clip(np.stack([r, g, b], -1), 0, 255).astype(np.uint8)


def decode(data: bytes, info=None):
  """Every stage of one file: {'coef', 'planes', 'upsampled', 'rgb', 'status'}."""
  info = info or J.parse(data)
  coef, status = coefficients(data, info)
  pls = []
  for c in range(len(info.comps)):
    blocks, st = idct(coef[c], info.qt[c])
    status |= st
    pls.append(planes(blocks))
  if len(pls) == 1:
    up = [pls[0][:info.H, :info.W].astype(np.int32)]
    rgb = np.repeat(up[0].astype(np.uint8)[..., None], 3, 2)
  else:
    h2, v2 = info.comps[0].h == 2, info.comps[0].v == 2
    up = [pls[0][:info.H, :info.W].astype(np.int32)] + [upsample(p, h2, v2, info.H, info.W) for p in pls[1:]]
    rgb = ycc_to_rgb(*up)
  return {'coef': coef, 'planes': pls, 'upsampled': up, 'rgb': rgb, 'status': status}
