"""Restatement of the device PNG decoder (twingan_b200/csrc/twg_png.cu) in Python and integer numpy.

  * `inflate(stream, size)`: RFC 1950 / 1951 bit by bit (canonical decoding as RFC 1951 3.2.2 describes it), with the
    kernel's checks in the kernel's order, so a corrupt stream gets the kernel's TWG_PNG_* bits.  Its bytes are held to
    zlib's in the CPU suite; `decode` takes zlib's bytes for a stream zlib finds clean, since Python decodes slowly.
    A bad code is found bit by bit here; the kernel peeks 15 bits and calls it truncation when fewer were left, which
    is the same verdict.
  * `unfilter(raw, info)`: None / Sub / Up / Average / Paeth, rows in order.
  * `to_rgb(rows, info)`: PIL's convert('RGB') of each colour type and bit depth.
It sits beside its suites rather than in oracle/, as tests/jenc_oracle.py does."""
from __future__ import annotations

import zlib

import numpy as np

from twingan_b200 import png as P

LEN_BASE = (3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227,
            258)
LEN_EXTRA = (0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0)
DIST_BASE = (1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097,
             6145, 8193, 12289, 16385, 24577)
DIST_EXTRA = (0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13)
CL_ORDER = (16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15)


class _Stop(Exception):
  def __init__(self, bit):
    self.bit = bit


class _Bits:
  def __init__(self, data):
    self.d, self.pos, self.nbits = data, 0, 8 * len(data)

  def take(self, k):
    if self.pos + k > self.nbits:
      raise _Stop(P.STATUS_TRUNCATED)
    v = 0
    for i in range(k):
      p = self.pos + i
      v |= ((self.d[p >> 3] >> (p & 7)) & 1) << i
    self.pos += k
    return v

  def align(self):
    self.pos = -(-self.pos // 8) * 8


def _code(lengths, code_lengths):
  """(count, symbols) of a canonical code, or _Stop(CODES) for a set zlib refuses (as the kernel's build)."""
  count = [0] * 16
  for l in lengths:
    count[l] += 1
  left, maxl = 1, 0
  for l in range(1, 16):
    left = (left << 1) - count[l]
    if left < 0:
      raise _Stop(P.STATUS_CODES)
    if count[l]:
      maxl = l
  if left > 0 and (code_lengths or maxl > 1):
    raise _Stop(P.STATUS_CODES)
  syms = [s for l in range(1, 16) for s, ls in enumerate(lengths) if ls == l]
  return count, syms


def _decode(bits, table):
  count, syms = table
  code = first = index = 0
  for l in range(1, 16):
    code |= bits.take(1)
    if code - count[l] < first:
      return syms[index + code - first]
    index += count[l]
    first = (first + count[l]) << 1
    code <<= 1
  raise _Stop(P.STATUS_SYMBOL)


_FIXED = ([8] * 144 + [9] * 112 + [7] * 24 + [8] * 8, [5] * 32)


def adler32(b: bytes) -> int:
  return zlib.adler32(b) & 0xFFFFFFFF


def inflate(stream: bytes, size: int):
  """(inflated bytes, TWG_PNG_* status) of one image's zlib stream into a region of `size` bytes."""
  out = bytearray()
  bits = _Bits(stream)
  try:
    cmf, flg = bits.take(8), bits.take(8)
    if (cmf & 15) != 8 or (cmf >> 4) > 7 or (cmf * 256 + flg) % 31 or flg & 0x20:
      raise _Stop(P.STATUS_HEADER)
    window = 1 << ((cmf >> 4) + 8)
    last = False
    while not last:
      last, btype = bits.take(1), bits.take(2)
      if btype == 3:
        raise _Stop(P.STATUS_BLOCK)
      if btype == 0:
        bits.align()
        n, nn = bits.take(16), bits.take(16)
        if n != (~nn & 0xFFFF):
          raise _Stop(P.STATUS_BLOCK)
        at = bits.pos // 8
        if at + n > len(stream):
          raise _Stop(P.STATUS_TRUNCATED)
        if len(out) + n > size:
          raise _Stop(P.STATUS_LONG)
        out += stream[at:at + n]
        bits.pos += 8 * n
        continue
      if btype == 1:
        lit, dist = _code(_FIXED[0], False), _code(_FIXED[1], False)
      else:
        nlit, ndist, ncl = bits.take(5) + 257, bits.take(5) + 1, bits.take(4) + 4
        if nlit > 286 or ndist > 30:
          raise _Stop(P.STATUS_CODES)
        cl = [0] * 19
        got = bits.take(3 * ncl)                       # one read, as the kernel's lanes take theirs at once
        for i in range(ncl):
          cl[CL_ORDER[i]] = (got >> (3 * i)) & 7
        clt = _code(cl, True)
        lens = []
        while len(lens) < nlit + ndist:
          s = _decode(bits, clt)
          if s < 16:
            rep, v = 1, s
          elif s == 16:
            if not lens:
              raise _Stop(P.STATUS_CODES)
            rep, v = 3 + bits.take(2), lens[-1]
          elif s == 17:
            rep, v = 3 + bits.take(3), 0
          else:
            rep, v = 11 + bits.take(7), 0
          if len(lens) + rep > nlit + ndist:
            raise _Stop(P.STATUS_CODES)
          lens += [v] * rep
        if lens[256] == 0:
          raise _Stop(P.STATUS_CODES)
        lit, dist = _code(lens[:nlit], False), _code(lens[nlit:], False)
      while True:
        s = _decode(bits, lit)
        if s < 256:
          if len(out) >= size:
            raise _Stop(P.STATUS_LONG)
          out.append(s)
          continue
        if s == 256:
          break
        if s > 285:
          raise _Stop(P.STATUS_SYMBOL)
        n = LEN_BASE[s - 257] + bits.take(LEN_EXTRA[s - 257])
        d = _decode(bits, dist)
        if d > 29:
          raise _Stop(P.STATUS_SYMBOL)
        off = DIST_BASE[d] + bits.take(DIST_EXTRA[d])
        if off > len(out) or off > window:
          raise _Stop(P.STATUS_DISTANCE)
        if len(out) + n > size:
          raise _Stop(P.STATUS_LONG)
        for _ in range(n):
          out.append(out[-off])
    bits.align()
    trailer = int.from_bytes(bytes(bits.take(8) for _ in range(4)), 'big')
  except _Stop as e:
    return bytes(out), e.bit
  st = 0
  if len(out) < size:
    st |= P.STATUS_SHORT
  if bits.pos < bits.nbits:
    st |= P.STATUS_TRAILING
  if adler32(bytes(out)) != trailer:
    st |= P.STATUS_ADLER
  return bytes(out), st


def unfilter(raw: bytes, info: P.PngInfo):
  """uint8 [H, row bytes] of the unfiltered rows, or None with STATUS_FILTER when a row's filter type is > 4."""
  H, rb = info.H, info.row_bytes
  bpp = max(1, P.CHANNELS[info.color_type] * info.depth // 8)
  a = np.frombuffer(raw, np.uint8).reshape(H, rb + 1)
  out = np.zeros((H, rb), np.int64)
  prev = np.zeros(rb, np.int64)
  for y in range(H):
    f, x = int(a[y, 0]), a[y, 1:].astype(np.int64)
    if f > 4:
      return None, P.STATUS_FILTER
    if f == 0:
      r = x
    elif f == 2:
      r = (x + prev) & 255
    elif f == 1:
      r = x.copy()
      for c in range(bpp):                           # a prefix sum mod 256 in each byte lane
        r[c::bpp] = np.cumsum(x[c::bpp]) & 255
    else:
      r, xs, ps = [0] * rb, x.tolist(), prev.tolist()
      for i in range(rb):
        left = r[i - bpp] if i >= bpp else 0
        up = ps[i]
        if f == 3:
          pred = (left + up) >> 1
        else:
          ul = ps[i - bpp] if i >= bpp else 0
          p = left + up - ul
          pa, pb, pc = abs(p - left), abs(p - up), abs(p - ul)
          pred = left if pa <= pb and pa <= pc else up if pb <= pc else ul
        r[i] = (xs[i] + pred) & 255
      r = np.asarray(r, np.int64)
    out[y] = r
    prev = r
  return out.astype(np.uint8), 0


def _samples(rows, depth, n):
  """[H, n] samples of `depth` bits (MSB first; 16-bit big-endian) of each row."""
  rows = rows.astype(np.int64)
  if depth == 8:
    return rows[:, :n]
  if depth == 16:
    return (rows[:, 0:2 * n:2] << 8) | rows[:, 1:2 * n:2]
  k = np.arange(n)
  bit = k * depth
  return (rows[:, bit >> 3] >> (8 - depth - (bit & 7))) & ((1 << depth) - 1)


def to_rgb(rows, info: P.PngInfo):
  """uint8 [H, W, 3]: PIL's convert('RGB') of the unfiltered rows of a mode that PngImagePlugin opens as
  1 / L;2 / L;4 / L / I;16 / RGB / RGB;16B / P;n / LA / LA;16B (RGBA) / RGBA / RGBA;16B."""
  ct, depth, W = info.color_type, info.depth, info.W
  ch = P.CHANNELS[ct]
  s = _samples(rows, depth, W * ch).reshape(info.H, W, ch)
  if ct == 0:
    v = s[..., 0]
    v = np.minimum(v, 255) if depth == 16 else v * (255 // ((1 << depth) - 1))
    return np.repeat(v[..., None], 3, 2).astype(np.uint8)
  if ct == 3:
    pal = np.zeros(P.PALETTE_BYTES, np.uint8)
    pal[:len(info.palette)] = np.frombuffer(info.palette, np.uint8)
    return pal.reshape(256, 3)[s[..., 0]]
  hi = s >> 8 if depth == 16 else s
  if ct == 4:
    return np.repeat(hi[..., :1], 3, 2).astype(np.uint8)
  return hi[..., :3].astype(np.uint8)


def stream_of(data: bytes, info: P.PngInfo) -> bytes:
  return b''.join(data[s:e] for s, e in info.idat)


def decode(data: bytes, info: P.PngInfo = None):
  """{'raw', 'rows', 'rgb', 'status'} of a file png.parse accepts.  A stream with a 32 KB window that zlib inflates
  cleanly to exactly the region's size, trailer checked and nothing after it, is taken from zlib; any other goes through
  `inflate`."""
  info = info or P.parse(data)
  stream = stream_of(data, info)
  d = zlib.decompressobj()
  try:
    raw = d.decompress(stream)
    # zlib resolves every distance from its output here, so the window the header declares binds only at 32 KB
    clean = d.eof and not d.unused_data and len(raw) == info.raw_bytes and stream[0] >> 4 == 7
  except zlib.error:
    clean = False
  if not clean:
    raw, st = inflate(stream, info.raw_bytes)
    if st:
      return {'raw': raw, 'rows': None, 'rgb': None, 'status': st}
  rows, st = unfilter(raw, info)
  if st:
    return {'raw': raw, 'rows': None, 'rgb': None, 'status': st}
  return {'raw': raw, 'rows': rows, 'rgb': to_rgb(rows, info), 'status': 0}
