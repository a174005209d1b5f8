"""Host side of the device JPEG decoder (csrc/twg_jpeg.cu): read a file's headers, decide whether the device decodes it,
and pack the descriptors of a batch; and of the device JPEG encoder (csrc/twg_jenc.cu): the header PIL writes before
the scan the device encodes.

A file goes to the device only if libjpeg (as PIL calls it) would decode it through the path the kernels restate:
  * baseline sequential Huffman: SOF0, or SOF1 with 8-bit samples; one scan (Ss 0, Se 63, Ah 0, Al 0) holding every
    component in frame order, ended by EOI;
  * 1 component, or 3 that libjpeg reads as YCbCr: a JFIF APP0, or an Adobe APP14 with transform 1, or neither marker
    and component ids 1, 2, 3 (jdapimin.c default_decompress_parms, nothing looser);
  * 4:4:4, 4:2:2 (luma 2x1) or 4:2:0 (luma 2x2), chroma 1x1;
  * every Huffman and quantisation table it uses defined before the scan, and every Huffman table valid as libjpeg's
    jpeg_make_d_derived_tbl checks it.
DQT (8- or 16-bit), DHT, DRI, any size and APPn / COM segments in any order are accepted.  Everything else -- progressive,
arithmetic, lossless, 12-bit, CMYK / YCCK, Adobe transform 0, other sampling, DNL, several scans, a scan not ended by EOI,
anything the parser does not recognise -- is left to PIL: `parse` raises `Unsupported` with the reason.

The segments of a scan (restart intervals when DRI is set, else the whole scan) are found here by their RSTn markers; the
device checks that each one ends in the marker it should (RSTn in sequence, EOI after the last).
"""
from __future__ import annotations

from typing import List, NamedTuple, Sequence, Tuple

import numpy as np

# descriptor row layouts (int64), shared with include/twgjpeg.h
SEG_FIELDS = 6      # {byte start, byte end, image, first MCU, MCUs, segment index in its image}
COMP_FIELDS = 10    # {block base, blocks wide, blocks high, plane offset, quant row, DC table, AC table, h, v, image}
IMAGE_FIELDS = 12   # {first comp, comps, MCUs wide, H, W, payload offset, first pixel, segments, hmax, vmax, 0, 0}
HUFF_LUT_BITS = 9
HUFF_WORDS = 1024   # int32 per table: lut[512] | maxcode[18] | valoff[18] | vals[256] | pad

# device status bits (TWG_JPEG_* of include/twgjpeg.h)
STATUS_BAD_CODE = 1
STATUS_MARKER = 2
STATUS_TRUNCATED = 4
STATUS_RESTART = 8
STATUS_COEF_RANGE = 16
STATUS_IDCT_RANGE = 32


class Unsupported(ValueError):
  """The file is not in the subset the device decodes (the reason is the message); PIL decodes it."""


class Component(NamedTuple):
  id: int
  h: int
  v: int
  tq: int


class JpegInfo(NamedTuple):
  H: int
  W: int
  comps: Tuple[Component, ...]
  qt: Tuple[np.ndarray, ...]          # per component: int32 [64], zig-zag order
  dc: Tuple[Tuple[bytes, bytes], ...]  # per component: (BITS[16], HUFFVAL)
  ac: Tuple[Tuple[bytes, bytes], ...]
  restart_interval: int
  mcux: int
  mcuy: int
  segments: Tuple[Tuple[int, int], ...]   # [start, end) byte ranges of the entropy-coded segments in the file
  scan_start: int
  eoi: int                             # offset of the FF D9 that ends the scan

  @property
  def hmax(self):
    return max(c.h for c in self.comps)

  @property
  def vmax(self):
    return max(c.v for c in self.comps)

  @property
  def mcus(self):
    return self.mcux * self.mcuy

  def block_dims(self):
    """(blocks wide, blocks high) of each component as coded."""
    if len(self.comps) == 1:
      return [(self.mcux, self.mcuy)]
    return [(self.mcux * c.h, self.mcuy * c.v) for c in self.comps]


def _u16(b, i):
  return (b[i] << 8) | b[i + 1]


def _huff_ok(bits: bytes, vals: bytes, is_dc: bool) -> bool:
  """jpeg_make_d_derived_tbl's checks: no code runs out of its length, DC symbols <= 15."""
  code = 0
  for l in range(1, 17):
    code += bits[l - 1]
    if code >= (1 << l):
      return False
    code <<= 1
  return not (is_dc and any(v > 15 for v in vals))


def read_dht(seg: bytes, huff: dict, check: bool) -> None:
  """The tables of one DHT segment into huff[(class, id)] = (BITS, HUFFVAL); with `check`, each is held to `_huff_ok`
  as it is defined (a progressive file checks only the tables its scans use, when they use them)."""
  i = 0
  while i < len(seg):
    if i + 17 > len(seg):
      raise Unsupported('bad DHT')
    tc, th = seg[i] >> 4, seg[i] & 15
    bits = bytes(seg[i + 1:i + 17])
    cnt = sum(bits)
    if tc > 1 or th > 3 or cnt > 256 or i + 17 + cnt > len(seg):
      raise Unsupported('bad DHT')
    vals = bytes(seg[i + 17:i + 17 + cnt])
    if check and not _huff_ok(bits, vals, tc == 0):
      raise Unsupported('invalid Huffman table')
    huff[(tc, th)] = (bits, vals)
    i += 17 + cnt


def read_dqt(seg: bytes, qt: dict) -> None:
  """The tables of one DQT segment (8- or 16-bit) into qt[id] = int32 [64], zig-zag order."""
  i = 0
  while i < len(seg):
    pq, tq = seg[i] >> 4, seg[i] & 15
    size = 64 * (pq + 1)
    if pq > 1 or tq > 3 or i + 1 + size > len(seg):
      raise Unsupported('bad DQT')
    raw = np.frombuffer(seg[i + 1:i + 1 + size], dtype='>u2' if pq else np.uint8)
    qt[tq] = raw.astype(np.int32)
    i += 1 + size


def read_dri(seg: bytes) -> int:
  if len(seg) != 2:
    raise Unsupported('bad DRI')
  return _u16(seg, 0)


def is_jfif(seg: bytes) -> bool:
  return len(seg) >= 14 and seg[:5] == b'JFIF\0'


def is_adobe(seg: bytes) -> bool:
  return len(seg) >= 12 and seg[:5] == b'Adobe'


def colour_and_sampling(comps: Tuple[Component, ...], jfif: bool, adobe: bool, transform) -> Tuple[Component, ...]:
  """The frame's components as decoded, or `Unsupported`: 3 components only when libjpeg reads them as YCbCr (a JFIF
  APP0, an Adobe APP14 with transform 1, or neither marker and ids 1, 2, 3) at 4:4:4, 4:2:2 or 4:2:0; a lone
  component is coded one block per MCU whatever its factors."""
  if len(comps) == 3:
    if not jfif:
      if adobe and transform != 1:
        raise Unsupported('Adobe transform %d' % transform)
      if not adobe and [c.id for c in comps] != [1, 2, 3]:
        raise Unsupported('component ids %s without JFIF or Adobe marker' % [c.id for c in comps])
    y, cb, cr = comps
    if (cb.h, cb.v, cr.h, cr.v) != (1, 1, 1, 1) or (y.h, y.v) not in ((1, 1), (2, 1), (2, 2)):
      raise Unsupported('sampling %s' % ['%dx%d' % (c.h, c.v) for c in comps])
    return comps
  return (comps[0]._replace(h=1, v=1),)


def parse(data: bytes) -> JpegInfo:
  """The header and segment layout of a JPEG file the device decodes; `Unsupported` otherwise."""
  b = memoryview(data).cast('B') if not isinstance(data, (bytes, bytearray)) else data
  n = len(b)
  if n < 4 or b[0] != 0xFF or b[1] != 0xD8:
    raise Unsupported('not a JPEG stream (no SOI)')
  pos = 2
  qt = {}
  huff = {}
  ri = 0
  frame = None
  jfif = adobe = False
  transform = None
  while True:
    if pos >= n or b[pos] != 0xFF:
      raise Unsupported('no marker at byte %d' % pos)
    while pos < n and b[pos] == 0xFF:
      pos += 1
    if pos >= n:
      raise Unsupported('truncated before the scan')
    m = b[pos]
    pos += 1
    if m == 0xD8 or m == 0xD9 or m == 0x01 or 0xD0 <= m <= 0xD7:
      raise Unsupported('marker %02X before the scan' % m)
    if pos + 2 > n:
      raise Unsupported('truncated marker segment')
    L = _u16(b, pos)
    if L < 2 or pos + L > n:
      raise Unsupported('marker %02X: bad length %d' % (m, L))
    seg = bytes(b[pos + 2:pos + L])
    pos += L
    if m in (0xC0, 0xC1):
      if frame is not None:
        raise Unsupported('two frame headers')
      if len(seg) < 6 or seg[0] != 8:
        raise Unsupported('SOF%d with %d-bit samples' % (m - 0xC0, seg[0] if seg else -1))
      H, W, nf = _u16(seg, 1), _u16(seg, 3), seg[5]
      if H == 0 or W == 0:
        raise Unsupported('image size %dx%d (DNL)' % (H, W))
      if nf not in (1, 3) or len(seg) != 6 + 3 * nf:
        raise Unsupported('%d components' % nf)
      comps = tuple(Component(seg[6 + 3 * i], seg[7 + 3 * i] >> 4, seg[7 + 3 * i] & 15, seg[8 + 3 * i]) for i in range(nf))
      frame = (H, W, comps)
    elif 0xC2 <= m <= 0xCF and m not in (0xC4, 0xC8, 0xCC):
      raise Unsupported('SOF%d (progressive, lossless or arithmetic)' % (m - 0xC0))
    elif m == 0xCC:
      raise Unsupported('arithmetic coding (DAC)')
    elif m == 0xC4:
      read_dht(seg, huff, check=True)
    elif m == 0xDB:
      read_dqt(seg, qt)
    elif m == 0xDD:
      ri = read_dri(seg)
    elif m == 0xE0:
      jfif = jfif or is_jfif(seg)
    elif m == 0xEE:
      if is_adobe(seg):
        adobe, transform = True, seg[11]
    elif 0xE1 <= m <= 0xEF or m == 0xFE:
      pass
    elif m == 0xDA:
      break
    else:
      raise Unsupported('marker %02X' % m)
  if frame is None:
    raise Unsupported('scan before the frame header')
  H, W, comps = frame
  # the scan header
  ns = seg[0] if seg else 0
  if ns != len(comps) or len(seg) != 4 + 2 * ns:
    raise Unsupported('a scan of %d of %d components' % (ns, len(comps)))
  if [seg[1 + 2 * i] for i in range(ns)] != [c.id for c in comps]:
    raise Unsupported('scan components not in frame order')
  if len({c.id for c in comps}) != len(comps):
    raise Unsupported('duplicate component ids')
  ss, se, ahal = seg[1 + 2 * ns], seg[2 + 2 * ns], seg[3 + 2 * ns]
  if ss != 0 or se != 63 or ahal != 0:
    raise Unsupported('not a sequential scan (Ss %d, Se %d, AhAl %02X)' % (ss, se, ahal))
  tables = [(seg[2 + 2 * i] >> 4, seg[2 + 2 * i] & 15) for i in range(ns)]
  comps = colour_and_sampling(comps, jfif, adobe, transform)
  for c in comps:
    if c.tq not in qt:
      raise Unsupported('quantisation table %d undefined' % c.tq)
  for td, ta in tables:
    if (0, td) not in huff or (1, ta) not in huff:
      raise Unsupported('Huffman table undefined')
  hmax, vmax = max(c.h for c in comps), max(c.v for c in comps)
  mcux, mcuy = -(-W // (8 * hmax)), -(-H // (8 * vmax))
  # the entropy-coded data: RSTn split it, the first other marker ends it
  scan_start = pos
  arr = np.frombuffer(bytes(b[scan_start:]), dtype=np.uint8)
  ff = np.flatnonzero(arr[:-1] == 0xFF)
  nxt = arr[ff + 1]
  is_marker = (nxt != 0) & (nxt != 0xFF)
  rst = (nxt >= 0xD0) & (nxt <= 0xD7)
  ends = np.flatnonzero(is_marker & ~rst)
  if not len(ends):
    raise Unsupported('the scan is not ended by a marker')
  eoi = int(ff[ends[0]])
  if nxt[ends[0]] != 0xD9:
    raise Unsupported('marker %02X after the scan (several scans or DNL)' % nxt[ends[0]])
  cuts = ff[is_marker & rst & (ff < eoi)].tolist()
  starts = [0] + [c + 2 for c in cuts]
  stops = cuts + [eoi]
  segments = tuple((scan_start + s, scan_start + e) for s, e in zip(starts, stops))
  return JpegInfo(H, W, comps, tuple(qt[c.tq] for c in comps), tuple(huff[(0, t[0])] for t in tables),
                  tuple(huff[(1, t[1])] for t in tables), ri, mcux, mcuy, segments, scan_start, scan_start + eoi)


def probe(data: bytes):
  """JpegInfo for a file the device decodes, else None."""
  try:
    return parse(data)
  except Unsupported:
    return None


def huff_table(bits: bytes, vals: bytes) -> np.ndarray:
  """The device form of one Huffman table, int32 [HUFF_WORDS]: lut[2^9] = (length << 8 | symbol) of every code of at most
  9 bits indexed by the next 9 bits of the stream (0: longer code), maxcode[l] (l = 1..16; -1 when no code has length l,
  maxcode[17] = INT_MAX), valoff[l] (symbol = vals[code + valoff[l]]), vals[256]."""
  t = np.zeros(HUFF_WORDS, np.int32)
  lut, maxcode, valoff, v = t[:512], t[512:530], t[530:548], t[548:804]
  v[:len(vals)] = np.frombuffer(vals, np.uint8)
  code = k = 0
  maxcode[:] = -1
  for l in range(1, 17):
    cnt = bits[l - 1]
    if cnt:
      valoff[l] = k - code
      for j in range(cnt):
        if l <= HUFF_LUT_BITS:
          lo = (code + j) << (HUFF_LUT_BITS - l)
          lut[lo:lo + (1 << (HUFF_LUT_BITS - l))] = (l << 8) | vals[k + j]
      code += cnt
      k += cnt
      maxcode[l] = code - 1
    code <<= 1
  maxcode[17] = 0x7FFFFFFF
  return t


class Batch(NamedTuple):
  """Descriptors of the JPEG images of one batch (host int tensors as numpy arrays; see include/twgjpeg.h)."""
  data: np.ndarray     # uint8: the scans, each through its EOI
  segs: np.ndarray     # int64 [S, SEG_FIELDS]
  comps: np.ndarray    # int64 [C, COMP_FIELDS]
  images: np.ndarray   # int64 [n, IMAGE_FIELDS]
  qt: np.ndarray       # int32 [Q, 64]
  huff: np.ndarray     # int32 [T, HUFF_WORDS]
  blocks: int          # coefficient blocks (scratch: 128 bytes each)
  plane_bytes: int     # sample planes (scratch)
  pixels: int


def pack(files: Sequence[bytes], infos: Sequence[JpegInfo], payload_offsets: Sequence[int]) -> Batch:
  """Descriptors for decoding files[i] (described by infos[i]) into a payload at byte payload_offsets[i]."""
  chunks, segs, comps, images, qts = [], [], [], [], []
  tables, table_rows = {}, []
  at = blocks = planes = pixels = 0

  def table(bv):
    if bv not in tables:
      tables[bv] = len(table_rows)
      table_rows.append(huff_table(*bv))
    return tables[bv]

  for i, (f, info, off) in enumerate(zip(files, infos, payload_offsets)):
    chunk = f[info.scan_start:info.eoi + 2]
    base = at - info.scan_start
    nseg = 1 if info.restart_interval == 0 else -(-info.mcus // info.restart_interval)
    per = info.mcus if info.restart_interval == 0 else info.restart_interval
    for s in range(nseg):
      a, e = info.segments[s] if s < len(info.segments) else (info.eoi, info.eoi)
      segs.append((a + base, e + base, i, s * per, min(per, info.mcus - s * per), s))
    first = len(comps)
    for c, (comp, (bw, bh)) in enumerate(zip(info.comps, info.block_dims())):
      comps.append((blocks, bw, bh, planes, len(qts), table(info.dc[c]), table(info.ac[c]), comp.h, comp.v, i))
      qts.append(info.qt[c])
      blocks += bw * bh
      planes += bw * bh * 64
    images.append((first, len(info.comps), info.mcux, info.H, info.W, off, pixels, nseg, info.hmax, info.vmax, 0, 0))
    pixels += info.H * info.W
    chunks.append(np.frombuffer(chunk, np.uint8))
    at += len(chunk)
  i64 = lambda rows, k: np.asarray(rows, np.int64).reshape(-1, k)
  return Batch(np.concatenate(chunks) if chunks else np.zeros(0, np.uint8), i64(segs, SEG_FIELDS),
               i64(comps, COMP_FIELDS), i64(images, IMAGE_FIELDS),
               np.asarray(qts, np.int32).reshape(-1, 64), np.asarray(table_rows, np.int32).reshape(-1, HUFF_WORDS),
               blocks, planes, pixels)


# ---- encoding (csrc/twg_jenc.cu): the file PIL writes for Image.fromarray(rgb).save(f, 'JPEG') ----------------------
#
# PIL's defaults are libjpeg's: baseline, quality 75, 4:2:0 (Y 2x2, Cb and Cr 1x1), the Annex K Huffman tables without
# optimisation, no restart markers, a JFIF 1.01 APP0 without units at density 1x1.  Only the frame size varies between
# files, so the header is assembled here and the device writes the entropy-coded scan that follows it.

# T.81 Annex K.1, tables K.1 and K.2 (natural order): the basis libjpeg's jpeg_set_quality scales
_STD_LUMA_QT = (16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56,
                14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
                49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99)
_STD_CHROMA_QT = (17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99,
                  47, 66, 99, 99, 99, 99, 99, 99) + (99,) * 32
# natural index of the k-th coefficient in zig-zag order
ZIGZAG = (0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,
          7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31,
          39, 46, 53, 60, 61, 54, 47, 55, 62, 63)
# T.81 Annex K.3 (tables K.3 - K.6): (BITS[16], HUFFVAL) of DC luma, AC luma, DC chroma, AC chroma
_AC_LUMA_VALS = bytes.fromhex(
    '01020300041105122131410613516107227114328191a1082342b1c11552d1f02433627282090a161718191a25262728292a3435363738'
    '393a434445464748494a535455565758595a636465666768696a737475767778797a838485868788898a92939495969798999aa2a3a4a5'
    'a6a7a8a9aab2b3b4b5b6b7b8b9bac2c3c4c5c6c7c8c9cad2d3d4d5d6d7d8d9dae1e2e3e4e5e6e7e8e9eaf1f2f3f4f5f6f7f8f9fa')
_AC_CHROMA_VALS = bytes.fromhex(
    '000102031104052131061241510761711322328108144291a1b1c109233352f0156272d10a162434e125f11718191a262728292a353637'
    '38393a434445464748494a535455565758595a636465666768696a737475767778797a82838485868788898a92939495969798999aa2a3'
    'a4a5a6a7a8a9aab2b3b4b5b6b7b8b9bac2c3c4c5c6c7c8c9cad2d3d4d5d6d7d8d9dae2e3e4e5e6e7e8e9eaf2f3f4f5f6f7f8f9fa')
STD_HUFF = (
    (bytes([0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0]), bytes(range(12))),
    (bytes([0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7D]), _AC_LUMA_VALS),
    (bytes([0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0]), bytes(range(12))),
    (bytes([0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77]), _AC_CHROMA_VALS),
)
ENCODE_QUALITY = 75


def encoder_qt(quality: int = ENCODE_QUALITY) -> np.ndarray:
  """int32 [2, 64] (luma, chroma) in zig-zag order: jcparam.c jpeg_set_quality's scaling of Annex K with baseline
  limits, (basis * s + 50) // 100 clamped to [1, 255], s = 5000 / q below 50, else 200 - 2 q."""
  s = 5000 // quality if quality < 50 else 200 - 2 * quality
  out = np.empty((2, 64), np.int32)
  for t, basis in enumerate((_STD_LUMA_QT, _STD_CHROMA_QT)):
    nat = np.clip((np.asarray(basis, np.int64) * s + 50) // 100, 1, 255)
    out[t] = nat[list(ZIGZAG)]
  return out


def _segment(marker: int, body: bytes) -> bytes:
  return bytes([0xFF, marker]) + (len(body) + 2).to_bytes(2, 'big') + body


def encoder_header(H: int, W: int) -> bytes:
  """The bytes PIL writes before the scan of an H x W RGB image: SOI, JFIF APP0, DQT luma and chroma, SOF0 (Y 2x2 on
  table 0, Cb and Cr 1x1 on table 1), DHT DC0 AC0 DC1 AC1, SOS of the three components."""
  if not (1 <= H <= 65535 and 1 <= W <= 65535):
    raise ValueError('a JPEG frame is 1..65535 pixels a side (got %dx%d)' % (H, W))
  qt = encoder_qt()
  out = [b'\xff\xd8', _segment(0xE0, b'JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00')]
  out += [_segment(0xDB, bytes([t]) + bytes(qt[t].astype(np.uint8))) for t in (0, 1)]
  out.append(_segment(0xC0, bytes([8]) + H.to_bytes(2, 'big') + W.to_bytes(2, 'big')
                      + bytes([3, 1, 0x22, 0, 2, 0x11, 1, 3, 0x11, 1])))
  out += [_segment(0xC4, bytes([cls]) + bits + vals) for cls, (bits, vals) in zip((0x00, 0x10, 0x01, 0x11), STD_HUFF)]
  out.append(_segment(0xDA, bytes([3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0])))
  return b''.join(out)


EOI = b'\xff\xd9'
