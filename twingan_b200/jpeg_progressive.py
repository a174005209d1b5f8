"""Host side of the device progressive JPEG decoder (csrc/twg_jpegp.cu): read a progressive file's headers and scans,
decide whether the device decodes it, and pack the descriptors of a batch.

A progressive file differs from a baseline one only in how its coefficients are entropy-coded: several scans each send
a band of coefficients (a spectral selection Ss..Se) of one or more components, to some bit precision (successive
approximation Ah, Al).  Once every coefficient of every component has been sent to its last bit, libjpeg (as PIL calls
it) does not smooth any block, and its pixels are those of a baseline file with the same coefficients: the baseline
inverse DCT and colour kernels (twgjpeg_idct, twgjpeg_color) turn the coefficient blocks into PIL's pixels unchanged.

A file goes to the device only if libjpeg would decode it without a warning, through the path the kernels restate:
  * SOF2 (progressive Huffman) with 8-bit samples; the components, colour space and sampling jpeg.parse accepts;
  * each scan as jdphuff.c's start_pass_phuff_decoder checks it (a DC scan has Se 0; an AC scan has one component and
    1 <= Ss <= Se <= 63; Ah 0 or Al = Ah - 1; Al <= 13; components in frame order), sent in an order its coef_bits
    bookkeeping accepts without JWRN_BOGUS_PROGRESSION (no AC scan of a component before its first DC scan, Ah the last
    Al of every coefficient of the band), no coefficient sent twice from its first bit, and every coefficient of every
    component complete (sent down to bit 0) after the last scan, so that libjpeg smooths no block;
  * DHT, DRI, APPn and COM between scans (a scan uses the tables and restart interval defined when it starts); every
    quantisation table defined before the first scan and no DQT after it (libjpeg latches a component's table at its
    first scan); the Huffman tables a scan uses defined and valid as jpeg_make_d_derived_tbl checks them;
  * each scan's entropy-coded data ended by the next marker segment, the last by EOI.
Everything else is left to PIL: `parse` raises `jpeg.Unsupported` with the reason.

Scans of one file depend on each other: a refinement scan reads what the earlier scans of its coefficients wrote.  Each
scan gets a level, 1 + the highest level of the earlier scans of its image that share a (component, coefficient) with
it (0 if none), so that the scans of one level write disjoint coefficients and read only what earlier levels wrote;
ops.jpeg_progressive_decode launches the entropy decoder once per level.
"""
from __future__ import annotations

from typing import List, NamedTuple, Sequence, Tuple

import numpy as np

from .jpeg import (COMP_FIELDS, HUFF_WORDS, IMAGE_FIELDS, SEG_FIELDS, Component, Unsupported, _huff_ok, _u16,
                   colour_and_sampling, huff_table, is_adobe, is_jfif, read_dht, read_dqt, read_dri)

# descriptor rows (int64), shared with include/twgjpegp.h.  A segment row is jpeg.SEG_FIELDS wide:
#   {byte start, byte end, scan row, first MCU, MCUs, the marker byte that must follow the segment}
SCAN_FIELDS = 16    # {image, Ss, Se, Ah, Al, comps, comp rows[3], table rows[3], grid wide, restart interval, level, 0}

# device status bits of the progressive decoder beyond jpeg.STATUS_* (TWG_JPEGP_* of include/twgjpegp.h)
STATUS_REFINE_SIZE = 64     # an AC refinement symbol whose size is neither 0 nor 1
STATUS_BAND = 128           # a coefficient written past the scan's Se
STATUS_VALUE_RANGE = 256    # a coefficient value outside int16 (s << Al, or a correction of +-(1 << Al))


class Scan(NamedTuple):
  comps: Tuple[int, ...]               # indices into the frame's components, in frame order
  ss: int
  se: int
  ah: int
  al: int
  tables: Tuple[Tuple[bytes, bytes], ...]   # per scan component: the (BITS, HUFFVAL) it decodes with; None: no table
  restart_interval: int
  grid: Tuple[int, int]                # MCUs (interleaved) or blocks (one component) wide, high
  segments: Tuple[Tuple[int, int], ...]    # [start, end) byte ranges of the entropy-coded segments found in the file
  end: int                             # offset of the FF of the marker that ends the scan
  end_marker: int                      # that marker's code (D9 for the last scan)
  level: int

  @property
  def mcus(self):
    return self.grid[0] * self.grid[1]

  @property
  def nseg(self):
    return 1 if self.restart_interval == 0 else -(-self.mcus // self.restart_interval)


class ProgressiveInfo(NamedTuple):
  H: int
  W: int
  comps: Tuple[Component, ...]
  qt: Tuple[np.ndarray, ...]           # per component: int32 [64], zig-zag order
  mcux: int
  mcuy: int
  scans: Tuple[Scan, ...]
  data_start: int                      # offset of the first scan's entropy-coded data
  eoi: int                             # offset of the FF D9 that ends the last scan

  @property
  def hmax(self):
    return max(c.h for c in self.comps)

  @property
  def vmax(self):
    return max(c.v for c in self.comps)

  @property
  def levels(self):
    return 1 + max(s.level for s in self.scans)

  def block_dims(self):
    """(blocks wide, blocks high) of each component in the MCU-padded layout jpeg.pack uses."""
    if len(self.comps) == 1:
      return [(self.mcux, self.mcuy)]
    return [(self.mcux * c.h, self.mcuy * c.v) for c in self.comps]

  def component_blocks(self, c):
    """(blocks wide, blocks high) a non-interleaved scan of component c walks (T.81 A.2.2): the blocks its samples
    cover, without the MCU padding."""
    comp = self.comps[c]
    cw = -(-self.W * comp.h // self.hmax)
    ch = -(-self.H * comp.v // self.vmax)
    return -(-cw // 8), -(-ch // 8)


def _scan_data(b, start: int):
  """(segments, end, end marker) of the entropy-coded data from `start`: RSTn split it, the first other marker ends it."""
  arr = np.frombuffer(bytes(b[start:]), dtype=np.uint8)
  ff = np.flatnonzero(arr[:-1] == 0xFF)
  nxt = arr[ff + 1]
  is_marker = (nxt != 0) & (nxt != 0xFF)
  rst = (nxt >= 0xD0) & (nxt <= 0xD7)
  ends = np.flatnonzero(is_marker & ~rst)
  if not len(ends):
    raise Unsupported('the scan is not ended by a marker')
  end = int(ff[ends[0]])
  cuts = ff[is_marker & rst & (ff < end)].tolist()
  starts = [0] + [c + 2 for c in cuts]
  stops = cuts + [end]
  return tuple((start + s, start + e) for s, e in zip(starts, stops)), start + end, int(nxt[ends[0]])


def parse(data: bytes) -> ProgressiveInfo:
  """The frame, scans and segment layout of a progressive JPEG file the device decodes; `Unsupported` otherwise."""
  b = memoryview(data).cast('B') if not isinstance(data, (bytes, bytearray)) else data
  n = len(b)
  if n < 4 or b[0] != 0xFF or b[1] != 0xD8:
    raise Unsupported('not a JPEG stream (no SOI)')
  pos = 2
  qt, huff = {}, {}
  ri = 0
  frame = comps = None
  jfif = adobe = False
  transform = None
  scans: List[Scan] = []
  coef_bits = None                     # libjpeg's coef_bits: per component and coefficient, the last Al sent; -1: none
  covered = []                         # per scan: the (component, coefficient) pairs it sends
  last_end = None                      # offset where the last scan's data ended
  while True:
    if pos >= n or b[pos] != 0xFF:
      raise Unsupported('no marker at byte %d' % pos)
    at = pos
    while pos < n and b[pos] == 0xFF:
      pos += 1
    if pos >= n:
      raise Unsupported('truncated before EOI')
    m = b[pos]
    pos += 1
    if m == 0xD9:
      if not scans:
        raise Unsupported('EOI before a scan')
      if at != last_end:
        raise Unsupported('the last scan is not ended by EOI')
      break
    if m == 0xD8 or m == 0x01 or 0xD0 <= m <= 0xD7:
      raise Unsupported('marker %02X outside a scan' % m)
    if pos + 2 > n:
      raise Unsupported('truncated marker segment')
    L = _u16(b, pos)
    if L < 2 or pos + L > n:
      raise Unsupported('marker %02X: bad length %d' % (m, L))
    seg = bytes(b[pos + 2:pos + L])
    pos += L
    if m == 0xC2:
      if frame is not None:
        raise Unsupported('two frame headers')
      if len(seg) < 6 or seg[0] != 8:
        raise Unsupported('SOF2 with %d-bit samples' % (seg[0] if seg else -1))
      H, W, nf = _u16(seg, 1), _u16(seg, 3), seg[5]
      if H == 0 or W == 0:
        raise Unsupported('image size %dx%d (DNL)' % (H, W))
      if nf not in (1, 3) or len(seg) != 6 + 3 * nf:
        raise Unsupported('%d components' % nf)
      frame = (H, W, tuple(Component(seg[6 + 3 * i], seg[7 + 3 * i] >> 4, seg[7 + 3 * i] & 15, seg[8 + 3 * i])
                           for i in range(nf)))
      if len({c.id for c in frame[2]}) != nf:
        raise Unsupported('duplicate component ids')
    elif 0xC0 <= m <= 0xCF and m not in (0xC4, 0xC8, 0xCC):
      raise Unsupported('SOF%d (not progressive Huffman)' % (m - 0xC0))
    elif m == 0xCC:
      raise Unsupported('arithmetic coding (DAC)')
    elif m == 0xDC:
      raise Unsupported('DNL')
    elif m == 0xC4:
      read_dht(seg, huff, check=False)
    elif m == 0xDB:
      if scans:
        raise Unsupported('DQT after the first scan')
      read_dqt(seg, qt)
    elif m == 0xDD:
      ri = read_dri(seg)
    elif m == 0xE0:
      jfif = jfif or (not scans and is_jfif(seg))
    elif m == 0xEE:
      if not scans and is_adobe(seg):
        adobe, transform = True, seg[11]
    elif 0xE1 <= m <= 0xEF or m == 0xFE:
      pass
    elif m == 0xDA:
      if frame is None:
        raise Unsupported('scan before the frame header')
      H, W, frame_comps = frame
      if comps is None:                # colour space, sampling and tables are fixed at the first scan
        comps = colour_and_sampling(frame_comps, jfif, adobe, transform)
        for c in comps:
          if c.tq not in qt:
            raise Unsupported('quantisation table %d undefined' % c.tq)
        hmax, vmax = max(c.h for c in comps), max(c.v for c in comps)
        mcux, mcuy = -(-W // (8 * hmax)), -(-H // (8 * vmax))
        coef_bits = np.full((len(comps), 64), -1, np.int64)
      scans.append(_scan(seg, comps, huff, ri, coef_bits, covered, (H, W, mcux, mcuy, hmax, vmax), pos, b))
      last_end = scans[-1].end
      pos = last_end
    else:
      raise Unsupported('marker %02X' % m)
  if (coef_bits != 0).any():
    c, k = np.argwhere(coef_bits != 0)[0]
    raise Unsupported('incomplete progression: coefficient %d of component %d ends at bit %d'
                      % (k, c, coef_bits[c, k]))
  return ProgressiveInfo(H, W, comps, tuple(qt[c.tq] for c in comps), mcux, mcuy, tuple(scans), scans[0].segments[0][0],
                         last_end)


def _scan(seg, comps, huff, ri, coef_bits, covered, geom, pos, b) -> Scan:
  """One scan header, checked as start_pass_phuff_decoder and the coef_bits bookkeeping check it."""
  H, W, mcux, mcuy, hmax, vmax = geom
  ns = seg[0] if seg else 0
  if not 1 <= ns <= len(comps) or len(seg) != 4 + 2 * ns:
    raise Unsupported('bad scan header (%d components)' % ns)
  ids = [c.id for c in comps]
  idx = []
  for i in range(ns):
    if seg[1 + 2 * i] not in ids:
      raise Unsupported('scan component id %d not in the frame' % seg[1 + 2 * i])
    idx.append(ids.index(seg[1 + 2 * i]))
  if idx != sorted(set(idx)):
    raise Unsupported('scan components not in frame order')
  ss, se, ah, al = seg[1 + 2 * ns], seg[2 + 2 * ns], seg[3 + 2 * ns] >> 4, seg[3 + 2 * ns] & 15
  if ss == 0:
    if se != 0:
      raise Unsupported('bad progression: a DC scan with Se %d' % se)
  else:
    if not ss <= se <= 63:
      raise Unsupported('bad progression: band %d..%d' % (ss, se))
    if ns != 1:
      raise Unsupported('bad progression: an AC scan of %d components' % ns)
  if ah != 0 and al != ah - 1:
    raise Unsupported('bad progression: Ah %d, Al %d' % (ah, al))
  if al > 13:
    raise Unsupported('bad progression: Al %d' % al)
  tables = []
  for i, c in enumerate(idx):
    td, ta = seg[2 + 2 * i] >> 4, seg[2 + 2 * i] & 15
    if ss == 0 and ah == 0:
      key = (0, td)
    elif ss > 0:
      key = (1, ta)
    else:
      tables.append(None)              # a DC refinement scan reads raw bits
      continue
    if key not in huff:
      raise Unsupported('Huffman table undefined')
    if not _huff_ok(*huff[key], key[0] == 0):
      raise Unsupported('invalid Huffman table')
    tables.append(huff[key])
  # jdphuff.c's coef_bits bookkeeping: decline whatever it warns about, and a second first scan of a coefficient
  band = range(ss, se + 1)
  for c in idx:
    if ss > 0 and coef_bits[c, 0] < 0:
      raise Unsupported('bogus progression: an AC scan of component %d before its DC scan' % c)
    for k in band:
      if ah == 0 and coef_bits[c, k] >= 0:
        raise Unsupported('a second first scan of coefficient %d of component %d' % (k, c))
      if ah != 0 and coef_bits[c, k] != ah:
        raise Unsupported('bogus progression: Ah %d for coefficient %d of component %d, last Al %d'
                          % (ah, k, c, coef_bits[c, k]))
  for c in idx:
    coef_bits[c, ss:se + 1] = al
  mine = {(c, k) for c in idx for k in band}
  level = 1 + max([s.level for s, cov in covered if cov & mine] or [-1])
  if ns == 1 and len(comps) > 1:
    cw, ch = -(-W * comps[idx[0]].h // hmax), -(-H * comps[idx[0]].v // vmax)
    grid = (-(-cw // 8), -(-ch // 8))
  else:
    grid = (mcux, mcuy)
  segments, end, end_marker = _scan_data(b, pos)
  s = Scan(tuple(idx), ss, se, ah, al, tuple(tables), ri, grid, segments, end, end_marker, level)
  covered.append((s, mine))
  return s


def probe(data: bytes):
  """ProgressiveInfo for a file the device decodes, else None."""
  try:
    return parse(data)
  except Unsupported:
    return None


class Batch(NamedTuple):
  """Descriptors of the progressive JPEG images of one batch (host numpy arrays; see include/twgjpegp.h)."""
  data: np.ndarray     # uint8: each file from its first scan's data through its EOI
  segs: np.ndarray     # int64 [S, SEG_FIELDS], sorted by level
  scans: np.ndarray    # int64 [scans, SCAN_FIELDS]
  comps: np.ndarray    # int64 [C, COMP_FIELDS], as jpeg.pack writes them
  images: np.ndarray   # int64 [n, IMAGE_FIELDS], as jpeg.pack writes them
  qt: np.ndarray       # int32 [Q, 64]
  huff: np.ndarray     # int32 [T, HUFF_WORDS]
  blocks: int          # coefficient blocks (scratch: 128 bytes each)
  plane_bytes: int     # sample planes (scratch)
  pixels: int
  levels: List[int]    # segment rows [levels[l], levels[l + 1]) are those of level l


def pack(files: Sequence[bytes], infos: Sequence[ProgressiveInfo], payload_offsets: Sequence[int]) -> Batch:
  """Descriptors for decoding files[i] (described by infos[i]) into a payload at byte payload_offsets[i]."""
  chunks, segs, scans, comps, images, qts = [], [], [], [], [], []
  tables, table_rows = {}, []
  at = blocks = planes = pixels = 0

  def table(bv):
    if bv is None:
      return -1
    if bv not in tables:
      tables[bv] = len(table_rows)
      table_rows.append(huff_table(*bv))
    return tables[bv]

  for i, (f, info, off) in enumerate(zip(files, infos, payload_offsets)):
    chunk = f[info.data_start:info.eoi + 2]
    base = at - info.data_start
    first = len(comps)
    for c, (comp, (bw, bh)) in enumerate(zip(info.comps, info.block_dims())):
      comps.append((blocks, bw, bh, planes, len(qts), 0, 0, comp.h, comp.v, i))
      qts.append(info.qt[c])
      blocks += bw * bh
      planes += bw * bh * 64
    nseg = 0
    for sc in info.scans:
      row = len(scans)
      rows = [first + c for c in sc.comps] + [-1] * (3 - len(sc.comps))
      trows = [table(t) for t in sc.tables] + [-1] * (3 - len(sc.comps))
      scans.append((i, sc.ss, sc.se, sc.ah, sc.al, len(sc.comps), *rows, *trows, sc.grid[0], sc.restart_interval,
                    sc.level, 0))
      per = sc.mcus if sc.restart_interval == 0 else sc.restart_interval
      for s in range(sc.nseg):
        a, e = sc.segments[s] if s < len(sc.segments) else (sc.end, sc.end)
        want = sc.end_marker if s == sc.nseg - 1 else 0xD0 + s % 8
        segs.append((sc.level, a + base, e + base, row, s * per, min(per, sc.mcus - s * per), want))
      nseg += sc.nseg
    images.append((first, len(info.comps), info.mcux, info.H, info.W, off, pixels, nseg, info.hmax, info.vmax, 0, 0))
    pixels += info.H * info.W
    chunks.append(np.frombuffer(chunk, np.uint8))
    at += len(chunk)
  segs.sort(key=lambda r: r[0])        # stable: each level keeps its scans' and segments' order
  nlev = 1 + max([r[0] for r in segs] or [-1])
  levels = [sum(1 for r in segs if r[0] < l) for l in range(nlev + 1)]
  i64 = lambda rows, k: np.asarray(rows, np.int64).reshape(-1, k)
  return Batch(np.concatenate(chunks) if chunks else np.zeros(0, np.uint8), i64([r[1:] for r in segs], SEG_FIELDS),
               i64(scans, SCAN_FIELDS), i64(comps, COMP_FIELDS), i64(images, IMAGE_FIELDS),
               np.asarray(qts, np.int32).reshape(-1, 64), np.asarray(table_rows, np.int32).reshape(-1, HUFF_WORDS),
               blocks, planes, pixels, levels)
