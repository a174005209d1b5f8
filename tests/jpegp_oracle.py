"""Restatement of the device progressive JPEG decoder (twingan_b200/csrc/twg_jpegp.cu) in Python, bit by bit, and a small
progressive re-encoder for the test suites.

`coefficients` decodes the scans of a file jpeg_progressive.parse accepts as ITU-T T.81 G.2 (with libjpeg-turbo's
jdphuff.c) does, making the kernel's checks in the kernel's order: the marker after each segment, a bit pattern that is
no code, a marker inside a segment, a segment that runs out, an AC refinement symbol of size > 1, a coefficient written
past Se, a value outside int16; the first of them stops the segment and flags the image.  `decode` then runs
oracle/jpeg_oracle.py's inverse DCT, upsampling and colour conversion, which the device shares with baseline files.

`reencode` writes the coefficients of a baseline file (decoded by jpeg_oracle.coefficients) as a progressive file under
any scan script, with flat canonical Huffman tables, so the suites can cover scripts PIL (which writes only libjpeg's
standard one) never writes: non-interleaved DC scans, deeper successive approximation, many bands, refinements split
differently from the first scans, restart intervals of one MCU, end-of-band runs cut by restarts.
"""
from __future__ import annotations

import numpy as np

from oracle import jpeg_oracle as JO
from twingan_b200 import jpeg as J
from twingan_b200 import jpeg_progressive as P


class _Stop(Exception):
  pass


def _decode_scan_segment(r, scan, info, coef, dc, ac, m0, m1):
  """The MCUs [m0, m1) of one segment of `scan` from the bit reader `r`; raises _Stop(status) at the first error."""
  ss, se, ah, al = scan.ss, scan.se, scan.ah, scan.al
  gridw = scan.grid[0]
  pred = [0] * len(scan.comps)
  eobrun = 0
  p1 = 1 << al

  def sym(codes):
    try:
      return r.symbol(codes)
    except JO._Stop as e:
      raise _Stop(e.args[0])

  def take(n):
    try:
      return r.take(n)
    except JO._Stop as e:
      raise _Stop(e.args[0])

  def check(v):
    if not -32768 <= v <= 32767:
      raise _Stop(P.STATUS_VALUE_RANGE)
    return v

  for m in range(m0, m1):
    my, mx = divmod(m, gridw)
    for i, c in enumerate(scan.comps):
      comp = info.comps[c]
      hv = [(0, 0)] if len(scan.comps) == 1 else [(by, bx) for by in range(comp.v) for bx in range(comp.h)]
      for by, bx in hv:
        blk = coef[c][my * (1 if len(scan.comps) == 1 else comp.v) + by, mx * (1 if len(scan.comps) == 1 else comp.h) + bx]
        if ss == 0 and ah == 0:
          t = sym(dc[i])
          pred[i] += JO._extend(take(t), t)
          check(pred[i])
          blk[0] = check(pred[i] << al)
        elif ss == 0:
          if take(1):
            blk[0] |= p1
        elif ah == 0:
          if eobrun > 0:
            eobrun -= 1
            continue
          k = ss
          while k <= se:
            rs = sym(ac[i])
            run, s = rs >> 4, rs & 15
            if s:
              k += run
              if k > se:
                raise _Stop(P.STATUS_BAND)
              blk[k] = check(JO._extend(take(s), s) << al)
            elif run == 15:
              k += 15
            else:
              eobrun = (1 << run) + take(run) - 1
              break
            k += 1
        else:
          k = ss
          if eobrun == 0:
            while k <= se:
              rs = sym(ac[i])
              run, s = rs >> 4, rs & 15
              if s:
                if s != 1:
                  raise _Stop(P.STATUS_REFINE_SIZE)
                s = p1 if take(1) else -p1
              elif run != 15:
                eobrun = (1 << run) + take(run)
                break
              while k <= se:
                if blk[k] != 0:
                  if take(1) and (int(blk[k]) & p1) == 0:
                    blk[k] = check(blk[k] + (p1 if blk[k] >= 0 else -p1))
                else:
                  run -= 1
                  if run < 0:
                    break
                k += 1
              if s:
                if k > se:
                  raise _Stop(P.STATUS_BAND)
                blk[k] = s
              k += 1
          if eobrun > 0:
            while k <= se:
              if blk[k] != 0 and take(1) and (int(blk[k]) & p1) == 0:
                blk[k] = check(blk[k] + (p1 if blk[k] >= 0 else -p1))
              k += 1
            eobrun -= 1


def coefficients(data: bytes, info: 'P.ProgressiveInfo'):
  """(per component int32 [blocks high, blocks wide, 64] zig-zag coefficients, status bits, the coefficients after each
  level).  The scans run level by level, in file order within a level, as the device runs them."""
  coef = [np.zeros((bh, bw, 64), np.int64) for bw, bh in info.block_dims()]
  status = 0
  after = []
  for level in range(info.levels):
    for scan in info.scans:
      if scan.level != level:
        continue
      dc = [JO._codes(*t) if scan.ss == 0 and scan.ah == 0 else None for t in scan.tables]
      ac = [JO._codes(*t) if scan.ss > 0 else None for t in scan.tables]
      per = scan.mcus if scan.restart_interval == 0 else scan.restart_interval
      for s in range(scan.nseg):
        a, e = scan.segments[s] if s < len(scan.segments) else (scan.end, scan.end)
        want = bytes([0xFF, scan.end_marker if s == scan.nseg - 1 else 0xD0 + s % 8])
        if data[e:e + 2] != want:
          status |= J.STATUS_RESTART
        r = JO._Bits(bytes(data[a:e]))
        try:
          _decode_scan_segment(r, scan, info, coef, dc, ac, s * per, min((s + 1) * per, scan.mcus))
        except _Stop as st:
          status |= st.args[0]
        status |= r.err
    after.append([c.astype(np.int32) for c in coef])
  return [c.astype(np.int32) for c in coef], status, after


def decode(data: bytes, info=None):
  """Every stage of one file: {'coef', 'levels', 'planes', 'rgb', 'status'}."""
  info = info or P.parse(data)
  coef, status, after = coefficients(data, info)
  pls = []
  for c in range(len(info.comps)):
    blocks, st = JO.idct(coef[c], info.qt[c])
    status |= st
    pls.append(JO.planes(blocks))
  if len(pls) == 1:
    rgb = np.repeat(pls[0][:info.H, :info.W][..., None], 3, 2)
  else:
    h2, v2 = info.comps[0].h == 2, info.comps[0].v == 2
    up = [pls[0][:info.H, :info.W].astype(np.int32)] + [JO.upsample(p, h2, v2, info.H, info.W) for p in pls[1:]]
    rgb = JO.ycc_to_rgb(*up)
  return {'coef': coef, 'levels': after, 'planes': pls, 'rgb': rgb, 'status': status}


# ---- the re-encoder ---------------------------------------------------------------------------------------------------

# flat canonical tables: every DC size 0..15 in 5 bits; every AC run/size with size 1..14, EOB0..EOB14 and ZRL in 8 bits
# (no code is all ones, as jpeg_make_d_derived_tbl requires)
DC_TABLE = (bytes([0] * 4 + [16] + [0] * 11), bytes(range(16)))
_AC_SYMBOLS = sorted([(r << 4) | s for r in range(16) for s in range(1, 15)] + [r << 4 for r in range(16)])
AC_TABLE = (bytes([0] * 7 + [len(_AC_SYMBOLS)] + [0] * 8), bytes(_AC_SYMBOLS))

# libjpeg's jpeg_simple_progression for YCbCr, the script PIL writes: (components, Ss, Se, Ah, Al)
STANDARD_SCRIPT = (((0, 1, 2), 0, 0, 0, 1), ((0,), 1, 5, 0, 2), ((2,), 1, 63, 0, 1), ((1,), 1, 63, 0, 1),
                   ((0,), 6, 63, 0, 2), ((0,), 1, 63, 2, 1), ((0, 1, 2), 0, 0, 1, 0), ((2,), 1, 63, 1, 0),
                   ((1,), 1, 63, 1, 0), ((0,), 1, 63, 1, 0))


def _codebook(bits, vals):
  return {v: (code, l) for code_str, v in JO._codes(bits, vals).items() for code, l in [(int(code_str, 2), len(code_str))]}


class _Writer(object):
  def __init__(self):
    self.bits = []

  def put(self, v, n):
    self.bits.extend((v >> (n - 1 - i)) & 1 for i in range(n))

  def flush(self) -> bytes:
    """The segment's bytes: padded with one bits, FF stuffed."""
    b = self.bits + [1] * (-len(self.bits) % 8)
    self.bits = []
    out = bytearray()
    for i in range(0, len(b), 8):
      x = int(''.join(map(str, b[i:i + 8])), 2)
      out.append(x)
      if x == 0xFF:
        out.append(0)
    return bytes(out)


def _magnitude(v):
  """(size, bits) of T.81 F.1.2.1's coding of v."""
  a = abs(v)
  n = a.bit_length()
  return n, (a if v >= 0 else (~a) & ((1 << n) - 1))


class _ScanEncoder(object):
  def __init__(self, w, dc, ac):
    self.w, self.dc, self.ac = w, dc, ac
    self.eobrun, self.be = 0, []

  def sym(self, book, s):
    code, l = book[s]
    self.w.put(code, l)

  def flush_eob(self):
    if self.eobrun:
      n = self.eobrun.bit_length() - 1
      self.sym(self.ac, n << 4)
      self.w.put(self.eobrun - (1 << n), n)
      for b in self.be:
        self.w.put(b, 1)
      self.eobrun, self.be = 0, []

  def count_eob(self, bits=()):
    self.eobrun += 1
    self.be += list(bits)
    if self.eobrun == 0x7FFF:
      self.flush_eob()

  def ac_first(self, blk, ss, se, al):
    r = 0
    for k in range(ss, se + 1):
      a = abs(int(blk[k])) >> al
      if a == 0:
        r += 1
        continue
      self.flush_eob()
      while r > 15:
        self.sym(self.ac, 0xF0)
        r -= 16
      n, bits = _magnitude(a if blk[k] > 0 else -a)
      self.sym(self.ac, (r << 4) | n)
      self.w.put(bits, n)
      r = 0
    if r:
      self.count_eob()

  def ac_refine(self, blk, ss, se, al):
    absv = [abs(int(blk[k])) >> al for k in range(ss, se + 1)]
    last_new = max([i for i, a in enumerate(absv) if a == 1] or [-1])
    r, br = 0, []
    for i, a in enumerate(absv):
      if a == 0:
        r += 1
        continue
      while r > 15 and i <= last_new:
        self.flush_eob()
        self.sym(self.ac, 0xF0)
        r -= 16
        for b in br:
          self.w.put(b, 1)
        br = []
      if a > 1:
        br.append(a & 1)
        continue
      self.flush_eob()
      self.sym(self.ac, (r << 4) | 1)
      self.w.put(1 if blk[ss + i] > 0 else 0, 1)
      for b in br:
        self.w.put(b, 1)
      br, r = [], 0
    if r or br:
      self.count_eob(br)


def _segment(marker, body):
  return bytes([0xFF, marker]) + (len(body) + 2).to_bytes(2, 'big') + body


def reencode(baseline: bytes, script, restart_interval: int = 0) -> bytes:
  """The coefficients of a baseline file as a progressive file whose scans follow `script`, a sequence of (component
  indices, Ss, Se, Ah, Al), with a DRI of `restart_interval` MCUs before every scan."""
  info = J.parse(baseline)
  coef, st = JO.coefficients(baseline, info)
  assert st == 0, st
  nc = len(info.comps)
  hmax, vmax = info.hmax, info.vmax
  out = [b'\xff\xd8', _segment(0xE0, b'JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00')]
  tq = sorted({c.tq for c in info.comps})
  for t in tq:
    q = info.qt[[c.tq for c in info.comps].index(t)]
    out.append(_segment(0xDB, bytes([t]) + bytes(q.astype(np.uint8))) if q.max() < 256 else
               _segment(0xDB, bytes([0x10 | t]) + q.astype('>u2').tobytes()))
  sof = bytes([8]) + info.H.to_bytes(2, 'big') + info.W.to_bytes(2, 'big') + bytes([nc])
  for c in info.comps:
    sof += bytes([c.id, (c.h << 4) | c.v, c.tq])
  out.append(_segment(0xC2, sof))
  out.append(_segment(0xC4, bytes([0x00]) + DC_TABLE[0] + DC_TABLE[1] + bytes([0x10]) + AC_TABLE[0] + AC_TABLE[1]))
  out.append(_segment(0xDD, restart_interval.to_bytes(2, 'big')))
  dc, ac = _codebook(*DC_TABLE), _codebook(*AC_TABLE)
  for comps, ss, se, ah, al in script:
    out.append(_segment(0xDA, bytes([len(comps)]) + b''.join(bytes([info.comps[c].id, 0x00]) for c in comps)
                        + bytes([ss, se, (ah << 4) | al])))
    if len(comps) == 1 and nc > 1:
      c = comps[0]
      cw, ch = -(-info.W * info.comps[c].h // hmax), -(-info.H * info.comps[c].v // vmax)
      gw, gh = -(-cw // 8), -(-ch // 8)
      units = [[(c, by, bx)] for by in range(gh) for bx in range(gw)]
    else:
      units = [[(c, my * info.comps[c].v + by, mx * info.comps[c].h + bx) for c in comps
                for by in range(info.comps[c].v) for bx in range(info.comps[c].h)]
               for my in range(info.mcuy) for mx in range(info.mcux)]
    w = _Writer()
    enc = _ScanEncoder(w, dc, ac)
    pred = {c: 0 for c in comps}
    data = bytearray()
    for u, blocks in enumerate(units):
      if restart_interval and u and u % restart_interval == 0:
        enc.flush_eob()
        data += w.flush() + bytes([0xFF, 0xD0 + (u // restart_interval - 1) % 8])
        pred = {c: 0 for c in comps}
      for c, by, bx in blocks:
        blk = coef[c][by, bx]
        if ss == 0 and ah == 0:
          v = int(blk[0]) >> al
          n, bits = _magnitude(v - pred[c])
          pred[c] = v
          enc.sym(dc, n)
          w.put(bits, n)
        elif ss == 0:
          w.put((int(blk[0]) >> al) & 1, 1)
        elif ah == 0:
          enc.ac_first(blk, ss, se, al)
        else:
          enc.ac_refine(blk, ss, se, al)
    enc.flush_eob()
    out.append(bytes(data) + w.flush())
  out.append(b'\xff\xd9')
  return b''.join(out)
