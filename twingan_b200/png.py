"""Host side of the device PNG decoder (csrc/twg_png.cu): read a file's chunks, decide whether the device decodes it,
and pack the descriptors of a batch.

PNG is lossless, so any correct inflate and unfiltering gives PIL's pixels; what is PIL's own is only the mapping of
colour type and bit depth to `convert('RGB')`.  The rule here is that the host may be stricter than PIL, never laxer:
a file `parse` declines goes to PIL exactly as before.  A file goes to the device when
  * it starts with the PNG signature and an IHDR of a size >= 1 x 1, compression 0, filter 0 and no interlace, with a
    legal colour type / bit depth (grey 1/2/4/8/16, RGB 8/16, palette 1/2/4/8, grey+alpha 8/16, RGBA 8/16);
  * every chunk's CRC is right, the IDAT chunks form one consecutive run of at least the 6 bytes of a zlib header and
    trailer, and IEND follows it as the file's last chunk;
  * a palette image has one PLTE of 1..256 entries before the IDAT run, and no tRNS (PIL's convert warns for those);
  * every other chunk before the IDAT run is one PIL reads without a change in pixels and without raising on its
    contents: tRNS of a grey (2 bytes) or RGB (6 bytes) image, gAMA, cHRM, sRGB, pHYs, tIME, bKGD, sBIT, tEXt, zTXt,
    iTXt, iCCP and eXIf -- the compressed ones (zTXt, iTXt, iCCP) are inflated here under PIL's MAX_TEXT_CHUNK, and the
    text total is held to its MAX_TEXT_MEMORY, as PngImagePlugin does.
Adam7 interlace, APNG (acTL / fcTL / fdAT), any other chunk and anything malformed raise `Unsupported` with the reason.
"""
from __future__ import annotations

import zlib
from typing import NamedTuple, Optional, Sequence, Tuple

import numpy as np

SIGNATURE = b'\x89PNG\r\n\x1a\n'
# descriptor row layout (int64), shared with include/twgpng.h
IMAGE_FIELDS = 12   # {stream start, stream end, inflated offset, inflated bytes, payload offset, H, W, colour type,
                    #  bit depth, row bytes, palette row (-1: none), first pixel}
PALETTE_BYTES = 256 * 3

# device status bits (TWG_PNG_* of include/twgpng.h)
STATUS_HEADER = 1        # zlib header: CM != 8, CINFO > 7, FCHECK, or FDICT set
STATUS_BLOCK = 2         # block type 3, or a stored block with LEN != ~NLEN
STATUS_CODES = 4         # a bad code set: over-subscribed or incomplete, too many symbols, a bad repeat
STATUS_SYMBOL = 8        # no code of its table, or an invalid literal/length or distance symbol
STATUS_DISTANCE = 16     # a distance before the start of the output or beyond the declared window
STATUS_TRUNCATED = 32    # the input ended before the final block and the Adler-32 trailer
STATUS_LONG = 64         # the stream inflates to more bytes than H x (1 + row bytes)
STATUS_SHORT = 128       # ... or to fewer
STATUS_TRAILING = 256    # bytes after the zlib stream in the IDAT run
STATUS_ADLER = 512       # the Adler-32 trailer does not match the inflated bytes
STATUS_FILTER = 1024     # a row's filter type is > 4

DEPTHS = {0: (1, 2, 4, 8, 16), 2: (8, 16), 3: (1, 2, 4, 8), 4: (8, 16), 6: (8, 16)}
CHANNELS = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}
# ancillary chunks PIL reads without a change in pixels (tRNS and the text / ICC chunks are checked further below)
_PASSIVE = {b'gAMA': 4, b'cHRM': 32, b'sRGB': None, b'pHYs': 9, b'tIME': None, b'bKGD': None, b'sBIT': None,
            b'eXIf': None}
_APNG = (b'acTL', b'fcTL', b'fdAT')


class Unsupported(ValueError):
  """The file is not in the subset the device decodes (the reason is the message); PIL decodes it."""


class PngInfo(NamedTuple):
  H: int
  W: int
  color_type: int
  depth: int
  palette: Optional[bytes]               # PLTE of a palette image
  idat: Tuple[Tuple[int, int], ...]       # [start, end) of each IDAT chunk's data in the file

  @property
  def row_bytes(self) -> int:
    return (self.W * CHANNELS[self.color_type] * self.depth + 7) // 8

  @property
  def raw_bytes(self) -> int:
    """The inflated size: a filter byte and the row bytes for each row."""
    return self.H * (1 + self.row_bytes)

  @property
  def stream_bytes(self) -> int:
    return sum(e - s for s, e in self.idat)


def _u32(b, i):
  return int.from_bytes(b[i:i + 4], 'big')


def _inflate_limited(s: bytes, limit: int) -> bytes:
  """PngImagePlugin._safe_zlib_decompress: ValueError past `limit` bytes; a zlib error leaves PIL with no value."""
  d = zlib.decompressobj()
  try:
    out = d.decompress(s, limit)
  except zlib.error:
    return b''
  if d.unconsumed_tail:
    raise Unsupported('compressed chunk inflates past PIL\'s MAX_TEXT_CHUNK')
  return out


def _text_chars(cid: bytes, s: bytes, limit: int) -> int:
  """What PngStream.chunk_tEXt / zTXt / iTXt add to its text memory (Unsupported where they raise)."""
  k, sep, v = s.partition(b'\0')
  if cid == b'tEXt':
    return len(v) if k else 0
  if cid == b'zTXt':
    if v and v[0] != 0:
      raise Unsupported('zTXt compression method %d' % v[0])
    v = _inflate_limited(v[1:], limit)
    return len(v) if k else 0
  # iTXt
  if not sep or len(v) < 2:
    return 0
  cf, cm, r = v[0], v[1], v[2:]
  parts = r.split(b'\0', 2)
  if len(parts) < 3:
    return 0
  v = parts[2]
  if cf != 0:
    if cm != 0:
      return 0
    v = _inflate_limited(v, limit)      # a zlib error: PIL keeps no text, as the empty string adds nothing
  try:
    parts[0].decode('utf-8', 'strict')
    parts[1].decode('utf-8', 'strict')
    return len(v.decode('utf-8', 'strict'))
  except UnicodeError:
    return 0


def parse(data: bytes) -> PngInfo:
  """The header and IDAT layout of a PNG file the device decodes; `Unsupported` otherwise."""
  from PIL import PngImagePlugin
  text_limit, text_memory_limit = PngImagePlugin.MAX_TEXT_CHUNK, PngImagePlugin.MAX_TEXT_MEMORY
  b = bytes(data)
  n = len(b)
  if b[:8] != SIGNATURE:
    raise Unsupported('not a PNG file')
  pos = 8
  ihdr = palette = None
  idat = []
  text_memory = 0
  while True:
    if pos + 12 > n:
      raise Unsupported('truncated chunk at byte %d' % pos)
    length, cid = _u32(b, pos), b[pos + 4:pos + 8]
    if length > 0x7FFFFFFF or pos + 12 + length > n:
      raise Unsupported('chunk %r runs past the end of the file' % cid)
    body = b[pos + 8:pos + 8 + length]
    if zlib.crc32(body, zlib.crc32(cid)) != _u32(b, pos + 8 + length):
      raise Unsupported('bad CRC in chunk %r' % cid)
    start, pos = pos + 8, pos + 12 + length
    if ihdr is None:
      if cid != b'IHDR' or length != 13:
        raise Unsupported('the first chunk is not a 13-byte IHDR')
      W, H, depth, ct, comp, filt, interlace = _u32(body, 0), _u32(body, 4), body[8], body[9], body[10], body[11], body[12]
      if not (1 <= W <= 0x7FFFFFFF and 1 <= H <= 0x7FFFFFFF):
        raise Unsupported('image size %dx%d' % (W, H))
      if depth not in DEPTHS.get(ct, ()):
        raise Unsupported('colour type %d at bit depth %d' % (ct, depth))
      if comp != 0 or filt != 0:
        raise Unsupported('compression method %d, filter method %d' % (comp, filt))
      if interlace != 0:
        raise Unsupported('interlaced (Adam7)')
      ihdr = (H, W, ct, depth)
      continue
    if cid == b'IDAT':
      if idat and idat[-1][1] + 4 != start - 8:
        raise Unsupported('IDAT chunks not consecutive')
      idat.append((start, start + length))
      continue
    if idat:
      if cid != b'IEND' or length != 0 or pos != n:
        raise Unsupported('%r after the IDAT run, or data after IEND' % cid)
      break
    ct = ihdr[2]
    if cid == b'PLTE':
      if ct != 3 or palette is not None or length % 3 or not 3 <= length <= PALETTE_BYTES:
        raise Unsupported('PLTE of %d bytes in a colour type %d image' % (length, ct))
      palette = body
    elif cid == b'tRNS':
      if ct == 3:
        raise Unsupported('palette image with tRNS')
      if (ct, length) not in ((0, 2), (2, 6)):
        raise Unsupported('tRNS of %d bytes in a colour type %d image' % (length, ct))
    elif cid in _PASSIVE:
      want = _PASSIVE[cid]
      if (want is not None and length != want) or (cid == b'sRGB' and length < 1):
        raise Unsupported('%r of %d bytes' % (cid, length))
    elif cid in (b'tEXt', b'zTXt', b'iTXt'):
      text_memory += _text_chars(cid, body, text_limit)
      if text_memory > text_memory_limit:
        raise Unsupported('text chunks past PIL\'s MAX_TEXT_MEMORY')
    elif cid == b'iCCP':
      i = body.find(b'\0')
      if i < 0 or i + 2 > len(body) or body[i + 1] != 0:
        raise Unsupported('iCCP without compression method 0')
      _inflate_limited(body[i + 2:], text_limit)
    elif cid in _APNG:
      raise Unsupported('APNG (%r)' % cid)
    else:
      raise Unsupported('chunk %r' % cid)
  H, W, ct, depth = ihdr
  if ct == 3 and palette is None:
    raise Unsupported('palette image without PLTE')
  if sum(e - s for s, e in idat) < 6:
    raise Unsupported('IDAT run shorter than a zlib header and trailer')
  return PngInfo(H, W, ct, depth, palette, tuple(idat))


def probe(data: bytes) -> Optional[PngInfo]:
  """PngInfo for a file the device decodes, else None."""
  try:
    return parse(data)
  except Unsupported:
    return None


class Batch(NamedTuple):
  """Descriptors of the PNG images of one batch (host arrays; see include/twgpng.h)."""
  data: np.ndarray       # uint8: each image's IDAT payloads back to back, one zlib stream per image
  images: np.ndarray     # int64 [n, IMAGE_FIELDS]
  palettes: np.ndarray   # uint8 [max(rows, 1), 768], zero-padded
  raw_bytes: int         # inflated scratch, each image's region 16-byte aligned
  pixels: int


def pack(files: Sequence[bytes], infos: Sequence[PngInfo], payload_offsets: Sequence[int]) -> Batch:
  """Descriptors for decoding files[i] (described by infos[i]) into a payload at byte payload_offsets[i]."""
  chunks, images, palettes = [], [], []
  at = raw = pixels = 0
  for f, info, off in zip(files, infos, payload_offsets):
    stream = b''.join(bytes(f[s:e]) for s, e in info.idat)
    prow = -1
    if info.palette is not None:
      prow = len(palettes)
      p = np.zeros(PALETTE_BYTES, np.uint8)
      p[:len(info.palette)] = np.frombuffer(info.palette, np.uint8)
      palettes.append(p)
    images.append((at, at + len(stream), raw, info.raw_bytes, off, info.H, info.W, info.color_type, info.depth,
                   info.row_bytes, prow, pixels))
    chunks.append(np.frombuffer(stream, np.uint8))
    at += len(stream)
    raw += -(-info.raw_bytes // 16) * 16
    pixels += info.H * info.W
  return Batch(np.concatenate(chunks) if chunks else np.zeros(0, np.uint8),
               np.asarray(images, np.int64).reshape(-1, IMAGE_FIELDS),
               np.stack(palettes) if palettes else np.zeros((1, PALETTE_BYTES), np.uint8), raw, pixels)
