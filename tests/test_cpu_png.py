"""CPU tests of the device PNG path's host side: which files twingan_b200/png.py sends to the device, the descriptors it
packs, and the restatement tests/png_oracle.py held to PIL and zlib on generated files, so the algorithm of
csrc/twg_png.cu is pinned without a GPU.  Also: the kernels compile without a spill, and include/twgpng.h gets the ABI
checks twg.h gets -- every symbol exported, every call from the package with the declared arity, every launching entry
owned by a GPU suite."""
import io
import os
import re
import subprocess
import zlib

import numpy as np
import pytest
from PIL import Image, PngImagePlugin

import __graft_entry__ as graft
from tests import png_oracle as PO
from tests.test_cpu_ptxas import _functions, _nvcc
from twingan_b200 import png as P

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
FIXTURES = ('ROJFO5Y2C4CT1SI51NBI8G8QVD42QK39_0.png', 'IVW7BL5WMJRWF8TMXF9RNYE2O1VIPF13_0.png')
KINDS = [(ct, d) for ct, ds in sorted(P.DEPTHS.items()) for d in ds]
WIDTHS = (1, 3, 7, 9, 17, 64, 1001)


def chunk(cid: bytes, body: bytes) -> bytes:
  return len(body).to_bytes(4, 'big') + cid + body + zlib.crc32(body, zlib.crc32(cid)).to_bytes(4, 'big')


def filtered(rows: np.ndarray, bpp: int, filters) -> bytes:
  """The scanlines of uint8 [H, row bytes] `rows`, row y filtered with filters[y % len(filters)]."""
  out = []
  prev = np.zeros(rows.shape[1], np.int64)
  for y, r in enumerate(rows.astype(np.int64)):
    f = filters[y % len(filters)]
    left = np.concatenate([np.zeros(bpp, np.int64), r[:-bpp]]) if len(r) > bpp else np.zeros(len(r), np.int64)
    ul = np.concatenate([np.zeros(bpp, np.int64), prev[:-bpp]]) if len(r) > bpp else np.zeros(len(r), np.int64)
    if len(r) <= bpp:
      left, ul = np.zeros(len(r), np.int64), np.zeros(len(r), np.int64)
    if f == 0:
      x = r
    elif f == 1:
      x = r - left
    elif f == 2:
      x = r - prev
    elif f == 3:
      x = r - ((left + prev) >> 1)
    else:
      p = left + prev - ul
      pa, pb, pc = abs(p - left), abs(p - prev), abs(p - ul)
      x = r - np.where((pa <= pb) & (pa <= pc), left, np.where(pb <= pc, prev, ul))
    out.append(bytes([f]) + bytes((x & 255).astype(np.uint8)))
    prev = r
  return b''.join(out)


def make_png(rows, W, ct, depth, filters=(0,), palette=None, extra=(), stream=None, split=None, level=6,
             strategy=zlib.Z_DEFAULT_STRATEGY, after_idat=(), interlace=0):
  """A PNG file of uint8 [H, row bytes] `rows`: extra chunks before the IDAT run, the zlib stream (given, or compressed
  at `level` / `strategy`) cut into IDAT chunks at `split` offsets, then `after_idat` and IEND."""
  H = rows.shape[0]
  bpp = max(1, P.CHANNELS[ct] * depth // 8)
  if stream is None:
    c = zlib.compressobj(level, zlib.DEFLATED, 15, 9, strategy)
    stream = c.compress(filtered(rows, bpp, filters)) + c.flush()
  cuts = [0] + sorted(split or []) + [len(stream)]
  ihdr = W.to_bytes(4, 'big') + H.to_bytes(4, 'big') + bytes([depth, ct, 0, 0, interlace])
  out = [P.SIGNATURE, chunk(b'IHDR', ihdr)]
  if palette is not None:
    out.append(chunk(b'PLTE', palette))
  out += [chunk(c, b) for c, b in extra]
  out += [chunk(b'IDAT', stream[a:b]) for a, b in zip(cuts, cuts[1:])]
  out += [chunk(c, b) for c, b in after_idat]
  out.append(chunk(b'IEND', b''))
  return b''.join(out)


def random_rows(H, W, ct, depth, seed):
  rb = (W * P.CHANNELS[ct] * depth + 7) // 8
  return np.random.default_rng(seed).integers(0, 256, (H, rb), dtype=np.uint8)


def smooth_rows(H, W, ct, depth, seed):
  """Rows of smooth content (long matches, every filter useful) for 8- and 16-bit samples; noise otherwise."""
  if depth < 8:
    return random_rows(H, W, ct, depth, seed)
  r = np.random.default_rng(seed)
  ch = P.CHANNELS[ct] * depth // 8
  y, x = np.mgrid[0:H, 0:W]
  base = (x * 3 + y * 5)[..., None] + r.integers(0, 4, (H, W, ch))
  return (base % 256).astype(np.uint8).reshape(H, W * ch)


def pil_rgb(data):
  with Image.open(io.BytesIO(data)) as im:
    return np.asarray(im.convert('RGB'))


def photo(h, w, seed):
  r = np.random.default_rng(seed)
  lo = r.integers(0, 256, (h // 8 + 2, w // 8 + 2, 3), dtype=np.uint8)
  a = np.asarray(Image.fromarray(lo).resize((w, h), Image.BILINEAR)).astype(np.int32)
  return np.clip(a + r.integers(-20, 21, a.shape), 0, 255).astype(np.uint8)


PALETTE = bytes(np.random.default_rng(0).integers(0, 256, 3 * 200, dtype=np.uint8))


def kind_file(ct, depth, W, H=5, seed=0, **kw):
  pal = PALETTE[:3 * (1 << depth) - 3] if ct == 3 else None      # one entry short: the last index reads the padding
  return make_png(random_rows(H, W, ct, depth, seed), W, ct, depth, palette=pal, **kw)


# ---- classification -------------------------------------------------------------------------------------------------

def test_every_legal_kind_is_accepted_and_others_declined():
  for ct, d in KINDS:
    info = P.parse(kind_file(ct, d, 9))
    assert (info.color_type, info.depth, info.W, info.H) == (ct, d, 9, 5)
  for ct, d in ((0, 3), (2, 4), (3, 16), (4, 4), (6, 1), (5, 8)):
    f = bytearray(make_png(random_rows(2, 4, 0, 8, 0), 2, 0, 8))
    f[24], f[25] = d, ct
    f[29:33] = zlib.crc32(bytes(f[12:29])).to_bytes(4, 'big')
    with pytest.raises(P.Unsupported, match='colour type'):
      P.parse(bytes(f))


def test_declined_files():
  a = photo(20, 24, 1)
  with pytest.raises(P.Unsupported, match='interlaced'):
    P.parse(make_png(random_rows(4, 4, 2, 8, 1), 4, 2, 8, interlace=1))
  b = io.BytesIO()
  Image.fromarray(a).save(b, 'PNG', save_all=True, append_images=[Image.fromarray(a[::-1].copy())])
  with pytest.raises(P.Unsupported, match='APNG'):
    P.parse(b.getvalue())
  p = Image.fromarray(a).convert('P')
  b = io.BytesIO()
  p.save(b, 'PNG', transparency=3)
  with pytest.raises(P.Unsupported, match='tRNS'):
    P.parse(b.getvalue())
  rows = random_rows(3, 5, 2, 8, 2)
  with pytest.raises(P.Unsupported, match='chunk'):
    P.parse(make_png(rows, 5, 2, 8, extra=[(b'vpAg', b'\0' * 9)]))
  good = make_png(rows, 5, 2, 8, split=[10])
  P.parse(good)
  bad_crc = bytearray(good)
  bad_crc[-20] ^= 1                                             # inside the last IDAT's data
  with pytest.raises(P.Unsupported, match='CRC'):
    P.parse(bytes(bad_crc))
  with pytest.raises(P.Unsupported):
    P.parse(good[:-12])                                         # no IEND
  with pytest.raises(P.Unsupported, match='after the IDAT run'):
    P.parse(good[:-12] + chunk(b'tEXt', b'k\0v') + good[-12:])   # a chunk after IDAT
  with pytest.raises(P.Unsupported, match='after IEND'):
    P.parse(good + chunk(b'tEXt', b'k\0v'))                     # a chunk after IEND
  with pytest.raises(P.Unsupported, match='after IEND'):
    P.parse(good + b'\0')
  with pytest.raises(P.Unsupported, match='after the IDAT run'):  # data between IDATs
    P.parse(_tEXt_between_idats(rows))
  with pytest.raises(P.Unsupported, match='without PLTE'):
    P.parse(make_png(random_rows(2, 2, 3, 8, 0), 2, 3, 8))
  for stream in (b'', zlib.compress(b'')[:5]):                 # no room for a zlib header and trailer
    with pytest.raises(P.Unsupported, match='shorter than'):
      P.parse(make_png(rows, 5, 2, 8, stream=stream))
  P.parse(make_png(rows, 5, 2, 8, stream=zlib.compress(b'')))     # 8 bytes: accepted, the device flags it short
  with pytest.raises(P.Unsupported, match='not a PNG'):
    P.parse(b'\xff\xd8\xff' + good)
  with pytest.raises(P.Unsupported):
    P.parse(good[:40])


def _tEXt_between_idats(rows):
  f = make_png(rows, 5, 2, 8, split=[10])
  i = f.index(b'IDAT') - 4
  n = int.from_bytes(f[i:i + 4], 'big')
  j = i + 12 + n
  return f[:j] + chunk(b'tEXt', b'k\0v') + f[j:]


ANCILLARY = [(b'sRGB', b'\0'), (b'gAMA', (45455).to_bytes(4, 'big')), (b'cHRM', bytes(range(32))),
             (b'pHYs', (2835).to_bytes(4, 'big') * 2 + b'\1'), (b'tIME', b'\x07\xe6\x01\x02\x03\x04\x05'),
             (b'bKGD', b'\0\1\0\2\0\3'), (b'sBIT', b'\5\6\7'), (b'tEXt', b'Comment\0hello'),
             (b'zTXt', b'Title\0\0' + zlib.compress(b'compressed text' * 50)),
             (b'iTXt', b'Desc\0\1\0en\0Desc\0' + zlib.compress('ünïcode'.encode())),
             (b'iTXt', b'Plain\0\0\0\0\0plain'), (b'iCCP', b'prof\0\0' + zlib.compress(b'\0' * 3000)),
             (b'eXIf', b'MM\0*\0\0\0\x08\0\0'), (b'tRNS', b'\0\1\0\2\0\3')]


def test_ancillary_chunks_leave_pils_pixels_alone():
  rows = smooth_rows(6, 11, 2, 8, 3)
  plain = make_png(rows, 11, 2, 8, filters=(4,))
  want = pil_rgb(plain)
  for cid, body in ANCILLARY:
    f = make_png(rows, 11, 2, 8, filters=(4,), extra=[(cid, body)])
    assert P.probe(f) is not None, cid
    assert np.array_equal(pil_rgb(f), want), cid
  f = make_png(rows, 11, 2, 8, filters=(4,), extra=ANCILLARY)
  assert P.probe(f) is not None and np.array_equal(pil_rgb(f), want)
  grey = random_rows(4, 6, 0, 16, 4)
  g = make_png(grey, 6, 0, 16, extra=[(b'tRNS', b'\0\7')])
  assert P.probe(g) is not None and np.array_equal(pil_rgb(g), pil_rgb(make_png(grey, 6, 0, 16)))


def test_chunks_pil_raises_on_are_declined():
  rows = smooth_rows(3, 4, 2, 8, 5)
  big = zlib.compress(b'a' * (PngImagePlugin.MAX_TEXT_CHUNK + 10))
  cases = [(b'zTXt', b'k\0\1' + zlib.compress(b'x')),              # unknown compression method
           (b'zTXt', b'k\0\0' + big), (b'iTXt', b'k\0\1\0\0\0' + big), (b'iCCP', b'p\0\0' + big),
           (b'iCCP', b'p\0\1' + zlib.compress(b'x')), (b'sRGB', b''), (b'pHYs', b'\0' * 8), (b'gAMA', b'\0' * 3),
           (b'tRNS', b'\0')]
  for cid, body in cases:
    f = make_png(rows, 4, 2, 8, extra=[(cid, body)])
    assert P.probe(f) is None, (cid, body[:8])
  mem = [(b'tEXt', b'k%d\0' % i + b'v' * (PngImagePlugin.MAX_TEXT_CHUNK // 2)) for i in range(140)]
  f = make_png(rows, 4, 2, 8, extra=mem)
  with pytest.raises(ValueError, match='MAX_TEXT_MEMORY'):
    pil_rgb(f)
  assert P.probe(f) is None


def test_pack_descriptors():
  files = [kind_file(2, 8, 7, H=3), kind_file(3, 4, 9, H=2), kind_file(0, 1, 17, H=4), kind_file(3, 8, 5, H=1)]
  infos = [P.parse(f) for f in files]
  b = P.pack(files, infos, [5, 1000, 2000, 3000])
  assert b.images.shape == (4, P.IMAGE_FIELDS)
  im = b.images
  assert im[:, 4].tolist() == [5, 1000, 2000, 3000]
  assert im[:, 5].tolist() == [3, 2, 4, 1] and im[:, 6].tolist() == [7, 9, 17, 5]
  assert im[:, 9].tolist() == [21, 5, 3, 5] and im[:, 3].tolist() == [3 * 22, 2 * 6, 4 * 4, 1 * 6]
  assert im[:, 10].tolist() == [-1, 0, -1, 1] and b.palettes.shape == (2, 768)
  assert im[:, 11].tolist() == [0, 21, 39, 107] and b.pixels == 112
  assert (im[:, 2] % 16 == 0).all() and (im[1:, 2] >= im[:-1, 2] + im[:-1, 3]).all() and b.raw_bytes >= im[-1, 2] + im[-1, 3]
  for row, f, info in zip(im, files, infos):                  # each stream is the IDAT payloads back to back
    assert b.data[row[0]:row[1]].tobytes() == PO.stream_of(f, info)
    assert zlib.decompress(b.data[row[0]:row[1]].tobytes()) and len(zlib.decompress(PO.stream_of(f, info))) == row[3]
  assert b.palettes[0, :len(infos[1].palette)].tobytes() == infos[1].palette and not b.palettes[0, len(infos[1].palette):].any()


# ---- the restatement against PIL and zlib -------------------------------------------------------------------------

def test_restatement_equals_pil_for_every_kind():
  n = 0
  for ct, d in KINDS:
    for W in WIDTHS:
      for H in ((1, 4) if W < 1000 else (3,)):
        f = kind_file(ct, d, W, H=H, seed=W * 31 + H + d, filters=(0, 1, 2, 3, 4))
        r = PO.decode(f)
        assert r['status'] == 0, (ct, d, W, H)
        assert np.array_equal(r['rgb'], pil_rgb(f)), (ct, d, W, H)
        n += 1
  assert n == len(KINDS) * 13


def test_grey16_clamps_and_16_bit_colour_takes_the_high_byte():
  rows = np.array([[0x00, 0x00, 0x00, 0xC8, 0x00, 0xFF, 0x01, 0x00, 0xFF, 0xFF]], np.uint8)
  assert PO.decode(make_png(rows, 5, 0, 16))['rgb'][0, :, 0].tolist() == [0, 200, 255, 255, 255]
  assert np.array_equal(pil_rgb(make_png(rows, 5, 0, 16))[0, :, 0], [0, 200, 255, 255, 255])
  f = make_png(np.array([[0x12, 0x34, 0xAB, 0xCD]], np.uint8), 1, 4, 16)       # grey+alpha 16: high byte of grey
  assert PO.decode(f)['rgb'].tolist() == pil_rgb(f).tolist() == [[[0x12] * 3]]


def test_filters_each_forced_and_mixed_per_row():
  for ct, d in ((2, 8), (6, 16), (0, 8), (0, 2), (4, 8), (3, 8), (2, 16)):
    for filters in ((0,), (1,), (2,), (3,), (4,), (0, 1, 2, 3, 4), (4, 2, 3, 1, 0, 4, 4)):
      rows = smooth_rows(9, 13, ct, d, 7)
      pal = PALETTE if ct == 3 else None
      f = make_png(rows, 13, ct, d, filters=filters, palette=pal)
      r = PO.decode(f)
      assert r['status'] == 0 and np.array_equal(r['rows'], rows), (ct, d, filters)
      assert np.array_equal(r['rgb'], pil_rgb(f)), (ct, d, filters)


def _streams():
  """(name, raw bytes, zlib stream) over levels, strategies and long distances."""
  rng = np.random.default_rng(11)
  text = (b'the quick brown fox jumps over the lazy dog ' * 40 + bytes(rng.integers(0, 256, 500, dtype=np.uint8)))
  far = bytes(rng.integers(0, 256, 300, dtype=np.uint8))
  long_dist = far + bytes(rng.integers(0, 256, 32768 - 300, dtype=np.uint8)) + far     # a match 32 768 back
  out = []
  for level in range(10):
    out.append(('level%d' % level, text, zlib.compress(text, level)))
  for name, strategy in (('fixed', zlib.Z_FIXED), ('rle', zlib.Z_RLE), ('huffman', zlib.Z_HUFFMAN_ONLY),
                         ('filtered', zlib.Z_FILTERED)):
    c = zlib.compressobj(9, zlib.DEFLATED, 15, 9, strategy)
    out.append((name, text, c.compress(text) + c.flush()))
  out.append(('distance32768', long_dist, zlib.compress(long_dist, 9)))
  c = zlib.compressobj(6)
  parts = c.compress(text[:700]) + c.flush(zlib.Z_FULL_FLUSH) + c.compress(text[700:]) + c.flush()  # empty stored block
  out.append(('full_flush', text, parts))
  return out


def test_inflate_restatement_equals_zlib():
  for name, raw, stream in _streams():
    got, st = PO.inflate(stream, len(raw))
    assert st == 0 and got == raw == zlib.decompress(stream), name


def test_streams_in_png_files_split_anywhere():
  rows = smooth_rows(40, 50, 2, 8, 9)
  want = pil_rgb(make_png(rows, 50, 2, 8))
  for level in (0, 1, 6, 9):
    for strategy in (zlib.Z_DEFAULT_STRATEGY, zlib.Z_FIXED, zlib.Z_RLE, zlib.Z_HUFFMAN_ONLY):
      for split in ([], [1], [2, 3], [5, 17, 100, 101]):          # inside the zlib header too
        f = make_png(rows, 50, 2, 8, filters=(1, 4), level=level, strategy=strategy, split=split)
        info = P.parse(f)
        assert len(info.idat) == len(split) + 1
        r = PO.decode(f, info)
        assert r['status'] == 0 and np.array_equal(r['rgb'], want), (level, strategy, split)
        assert np.array_equal(pil_rgb(f), want)


def test_pil_written_and_fixture_files():
  for a, mode in ((photo(37, 53, 1), None), (photo(20, 30, 2)[..., 0].copy(), None), (photo(9, 11, 3), 'P')):
    img = Image.fromarray(a).convert('P') if mode == 'P' else Image.fromarray(a)
    for kw in ({}, {'optimize': True}, {'compress_level': 1}, {'compress_level': 9}):
      b = io.BytesIO()
      img.save(b, 'PNG', **kw)
      f = b.getvalue()
      r = PO.decode(f)
      assert r['status'] == 0 and np.array_equal(r['rgb'], pil_rgb(f)), (a.shape, mode, kw)
  for fn in FIXTURES:
    f = open(os.path.join(GOLDEN, fn), 'rb').read()
    info = P.parse(f)
    assert info.color_type == 2 and info.depth == 8 and len(info.idat) >= 2
    stream = PO.stream_of(f, info)
    assert len(stream) > 100000
    r = PO.decode(f, info)
    assert r['status'] == 0 and np.array_equal(r['rgb'], pil_rgb(f)), fn


# ---- corrupt streams ----------------------------------------------------------------------------------------------

def corrupt_cases():
  """(name, rows, W, ct, depth, zlib stream, expected status) of files png.parse accepts whose data is damaged."""
  rows = smooth_rows(12, 20, 2, 8, 13)
  raw = filtered(rows, 3, (1, 4))
  good = zlib.compress(raw, 6)
  size = len(raw)
  cases = []

  def add(name, stream, want, r=rows):
    cases.append((name, r, 20, 2, 8, stream, want))

  add('cm7', bytes([0x77]) + good[1:], P.STATUS_HEADER)
  add('cinfo8', bytes([0x88, (31 - (0x88 * 256) % 31) % 31]) + good[2:], P.STATUS_HEADER)
  add('fcheck', good[:1] + bytes([good[1] ^ 1]) + good[2:], P.STATUS_HEADER)
  add('fdict', bytes([0x78, 0xBB]) + good[2:], P.STATUS_HEADER)   # 0x78BB % 31 == 0 with FDICT
  add('btype3', good[:2] + bytes([0x07]) + good[3:], P.STATUS_BLOCK)
  stored = zlib.compress(raw, 0)
  bad_nlen = bytearray(stored)
  bad_nlen[5] ^= 0xFF
  add('stored_nlen', bytes(bad_nlen), P.STATUS_BLOCK)
  add('stored_cut', stored[:200], P.STATUS_TRUNCATED)
  add('truncated', good[:len(good) // 2], P.STATUS_TRUNCATED)
  add('no_trailer', good[:-4], P.STATUS_TRUNCATED)
  add('adler', good[:-1] + bytes([good[-1] ^ 1]), P.STATUS_ADLER)
  add('trailing', good + b'\0\0', P.STATUS_TRAILING)
  add('long', zlib.compress(raw + b'\0' * 40), P.STATUS_LONG)
  add('long_stored', zlib.compress(raw + b'\1' * 40, 0), P.STATUS_LONG)
  short = zlib.compress(raw[:-21])
  add('short', short, P.STATUS_SHORT)
  # hand-assembled deflate bodies
  def z(body: bytes, data=b'') -> bytes:
    return b'\x78\x01' + body + zlib.adler32(data).to_bytes(4, 'big')
  # fixed block: literal 'a' (0x61 -> code 0x30 + 0x61 = 0x91, 8 bits), then length symbol 286 (invalid)
  add('lit286', z(_bits([(1, 1), (1, 2), (_rev(0x91, 8), 8), (_rev(0xC6, 8), 8)]) + b'\0' * 4), P.STATUS_SYMBOL)
  # fixed block: length 3 (sym 257, 7-bit code 0000001) with distance code 30 (invalid)
  add('dist30', z(_bits([(1, 1), (1, 2), (_rev(0x91, 8), 8), (_rev(1, 7), 7), (_rev(30, 5), 5)]) + b'\0' * 4),
      P.STATUS_SYMBOL)
  # fixed block: 'a', then a match of 3 at distance 2 (before the start)
  add('dist_far', z(_bits([(1, 1), (1, 2), (_rev(0x91, 8), 8), (_rev(1, 7), 7), (_rev(1, 5), 5)]) + b'\0' * 4),
      P.STATUS_DISTANCE)
  # a window of 256 bytes (CINFO 0) and a match 300 back
  blob = bytes(np.random.default_rng(3).integers(0, 256, size, dtype=np.uint8))
  c = zlib.compressobj(9, zlib.DEFLATED, 15)
  far = c.compress(blob[:300] + blob[:300] + blob[600:size]) + c.flush()
  add('window', bytes([0x08, (31 - (0x08 * 256) % 31) % 31]) + far[2:], P.STATUS_DISTANCE,
      r=np.frombuffer(blob, np.uint8)[:size].reshape(12, 61)[:, 1:].copy())
  # dynamic block headers: HLIT 287 (too many), an over-subscribed code-length code, a repeat with nothing before
  add('hlit', z(_bits([(1, 1), (2, 2), (30, 5), (0, 5), (15, 4)]) + b'\0' * 20), P.STATUS_CODES)
  add('cl_over', z(_bits([(1, 1), (2, 2), (0, 5), (0, 5), (0, 4)] + [(1, 3)] * 4) + b'\0' * 20), P.STATUS_CODES)
  # code-length code: symbols 16 and 18 of length 1 (complete); the first code, 16, repeats nothing
  cl = [(0, 5), (0, 5), (0, 4)]                        # HLIT 257, HDIST 1, HCLEN 4: lengths of 16, 17, 18, 0
  add('repeat_first', z(_bits([(1, 1), (2, 2)] + cl + [(1, 3), (0, 3), (1, 3), (0, 3)] + [(0, 1)] + [(0, 2)])
                        + b'\0' * 20), P.STATUS_CODES)
  # filter type 5 on the second row
  bad_rows = bytearray(raw)
  bad_rows[61] = 5
  add('filter5', zlib.compress(bytes(bad_rows)), P.STATUS_FILTER)
  return cases


def _rev(v, n):
  return int(format(v, '0%db' % n)[::-1], 2)


def _bits(fields):
  """Pack (value, width) fields LSB first (deflate's bit order; Huffman codes passed already reversed)."""
  acc = n = 0
  for v, w in fields:
    acc |= v << n
    n += w
  return acc.to_bytes((n + 7) // 8, 'little')


def corrupt_files():
  out = []
  for name, rows, W, ct, depth, stream, want in corrupt_cases():
    f = make_png(rows, W, ct, depth, stream=stream)
    assert P.probe(f) is not None, name
    out.append((name, f, want))
  return out


def test_corrupt_streams_are_classified():
  for name, f, want in corrupt_files():
    assert PO.decode(f)['status'] == want, (name, PO.decode(f)['status'], want)


# ---- compile and ABI audits -----------------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def report(tmp_path_factory):
  nvcc = _nvcc()
  if not nvcc:
    pytest.skip('nvcc not found')
  out = tmp_path_factory.mktemp('ptxas_png')
  cmd = [nvcc] + graft.NVCC_FLAGS + ['-Xptxas', '-v', '-c', '-o', str(out / 'twg_png.o'),
                                     os.path.join(graft.CSRC, 'twg_png.cu')]
  r = subprocess.run(cmd, cwd=str(out), capture_output=True, text=True)
  assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
  return r.stdout + r.stderr


def test_png_kernels_do_not_spill(report):
  fns = {f: s for f, s in _functions(report).items() if re.match(r'_ZN3twg\d+k_png_', f)}
  assert len(fns) == 3, sorted(fns)
  spilling = {f: s for f, s in fns.items() if s != (0, 0)}
  assert not spilling, spilling


def test_png_entries_reject_bad_arguments_without_gpu(built_lib):
  L = built_lib
  assert L.try_call('twgpng_inflate', None, 16, 1, 16, 16, None) == -1
  assert 'null' in L.last_error()
  assert L.try_call('twgpng_inflate', 16, 16, 0, 16, 16, None) == -1
  assert L.try_call('twgpng_unfilter', 16, None, 1, 16, None) == -1
  assert L.try_call('twgpng_unfilter', 16, 16, 0, 16, None) == -1
  assert L.try_call('twgpng_rgb', 16, 16, 1, 16, 0, 16, 16, None) == -1
  assert L.try_call('twgpng_rgb', 16, 16, 1, None, 1, 16, 16, None) == -1


def test_png_header_symbols_are_exported_and_owned(built_lib):
  from tests.test_gpu_png import OWNED_ENTRIES
  from twingan_b200 import _lib
  protos = _lib.parse_header(_lib.PNG_HEADER, _lib.PNG_PREFIX)
  hdr = open(_lib.PNG_HEADER).read()
  assert set(re.findall(r'\b(twgpng_\w+)\s*\(', hdr)) == set(protos) and protos
  assert not re.findall(r'\bint\s+(twg_\w+)\s*\(', hdr)
  for name in protos:
    assert hasattr(built_lib.cdll, name), name
  launching = {n for n, (_, args) in protos.items() if 'twg_stream_t' in args}
  assert launching == OWNED_ENTRIES, launching ^ OWNED_ENTRIES


def test_every_png_library_call_matches_the_header_arity():
  import ast
  from twingan_b200 import _lib
  protos = _lib.parse_header(_lib.PNG_HEADER, _lib.PNG_PREFIX)
  pkg = os.path.dirname(graft.CSRC)
  seen = 0
  for fn in sorted(os.listdir(pkg)):
    if not fn.endswith('.py'):
      continue
    for node in ast.walk(ast.parse(open(os.path.join(pkg, fn)).read())):
      if isinstance(node, ast.Call):
        named = [i for i, a in enumerate(node.args) if isinstance(a, ast.Constant) and str(a.value).startswith('twgpng_')]
        if named:
          name, args = node.args[named[0]].value, node.args[named[0] + 1:]
          assert name in protos and len(args) == len(protos[name][1]), (fn, node.lineno, name)
          seen += 1
  assert seen == len(protos), seen
