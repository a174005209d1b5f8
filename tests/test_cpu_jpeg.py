"""CPU tests of the device JPEG path's host side: which files twingan_b200/jpeg.py sends to the device, the descriptors it
packs, and the integer restatement oracle/jpeg_oracle.py held bit for bit to PIL (libjpeg-turbo) on generated files, so
the algorithm the kernels of csrc/twg_jpeg.cu implement is pinned without a GPU.  Also: the kernels compile without a
spill, and the ABI of include/twgjpeg.h gets the checks twg.h gets -- every symbol exported, every call from the package
with the declared arity, every launching entry owned by a GPU suite."""
import io
import os
import re
import subprocess

import numpy as np
import pytest
from PIL import Image

import __graft_entry__ as graft
from oracle import jpeg_oracle as JO
from tests.test_cpu_ptxas import _functions, _nvcc
from twingan_b200 import jpeg as J

SIZES = [(1, 1), (7, 9), (8, 8), (15, 17), (16, 16), (17, 33), (255, 257)]


def photo(h, w, seed):
  """Smooth content with noise, like a photograph."""
  r = np.random.default_rng(seed)
  lo = r.integers(0, 256, (h // 8 + 2, w // 8 + 2, 3), dtype=np.uint8)
  a = np.asarray(Image.fromarray(lo).resize((w, h), Image.BILINEAR)).astype(np.int32)
  return np.clip(a + r.integers(-20, 21, a.shape), 0, 255).astype(np.uint8)


def encode(a, **kw):
  b = io.BytesIO()
  Image.fromarray(a).save(b, 'JPEG', **kw)
  return b.getvalue()


def pil_rgb(data):
  with Image.open(io.BytesIO(data)) as im:
    return np.asarray(im.convert('RGB'))


def _swap_app0_for_adobe(data, transform):
  """The same stream with its JFIF APP0 replaced by an Adobe APP14 carrying `transform`."""
  assert data[2:4] == b'\xff\xe0'
  n = (data[4] << 8) | data[5]
  app14 = b'\xff\xee\x00\x0eAdobe\x00\x64\x00\x00\x00\x00' + bytes([transform])
  return data[:2] + app14 + data[4 + n:]


def _with_comments(data, k):
  coms = b''.join(b'\xff\xfe' + (len(c) + 2).to_bytes(2, 'big') + c for c in (b'comment %d ' % i * 40 for i in range(k)))
  return data[:2] + coms + data[2:]


def test_classification():
  a = photo(40, 56, 1)
  dev = lambda d: J.probe(d) is not None
  for ss in (0, 1, 2):
    info = J.parse(encode(a, quality=80, subsampling=ss))
    assert (info.comps[0].h, info.comps[0].v) == {0: (1, 1), 1: (2, 1), 2: (2, 2)}[ss]
  assert dev(encode(a, optimize=True))
  assert dev(encode(a[..., 0].copy()))                                      # grey
  rb = J.parse(encode(a, restart_marker_blocks=3))
  assert rb.restart_interval == 3 and len(rb.segments) == -(-rb.mcus // 3)
  rr = J.parse(encode(a, restart_marker_rows=1, subsampling=2))
  assert rr.restart_interval == rr.mcux and len(rr.segments) == rr.mcuy
  assert dev(_with_comments(encode(a, comment=b'x' * 1000), 50))
  assert dev(_swap_app0_for_adobe(encode(a), 1))
  with pytest.raises(J.Unsupported, match='progressive'):
    J.parse(encode(a, progressive=True))
  with pytest.raises(J.Unsupported, match='components'):
    J.parse(_cmyk(a))
  with pytest.raises(J.Unsupported, match='Adobe transform 0'):
    J.parse(_swap_app0_for_adobe(encode(a), 0))
  d = encode(a)
  for cut in (len(d) - 2, len(d) // 2, 100):
    with pytest.raises(J.Unsupported):
      J.parse(d[:cut])
  with pytest.raises(J.Unsupported):
    J.parse(b'\x89PNG\r\n\x1a\n' + d)
  # no JFIF / Adobe marker: only component ids 1, 2, 3 read as YCbCr
  n = (d[4] << 8) | d[5]
  bare = d[:2] + d[4 + n:]
  assert dev(bare)
  sof = bare.index(b'\xff\xc0')
  rgb_ids = bytearray(bare)
  sos = bare.index(b'\xff\xda')
  for k, cid in enumerate(b'RGB'):
    rgb_ids[sof + 10 + 3 * k] = rgb_ids[sos + 5 + 2 * k] = cid
  with pytest.raises(J.Unsupported, match='component ids'):
    J.parse(bytes(rgb_ids))
  # other sampling factors
  with pytest.raises(J.Unsupported, match='sampling'):
    bad = bytearray(d)
    s = bytes(bad).index(b'\xff\xc0')
    bad[s + 11] = 0x12
    J.parse(bytes(bad))


def _cmyk(a):
  b = io.BytesIO()
  Image.fromarray(a).convert('CMYK').save(b, 'JPEG')
  return b.getvalue()


def test_pack_descriptors():
  files = [encode(photo(17, 33, 2), subsampling=2, restart_marker_blocks=2), encode(photo(8, 8, 3)[..., 0].copy()),
           encode(photo(15, 17, 4), subsampling=1)]
  infos = [J.parse(f) for f in files]
  b = J.pack(files, infos, [5, 1000, 2000])
  assert b.images.shape == (3, J.IMAGE_FIELDS) and b.segs.shape[1] == J.SEG_FIELDS
  assert b.comps[:, 0].tolist() == sorted(b.comps[:, 0].tolist()) and b.blocks == int((b.comps[:, 1] * b.comps[:, 2]).sum())
  assert (b.comps[:, 3] % 16 == 0).all() and b.plane_bytes == b.blocks * 64
  assert b.images[:, 5].tolist() == [5, 1000, 2000] and b.pixels == 17 * 33 + 64 + 15 * 17
  for s in b.segs:                                      # every segment is followed by its marker in the packed data
    img, idx = int(s[2]), int(s[5])
    want = 0xD9 if idx == b.images[img, 7] - 1 else 0xD0 + idx % 8
    assert b.data[s[1]] == 0xFF and b.data[s[1] + 1] == want
  assert len(b.huff) == 4                               # PIL's standard tables, shared across the three files
  # the device Huffman tables decode what the canonical code says
  bits, vals = infos[0].ac[0]
  t = J.huff_table(bits, vals)
  code = k = 0
  for l in range(1, 17):
    for _ in range(bits[l - 1]):
      if l <= 9:
        assert t[code << (9 - l)] == (l << 8) | vals[k]
      else:
        assert code <= t[512 + l] and t[548 + code + t[530 + l]] == vals[k]
      code, k = code + 1, k + 1
    code <<= 1


def _corpus():
  for h, w in SIZES:
    for q in (1, 10, 50, 75, 90, 100):
      for ss in (0, 1, 2):
        extra = ({}, {'restart_marker_blocks': 3}, {'restart_marker_rows': 1})[(h + q + ss) % 3]
        yield (h, w, q, ss, extra)
  for q in range(1, 101, 3):
    yield (24, 40, q, q % 3, {})
  for ss, extra in ((2, {}), (1, {'restart_marker_rows': 2}), (0, {'restart_marker_blocks': 7})):
    yield (1024, 768, 85, ss, extra)
  yield (768, 1024, 95, 2, {'restart_marker_blocks': 1})


def test_oracle_equals_pil_bit_for_bit():
  n = 0
  for h, w, q, ss, extra in _corpus():
    a = photo(h, w, h * 7 + w + q)
    for grey in ((False, True) if (h, w) in ((7, 9), (255, 257)) else (False,)):
      d = encode(a[..., 0].copy() if grey else a, quality=q, subsampling=ss, **extra)
      r = JO.decode(d)
      assert r['status'] == 0, (h, w, q, ss, extra, r['status'])
      assert np.array_equal(r['rgb'], pil_rgb(d)), (h, w, q, ss, extra, grey)
      n += 1
  assert n > 150


def test_oracle_flags_corrupt_streams():
  a = photo(64, 96, 9)
  d = encode(a, restart_marker_blocks=2)
  info = J.parse(d)
  e0 = info.segments[0][1]
  cut = d[:info.segments[3][0] + 3] + b'\xff\xd9'               # truncated mid-segment, EOI appended
  assert JO.decode(cut, J.parse(cut))['status'] & (J.STATUS_TRUNCATED | J.STATUS_RESTART)
  swapped = bytearray(d)                                          # RST1 where RST0 belongs
  swapped[e0 + 1] = 0xD1
  assert JO.decode(bytes(swapped))['status'] & J.STATUS_RESTART
  fill = bytearray(d)                                             # a fill byte before RST0: FF inside the segment
  fill[e0 - 1] = 0xFF
  assert JO.decode(bytes(fill))['status'] & J.STATUS_MARKER


@pytest.fixture(scope='module')
def report(tmp_path_factory):
  nvcc = _nvcc()
  if not nvcc:
    pytest.skip('nvcc not found')
  out = tmp_path_factory.mktemp('ptxas_jpeg')
  cmd = [nvcc] + graft.NVCC_FLAGS + ['-Xptxas', '-v', '-c', '-o', str(out / 'twg_jpeg.o'),
                                     os.path.join(graft.CSRC, 'twg_jpeg.cu')]
  r = subprocess.run(cmd, cwd=str(out), capture_output=True, text=True)
  assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
  return r.stdout + r.stderr


def test_jpeg_kernels_do_not_spill(report):
  fns = {f: s for f, s in _functions(report).items() if re.match(r'_ZN3twg\d+k_jpeg_', f)}
  assert len(fns) == 3, sorted(fns)
  spilling = {f: s for f, s in fns.items() if s != (0, 0)}
  assert not spilling, spilling


def test_jpeg_entries_reject_bad_arguments_without_gpu(built_lib):
  L = built_lib
  assert L.try_call('twgjpeg_entropy', None, 16, 1, 16, 1, 16, 16, 16, 16, None) == -1
  assert 'null' in L.last_error()
  assert L.try_call('twgjpeg_entropy', 16, 16, 0, 16, 1, 16, 16, 16, 16, None) == -1
  assert L.try_call('twgjpeg_entropy', 16, 16, 1, 16, 1, 16, 16, 18, 16, None) == -1    # misaligned coefficients
  assert L.try_call('twgjpeg_idct', 16, 16, 1, 0, 16, 16, 16, None) == -1
  assert L.try_call('twgjpeg_idct', 16, 16, 1, 1, 16, 20, 16, None) == -1
  assert 'aligned' in L.last_error()
  assert L.try_call('twgjpeg_color', 16, 16, 0, 16, 1, 16, None) == -1


def test_jpeg_header_symbols_are_exported_and_owned(built_lib):
  from tests.test_gpu_jpeg import OWNED_ENTRIES
  from twingan_b200 import _lib
  protos = _lib.parse_header(_lib.JPEG_HEADER, _lib.JPEG_PREFIX)
  hdr = open(_lib.JPEG_HEADER).read()
  assert set(re.findall(r'\b(twgjpeg_\w+)\s*\(', hdr)) == set(protos) and protos
  assert not re.findall(r'\bint\s+(twg_\w+)\s*\(', hdr)          # the prefix keeps the two ABIs apart
  for name in protos:
    assert hasattr(built_lib.cdll, name), name
  launching = {n for n, (_, args) in protos.items() if 'twg_stream_t' in args}
  assert launching == OWNED_ENTRIES, launching ^ OWNED_ENTRIES


def test_every_jpeg_library_call_matches_the_header_arity():
  """As test_cpu_abi_host does for twg.h: every call in the package naming a twgjpeg_ entry passes as many arguments as
  include/twgjpeg.h declares."""
  import ast
  from twingan_b200 import _lib
  protos = _lib.parse_header(_lib.JPEG_HEADER, _lib.JPEG_PREFIX)
  pkg = os.path.join(os.path.dirname(graft.CSRC))
  seen = 0
  for fn in sorted(os.listdir(pkg)):
    if not fn.endswith('.py'):
      continue
    for node in ast.walk(ast.parse(open(os.path.join(pkg, fn)).read())):
      if isinstance(node, ast.Call):
        named = [i for i, a in enumerate(node.args) if isinstance(a, ast.Constant) and str(a.value).startswith('twgjpeg_')]
        if named:
          name, args = node.args[named[0]].value, node.args[named[0] + 1:]
          assert name in protos and len(args) == len(protos[name][1]), (fn, node.lineno, name)
          seen += 1
  assert seen == len(protos), seen
