"""CPU tests of the device JPEG encoder's host side and algorithm: the integer restatement tests/jenc_oracle.py held byte
for byte to PIL (libjpeg-turbo) at every output size translate writes, the header twingan_b200/jpeg.py assembles, and the
rounded-division quantisation held to libjpeg-turbo's reciprocal method over the forward DCT's whole range, so the
algorithm the kernels of csrc/twg_jenc.cu implement is pinned without a GPU.  Also: the kernels compile without a spill,
and the ABI of include/twgjenc.h gets the checks twg.h and twgjpeg.h get."""
import io
import os
import re
import subprocess

import numpy as np
import pytest
from PIL import Image

import __graft_entry__ as graft
from tests import jenc_oracle as E
from tests.test_cpu_ptxas import _functions, _nvcc
from twingan_b200 import jpeg as J

HWS = [4, 8, 16, 32, 64, 128, 256]


def pil_jpeg(a):
  b = io.BytesIO()
  Image.fromarray(a).save(b, 'JPEG')
  return b.getvalue()


def inputs(h, w, seed=0):
  """{name: uint8 [h, w, 3]}: seeded noise, smooth gradients, flat colours and per-pixel 0/255 checkerboards (the
  longest codes and many stuffed 0xFF bytes)."""
  r = np.random.default_rng(seed + 1000 * h + w)
  yy, xx = np.mgrid[0:h, 0:w]
  grad = np.stack([xx * 255 // max(w - 1, 1), yy * 255 // max(h - 1, 1), (xx + yy) * 255 // max(h + w - 2, 1)], -1)
  board = ((yy + xx) % 2 * 255).astype(np.uint8)
  return {'noise': r.integers(0, 256, (h, w, 3), dtype=np.uint8), 'gradient': grad.astype(np.uint8),
          'zeros': np.zeros((h, w, 3), np.uint8), 'ones': np.full((h, w, 3), 255, np.uint8),
          'flat': np.broadcast_to(np.array([200, 30, 90], np.uint8), (h, w, 3)).copy(),
          'checker': np.repeat(board[..., None], 3, 2),
          'checker_rgb': np.stack([board, 255 - board, board], -1)}


@pytest.mark.parametrize('hw', HWS)
def test_oracle_equals_pil_byte_for_byte(hw):
  for name, a in inputs(hw, hw).items():
    assert E.encode(a)['file'] == pil_jpeg(a), (hw, name)


def test_oracle_equals_pil_at_other_sizes():
  """Partial MCUs in both directions, odd heights (a row pair padded before downsampling)."""
  for h, w in ((1, 1), (3, 5), (5, 13), (9, 17), (17, 9), (24, 40), (31, 33), (40, 24)):
    for name, a in inputs(h, w).items():
      assert E.encode(a)['file'] == pil_jpeg(a), (h, w, name)


def test_checkerboards_stuff_many_bytes():
  scans = {name: E.encode(inputs(64, 64)[name])['scan'] for name in ('checker', 'checker_rgb')}
  assert scans['checker'].count(b'\xff\x00') > 100 and scans['checker_rgb'].count(b'\xff\x00') >= 8


@pytest.mark.parametrize('hw', [4, 8, 256])
def test_header_equals_pil(hw):
  head = J.encoder_header(hw, hw)
  assert len(head) == 623
  assert pil_jpeg(inputs(hw, hw)['noise'])[:len(head)] == head
  info = J.parse(head + b'\x00' + J.EOI)
  assert (info.H, info.W) == (hw, hw) and [(c.h, c.v) for c in info.comps] == [(2, 2), (1, 1), (1, 1)]


def test_quantisation_tables_are_libjpeg_quality_75():
  head = pil_jpeg(inputs(8, 8)['noise'])
  qt = J.encoder_qt()
  i = head.index(b'\xff\xdb')
  assert head[i + 5:i + 69] == bytes(qt[0].astype(np.uint8)) and head[i + 74:i + 138] == bytes(qt[1].astype(np.uint8))


def _fdct_extremes():
  """The forward DCT of the 64 sign patterns of the DCT basis at full swing (127 / -128): every coefficient at its
  largest magnitude."""
  k = np.arange(8)
  basis = np.cos((2 * k[:, None] + 1) * k[None, :] * np.pi / 16)      # [x, u]
  pats = []
  for u in range(8):
    for v in range(8):
      s = np.outer(basis[:, v], basis[:, u]) >= 0                       # [y, x]
      pats += [np.where(s, 255, 0), np.where(s, 0, 255)]
  return E.fdct(np.asarray(pats))


def test_quantisation_restatement_equals_the_reciprocal_method_exhaustively():
  bound = int(np.abs(_fdct_extremes()).max())
  assert 8000 < bound < 16384, bound
  c = np.arange(-16383, 16384, dtype=np.int64)
  for q in range(1, 256):
    d = q << 3
    assert np.array_equal(E.quantise(c, d), E.quantise_reciprocal(c, d)), d


# ---- the ABI of include/twgjenc.h --------------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def report(tmp_path_factory):
  nvcc = _nvcc()
  if not nvcc:
    pytest.skip('nvcc not found')
  out = tmp_path_factory.mktemp('ptxas_jenc')
  cmd = [nvcc] + graft.NVCC_FLAGS + ['-Xptxas', '-v', '-c', '-o', str(out / 'twg_jenc.o'),
                                     os.path.join(graft.CSRC, 'twg_jenc.cu')]
  r = subprocess.run(cmd, cwd=str(out), capture_output=True, text=True)
  assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
  return r.stdout + r.stderr


def test_jenc_kernels_do_not_spill(report):
  fns = {f: s for f, s in _functions(report).items() if re.search(r'\d+k_jenc_\w+', f)}
  assert len(fns) == 5, sorted(fns)
  spilling = {f: s for f, s in fns.items() if s != (0, 0)}
  assert not spilling, spilling


def test_jenc_entries_reject_bad_arguments_without_gpu(built_lib):
  L = built_lib
  assert L.try_call('twgjenc_dct', None, 1, 8, 8, 16, 16, None) == -1
  assert 'null' in L.last_error()
  assert L.try_call('twgjenc_dct', 16, 0, 8, 8, 16, 16, None) == -1
  assert L.try_call('twgjenc_dct', 16, 1, 8, 70000, 16, 16, None) == -1
  assert L.try_call('twgjenc_dct', 16, 1, 8192, 8192, 16, 16, None) == -1                  # h * w > 2^25
  assert L.try_call('twgjenc_dct', 16, 1, 8, 8, 16, 18, None) == -1                        # misaligned coefficients
  assert 'aligned' in L.last_error()
  assert L.try_call('twgjenc_bits', 16, 1, 0, 8, 16, None) == -1
  assert L.try_call('twgjenc_pack', 16, 16, 1, 8, 8, 20, 16, 16, None) == -1
  assert L.try_call('twgjenc_pack', 16, None, 1, 8, 8, 16, 16, 16, None) == -1
  assert L.cdll.twgjenc_workspace_bytes(0, 8, 8) == -1 and L.cdll.twgjenc_scan_capacity(1, 0, 8) == -1
  assert L.cdll.twgjenc_scan_capacity(2, 256, 256) >= 2 * 2 * 6 * 256 * 208


def test_jenc_header_symbols_are_exported_and_owned(built_lib):
  from tests.test_gpu_jenc import OWNED_ENTRIES
  from twingan_b200 import _lib
  protos = _lib.parse_header(_lib.JENC_HEADER, _lib.JENC_PREFIX)
  hdr = open(_lib.JENC_HEADER).read()
  assert set(re.findall(r'\b(twgjenc_\w+)\s*\(', hdr)) == set(protos) and protos
  assert not re.findall(r'\b(?:int|int64_t)\s+(twg_\w+|twgjpeg_\w+)\s*\(', hdr)
  for name in protos:
    assert hasattr(built_lib.cdll, name), name
  launching = {n for n, (_, args) in protos.items() if 'twg_stream_t' in args}
  assert launching == OWNED_ENTRIES, launching ^ OWNED_ENTRIES


def test_every_jenc_library_call_matches_the_header_arity():
  """Every call in the package naming a twgjenc_ entry -- `lib().call('twgjenc_...', ...)` or `.cdll.twgjenc_...(...)` --
  passes as many arguments as include/twgjenc.h declares."""
  import ast
  from twingan_b200 import _lib
  protos = _lib.parse_header(_lib.JENC_HEADER, _lib.JENC_PREFIX)
  pkg = os.path.dirname(graft.CSRC)
  seen = set()
  for fn in sorted(os.listdir(pkg)):
    if not fn.endswith('.py'):
      continue
    for node in ast.walk(ast.parse(open(os.path.join(pkg, fn)).read())):
      if not isinstance(node, ast.Call):
        continue
      named = [i for i, a in enumerate(node.args) if isinstance(a, ast.Constant) and str(a.value).startswith('twgjenc_')]
      f = node.func
      if named:
        name, args = node.args[named[0]].value, node.args[named[0] + 1:]
      elif isinstance(f, ast.Attribute) and f.attr.startswith('twgjenc_'):
        name, args = f.attr, node.args
      else:
        continue
      assert name in protos and len(args) == len(protos[name][1]), (fn, node.lineno, name)
      seen.add(name)
  assert seen == set(protos), set(protos) - seen
