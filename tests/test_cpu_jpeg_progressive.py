"""CPU tests of the device progressive JPEG path's host side: which files twingan_b200/jpeg_progressive.py sends to the
device and why it declines the others, the descriptors and scan levels it packs, and the restatement tests/jpegp_oracle.py
held bit for bit to PIL (libjpeg-turbo) on PIL's progressive files and on files the re-encoder writes under other scan
scripts, so the algorithm csrc/twg_jpegp.cu implements is pinned without a GPU.  Also: the kernel compiles without a
spill, and the ABI of include/twgjpegp.h gets the checks the other headers get."""
import os
import re
import subprocess

import numpy as np
import pytest

import __graft_entry__ as graft
from oracle import jpeg_oracle as JO
from tests import jpegp_oracle as PO
from tests.test_cpu_jpeg import SIZES, encode, photo, pil_rgb
from tests.test_cpu_ptxas import _functions, _nvcc
from twingan_b200 import jpeg as J
from twingan_b200 import jpeg_progressive as P

EW = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'ew.jpg')

# scan scripts PIL never writes: (name, script for a 3-component frame, restart interval)
Y, CB, CR = (0,), (1,), (2,)
SCRIPTS = [
    ('standard', PO.STANDARD_SCRIPT, 0),
    ('standard_rst1', PO.STANDARD_SCRIPT, 1),
    ('dc_apart', [(Y, 0, 0, 0, 0), (CB, 0, 0, 0, 0), (CR, 0, 0, 0, 0), (Y, 1, 63, 0, 0), (CB, 1, 63, 0, 0),
                  (CR, 1, 63, 0, 0)], 0),
    ('cbcr_dc_deep', [(Y, 0, 0, 0, 4), ((1, 2), 0, 0, 0, 3), (Y, 0, 0, 4, 3), ((1, 2), 0, 0, 3, 2), (Y, 0, 0, 3, 2),
                      ((0, 1, 2), 0, 0, 2, 1), ((0, 1, 2), 0, 0, 1, 0), (Y, 1, 63, 0, 3), (Y, 1, 63, 3, 2),
                      (Y, 1, 63, 2, 1), (Y, 1, 63, 1, 0), (CB, 1, 63, 0, 1), (CB, 1, 63, 1, 0), (CR, 1, 63, 0, 0)], 3),
    ('bands', [((0, 1, 2), 0, 0, 0, 0)] + [(c, a, b, 0, 0) for c in (Y, CB, CR)
                                           for a, b in ((1, 1), (2, 3), (4, 9), (10, 20), (21, 40), (41, 63))], 2),
    ('split_refine', [((0, 1, 2), 0, 0, 0, 2), (Y, 1, 5, 0, 2), (Y, 6, 63, 0, 2), (CB, 1, 63, 0, 1), (CR, 1, 63, 0, 1),
                      (Y, 1, 30, 2, 1), (Y, 31, 63, 2, 1), ((0, 1, 2), 0, 0, 2, 1), ((0, 1, 2), 0, 0, 1, 0),
                      (Y, 1, 2, 1, 0), (Y, 3, 63, 1, 0), (CB, 1, 40, 1, 0), (CB, 41, 63, 1, 0), (CR, 1, 63, 1, 0)], 0),
    ('eob_runs_rst', [((0, 1, 2), 0, 0, 0, 1), (Y, 1, 63, 0, 3), (CB, 1, 63, 0, 2), (CR, 1, 63, 0, 2),
                      (Y, 1, 63, 3, 2), (Y, 1, 63, 2, 1), ((0, 1, 2), 0, 0, 1, 0), (CB, 1, 63, 2, 1),
                      (CR, 1, 63, 2, 1), (Y, 1, 63, 1, 0), (CB, 1, 63, 1, 0), (CR, 1, 63, 1, 0)], 5),
]
GREY_SCRIPT = [((0,), 0, 0, 0, 2), ((0,), 1, 63, 0, 2), ((0,), 0, 0, 2, 1), ((0,), 1, 63, 2, 1), ((0,), 0, 0, 1, 0),
               ((0,), 1, 63, 1, 0)]


def pil_corpus():
  """(name, bytes) of progressive files PIL writes: every sampling, grey, optimize, restart markers, many sizes."""
  out = []
  for h, w in SIZES:
    for q in (1, 10, 50, 75, 90, 97):      # PIL's buffer for a progressive file cannot hold every 257-wide q100 one
      for ss in (0, 1, 2):
        extra = ({}, {'restart_marker_blocks': 3}, {'restart_marker_rows': 1}, {'optimize': True})[(h + q + ss) % 4]
        out.append(('%dx%d_q%d_ss%d_%s' % (h, w, q, ss, extra), encode(photo(h, w, h + w + q), quality=q,
                                                                          subsampling=ss, progressive=True, **extra)))
  for q in range(1, 101, 4):
    out.append(('24x40_q%d' % q, encode(photo(24, 40, q), quality=q, subsampling=q % 3, progressive=True)))
  for h, w in ((7, 9), (255, 257), (16, 16)):
    out.append(('grey_%dx%d' % (h, w), encode(photo(h, w, 6)[..., 0].copy(), quality=70, progressive=True)))
  out.append(('grey_rst', encode(photo(33, 20, 7)[..., 0].copy(), progressive=True, restart_marker_blocks=1)))
  return out


def reencoded_corpus(with_base=False):
  """(name, bytes) of baseline files re-encoded under SCRIPTS (and a grey script), each at every sampling; with
  `with_base`, (name, bytes, the baseline file)."""
  out = []
  for name, script, ri in SCRIPTS:
    for ss in (0, 1, 2):
      base = encode(photo(35, 53, ss + len(name)), quality=90, subsampling=ss)
      out.append(('%s_ss%d' % (name, ss), PO.reencode(base, script, ri), base))
  base = encode(photo(29, 37, 9)[..., 0].copy(), quality=80)
  out.append(('grey_script', PO.reencode(base, GREY_SCRIPT, 2), base))
  return out if with_base else [(n, f) for n, f, _ in out]


def test_accepts_pil_progressive_files_and_the_reference_demo_input():
  a = photo(40, 56, 1)
  for ss in (0, 1, 2):
    info = P.parse(encode(a, quality=80, subsampling=ss, progressive=True))
    assert (info.comps[0].h, info.comps[0].v) == {0: (1, 1), 1: (2, 1), 2: (2, 2)}[ss]
    assert len(info.scans) == 10 and info.levels == 3
  for kw in ({'optimize': True}, {'restart_marker_blocks': 3}, {'restart_marker_rows': 1}):
    assert P.probe(encode(a, progressive=True, **kw)) is not None, kw
  grey = P.parse(encode(a[..., 0].copy(), progressive=True))
  assert len(grey.comps) == 1 and [s.level for s in grey.scans] == [0, 0, 0, 1, 1, 2]
  ew = P.parse(open(EW, 'rb').read())
  assert (ew.H, ew.W, len(ew.scans), ew.levels) == (864, 720, 10, 3)
  # the baseline parser keeps declining them, with the same message
  with pytest.raises(J.Unsupported, match='progressive'):
    J.parse(open(EW, 'rb').read())
  # and this one declines baseline files
  with pytest.raises(J.Unsupported, match='not progressive'):
    P.parse(encode(a))


def _scan_at(data, k):
  """Offset of the k-th SOS marker."""
  at = -1
  for _ in range(k + 1):
    at = data.index(b'\xff\xda', at + 1)
  return at


def _insert_before_scan(data, k, segment):
  at = _scan_at(data, k)
  return data[:at] + segment + data[at:]


def _script_file(script, ri=0, grey=False):
  a = photo(24, 32, 3)
  return PO.reencode(encode(a[..., 0].copy() if grey else a, quality=90), script, ri)


def test_declines_each_unsupported_progression_with_its_reason():
  full_y = [((0, 1, 2), 0, 0, 0, 0), (CB, 1, 63, 0, 0), (CR, 1, 63, 0, 0)]
  cases = {
      'AC scan of component 0 before its DC scan': [(Y, 1, 63, 0, 0)] + full_y,
      'bogus progression: Ah 2': [((0, 1, 2), 0, 0, 0, 1), (Y, 1, 63, 0, 1), (Y, 1, 63, 2, 1)],
      'a second first scan': full_y + [(Y, 1, 63, 0, 0), (Y, 1, 63, 0, 0)],
      'incomplete progression': [((0, 1, 2), 0, 0, 0, 1), (Y, 1, 63, 0, 0), (CB, 1, 63, 0, 0), (CR, 1, 63, 0, 0)],
      'AC scan of 2 components': [((0, 1, 2), 0, 0, 0, 0), ((1, 2), 1, 63, 0, 0), (Y, 1, 63, 0, 0)],
      'DC scan with Se 5': [((0, 1, 2), 0, 5, 0, 0)],
      'band 9..3': full_y + [(Y, 9, 3, 0, 0)],
      'Ah 3, Al 1': [((0, 1, 2), 0, 0, 0, 3), ((0, 1, 2), 0, 0, 3, 1)],
      'Al 14': [((0, 1, 2), 0, 0, 0, 14)],
      'not in frame order': [((2, 1, 0), 0, 0, 0, 0)],
  }
  for reason, script in cases.items():
    f = _script_file(script)
    with pytest.raises(J.Unsupported) as e:
      P.parse(f)
    assert reason.split(':')[0].split(' of component')[0] in str(e.value) or reason in str(e.value), (reason, e.value)
  good = _script_file(PO.STANDARD_SCRIPT)
  assert P.probe(good) is not None
  dqt = J._segment(0xDB, bytes([0]) + bytes(range(1, 65)))
  with pytest.raises(J.Unsupported, match='DQT after the first scan'):
    P.parse(_insert_before_scan(good, 3, dqt))
  with pytest.raises(J.Unsupported, match='DNL'):
    P.parse(_insert_before_scan(good, 3, J._segment(0xDC, b'\x00\x18')))
  with pytest.raises(J.Unsupported, match='not ended by a marker'):
    P.parse(good[:-2])
  with pytest.raises(J.Unsupported, match='not ended by EOI'):
    P.parse(good[:-2] + J._segment(0xFE, b'late') + b'\xff\xd9')
  with pytest.raises(J.Unsupported, match='two frame headers'):
    sof = good.index(b'\xff\xc2')
    n = int.from_bytes(good[sof + 2:sof + 4], 'big')
    P.parse(_insert_before_scan(good, 0, good[sof:sof + 2 + n]))
  # markers between scans: DHT (a scan uses the tables it starts with), DRI, COM and APPn are accepted
  dht = J._segment(0xC4, bytes([0x11]) + PO.AC_TABLE[0] + PO.AC_TABLE[1])
  for seg in (dht, J._segment(0xDD, b'\x00\x02'), J._segment(0xFE, b'note'), J._segment(0xE5, b'app5')):
    assert P.probe(_insert_before_scan(good, 4, seg)) is not None
  # an undefined table is declined only when a scan uses it, an invalid one too
  bad_dht = J._segment(0xC4, bytes([0x13]) + bytes([0, 2] + [0] * 14) + b'\x00\x01')    # two 2-bit codes: fine
  assert P.probe(_insert_before_scan(good, 2, bad_dht)) is not None
  all_ones = J._segment(0xC4, bytes([0x11]) + bytes([2] + [0] * 15) + b'\x00\x01')     # 1-bit codes 0 and 1
  with pytest.raises(J.Unsupported, match='invalid Huffman table'):
    P.parse(_insert_before_scan(good, 2, all_ones).replace(b'\xff\xda\x00\x08\x01\x03\x00', b'\xff\xda\x00\x08\x01\x03\x01'))


def test_descriptors_levels_grids_and_segments():
  a = photo(41, 67, 2)
  files = [encode(a, subsampling=2, progressive=True, restart_marker_blocks=2),
           encode(a[..., 0].copy(), progressive=True),
           _script_file(SCRIPTS[3][1], SCRIPTS[3][2])]
  infos = [P.parse(f) for f in files]
  b = P.pack(files, infos, [5, 100000, 200000])
  assert b.scans.shape == (sum(len(i.scans) for i in infos), P.SCAN_FIELDS)
  assert b.segs.shape[1] == J.SEG_FIELDS and b.levels[0] == 0 and b.levels[-1] == len(b.segs)
  assert len(b.levels) - 1 == max(i.levels for i in infos)
  assert b.blocks == int((b.comps[:, 1] * b.comps[:, 2]).sum()) and b.plane_bytes == b.blocks * 64
  lev = b.segs[:, 2]
  for l in range(len(b.levels) - 1):                        # segment rows sorted by level
    assert (b.scans[lev[b.levels[l]:b.levels[l + 1]], 14] == l).all()
  for info in infos:                                        # no two scans of a level share a coefficient
    for l in range(info.levels):
      seen = set()
      for s in info.scans:
        if s.level == l:
          mine = {(c, k) for c in s.comps for k in range(s.ss, s.se + 1)}
          assert not seen & mine
          seen |= mine
  # PIL 4:2:0 41x67: the interleaved DC scan walks 5 x 3 MCUs, a chroma scan 5 x 3 blocks, a luma scan 9 x 6
  grids = {(s.comps, s.ss): s.grid for s in infos[0].scans}
  assert grids[((0, 1, 2), 0)] == (5, 3) and grids[((1,), 1)] == (5, 3) and grids[((0,), 1)] == (9, 6)
  assert infos[0].block_dims()[0] == (10, 6)                # the padded layout holds a dummy column of blocks
  for s in b.segs:                                          # every segment is followed by its marker in the packed data
    assert b.data[s[1]] == 0xFF and b.data[s[1] + 1] == s[5]
  # the scans' comp rows point into the image's own rows
  for row in b.scans:
    img = row[0]
    first, n = b.images[img, 0], b.images[img, 1]
    assert all(first <= c < first + n for c in row[6:6 + row[5]])


def test_restatement_equals_pil_bit_for_bit():
  n = 0
  for name, f in pil_corpus() + [('ew', open(EW, 'rb').read())]:
    r = PO.decode(f)
    assert r['status'] == 0, (name, r['status'])
    assert np.array_equal(r['rgb'], pil_rgb(f)), name
    n += 1
  assert n > 150, n


def test_reencoded_scripts_hold_to_pil_and_the_restatement():
  """Each re-encoded file decodes in PIL to the pixels of the baseline file it came from (checking the re-encoder and
  that libjpeg smooths nothing once a progression is complete), and the restatement decodes it to the same."""
  corpus = reencoded_corpus(with_base=True)
  for name, f, base in corpus:
    info = P.parse(f)
    assert np.array_equal(pil_rgb(f), pil_rgb(base)), name
    r = PO.decode(f, info)
    assert r['status'] == 0 and np.array_equal(r['rgb'], pil_rgb(f)), name
    bi = J.parse(base)
    coef, _ = JO.coefficients(base, bi)
    for k in range(len(coef)):                      # the dummy blocks of the MCU padding only a baseline file codes
      gw, gh = info.component_blocks(k)
      assert np.array_equal(r['coef'][k][:gh, :gw], coef[k][:gh, :gw]), (name, k)
  levels = {name: P.parse(f).levels for name, f, _ in corpus}
  assert levels['standard_ss2'] == 3 and levels['bands_ss0'] == 1 and levels['cbcr_dc_deep_ss1'] > 3


def corrupt_files():
  """(name, bytes) of progressive streams the parser accepts but whose data is damaged."""
  d = encode(photo(64, 96, 21), quality=90, subsampling=2, progressive=True, restart_marker_blocks=2)
  info = P.parse(d)
  sc = info.scans
  out = []
  swapped = bytearray(d)
  swapped[sc[1].segments[0][1] + 1] = 0xD3                                 # RST out of sequence
  out.append(('rst_order', bytes(swapped)))
  fill = bytearray(d)
  fill[sc[2].segments[1][1] - 1] = 0xFF                                    # FF right before an RST marker
  out.append(('fill', bytes(fill)))
  ones = bytearray(d)
  a, e = sc[4].segments[0]
  ones[a:a + 8] = b'\xff\x00' * 4                                          # 32 one bits: no code is all ones
  out.append(('bad_code', bytes(ones)))
  short = bytearray(d)                                                     # a refinement segment cut short
  a, e = sc[9].segments[0]
  out.append(('short', bytes(short[:a + 3]) + bytes(short[e:])))
  # values out of range: a DC first scan at Al 13 of large differences
  big = PO.reencode(encode(photo(16, 16, 5), quality=100), [((0, 1, 2), 0, 0, 0, 0), (Y, 1, 63, 0, 0),
                                                            (CB, 1, 63, 0, 0), (CR, 1, 63, 0, 0)])
  out.append(('value_range', _dc_shift(big)))
  for name, f in out:
    assert P.probe(f) is not None, name
  return out


def _dc_shift(f):
  """The file with its first scan's Al raised to 13 and a refinement of DC bits 12..0 the parser accepts: the DC values
  shifted left by 13 leave int16."""
  at = _scan_at(f, 0)
  g = bytearray(f)
  g[at + 2 + 2 + 1 + 6 + 2] = 0x0D                                          # Ah 0, Al 13
  refine = b''.join(J._segment(0xDA, bytes([3, 1, 0, 2, 0, 3, 0, 0, 0, (k + 1) << 4 | k])) + b'\x00'
                    for k in range(12, -1, -1))
  eoi = len(g) - 2
  return bytes(g[:eoi]) + refine + b'\xff\xd9'


# the status bit each damaged stream must raise (the decoders stop at the first error, the device reading ahead of the
# restatement, so later bits may differ)
CORRUPT_STATUS = {'rst_order': J.STATUS_RESTART, 'fill': J.STATUS_MARKER, 'bad_code': J.STATUS_BAD_CODE,
                  'short': J.STATUS_TRUNCATED | J.STATUS_RESTART, 'value_range': P.STATUS_VALUE_RANGE}


def test_restatement_flags_corrupt_streams():
  for name, f in corrupt_files():
    st = PO.decode(f)['status']
    assert st & CORRUPT_STATUS[name], (name, st)


@pytest.fixture(scope='module')
def report(tmp_path_factory):
  nvcc = _nvcc()
  if not nvcc:
    pytest.skip('nvcc not found')
  out = tmp_path_factory.mktemp('ptxas_jpegp')
  cmd = [nvcc] + graft.NVCC_FLAGS + ['-Xptxas', '-v', '-c', '-o', str(out / 'twg_jpegp.o'),
                                     os.path.join(graft.CSRC, 'twg_jpegp.cu')]
  r = subprocess.run(cmd, cwd=str(out), capture_output=True, text=True)
  assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
  return r.stdout + r.stderr


def test_progressive_kernel_does_not_spill(report):
  fns = {f: s for f, s in _functions(report).items() if re.match(r'_ZN3twg\d+k_jpegp_', f)}
  assert len(fns) == 1, sorted(fns)
  assert all(s == (0, 0) for s in fns.values()), fns


def test_progressive_entries_reject_bad_arguments_without_gpu(built_lib):
  L = built_lib
  assert L.try_call('twgjpegp_reset', None, 1, 16, 1, None) == -1
  assert 'null' in L.last_error()
  assert L.try_call('twgjpegp_reset', 16, 0, 16, 1, None) == -1
  assert L.try_call('twgjpegp_reset', 18, 1, 16, 1, None) == -1
  assert 'aligned' in L.last_error()
  assert L.try_call('twgjpegp_entropy', 16, 16, 0, 16, 16, 16, 16, 16, None) == -1
  assert L.try_call('twgjpegp_entropy', None, 16, 1, 16, 16, 16, 16, 16, None) == -1


def test_progressive_header_symbols_are_exported_and_owned(built_lib):
  from tests.test_gpu_jpeg_progressive import OWNED_ENTRIES
  from twingan_b200 import _lib
  protos = _lib.parse_header(_lib.JPEGP_HEADER, _lib.JPEGP_PREFIX)
  hdr = open(_lib.JPEGP_HEADER).read()
  assert set(re.findall(r'\b(twgjpegp_\w+)\s*\(', hdr)) == set(protos) and protos
  assert not re.findall(r'\bint\s+(twg_\w+|twgjpeg_\w+)\s*\(', hdr)
  for name in protos:
    assert hasattr(built_lib.cdll, name), name
  launching = {n for n, (_, args) in protos.items() if 'twg_stream_t' in args}
  assert launching == OWNED_ENTRIES, launching ^ OWNED_ENTRIES
  assert P.STATUS_REFINE_SIZE == 64 and P.STATUS_BAND == 128 and P.STATUS_VALUE_RANGE == 256
  for name, v in (('REFINE_SIZE', 64), ('BAND', 128), ('VALUE_RANGE', 256)):
    assert re.search(r'#define TWG_JPEGP_%s %d\b' % (name, v), hdr), name


def test_every_progressive_library_call_matches_the_header_arity():
  import ast
  from twingan_b200 import _lib
  protos = _lib.parse_header(_lib.JPEGP_HEADER, _lib.JPEGP_PREFIX)
  pkg = os.path.dirname(graft.CSRC)
  seen = 0
  for fn in sorted(os.listdir(pkg)):
    if not fn.endswith('.py'):
      continue
    for node in ast.walk(ast.parse(open(os.path.join(pkg, fn)).read())):
      if isinstance(node, ast.Call):
        named = [i for i, a in enumerate(node.args) if isinstance(a, ast.Constant) and str(a.value).startswith('twgjpegp_')]
        if named:
          name, args = node.args[named[0]].value, node.args[named[0] + 1:]
          assert name in protos and len(args) == len(protos[name][1]), (fn, node.lineno, name)
          seen += 1
  assert seen == len(protos), seen
