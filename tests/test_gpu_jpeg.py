"""Device JPEG decoding (csrc/twg_jpeg.cu through ops.jpeg_decode) against PIL bit for bit, stage by stage against the
integer restatement oracle/jpeg_oracle.py, and through `translate_files`: mixed batches give the same files as decoding
everything with PIL, and corrupt streams come back flagged and end as PIL ends them."""
import io
import os

import numpy as np
import pytest
import torch
from PIL import Image

from oracle import jpeg_oracle as JO
from tests.test_cpu_jpeg import SIZES, encode, photo, pil_rgb

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
# the launching entries of include/twgjpeg.h this suite holds to PIL and to the restatement (audited in test_cpu_jpeg)
OWNED_ENTRIES = {'twgjpeg_entropy', 'twgjpeg_idct', 'twgjpeg_color'}


def _device_decode(files, lead=7):
  """Decode `files` in one batch into a payload (images at odd offsets, `lead` bytes first); returns (images, status)."""
  from twingan_b200 import jpeg as J, ops
  infos = [J.parse(f) for f in files]
  offs, at = [], lead
  for i in infos:
    offs.append(at)
    at += i.H * i.W * 3 + 1
  b = J.pack(files, infos, offs)
  payload = torch.full((at,), 0xAB, dtype=torch.uint8, device=DEV)
  t = [torch.from_numpy(a).to(DEV) for a in (b.data, b.segs, b.comps, b.images, b.qt, b.huff)]
  status = ops.jpeg_decode(payload, *t, b.blocks, b.plane_bytes, b.pixels).cpu().numpy()
  host = payload.cpu().numpy()
  assert host[:lead].tolist() == [0xAB] * lead                      # nothing outside the regions is written
  assert all(host[o + i.H * i.W * 3] == 0xAB for o, i in zip(offs, infos))
  return [host[o:o + i.H * i.W * 3].reshape(i.H, i.W, 3) for o, i in zip(offs, infos)], status


def _corpus():
  out = []
  for h, w in SIZES:
    for q in (1, 10, 50, 75, 90, 100):
      for ss in (0, 1, 2):
        extra = ({}, {'restart_marker_blocks': 3}, {'restart_marker_rows': 1})[(h + q + ss) % 3]
        out.append(encode(photo(h, w, h + w + q), quality=q, subsampling=ss, **extra))
  for q in range(1, 101, 3):
    out.append(encode(photo(24, 40, q), quality=q, subsampling=q % 3))
  for ss, extra in ((2, {}), (1, {'restart_marker_rows': 2}), (0, {'restart_marker_blocks': 7}), (2, {'optimize': True})):
    out.append(encode(photo(1024, 768, ss), quality=85, subsampling=ss, **extra))
  out.append(encode(photo(255, 257, 5)[..., 0].copy(), quality=70))
  out.append(encode(photo(7, 9, 6)[..., 0].copy(), quality=20, restart_marker_blocks=1))
  return out


def test_device_decode_equals_pil_one_by_one_and_mixed(built_lib):
  files = _corpus()
  for f in files[::7]:
    got, st = _device_decode([f])
    assert st.tolist() == [0] and np.array_equal(got[0], pil_rgb(f))
  got, st = _device_decode(files)
  assert not st.any(), np.flatnonzero(st)
  bad = [i for i, (g, f) in enumerate(zip(got, files)) if not np.array_equal(g, pil_rgb(f))]
  assert not bad, bad


@pytest.mark.parametrize('extra', [{}, {'restart_marker_rows': 4}])
def test_device_decode_of_a_4000x3000_photo(built_lib, extra):
  f = encode(photo(3000, 4000, 11), quality=92, subsampling=2, **extra)
  small = encode(photo(17, 33, 12), quality=60, subsampling=1)
  got, st = _device_decode([small, f])
  assert not st.any()
  assert np.array_equal(got[1], pil_rgb(f)) and np.array_equal(got[0], pil_rgb(small))


def test_stages_equal_the_restatement(built_lib):
  """Coefficients and sample planes of the device against the oracle's, for one file of each sampling."""
  from twingan_b200 import jpeg as J
  from twingan_b200._lib import lib
  st = lambda: torch.cuda.current_stream().cuda_stream
  for ss in (0, 1, 2):
    f = encode(photo(41, 67, ss), quality=83, subsampling=ss, restart_marker_blocks=2)
    info = J.parse(f)
    b = J.pack([f], [info], [0])
    data, segs, comps, images, qt, huff = [torch.from_numpy(a).to(DEV) for a in (b.data, b.segs, b.comps, b.images,
                                                                                 b.qt, b.huff)]
    coefs = torch.empty(b.blocks * 64, dtype=torch.int16, device=DEV)
    planes = torch.empty(b.plane_bytes, dtype=torch.uint8, device=DEV)
    status = torch.empty(1, dtype=torch.int32, device=DEV)
    lib().call('twgjpeg_entropy', data.data_ptr(), segs.data_ptr(), len(b.segs), images.data_ptr(), 1,
               comps.data_ptr(), huff.data_ptr(), coefs.data_ptr(), status.data_ptr(), st())
    lib().call('twgjpeg_idct', coefs.data_ptr(), comps.data_ptr(), len(b.comps), b.blocks, qt.data_ptr(),
               planes.data_ptr(), status.data_ptr(), st())
    ref = JO.decode(f)
    assert status.item() == 0
    c, p = coefs.cpu().numpy(), planes.cpu().numpy()
    for k, row in enumerate(b.comps):
      n = int(row[1] * row[2])
      assert np.array_equal(c[row[0] * 64:(row[0] + n) * 64].reshape(ref['coef'][k].shape), ref['coef'][k]), (ss, k)
      assert np.array_equal(p[row[3]:row[3] + n * 64].reshape(ref['planes'][k].shape), ref['planes'][k]), (ss, k)


def _corrupt_files():
  """(name, bytes) of streams the parser accepts but whose data is damaged."""
  from twingan_b200 import jpeg as J
  d = encode(photo(64, 96, 21), quality=90, subsampling=2, restart_marker_blocks=2)
  info = J.parse(d)
  segs = info.segments
  out = [('cut_eoi', d[:segs[3][0] + 5] + b'\xff\xd9'),                     # truncated mid-segment, EOI appended
         ('cut_at_rst', d[:segs[5][0] - 2] + b'\xff\xd9')]
  swapped = bytearray(d)
  swapped[segs[0][1] + 1] = 0xD3                                            # RST out of sequence
  out.append(('rst_order', bytes(swapped)))
  fill = bytearray(d)
  fill[segs[2][1] - 1] = 0xFF                                               # FF right before an RST marker
  out.append(('fill', bytes(fill)))
  plain = encode(photo(48, 40, 22), quality=75)
  pi = J.parse(plain)
  ones = bytearray(plain)
  s0 = pi.segments[0][0]
  ones[s0 + 10:s0 + 30] = b'\xff\x00' * 10                                   # 80 one bits: no code is all ones
  out.append(('bad_code', bytes(ones)))
  out.append(('short', plain[:s0 + 40] + b'\xff\xd9'))
  for name, f in out:
    assert J.probe(f) is not None, name
  return out


def test_corrupt_streams_are_flagged(built_lib):
  files = _corrupt_files()
  _, st = _device_decode([f for _, f in files])
  assert all(st), dict(zip([n for n, _ in files], st.tolist()))


# ---- through translate_files ------------------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def model():
  from twingan_b200 import ops, twingan
  ops.set_precision(1)
  return twingan.GanModel(twingan.Flags(train_image_size=32, pggan_max_num_channels=32), device=DEV, seed=5)


def _host_path(model, paths, outs, batch_size):
  """The host-decode path: PIL decodes every file, then the same kernels and model."""
  from twingan_b200 import translate
  arrs = translate.translate_arrays(model, [translate.decode(p) for p in paths], batch_size=batch_size)
  for a, o in zip(arrs, outs):
    translate.save(a, o)


def _files(d):
  return {fn: open(os.path.join(d, fn), 'rb').read() for fn in sorted(os.listdir(d))}


def test_translate_files_of_a_mixed_batch_equals_the_host_path(built_lib, model, tmp_path):
  from twingan_b200 import jpeg as J, translate
  src = tmp_path / 'in'
  src.mkdir()
  items = {'a.jpg': encode(photo(368, 371, 1), quality=90), 'b.jpg': encode(photo(300, 200, 2), subsampling=1),
           'c.jpg': encode(photo(77, 93, 3), subsampling=0, restart_marker_rows=1),
           'd.jpg': encode(photo(120, 80, 4), progressive=True),
           'e.jpeg': encode(photo(50, 61, 5)[..., 0].copy()), 'g.jpg': encode(photo(1024, 768, 6), quality=95)}
  for name, data in items.items():
    (src / name).write_bytes(data)
  Image.fromarray(photo(90, 64, 7)).save(str(src / 'f.png'))
  assert J.probe(items['d.jpg']) is None and all(J.probe(items[k]) for k in ('a.jpg', 'b.jpg', 'c.jpg', 'e.jpeg', 'g.jpg'))
  for bs, ext in ((3, '.png'), (8, '.jpg')):
    ins, outs = translate.list_images(str(src), str(tmp_path / ('dev%d' % bs)))
    outs = [os.path.splitext(o)[0] + ext for o in outs]
    assert translate.translate_files(model, ins, outs, batch_size=bs, num_decode_threads=2) == 7
    want = tmp_path / ('host%d' % bs)
    want.mkdir()
    _host_path(model, ins, [str(want / os.path.basename(o)) for o in outs], bs)
    assert _files(str(tmp_path / ('dev%d' % bs))) == _files(str(want)), bs


def test_translate_files_with_corrupt_jpegs_ends_as_pil_does(built_lib, model, tmp_path):
  from twingan_b200 import translate
  good = tmp_path / 'good.jpg'
  good.write_bytes(encode(photo(40, 40, 30)))
  for name, data in _corrupt_files():
    p = tmp_path / (name + '.jpg')
    p.write_bytes(data)
    try:
      want = translate.decode(str(p))
    except ValueError as e:
      with pytest.raises(ValueError) as got:
        translate.translate_files(model, [str(good), str(p)], [str(tmp_path / 'o1.png'), str(tmp_path / 'o2.png')])
      assert str(got.value) == str(e), name
      continue
    outs = [str(tmp_path / ('%s_%d.png' % (name, k))) for k in range(2)]
    assert translate.translate_files(model, [str(good), str(p)], outs) == 2
    ref = translate.translate_arrays(model, [translate.decode(str(good)), want])
    for o, r in zip(outs, ref):
      with Image.open(o) as im:
        assert np.array_equal(np.asarray(im), r), name
