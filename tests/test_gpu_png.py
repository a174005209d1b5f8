"""Device PNG decoding (csrc/twg_png.cu through ops.png_decode) against PIL and the restatement tests/png_oracle.py stage
by stage, and through `translate_files`: directories mixing every accepted PNG kind, declined PNGs and JPEGs give the
same files as decoding everything with PIL, and corrupt streams come back flagged and end as PIL ends them."""
import io
import os
import zlib

import numpy as np
import pytest
import torch
from PIL import Image

from tests import png_oracle as PO
from tests.test_cpu_png import (FIXTURES, GOLDEN, KINDS, WIDTHS, corrupt_files, kind_file, make_png, photo, pil_rgb,
                                smooth_rows, _streams, ANCILLARY)

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
# the launching entries of include/twgpng.h this suite holds to PIL and to the restatement (audited in test_cpu_png)
OWNED_ENTRIES = {'twgpng_inflate', 'twgpng_unfilter', 'twgpng_rgb'}


def _fixture(fn):
  return open(os.path.join(GOLDEN, fn), 'rb').read()


def _stages(files, lead=5):
  """Run the three entries on `files` in one batch (images at odd payload offsets, `lead` bytes first); returns
  (status, inflated regions, unfiltered regions, images)."""
  from twingan_b200 import png as P
  from twingan_b200._lib import lib
  infos = [P.parse(f) for f in files]
  offs, at = [], lead
  for i in infos:
    offs.append(at)
    at += i.H * i.W * 3 + 1
  b = P.pack(files, infos, offs)
  data, images, pals = (torch.from_numpy(a).to(DEV) for a in (b.data, b.images, b.palettes))
  raw = torch.full((b.raw_bytes + 16,), 0xCD, dtype=torch.uint8, device=DEV)
  payload = torch.full((at,), 0xAB, dtype=torch.uint8, device=DEV)
  status = torch.empty(len(files), dtype=torch.int32, device=DEV)
  st = torch.cuda.current_stream().cuda_stream
  n = len(files)
  lib().call('twgpng_inflate', data.data_ptr(), images.data_ptr(), n, raw.data_ptr(), status.data_ptr(), st)
  inflated = raw.cpu().numpy()
  lib().call('twgpng_unfilter', raw.data_ptr(), images.data_ptr(), n, status.data_ptr(), st)
  unfiltered = raw.cpu().numpy()
  lib().call('twgpng_rgb', raw.data_ptr(), images.data_ptr(), n, pals.data_ptr(), b.pixels, status.data_ptr(),
             payload.data_ptr(), st)
  host = payload.cpu().numpy()
  assert host[:lead].tolist() == [0xAB] * lead                       # nothing outside the regions is written
  assert all(host[o + i.H * i.W * 3] == 0xAB for o, i in zip(offs, infos))
  assert (inflated[b.raw_bytes:] == 0xCD).all()
  regions = [(int(r[2]), int(r[3])) for r in b.images]
  return (status.cpu().numpy(), [inflated[o:o + s].tobytes() for o, s in regions],
          [unfiltered[o:o + s] for o, s in regions],
          [host[o:o + i.H * i.W * 3].reshape(i.H, i.W, 3) for o, i in zip(offs, infos)])


def _corpus():
  out = []
  for ct, d in KINDS:
    for W in WIDTHS:
      out.append(kind_file(ct, d, W, H=4 if W < 1000 else 2, seed=W + d, filters=(0, 1, 2, 3, 4)))
    out.append(kind_file(ct, d, 1, H=1))
  for k, (name, raw, stream) in enumerate(_streams()):             # levels, strategies, a 32 768 distance
    W = 61
    rows = len(raw) // (W * 3 + 1)
    body = raw[:rows * (W * 3 + 1)]
    body = bytes(v if i % (W * 3 + 1) else v % 5 for i, v in enumerate(body))   # valid filter bytes
    c = zlib.compressobj(9 if 'level' not in name else int(name[5:]), zlib.DEFLATED, 15, 9,
                         {'fixed': zlib.Z_FIXED, 'rle': zlib.Z_RLE, 'huffman': zlib.Z_HUFFMAN_ONLY}.get(name, 0))
    out.append(make_png(np.zeros((rows, W * 3), np.uint8), W, 2, 8, stream=c.compress(body) + c.flush(),
                        split=[1, 2, 50]))
  rows = smooth_rows(64, 96, 6, 16, 3)
  out.append(make_png(rows, 96, 6, 16, filters=(4, 3, 1, 2, 0), extra=ANCILLARY[:-1]))
  for a in (photo(368, 371, 1), photo(77, 93, 2)[..., 0].copy()):
    b = io.BytesIO()
    Image.fromarray(a).save(b, 'PNG')
    out.append(b.getvalue())
  out += [_fixture(fn) for fn in FIXTURES]
  return out


def test_stages_equal_zlib_the_restatement_and_pil(built_lib):
  files = _corpus()
  st, inflated, unfiltered, got = _stages(files)
  assert not st.any(), {i: int(s) for i, s in enumerate(st) if s}
  for i, f in enumerate(files):
    ref = PO.decode(f)
    assert inflated[i] == ref['raw'], i
    assert np.array_equal(unfiltered[i].reshape(-1, ref['rows'].shape[1] + 1)[:, 1:], ref['rows']), i
    assert np.array_equal(got[i], ref['rgb']) and np.array_equal(got[i], pil_rgb(f)), i


def test_one_by_one_and_the_fixtures(built_lib):
  files = _corpus()
  for f in files[::5] + [_fixture(fn) for fn in FIXTURES]:
    st, inflated, _, got = _stages([f])
    assert st.tolist() == [0] and np.array_equal(got[0], pil_rgb(f))
    from twingan_b200 import png as P
    assert inflated[0] == zlib.decompress(PO.stream_of(f, P.parse(f)))


def test_ops_png_decode_on_concurrent_streams(built_lib):
  """Batches decoded on several streams at once (as translate's decoder runs them) each get PIL's pixels."""
  from twingan_b200 import ops, png as P
  files = [_fixture(fn) for fn in FIXTURES] + _corpus()[::9]
  infos = [P.parse(f) for f in files]
  offs = np.cumsum([0] + [i.H * i.W * 3 for i in infos])
  b = P.pack(files, infos, offs[:-1].tolist())
  t = [torch.from_numpy(a).to(DEV) for a in (b.data, b.images, b.palettes)]
  torch.cuda.synchronize()
  runs = []
  for _ in range(4):
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
      payload = torch.empty(int(offs[-1]), dtype=torch.uint8, device=DEV)
      runs.append((payload, ops.png_decode(payload, *t, b.raw_bytes, b.pixels)))
  torch.cuda.synchronize()
  for payload, status in runs:
    assert not status.any().item()
    host = payload.cpu().numpy()
    for o, i, f in zip(offs, infos, files):
      assert np.array_equal(host[o:o + i.H * i.W * 3].reshape(i.H, i.W, 3), pil_rgb(f))


def test_corrupt_streams_are_flagged_with_the_restatements_bit(built_lib):
  cases = corrupt_files()
  good = _fixture(FIXTURES[0])
  st, _, _, got = _stages([good] + [f for _, f, _ in cases] + [good])
  want = {name: w for name, _, w in cases}
  assert dict(zip(want, st[1:-1].tolist())) == want
  assert st[0] == 0 and st[-1] == 0 and np.array_equal(got[0], pil_rgb(good)) and np.array_equal(got[-1], got[0])


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


def test_translate_files_of_mixed_directories_equals_the_host_path(built_lib, model, tmp_path):
  from twingan_b200 import jpeg as J, png as P, translate
  src = tmp_path / 'in'
  src.mkdir()
  items = {}
  for ct, d in KINDS:
    items['k%d_%d.png' % (ct, d)] = kind_file(ct, d, 37, H=29, seed=ct * 17 + d, filters=(0, 1, 2, 3, 4))
  a = photo(120, 80, 4)
  # a 1 x 1 image is its own Adam7 pass 1, so the same stream serves an interlaced file (PIL writes none)
  items['interlaced.png'] = make_png(np.array([[0, 9, 99, 199]], np.uint8)[:, 1:], 1, 2, 8, interlace=1)
  for name, kw in (('plain.png', {}), ('optimized.png', {'optimize': True})):
    b = io.BytesIO()
    Image.fromarray(a).save(b, 'PNG', **kw)
    items[name] = b.getvalue()
  b = io.BytesIO()
  Image.fromarray(a).convert('P').save(b, 'PNG', transparency=2)
  items['ptrns.png'] = b.getvalue()
  for name, kw in (('base.jpg', {'quality': 90}), ('prog.jpg', {'progressive': True})):
    b = io.BytesIO()
    Image.fromarray(photo(70, 90, 5)).save(b, 'JPEG', **kw)
    items[name] = b.getvalue()
  for fn in FIXTURES:
    items[fn] = _fixture(fn)
  for name, data in items.items():
    (src / name).write_bytes(data)
  assert P.probe(items['interlaced.png']) is None and P.probe(items['ptrns.png']) is None
  assert P.probe(items['plain.png']) and J.probe(items['base.jpg']) and J.probe(items['prog.jpg']) is None
  n = len(items)
  for bs in (1, 3, 64):
    for ext in ('.png', '.jpg'):
      tag = '%d%s' % (bs, ext.replace('.', '_'))
      ins, outs = translate.list_images(str(src), str(tmp_path / ('dev' + tag)))
      outs = [os.path.splitext(o)[0] + ext for o in outs]
      assert translate.translate_files(model, ins, outs, batch_size=bs, num_decode_threads=3) == n
      want = tmp_path / ('host' + tag)
      want.mkdir()
      _host_path(model, ins, [str(want / os.path.basename(o)) for o in outs], bs)
      assert _files(str(tmp_path / ('dev' + tag))) == _files(str(want)), tag


def test_translate_files_with_corrupt_pngs_ends_as_pil_does(built_lib, model, tmp_path):
  from twingan_b200 import translate
  good = tmp_path / 'good.png'
  good.write_bytes(_fixture(FIXTURES[0]))
  seen_error = seen_pixels = 0
  for name, data, _ in corrupt_files():
    p = tmp_path / (name + '.png')
    p.write_bytes(data)
    try:
      want = translate.decode(str(p))
    except ValueError as e:
      with pytest.raises(ValueError) as got:
        translate.translate_files(model, [str(good), str(p)], [str(tmp_path / 'o1.png'), str(tmp_path / 'o2.png')])
      assert str(got.value) == str(e), name
      seen_error += 1
      continue
    outs = [str(tmp_path / ('%s_%d.png' % (name, k))) for k in range(2)]
    assert translate.translate_files(model, [str(good), str(p)], outs) == 2
    ref = translate.translate_arrays(model, [translate.decode(str(good)), want])
    for o, r in zip(outs, ref):
      with Image.open(o) as im:
        assert np.array_equal(np.asarray(im), r), name
    seen_pixels += 1
  assert seen_error and seen_pixels
  empty = tmp_path / 'empty_idat.png'                              # png.parse declines it: PIL's error, every batch size
  empty.write_bytes(make_png(np.zeros((2, 6), np.uint8), 2, 2, 8, stream=b''))
  with pytest.raises(ValueError) as want:
    translate.decode(str(empty))
  for bs in (1, 2):
    with pytest.raises(ValueError) as got:
      translate.translate_files(model, [str(empty), str(good)], [str(tmp_path / 'e1.png'), str(tmp_path / 'e2.png')],
                                batch_size=bs)
    assert str(got.value) == str(want.value)
