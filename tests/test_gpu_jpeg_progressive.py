"""Device progressive JPEG decoding (csrc/twg_jpegp.cu, then twg_jpeg.cu's IDCT and colour stages, through
ops.jpeg_progressive_decode) against PIL bit for bit, level by level against the restatement tests/jpegp_oracle.py, on
several streams at once, and through `translate_files`: directories mixing baseline, progressive, PNG and declined files
give the same output files as decoding everything with PIL, and corrupt streams come back flagged and end as PIL ends
them."""
import os

import numpy as np
import pytest
import torch
from PIL import Image

from tests import jpegp_oracle as PO
from tests.test_cpu_jpeg import encode, photo, pil_rgb
from tests.test_cpu_jpeg_progressive import CORRUPT_STATUS, EW, corrupt_files, pil_corpus, reencoded_corpus

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
# the launching entries of include/twgjpegp.h this suite holds to PIL and to the restatement (audited in
# test_cpu_jpeg_progressive)
OWNED_ENTRIES = {'twgjpegp_reset', 'twgjpegp_entropy'}


def _tensors(b):
  return [torch.from_numpy(a).to(DEV) for a in (b.data, b.segs, b.scans, b.comps, b.images, b.qt, b.huff)]


def _device_decode(files, lead=7):
  """Decode `files` in one batch into a payload (images at odd offsets, `lead` bytes first); returns (images, status)."""
  from twingan_b200 import jpeg_progressive as P, ops
  infos = [P.parse(f) for f in files]
  offs, at = [], lead
  for i in infos:
    offs.append(at)
    at += i.H * i.W * 3 + 1
  b = P.pack(files, infos, offs)
  payload = torch.full((at,), 0xAB, dtype=torch.uint8, device=DEV)
  status = ops.jpeg_progressive_decode(payload, *_tensors(b), b.blocks, b.plane_bytes, b.pixels, b.levels)
  status = status.cpu().numpy()
  host = payload.cpu().numpy()
  assert host[:lead].tolist() == [0xAB] * lead                      # nothing outside the regions is written
  assert all(host[o + i.H * i.W * 3] == 0xAB for o, i in zip(offs, infos))
  return [host[o:o + i.H * i.W * 3].reshape(i.H, i.W, 3) for o, i in zip(offs, infos)], status


def _all_files():
  return [f for _, f in pil_corpus()] + [f for _, f in reencoded_corpus()] + [open(EW, 'rb').read()]


def test_device_decode_equals_pil_one_by_one_and_mixed(built_lib):
  files = _all_files()
  for f in files[::5] + [files[-1]]:
    got, st = _device_decode([f])
    assert st.tolist() == [0] and np.array_equal(got[0], pil_rgb(f))
  got, st = _device_decode(files)
  assert not st.any(), np.flatnonzero(st)
  bad = [i for i, (g, f) in enumerate(zip(got, files)) if not np.array_equal(g, pil_rgb(f))]
  assert not bad, bad


@pytest.mark.parametrize('extra', [{}, {'restart_marker_rows': 4}])
def test_device_decode_of_a_4000x3000_photo(built_lib, extra):
  f = encode(photo(3000, 4000, 11), quality=92, subsampling=2, progressive=True, **extra)
  small = encode(photo(17, 33, 12), quality=60, subsampling=1, progressive=True)
  got, st = _device_decode([small, f])
  assert not st.any()
  assert np.array_equal(got[1], pil_rgb(f)) and np.array_equal(got[0], pil_rgb(small))


def test_levels_and_planes_equal_the_restatement(built_lib):
  """Coefficients after each level and sample planes of the device against the restatement's, for one PIL file of each
  sampling and grey, and a re-encoded script with restarts."""
  from twingan_b200 import jpeg_progressive as P
  from twingan_b200._lib import lib
  st = lambda: torch.cuda.current_stream().cuda_stream
  files = [encode(photo(41, 67, ss), quality=83, subsampling=ss, progressive=True, restart_marker_blocks=2)
           for ss in (0, 1, 2)]
  files.append(encode(photo(30, 45, 3)[..., 0].copy(), quality=70, progressive=True))
  files.append(PO.reencode(encode(photo(41, 67, 4), quality=88, subsampling=2), PO.STANDARD_SCRIPT, 1))
  for n, f in enumerate(files):
    info = P.parse(f)
    b = P.pack([f], [info], [0])
    data, segs, scans, comps, images, qt, huff = _tensors(b)
    coefs = torch.empty(b.blocks * 64, dtype=torch.int16, device=DEV)
    planes = torch.empty(b.plane_bytes, dtype=torch.uint8, device=DEV)
    status = torch.empty(1, dtype=torch.int32, device=DEV)
    ref = PO.decode(f)
    lib().call('twgjpegp_reset', coefs.data_ptr(), b.blocks, status.data_ptr(), 1, st())
    for level, (a, e) in enumerate(zip(b.levels, b.levels[1:])):
      lib().call('twgjpegp_entropy', data.data_ptr(), segs[a:].data_ptr(), e - a, scans.data_ptr(), comps.data_ptr(),
                 huff.data_ptr(), coefs.data_ptr(), status.data_ptr(), st())
      c = coefs.cpu().numpy()
      for k, row in enumerate(b.comps):
        want = ref['levels'][level][k]
        assert np.array_equal(c[row[0] * 64:(row[0] + want.size // 64) * 64].reshape(want.shape), want), (n, level, k)
    lib().call('twgjpeg_idct', coefs.data_ptr(), comps.data_ptr(), len(b.comps), b.blocks, qt.data_ptr(),
               planes.data_ptr(), status.data_ptr(), st())
    assert status.item() == 0 and ref['status'] == 0
    p = planes.cpu().numpy()
    for k, row in enumerate(b.comps):
      want = ref['planes'][k]
      assert np.array_equal(p[row[3]:row[3] + want.size].reshape(want.shape), want), (n, k)


def test_decoding_on_several_streams_at_once(built_lib):
  from twingan_b200 import jpeg_progressive as P, ops
  files = _all_files()
  groups = [files[k::4] for k in range(4)]
  streams = [torch.cuda.Stream(device=DEV) for _ in groups]
  jobs = []
  for g, s in zip(groups, streams):
    infos = [P.parse(f) for f in g]
    offs = np.cumsum([0] + [i.H * i.W * 3 for i in infos])
    b = P.pack(g, infos, offs[:-1].tolist())
    with torch.cuda.stream(s):
      payload = torch.empty(int(offs[-1]), dtype=torch.uint8, device=DEV)
      t = [x.to(DEV, non_blocking=True) for x in (torch.from_numpy(a) for a in (b.data, b.segs, b.scans, b.comps,
                                                                                 b.images, b.qt, b.huff))]
      status = ops.jpeg_progressive_decode(payload, *t, b.blocks, b.plane_bytes, b.pixels, b.levels)
    jobs.append((g, infos, offs, payload, status))
  torch.cuda.synchronize()
  for g, infos, offs, payload, status in jobs:
    assert not status.cpu().any()
    host = payload.cpu().numpy()
    for f, i, o in zip(g, infos, offs):
      assert np.array_equal(host[o:o + i.H * i.W * 3].reshape(i.H, i.W, 3), pil_rgb(f))


def test_corrupt_streams_are_flagged(built_lib):
  files = corrupt_files()
  _, st = _device_decode([f for _, f in files])
  assert all(st), dict(zip([n for n, _ in files], st.tolist()))
  for (name, f), s in zip(files, st):
    assert s & CORRUPT_STATUS[name], (name, s)


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
  from twingan_b200 import jpeg as J, jpeg_progressive as P, translate
  src = tmp_path / 'in'
  src.mkdir()
  items = {'a.jpg': encode(photo(368, 371, 1), quality=90), 'b.jpg': encode(photo(120, 80, 4), progressive=True),
           'c.jpg': encode(photo(77, 93, 3), subsampling=0, progressive=True, restart_marker_rows=1),
           'd.jpg': open(EW, 'rb').read(),
           'e.jpeg': encode(photo(50, 61, 5)[..., 0].copy(), progressive=True),
           'g.jpg': PO.reencode(encode(photo(64, 80, 6), quality=95), PO.STANDARD_SCRIPT, 1),
           # declined: an incomplete progression, which libjpeg decodes by smoothing blocks
           'h.jpg': PO.reencode(encode(photo(40, 48, 8)), [((0, 1, 2), 0, 0, 0, 1), ((0,), 1, 63, 0, 0),
                                                             ((1,), 1, 63, 0, 0), ((2,), 1, 63, 0, 0)])}
  for name, data in items.items():
    (src / name).write_bytes(data)
  Image.fromarray(photo(90, 64, 7)).save(str(src / 'f.png'))
  progressive = [k for k in items if P.probe(items[k]) is not None]
  assert sorted(progressive) == ['b.jpg', 'c.jpg', 'd.jpg', 'e.jpeg', 'g.jpg'] and J.probe(items['a.jpg'])
  assert P.probe(items['h.jpg']) is None and J.probe(items['h.jpg']) is None
  # the progressive files go to the device, and it decodes them exactly
  ins, _ = translate.list_images(str(src), str(tmp_path / 'x'))
  tensors, (count, jpegs, pngs, jpegps) = translate._produce_batch(ins, len(ins), translate.ThreadPoolExecutor(2))
  assert sorted(os.path.basename(p) for p in jpegps.paths) == progressive
  dev = [t.to(DEV) for t in tensors]
  payload, _, handle = translate._DeviceDecoder(DEV, 1).start(dev[0], dev[1], dev[2:], jpegs, pngs, jpegps)
  host, done, _ = handle
  done.synchronize()
  assert not host.any(), host
  for bs in (1, 3, 64):
    for ext in ('.png', '.jpg'):
      name = 'dev%d%s' % (bs, ext)
      ins, outs = translate.list_images(str(src), str(tmp_path / name))
      outs = [os.path.splitext(o)[0] + ext for o in outs]
      assert translate.translate_files(model, ins, outs, batch_size=bs, num_decode_threads=2) == len(ins)
      want = tmp_path / ('host%d%s' % (bs, ext))
      want.mkdir()
      _host_path(model, ins, [str(want / os.path.basename(o)) for o in outs], bs)
      assert _files(str(tmp_path / name)) == _files(str(want)), (bs, ext)


def test_translate_files_with_corrupt_progressive_jpegs_ends_as_pil_does(built_lib, model, tmp_path):
  from twingan_b200 import translate
  good = tmp_path / 'good.jpg'
  good.write_bytes(encode(photo(40, 40, 30), progressive=True))
  for name, data in corrupt_files():
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
