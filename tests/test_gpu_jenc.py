"""Device JPEG encoding (csrc/twg_jenc.cu through ops.jpeg_encode) against PIL byte for byte, stage by stage against the
integer restatement tests/jenc_oracle.py, and through `translate_files`: mixed .png / .jpg / .jpeg outputs are the files
PIL writes for `translate_arrays`' images, and a device-encoded file decodes on the device as PIL decodes it."""
import os

import numpy as np
import pytest
import torch
from PIL import Image

from tests import jenc_oracle as E
from tests.test_cpu_jenc import HWS, inputs, pil_jpeg

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
# the launching entries of include/twgjenc.h this suite holds to PIL and to the restatement (audited in test_cpu_jenc)
OWNED_ENTRIES = {'twgjenc_dct', 'twgjenc_bits', 'twgjenc_pack'}


def _device_files(arrs):
  """PIL-format files of the uint8 [h, w, 3] arrays (one size), encoded in one batch on the device."""
  from twingan_b200 import jpeg as J, ops
  x = torch.from_numpy(np.stack(arrs)).to(DEV)
  scans, offsets = ops.jpeg_encode(x)
  buf, off = scans.cpu().numpy(), offsets.cpu().tolist()
  head = J.encoder_header(*arrs[0].shape[:2])
  return [head + buf[off[i]:off[i + 1]].tobytes() + J.EOI for i in range(len(arrs))]


def _batch(hw, n, seed=0):
  pool = [a for s in range(-(-n // 7)) for a in inputs(hw, hw, seed + s).values()]
  return pool[:n]


@pytest.mark.parametrize('n', [1, 7, 64])
@pytest.mark.parametrize('hw', HWS)
def test_device_files_equal_pil(built_lib, hw, n):
  arrs = _batch(hw, n)
  got = _device_files(arrs)
  bad = [i for i, (g, a) in enumerate(zip(got, arrs)) if g != pil_jpeg(a)]
  assert not bad, bad


def test_stages_equal_the_restatement(built_lib):
  """Coefficients, per-block code lengths and the final scan of the device against the restatement's."""
  from twingan_b200 import jpeg as J
  from twingan_b200._lib import lib
  st = lambda: torch.cuda.current_stream().cuda_stream
  L = lib()
  qt = torch.from_numpy(J.encoder_qt()).to(DEV)
  for hw in (4, 8, 24, 64):
    arrs = list(inputs(hw, hw, 3).values())
    n = len(arrs)
    x = torch.from_numpy(np.stack(arrs)).to(DEV)
    blocks = 6 * (-(-hw // 16)) ** 2
    coefs = torch.empty(n * blocks * 64, dtype=torch.int16, device=DEV)
    bitpos = torch.empty(n * (blocks + 1), dtype=torch.int32, device=DEV)
    work = torch.empty(L.cdll.twgjenc_workspace_bytes(n, hw, hw), dtype=torch.uint8, device=DEV)
    out = torch.empty(L.cdll.twgjenc_scan_capacity(n, hw, hw), dtype=torch.uint8, device=DEV)
    offsets = torch.empty(n + 1, dtype=torch.int64, device=DEV)
    L.call('twgjenc_dct', x.data_ptr(), n, hw, hw, qt.data_ptr(), coefs.data_ptr(), st())
    L.call('twgjenc_bits', coefs.data_ptr(), n, hw, hw, bitpos.data_ptr(), st())
    L.call('twgjenc_pack', coefs.data_ptr(), bitpos.data_ptr(), n, hw, hw, work.data_ptr(), out.data_ptr(),
           offsets.data_ptr(), st())
    c = coefs.cpu().numpy().reshape(n, blocks // 6, 6, 64)
    pos = bitpos.cpu().numpy().reshape(n, blocks + 1)
    buf, off = out.cpu().numpy(), offsets.cpu().tolist()
    for i, a in enumerate(arrs):
      ref = E.encode(a)
      assert np.array_equal(c[i], ref['coef']), (hw, i)
      assert pos[i, 0] == 0 and np.array_equal(np.diff(pos[i]), ref['lengths']), (hw, i)
      assert buf[off[i]:off[i + 1]].tobytes() == ref['scan'], (hw, i)


def test_two_runs_give_identical_bytes(built_lib):
  arrs = _batch(256, 64, 5)
  assert _device_files(arrs) == _device_files(arrs)


def test_device_file_round_trip(built_lib):
  """A device-encoded file is one the device decoder takes, and decoding it there equals PIL's decode."""
  from twingan_b200 import jpeg as J
  from tests.test_gpu_jpeg import _device_decode
  from tests.test_cpu_jpeg import pil_rgb
  for hw in (8, 64, 256):
    files = _device_files(list(inputs(hw, hw, 9).values()))
    assert all(J.probe(f) is not None for f in files)
    got, st = _device_decode(files)
    assert not st.any()
    for g, f in zip(got, files):
      assert np.array_equal(g, pil_rgb(f)), hw


# ---- through translate_files ------------------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def model():
  from twingan_b200 import ops, twingan
  ops.set_precision(1)
  return twingan.GanModel(twingan.Flags(train_image_size=32, pggan_max_num_channels=32), device=DEV, seed=7)


def _files(d):
  return {fn: open(os.path.join(d, fn), 'rb').read() for fn in sorted(os.listdir(d))}


@pytest.mark.parametrize('direction', ['t', 's'])
@pytest.mark.parametrize('use_graph', [True, False])
def test_translate_files_of_mixed_outputs_equal_pil(built_lib, model, tmp_path, direction, use_graph):
  from tests.test_cpu_jpeg import encode, photo
  from twingan_b200 import translate
  src = tmp_path / 'in'
  src.mkdir()
  for i in range(9):
    (src / ('%d.jpg' % i)).write_bytes(encode(photo(40 + 7 * i, 50 - 3 * i, i)))
  ins, _ = translate.list_images(str(src), str(tmp_path))
  exts = ['.png', '.jpg', '.JPEG', '.jpg', '.jpg', '.png', '.jpeg', '.jpg', '.jpg']
  ref = translate.translate_arrays(model, [translate.decode(p) for p in ins], direction, use_graph=use_graph)
  want = tmp_path / 'want'
  want.mkdir()
  for k, (a, e) in enumerate(zip(ref, exts)):
    translate.save(a, str(want / ('%d%s' % (k, e))))
  for bs in (1, 7, 64):
    d = tmp_path / ('got%d' % bs)
    outs = [str(d / ('%d%s' % (k, e))) for k, e in enumerate(exts)]
    assert translate.translate_files(model, ins, outs, direction, batch_size=bs, num_decode_threads=2,
                                     use_graph=use_graph) == 9
    assert _files(str(d)) == _files(str(want)), bs
  all_jpeg = tmp_path / 'all_jpeg'
  outs = [str(all_jpeg / ('%d.jpg' % k)) for k in range(9)]
  translate.translate_files(model, ins, outs, direction, batch_size=4, use_graph=use_graph)
  for k, o in enumerate(outs):
    assert open(o, 'rb').read() == pil_jpeg(ref[k]), k
