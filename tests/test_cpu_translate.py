"""CPU tests of image translation (twingan_b200/translate.py, the front and back end in ops and csrc/twg_image.cu,
oracle/translate_oracle.py): the fp64 restatement against hand-computed cases and the training path's resize, the
quantisation rule, the host packer, path walking, tensor-name pairing, model-path resolution, the ABI's argument checks
and ptxas's report."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import __graft_entry__ as graft
from oracle import translate_oracle as O
from twingan_b200 import ops, pggan_runner, translate


def test_restatement_is_the_identity_at_equal_size():
  rng = np.random.default_rng(0)
  for h in (1, 5, 32):
    img = rng.integers(0, 256, (h, h, 3), dtype=np.uint8)
    got = O.resize(img, h)
    assert np.array_equal(got, img.astype(np.float64) * O.INV255)
    # rounded to fp32 it is convert_image_dtype's product: a multiply by fl32(1/255), not a division
    assert np.array_equal(got.astype(np.float32), img.astype(np.float32) * np.float32(1 / 255))


def test_restatement_matches_hand_computed_cases():
  # 2x2 -> 4x4: scale 0.5, source rows / columns 0, .5, 1, 1.5 -> taps (0,1,0), (0,1,.5), (1,1,0), (1,1,.5)
  img = np.array([[[0, 0, 0], [255, 51, 0]], [[102, 0, 255], [255, 255, 255]]], np.uint8)
  p = img.astype(np.float64) * O.INV255
  out = O.resize(img, 4)
  pos = [(0, 1, 0.0), (0, 1, 0.5), (1, 1, 0.0), (1, 1, 0.5)]
  for y, (y0, y1, ly) in enumerate(pos):
    for x, (x0, x1, lx) in enumerate(pos):
      top = p[y0, x0] + (p[y0, x1] - p[y0, x0]) * lx
      bot = p[y1, x0] + (p[y1, x1] - p[y1, x0]) * lx
      assert np.array_equal(out[y, x], top + (bot - top) * ly), (y, x)
  # 5x3 -> 2x2: rows at 0 and 2.5 (taps 0,1 / 2,3 at .5), columns at 0 and 1.5 (taps 0,1 / 1,2 at .5)
  img = np.arange(45, dtype=np.uint8).reshape(5, 3, 3) * 5
  p = img.astype(np.float64) * O.INV255
  out = O.resize(img, 2)
  assert np.array_equal(out[0, 0], p[0, 0])
  assert np.allclose(out[0, 1], (p[0, 1] + p[0, 2]) / 2, atol=1e-15)
  assert np.allclose(out[1, 0], (p[2, 0] + p[3, 0]) / 2, atol=1e-15)
  assert np.allclose(out[1, 1], (p[2, 1] + p[2, 2] + p[3, 1] + p[3, 2]) / 4, atol=1e-15)


def test_restatement_agrees_with_the_training_resize():
  from twingan_b200 import image_only
  rng = np.random.default_rng(1)
  for (h, w), hw in (((368, 371), 256), ((37, 1000), 32), ((7, 5), 16), ((300, 200), 256)):
    img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    want = image_only.resize_bilinear_tf1(torch.from_numpy(img).double() / 255.0, hw, hw).numpy()
    assert np.abs(O.resize(img, hw) - want).max() < 1e-4, (h, w, hw)


def test_quantisation_is_numpys_clip_and_truncation():
  eps = np.float32(1e-7)
  k = np.arange(256, dtype=np.float32) / np.float32(255)
  x = np.concatenate([np.array([-1.0, -1e-9, -0.0, 0.0, 1.0, 1.0000001, 2.0, 1e30, -1e30, np.inf, -np.inf], np.float32),
                      k, k - eps, k + eps, np.nextafter(k, np.float32(-1)), np.nextafter(k, np.float32(2))]).astype(np.float32)
  want = np.clip(x * np.float32(255), 0, 255).astype(np.uint8)
  assert np.array_equal(O.to_u8(x), want)
  assert O.to_u8(np.float32(254.9999 / 255))[()] == 254          # truncation, not rounding
  assert O.to_u8(np.array([np.nan], np.float32))[0] == 0


def test_pack_images_builds_the_table_and_rejects_bad_images():
  a = np.zeros((2, 3, 3), np.uint8)
  b = np.full((5, 1, 3), 7, np.uint8)
  c = np.arange(12, dtype=np.uint8).reshape(1, 4, 3)
  payload, table = ops.pack_images([a, b, torch.from_numpy(c)])
  assert payload.dtype == torch.uint8 and payload.numel() == 18 + 15 + 12
  assert table.dtype == torch.int64 and table.tolist() == [[0, 2, 3], [18, 5, 1], [33, 1, 4]]
  assert bytes(payload[33:].numpy()) == bytes(c.reshape(-1))
  with pytest.raises(ValueError, match='empty'):
    ops.pack_images([a, np.zeros((0, 4, 3), np.uint8)])
  with pytest.raises(ValueError, match='uint8'):
    ops.pack_images([np.zeros((4, 4, 3), np.float32)])
  with pytest.raises(ValueError, match=r'\[H, W, 3\]'):
    ops.pack_images([np.zeros((4, 4), np.uint8)])
  with pytest.raises(ValueError, match=r'\[H, W, 3\]'):
    ops.pack_images([np.zeros((4, 4, 4), np.uint8)])
  with pytest.raises(ValueError, match='no images'):
    ops.pack_images([])
  # a table whose sizes do not fit the payload
  ops.check_table(table, payload.numel())
  for bad in ([[0, 2, 3], [18, 5, 1], [34, 1, 4]], [[0, 2, 3], [18, 0, 1], [33, 1, 4]], [[-1, 2, 3]]):
    with pytest.raises(ValueError, match='does not fit'):
      ops.check_table(torch.tensor(bad, dtype=torch.int64), payload.numel())
  with pytest.raises(ValueError, match='int64'):
    ops.check_table(table.int(), payload.numel())


def _touch(path, data=b''):
  os.makedirs(os.path.dirname(path), exist_ok=True)
  with open(path, 'wb') as f:
    f.write(data)


def test_path_walking(tmp_path):
  d = str(tmp_path / 'in')
  for rel in ('b.png', 'A.JPG', 'sub/c.Jpeg', 'sub/deeper/a0.png', 'notes.txt', 'sub/x.gif', 'sub/y.png.bak'):
    _touch(os.path.join(d, rel))
  ins, outs = translate.list_images(d, '/out')
  want = sorted(os.path.join(d, r) for r in ('b.png', 'A.JPG', 'sub/c.Jpeg', 'sub/deeper/a0.png'))
  assert ins == want
  assert outs == [os.path.join('/out', os.path.basename(p)) for p in want]
  # single-file mode: the output path is the file
  assert translate.list_images(os.path.join(d, 'b.png'), '/o/x.jpg') == ([os.path.join(d, 'b.png')], ['/o/x.jpg'])
  _touch(os.path.join(d, 'sub', 'b.png'))
  with pytest.raises(ValueError, match='both be written'):
    translate.list_images(d, '/out')
  e = str(tmp_path / 'empty')
  _touch(os.path.join(e, 'readme.txt'))
  with pytest.raises(ValueError, match=re.escape(e)):
    translate.list_images(e, '/out')
  with pytest.raises(FileNotFoundError):
    translate.list_images(str(tmp_path / 'missing'), '/out')


def test_undecodable_file_names_the_path(tmp_path):
  p = str(tmp_path / 'bad.png')
  _touch(p, b'not an image')
  with pytest.raises(ValueError, match=re.escape(p)):
    translate.decode(p)


def test_tensor_name_pairing():
  for v in ('source', 'target', 'rand', 'ph'):
    assert translate.direction_of('sources_ph', 'custom_generated_t_style_%s' % v) == 't'
    assert translate.direction_of('targets_ph:0', 'custom_generated_s_style_%s:0' % v) == 's'
    with pytest.raises(ValueError, match='not computed from'):
      translate.direction_of('sources_ph', 'custom_generated_s_style_%s' % v)
    with pytest.raises(ValueError, match='not computed from'):
      translate.direction_of('targets_ph', 'custom_generated_t_style_%s' % v)
  for i, o in (('images_ph', 'custom_generated_t_style_source'), ('sources_ph', 'generated_t'),
               ('sources_ph', 'custom_generated_t_style_source:1')):
    with pytest.raises(ValueError, match='unknown'):
      translate.direction_of(i, o)
  a = translate._parser().parse_args(['--model_path', 'm', '--input_image_path', 'i', '--output_image_path', 'o'])
  assert translate.direction_of(a.input_tensor_name, a.output_tensor_name) == 't'


def test_cli_rejects_bad_arguments_before_any_work(tmp_path, capsys):
  d = str(tmp_path / 'in')
  _touch(os.path.join(d, 'a.png'))
  _touch(os.path.join(d, 'sub', 'a.png'))
  base = ['--model_path', str(tmp_path / 'missing.pt'), '--input_image_path', d, '--output_image_path', str(tmp_path / 'o')]

  def fails(extra, pattern):
    with pytest.raises(SystemExit) as e:
      translate.main(base + extra)
    assert e.value.code == 2
    err = capsys.readouterr().err
    assert re.search(pattern, err), err

  fails(['--output_tensor_name', 'custom_generated_s_style_source'], 'not computed from')
  fails(['--input_tensor_name', 'foo'], 'unknown input tensor')
  fails(['--batch_size', '0'], 'must be positive')
  fails(['--image_hw', '48'], 'power of two')
  fails([], 'both be written')
  assert not os.path.exists(str(tmp_path / 'o'))


def test_model_path_resolution(tmp_path):
  d = tmp_path / 'train'
  d.mkdir()
  for s in (3, 12, 7):
    (d / ('model.ckpt-%d.pt' % s)).write_bytes(b'x')
  assert pggan_runner.resolve_model_path(str(d)) == ('pt', str(d / 'model.ckpt-12.pt'))
  assert pggan_runner.resolve_model_path(str(d / 'model.ckpt-3.pt')) == ('pt', str(d / 'model.ckpt-3.pt'))
  # a TensorFlow prefix, and a directory with a TensorFlow `checkpoint` state file (relative and absolute paths)
  tf = tmp_path / 'tf'
  tf.mkdir()
  (tf / 'model.ckpt-40.index').write_bytes(b'')
  (tf / 'model.ckpt-40.data-00000-of-00001').write_bytes(b'')
  prefix = str(tf / 'model.ckpt-40')
  assert pggan_runner.resolve_model_path(prefix) == ('tf', prefix)
  (tf / 'checkpoint').write_text('model_checkpoint_path: "model.ckpt-40"\nall_model_checkpoint_paths: "model.ckpt-40"\n')
  assert pggan_runner.resolve_model_path(str(tf)) == ('tf', prefix)
  other = tmp_path / 'elsewhere'
  other.mkdir()
  (other / 'checkpoint').write_text('model_checkpoint_path: "%s"\n' % prefix)
  assert pggan_runner.resolve_model_path(str(other)) == ('tf', prefix)
  (other / 'checkpoint').write_text('model_checkpoint_path: "model.ckpt-99"\n')
  with pytest.raises(FileNotFoundError, match='no .index'):
    pggan_runner.resolve_model_path(str(other))
  # refused and missing forms
  for p in (str(tmp_path / 'frozen.pb'), str(tf / 'model.ckpt-40.meta'), str(tmp_path / 'g.pbtxt')):
    with pytest.raises(ValueError, match='not supported'):
      pggan_runner.resolve_model_path(p)
  with pytest.raises(FileNotFoundError, match='no checkpoint'):
    pggan_runner.resolve_model_path(str(tmp_path / 'missing.pt'))
  (tmp_path / 'nothing').mkdir()
  with pytest.raises(FileNotFoundError, match='no checkpoint in directory'):
    pggan_runner.resolve_model_path(str(tmp_path / 'nothing'))
  assert pggan_runner.step_of(prefix) == 40 and pggan_runner.step_of(str(d / 'model.ckpt-12.pt')) == 12
  assert pggan_runner.step_of('/a/model', 5) == 5


def test_tf_checkpoint_needs_an_image_size(tmp_path):
  from twingan_b200 import twingan
  (tmp_path / 'm.index').write_bytes(b'')
  with pytest.raises(ValueError, match='does not record its image size'):
    pggan_runner.load_for_inference(str(tmp_path / 'm'), twingan.Flags(train_image_size=None))


def test_abi_entries_reject_bad_arguments_without_gpu(built_lib):
  L = built_lib
  assert L.try_call('twg_images_u8_to_batch', None, 16, 16, 1, 32, None) == -1
  assert 'null' in L.last_error()
  assert L.try_call('twg_images_u8_to_batch', 16, 16, 16, 0, 32, None) == -1           # empty batch
  assert L.try_call('twg_images_u8_to_batch', 16, 16, 16, 1, 0, None) == -1            # hw = 0
  assert L.try_call('twg_images_u8_to_batch', 16, 16, 20, 1, 32, None) == -1           # misaligned output
  assert 'aligned' in L.last_error()
  assert L.try_call('twg_batch_to_u8', None, 16, 10, None) == -1
  assert L.try_call('twg_batch_to_u8', 16, 16, 0, None) == -1


def test_image_kernels_do_not_spill(tmp_path):
  nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
  nvcc = nvcc if os.path.exists(nvcc) else shutil.which('nvcc')
  if not nvcc:
    pytest.skip('nvcc not found')
  cmd = [nvcc] + graft.NVCC_FLAGS + ['-Xptxas', '-v', '-c', '-o', str(tmp_path / 'twg_image.o'),
                                     os.path.join(graft.CSRC, 'twg_image.cu')]
  r = subprocess.run(cmd, cwd=str(tmp_path), capture_output=True, text=True)
  assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
  report = r.stdout + r.stderr
  fns = re.findall(r"Compiling entry function '(\w+)'", report)
  spills = re.findall(r'(\d+) bytes spill stores, (\d+) bytes spill loads', report)
  assert len(fns) == len(spills) == 2, (fns, spills)
  assert all(s == ('0', '0') for s in spills), list(zip(fns, spills))
  assert re.search(r'(\d+) bytes stack frame', report) and set(re.findall(r'(\d+) bytes stack frame', report)) == {'0'}
