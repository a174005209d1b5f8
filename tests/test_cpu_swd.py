"""CPU tests of the sliced Wasserstein evaluation (twingan_b200/swd.py, oracle/swd_oracle.py, csrc/twg_swd.cu): the fp64
restatement's pyramid and sliced W1 against independent definitions, the descriptor component order, the draws, the
reference's result-file layout, the CLI's argument checks, the ABI's argument checks and ptxas's report."""
import io
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import __graft_entry__ as graft
from oracle import swd_oracle as O
from twingan_b200 import swd


def test_oracle_pyramid_collapses_back_to_the_image():
  rng = np.random.default_rng(0)
  for R in (16, 32, 256):
    x = rng.random((2, R, R, 3))
    levels = int(np.log2(R)) - 3
    p = O.laplacian_pyramid(x, levels)
    assert [a.shape for a in p] == [(2, R >> l, R >> l, 3) for l in range(levels)]
    assert np.abs(O.collapse(p) - x).max() < 1e-14


def test_oracle_pyramid_is_mirror_bordered_pyr_down():
  """pyr_down at a border pixel, written out by hand: mirror reflection d c b | a b c d."""
  rng = np.random.default_rng(1)
  x = rng.random((1, 8, 8, 1))
  g = np.array([1., 4., 6., 4., 1.]) / 16.0
  m = lambda i: abs(i) if i < 8 else 14 - i
  want = sum(g[a] * g[b] * x[0, m(a - 2), m(b - 2), 0] for a in range(5) for b in range(5))
  assert abs(O.pyr_down(x)[0, 0, 0, 0] - want) < 1e-15


def test_sorted_l1_per_direction_is_scipy_wasserstein_distance():
  from scipy.stats import wasserstein_distance
  rng = np.random.default_rng(2)
  a, b = rng.normal(size=(500, 147)), rng.normal(0.3, 1.2, size=(500, 147))
  dirs = rng.normal(size=(3, 147, 4))
  dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
  for r in range(3):
    for j in range(4):
      d = dirs[r:r + 1, :, j:j + 1]
      want = wasserstein_distance(a @ d[0, :, 0], b @ d[0, :, 0])
      assert abs(O.sliced_wasserstein(a, b, d) - want) < 1e-12 * max(1.0, want)


def test_descriptor_components_are_in_nchw_order():
  n, R, s = 2, 16, 7
  img = np.arange(n * R * R * 3, dtype=np.float64).reshape(n, R, R, 3)     # every value names its (n, y, x, c)
  nchw = img.transpose(0, 3, 1, 2)
  centres = np.array([[[3, 3], [12, 5], [7, 12]], [[3, 12], [12, 12], [8, 9]]])
  d = O.descriptors(img, centres, s)
  assert d.shape == (n * 3, 3 * s * s)
  for i in range(n):
    for k in range(3):
      cy, cx = centres[i, k]
      for c in range(3):
        for dy in range(s):
          for dx in range(s):
            assert d[i * 3 + k, c * 49 + dy * 7 + dx] == nchw[i, c, cy - 3 + dy, cx - 3 + dx]


def test_normalise_is_per_channel_population_std():
  rng = np.random.default_rng(3)
  d = rng.normal(2.0, 3.0, size=(100, 147))
  d[:, :49] = 5.0                                 # a constant channel normalises to 0
  z = O.normalise(d).reshape(100, 3, 49)
  assert np.all(z[:, 0] == 0)
  for c in (1, 2):
    assert abs(z[:, c].mean()) < 1e-12 and abs(z[:, c].std() - 1) < 1e-12


def test_draws_are_seeded_in_range_and_unit():
  a = swd.make_draws(64, 6, seed=5)
  b = swd.make_draws(64, 6, seed=5)
  assert swd.resolutions(64) == [64, 32, 16] and swd.resolutions(16) == [16]
  assert len(a['centres']) == 3 and len(a['dirs']) == 3
  for l, r in enumerate((64, 32, 16)):
    c = a['centres'][l]
    assert c.dtype == torch.int32 and tuple(c.shape) == (6, 128, 2)
    assert int(c.min()) == 3 and int(c.max()) == r - 4       # uniform integers in [3, R_l - 4]
    assert torch.equal(c, b['centres'][l])
    d = a['dirs'][l]
    assert d.dtype == torch.float32 and tuple(d.shape) == (4, 147, 128)
    assert float((d.double().square().sum(dim=1) - 1).abs().max()) < 1e-6
    assert torch.equal(d, b['dirs'][l])
  assert not torch.equal(a['dirs'][0], swd.make_draws(64, 6, seed=6)['dirs'][0])
  for bad in (8, 24, 0):
    with pytest.raises(ValueError):
      swd.resolutions(bad)


def test_result_file_matches_the_reference_layout(tmp_path):
  result = {'SWDx1e3_64': 12.5, 'SWDx1e3_32': 7.25, 'SWDx1e3_16': 3.0, 'SWDx1e3_avg': 22.75 / 3,
            'real_SWDx1e3_64': 1.5, 'real_SWDx1e3_32': 2.0, 'real_SWDx1e3_16': 1.0, 'real_SWDx1e3_avg': 1.5}
  path = swd.write_result(str(tmp_path), 1200, 8192, result, is_training=True)
  assert os.path.basename(path) == 'swd_train_step_1200_8192_images.txt'
  # image_generation.py:919-924 on the same numbers
  want = ('swd sliced wasserstein score evaluated on 8192 images.\n'
          'res\treal\tfake\n'
          '64\t1.500000\t12.500000\n'
          '32\t2.000000\t7.250000\n'
          '16\t1.000000\t3.000000\n'
          'Average\t1.500000\t7.583333\n')
  assert open(path, 'rb').read() == want.encode()
  assert os.path.basename(swd.write_result(str(tmp_path), 7, 16, result, False)) == 'swd_eval_step_7_16_images.txt'
  with pytest.raises(ValueError):
    swd.write_result(str(tmp_path), 1, 16, {k: v for k, v in result.items() if not k.startswith('real_')}, False)


def test_constructor_rejects_bad_arguments_before_touching_a_device():
  with pytest.raises(ValueError, match='power of two'):
    swd.SlicedWasserstein(8, 4, 'cuda', 0)
  with pytest.raises(ValueError, match='even'):
    swd.SlicedWasserstein(16, 5, 'cuda', 0)
  with pytest.raises(ValueError, match='CUDA'):
    swd.SlicedWasserstein(16, 5, 'cpu', 0, real_floor=False)


class _Images(object):
  def __init__(self, n):
    self.n = n

  def __len__(self):
    return self.n

  def image(self, i):
    return np.full((16, 16, 3), i, np.uint8)


def test_evaluate_translation_rejects_small_datasets_and_sizes():
  class M:
    class flags:
      train_image_size = 16
    device = torch.device('cuda')
  with pytest.raises(ValueError, match='fewer'):
    swd.evaluate_translation(M, _Images(3), _Images(10), 4)
  with pytest.raises(ValueError, match='fewer'):
    swd.evaluate_translation(M, _Images(10), _Images(3), 4)
  M.flags.train_image_size = 8
  with pytest.raises(ValueError, match='at least 16'):
    swd.evaluate_translation(M, _Images(10), _Images(10), 4)


def _write_dataset(d, n, split='train'):
  from PIL import Image
  from twingan_b200 import image_only
  recs = []
  for i in range(n):
    buf = io.BytesIO()
    Image.fromarray(np.full((20, 20, 3), 10 * i, np.uint8)).save(buf, format='PNG')
    recs.append(image_only.image_only_example('%d.png' % i, buf.getvalue(), 'PNG'))
  image_only.write_records(os.path.join(d, '%s-00000-of-00001' % split), recs)
  return d


def test_cli_rejects_bad_arguments(tmp_path, capsys):
  from twingan_b200 import swd_eval
  src = _write_dataset(str(tmp_path / 'a'), 6)
  tgt = _write_dataset(str(tmp_path / 'b'), 3)
  base = ['--checkpoint_path', str(tmp_path / 'missing.pt'), '--dataset_dir', src, '--unpaired_target_dataset_dir', tgt,
          '--eval_dir', str(tmp_path / 'eval')]

  def fails(extra, pattern):
    with pytest.raises(SystemExit) as e:
      swd_eval.main(base + extra)
    assert e.value.code == 2
    err = capsys.readouterr().err
    assert re.search(pattern, err), err

  fails(['--train_image_size', '8', '--swd_num_images', '2'], 'train_image_size.*at least 16')
  fails(['--train_image_size', '48', '--swd_num_images', '2'], 'power of two')
  fails(['--train_image_size', '16', '--swd_num_images', '3'], 'swd_num_images must be even')
  fails(['--train_image_size', '16', '--swd_num_images', '4'], 'unpaired_target_dataset_dir has 3 train images, fewer')
  with pytest.raises(SystemExit):
    swd_eval.main(['--dataset_dir', src])                         # required flags
  capsys.readouterr()
  # arguments and datasets pass: the missing checkpoint is what stops it
  with pytest.raises(FileNotFoundError, match='no checkpoint'):
    swd_eval.main(base[:5] + [src] + base[6:] + ['--train_image_size', '16', '--swd_num_images', '4'])


def test_abi_entries_reject_bad_arguments_without_gpu(built_lib):
  L = built_lib
  assert L.try_call('twg_swd_pyramid', None, None, 1, 16, 1, None) == -1
  assert L.try_call('twg_swd_pyramid', 8, 8, 1, 24, 1, None) == -1                 # not a power of two
  assert L.try_call('twg_swd_pyramid', 8, 8, 1, 16, 4, None) == -1                 # 16 >> 3 < 4
  assert L.try_call('twg_swd_gather', 8, 8, 8, 1, 16, 128, 6, None) == -1          # even neighbourhood
  assert L.try_call('twg_swd_stats', 8, 8, 0, 7, None) == -1
  assert L.try_call('twg_swd_project', 8, 8, 8, 8, 100, 7, 100, None) == -1        # ndirs not a multiple of 128
  assert L.try_call('twg_swd_sort', 8, 8, 0, 10, None) == -1
  assert L.try_call('twg_swd_sort', 8, 8, 1, 1 << 31, None) == -1
  assert L.try_call('twg_swd_sorted_l1', 8, 8, 8, 0, None) == -1
  assert L.cdll.twg_swd_sort_workspace(0, 10) < 0
  # alternate key buffer + per-tile digit counts (2048-key tiles, 256 digits) + per-segment digit bases, 4 bytes each
  assert L.cdll.twg_swd_sort_workspace(128, (1 << 20) + 3) == 4 * (128 * ((1 << 20) + 3) + 128 * 513 * 256 + 128 * 256)


def test_swd_kernels_do_not_spill(tmp_path):
  nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
  nvcc = nvcc if os.path.exists(nvcc) else shutil.which('nvcc')
  if not nvcc:
    pytest.skip('nvcc not found')
  cmd = [nvcc] + graft.NVCC_FLAGS + ['-Xptxas', '-v', '-c', '-o', str(tmp_path / 'twg_swd.o'),
                                     os.path.join(graft.CSRC, 'twg_swd.cu')]
  r = subprocess.run(cmd, cwd=str(tmp_path), capture_output=True, text=True)
  assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
  report = r.stdout + r.stderr
  fns = re.findall(r"Compiling entry function '(\w+)'", report)
  spills = re.findall(r'(\d+) bytes spill stores, (\d+) bytes spill loads', report)
  assert len(fns) == len(spills) >= 10, (fns, spills)
  assert all(s == ('0', '0') for s in spills), list(zip(fns, spills))
