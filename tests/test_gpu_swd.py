"""The sliced Wasserstein evaluation on the device (csrc/twg_swd.cu through twingan_b200/swd.py) against the fp64
restatement in oracle/swd_oracle.py on the same draws, and its properties: exact zero for identical sets, bit-identical
repeats, growth with the distance between the sets, and training that is left exactly as it would run without it."""
import math

import numpy as np
import pytest
import torch

from oracle import swd_oracle as O

pytestmark = pytest.mark.gpu
ULP1 = 2.0 ** -23          # fp32 ulp at 1.0, the scale of images in [0, 1]


def _lib():
  from twingan_b200._lib import lib
  return lib()


def _st():
  return torch.cuda.current_stream().cuda_stream


def _device_pyramid(x, levels):
  N, R = x.shape[0], x.shape[1]
  pyr = torch.empty(sum(N * (R >> l) ** 2 * 3 for l in range(levels)), device='cuda')
  _lib().call('twg_swd_pyramid', x.data_ptr(), pyr.data_ptr(), N, R, levels, _st())
  out, off = [], 0
  for l in range(levels):
    r = R >> l
    out.append(pyr[off:off + N * r * r * 3].view(N, r, r, 3))
    off += N * r * r * 3
  return out


@pytest.mark.parametrize('R', [16, 32, 256])
def test_pyramid_matches_fp64(R):
  g = torch.Generator().manual_seed(R)
  x = torch.rand((3, R, R, 3), generator=g)
  levels = int(math.log2(R)) - 3
  got = _device_pyramid(x.cuda(), levels)
  want = O.laplacian_pyramid(x.double().numpy(), levels)
  for l in range(levels):
    err = float(np.abs(got[l].cpu().double().numpy() - want[l]).max())
    print('R=%d level %d: max |err| = %.3g (%.2f ulp of 1.0)' % (R, l, err, err / ULP1))
    assert err <= 4 * ULP1, (R, l, err)


def test_gather_is_bit_identical_to_indexing_the_pyramid():
  from twingan_b200 import swd
  N, R, s, k = 5, 64, 7, 128
  x = torch.rand((N, R, R, 3), device='cuda', generator=torch.Generator(device='cuda').manual_seed(1))
  draws = swd.make_draws(R, N, seed=3)
  pyr = _device_pyramid(x, 3)
  for l, r in enumerate((64, 32, 16)):
    cen = draws['centres'][l].cuda()
    desc = torch.empty((N * k, 3 * s * s), device='cuda')
    _lib().call('twg_swd_gather', pyr[l].data_ptr(), cen.data_ptr(), desc.data_ptr(), N, r, k, s, _st())
    off = torch.arange(s, device='cuda') - 3
    c = cen.long()
    ys = c[:, :, 0, None, None] + off[:, None]
    xs = c[:, :, 1, None, None] + off[None, :]
    want = pyr[l][torch.arange(N, device='cuda')[:, None, None, None], ys, xs, :]        # [N, k, s, s, 3]
    want = want.permute(0, 1, 4, 2, 3).reshape(N * k, -1)
    assert torch.equal(desc, want), l


def _sort(x):
  segs, n = x.shape
  ws = torch.empty(int(_lib().cdll.twg_swd_sort_workspace(segs, n)), device='cuda', dtype=torch.uint8)
  y = x.clone()
  _lib().call('twg_swd_sort', y.data_ptr(), ws.data_ptr(), segs, n, _st())
  return y


def test_sort_equals_torch_sort():
  g = torch.Generator(device='cuda').manual_seed(2)
  cases = {
      'normal, ragged tile': torch.randn((3, 5000), device='cuda', generator=g),
      'duplicates': torch.randint(-4, 5, (7, 3001), device='cuda', generator=g).float() * 0.5,
      'signed zeros and negatives': torch.tensor([0.0, -0.0, -1.0, 1.0, -0.0, 0.0, -3.5, 2.0] * 300, device='cuda').view(2, -1),
      'subnormals': torch.cat([torch.tensor([1e-45, -1e-45, 1e-40, -1e-40, 1.2e-38, -1.2e-38, 0.0, -0.0], device='cuda').repeat(100),
                               torch.randn(211, device='cuda', generator=g) * 1e-39]).view(1, -1),
      'large magnitudes': (torch.randn((4, 2049), device='cuda', generator=g) * 1e30),
      'one key': torch.randn((5, 1), device='cuda', generator=g),
      '2^20 + 3 keys': torch.randn((1, (1 << 20) + 3), device='cuda', generator=g),
      '128 columns': torch.randn((128, 4099), device='cuda', generator=g),
  }
  for name, x in cases.items():
    got = _sort(x)
    want = torch.sort(x, dim=1).values
    assert torch.equal(got, want), name
    neg = torch.signbit(got) & (got == 0)                          # -0 sorts before +0 within the zeros
    pos = ~torch.signbit(got) & (got == 0)
    if bool(neg.any()) and bool(pos.any()):
      idx = torch.arange(got.shape[1], device='cuda').expand_as(got)
      for r in range(got.shape[0]):
        if bool(neg[r].any()) and bool(pos[r].any()):
          assert int(idx[r][neg[r]].max()) < int(idx[r][pos[r]].min()), name


def _images(n, R, seed):
  """Two sets with different statistics: smooth random images (real) and noisier, darker ones (fake)."""
  g = torch.Generator().manual_seed(seed)
  lo = torch.rand((n, 3, R // 4, R // 4), generator=g)
  real = torch.nn.functional.interpolate(lo, size=(R, R), mode='bilinear', align_corners=False).permute(0, 2, 3, 1)
  fake = 0.5 * real + 0.5 * torch.rand((n, R, R, 3), generator=g) ** 2
  return real.contiguous(), fake.contiguous()


def _device_swd(real, fake, seed, batch=None, **kw):
  from twingan_b200 import swd
  n, R = real.shape[0], real.shape[1]
  m = swd.SlicedWasserstein(R, n, 'cuda', seed, **kw)
  batch = batch or n
  for i in range(0, n, batch):
    m.feed('real', real[i:i + batch].cuda())
    m.feed('fake', fake[i:i + batch].cuda())
  return m.result()


@pytest.mark.parametrize('n,R', [(64, 64), (512, 128)])
def test_swd_matches_fp64_on_the_same_draws(n, R):
  from twingan_b200 import swd
  real, fake = _images(n, R, seed=n)
  got = _device_swd(real, fake, seed=7, batch=45)               # batches of 45: the last one partial
  want = O.swd(real.numpy(), fake.numpy(), swd.make_draws(R, n, 7))
  assert set(got) == set(want)
  worst = 0.0
  for k in sorted(want):
    rel = abs(got[k] - want[k]) / abs(want[k])
    worst = max(worst, rel)
    print('n=%d R=%d %s: device %.9g fp64 %.9g rel %.2e' % (n, R, k, got[k], want[k], rel))
    assert rel < 1e-5, (k, got[k], want[k], rel)
  print('n=%d R=%d worst relative error %.2e' % (n, R, worst))


def test_identical_sets_score_zero_and_repeats_are_bit_identical():
  real, fake = _images(64, 64, seed=3)
  same = _device_swd(real, real, seed=1, real_floor=False)
  assert all(v == 0.0 for v in same.values()), same
  a = _device_swd(real, fake, seed=1)
  b = _device_swd(real, fake, seed=1, batch=7)
  assert a == b                                                  # bit-identical floats, whatever the batching


def test_swd_grows_with_noise_on_the_fakes():
  real, _ = _images(64, 64, seed=4)
  noise = torch.randn(real.shape, generator=torch.Generator().manual_seed(5))
  vals = [_device_swd(real, real + s * noise, seed=2, real_floor=False)['SWDx1e3_avg']
          for s in (0.0, 0.01, 0.03, 0.1, 0.3)]
  print('SWDx1e3_avg vs sigma:', vals)
  assert vals[0] == 0.0 and all(b > a for a, b in zip(vals, vals[1:])), vals


class _Images(object):
  """uint8 HWC images made on the fly from a seed (len() and image(i) like image_only.ImageOnlyDataset)."""

  def __init__(self, n, seed, hw=20):
    self.imgs = (torch.rand((n, hw, hw, 3), generator=torch.Generator().manual_seed(seed)) * 255).to(torch.uint8).numpy()

  def __len__(self):
    return len(self.imgs)

  def image(self, i):
    return self.imgs[i]


def _train(eval_fn, every):
  from twingan_b200 import pggan_runner as R
  from twingan_b200 import twingan
  flags = twingan.Flags(train_image_size=16, pggan_max_num_channels=32, learning_rate=1e-3)
  model = twingan.GanModel(flags, device='cuda', seed=11)
  gen = torch.Generator(device='cuda').manual_seed(5)
  dragan = torch.Generator(device='cuda').manual_seed(6)

  def batch_fn(stage, step):
    shape = (stage.batch_size, stage.hw, stage.hw, 3)
    return torch.rand(shape, device='cuda', generator=gen), torch.rand(shape, device='cuda', generator=gen)
  log = []
  R.run_stage(model, R.Stage(16, False, 4, 6, '16'), batch_fn, dragan_generator=dragan,
              log_fn=lambda s, l: log.append((s, l)), eval_every_n_iter_in_training=every, eval_fn=eval_fn)
  torch.cuda.synchronize()
  return model, log


def test_training_with_evaluation_is_bit_identical_to_training_without(tmp_path):
  from twingan_b200 import swd
  calls = []
  inner = swd.make_eval_fn(_Images(12, 1), _Images(12, 2), 8, str(tmp_path))

  def eval_fn(model, step):
    calls.append((step, inner(model, step)))
  m0, log0 = _train(None, 0)
  m1, log1 = _train(eval_fn, 2)
  assert [s for s, _ in calls] == [2, 4, 6]
  for s, res in calls:
    assert res is not None and all(math.isfinite(v) for v in res.values()), (s, res)
    assert (tmp_path / ('swd_train_step_%d_8_images.txt' % s)).exists()
  assert log0 == log1                                            # losses, float for float
  assert torch.equal(m0.variables.flat, m1.variables.flat)
  assert torch.equal(m0.variables.state, m1.variables.state)
  assert torch.equal(m0.variables.adam_m, m1.variables.adam_m) and torch.equal(m0.variables.adam_v, m1.variables.adam_v)
  # an existing result file is not recomputed during training (image_generation.py:884-886)
  assert inner(m1, 2) is None


def test_cli_evaluates_a_product_checkpoint(tmp_path):
  import io
  from PIL import Image
  from twingan_b200 import image_only, pggan_runner, swd_eval, twingan
  for name, seed in (('a', 1), ('b', 2)):
    imgs = _Images(6, seed).imgs
    recs = []
    for i, im in enumerate(imgs):
      buf = io.BytesIO()
      Image.fromarray(im).save(buf, format='PNG')
      recs.append(image_only.image_only_example('%d.png' % i, buf.getvalue(), 'PNG'))
    image_only.write_records(str(tmp_path / name / 'train-00000-of-00001'), recs)
  model = twingan.GanModel(twingan.Flags(train_image_size=16, pggan_max_num_channels=32), device='cuda')
  ckpt = pggan_runner.save_checkpoint(model, str(tmp_path / 'train'), 3)
  res = swd_eval.main(['--checkpoint_path', ckpt, '--dataset_dir', str(tmp_path / 'a'), '--unpaired_target_dataset_dir',
                       str(tmp_path / 'b'), '--train_image_size', '16', '--swd_num_images', '4', '--pggan_max_num_channels',
                       '32', '--eval_dir', str(tmp_path / 'eval')])
  text = (tmp_path / 'eval' / 'swd_eval_step_3_4_images.txt').read_text().splitlines()
  assert text[:2] == ['swd sliced wasserstein score evaluated on 4 images.', 'res\treal\tfake']
  assert text[2].startswith('16\t') and text[3].startswith('Average\t') and len(text) == 4
  assert float(text[2].split('\t')[2]) == pytest.approx(res['SWDx1e3_16'], abs=1e-6)
