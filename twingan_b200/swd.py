"""Sliced Wasserstein distance (SWD) of translated images on the device -- the reference's `--calc_swd` evaluation
(image_generation.py:868-927, twingan.py:679-680, 762-763), whose library the reference does not ship (:926-927).

The metric is PGGAN's (Karras et al., ICLR 2018, section 5 and appendix D):
  1. a Laplacian pyramid per image, levels R, R/2, ..., 16 (the last one Gaussian);
  2. per image and level, `nhoods_per_image` neighbourhoods of nhood_size x nhood_size pixels at uniformly drawn centres,
     each a descriptor of 3 * nhood_size^2 components in NCHW order;
  3. per set and level, every channel normalised to zero mean and unit population std over all its descriptor values;
  4. per level and repeat, both sets projected onto `dirs_per_repeat` random unit directions, every projection column
     sorted, and the mean absolute difference of the sorted columns taken; a level's value is the mean over the repeats,
     x 1e3.
The kernels are in csrc/twg_swd.cu (twg_swd_* in include/twg.h).  Every random draw (centres, directions) comes from one
seeded host torch.Generator (`make_draws`), so an evaluation is reproducible bit for bit and a restatement in fp64 can
consume exactly the same draws.  The same centres serve both sets (image i of either set is sampled at the same
positions), so two identical sets score exactly 0.
"""
from __future__ import annotations

import math
import os
from typing import Dict, List, Optional

import torch

from ._lib import lib

KINDS = ('real', 'fake')


def resolutions(resolution: int) -> List[int]:
  """The pyramid levels of an R x R image: R, R/2, ..., 16 (image_generation.py:913-916)."""
  check_resolution(resolution)
  return [resolution >> l for l in range(int(math.log2(resolution)) - 3)]


def check_resolution(resolution: int) -> None:
  if resolution < 16 or resolution & (resolution - 1):
    raise ValueError('SWD needs a square image size that is a power of two and at least 16, got %r' % (resolution,))


def make_draws(resolution: int, num_images: int, seed: int, nhood_size: int = 7, nhoods_per_image: int = 128,
               dir_repeats: int = 4, dirs_per_repeat: int = 128) -> Dict[str, list]:
  """All random draws of one evaluation from one generator seeded with `seed`, in this order:
  'centres'[l]: int32 [num_images, nhoods_per_image, 2] = {y, x}, uniform in [h, R_l - 1 - h], h = nhood_size // 2, for
  every level l in turn; then 'dirs'[l]: fp32 [dir_repeats, 3 * nhood_size^2, dirs_per_repeat], N(0, 1) draws whose
  columns are normalised to unit L2 norm in fp64 and then rounded to fp32."""
  gen = torch.Generator().manual_seed(int(seed))
  h = nhood_size // 2
  res = resolutions(resolution)
  centres = [torch.randint(h, r - h, (num_images, nhoods_per_image, 2), generator=gen, dtype=torch.int32) for r in res]
  dirs = []
  for _ in res:
    d = torch.randn((dir_repeats, 3 * nhood_size * nhood_size, dirs_per_repeat), generator=gen, dtype=torch.float64)
    dirs.append((d / d.square().sum(dim=1, keepdim=True).sqrt()).to(torch.float32))
  return {'centres': centres, 'dirs': dirs}


class SlicedWasserstein(object):
  """SWD between a set of real and a set of fake NHWC fp32 RGB images, `num_images` each, fed in batches of any size.

  `result()` gives {'SWDx1e3_<res>': ..., 'SWDx1e3_avg': ...} and, with `real_floor`, the same keys prefixed 'real_' for
  the real-vs-real floor: this project's definition of the `real` column of the reference's result file (the reference's
  library is not public), the SWD between the first and the second half of the real set with the same directions, each
  half normalised on its own (step 3).  It needs an even `num_images`.

  Memory: the descriptors are kept on the device in fp32, 3 * nhood_size^2 * nhoods_per_image * 4 bytes per image, level
  and set (about 3 GB per set at 8192 images of 256^2); `result()` works through the levels one at a time."""

  def __init__(self, resolution: int, num_images: int, device, seed: int, nhood_size: int = 7,
               nhoods_per_image: int = 128, dir_repeats: int = 4, dirs_per_repeat: int = 128, real_floor: bool = True):
    check_resolution(resolution)
    if num_images < 1:
      raise ValueError('num_images must be positive, got %r' % (num_images,))
    if real_floor and num_images % 2:
      raise ValueError('the real-vs-real floor compares the two halves of the real set: num_images must be even, got %d'
                       % num_images)
    if nhood_size < 1 or nhood_size % 2 == 0 or nhood_size > 16:
      raise ValueError('nhood_size must be odd and at most 16 (the smallest level), got %r' % (nhood_size,))
    if nhoods_per_image < 1 or dir_repeats < 1 or dirs_per_repeat < 1 or dirs_per_repeat % 128:
      raise ValueError('nhoods_per_image and dir_repeats must be positive and dirs_per_repeat a multiple of 128')
    self.device = torch.device(device)
    if self.device.type != 'cuda':
      raise ValueError('SlicedWasserstein runs on a CUDA device (there is no CPU path)')
    self.resolution, self.num_images, self.seed = int(resolution), int(num_images), int(seed)
    self.nhood_size, self.nhoods = int(nhood_size), int(nhoods_per_image)
    self.dir_repeats, self.dirs_per_repeat = int(dir_repeats), int(dirs_per_repeat)
    self.real_floor = bool(real_floor)
    self.resolutions = resolutions(resolution)
    draws = make_draws(resolution, num_images, seed, nhood_size, nhoods_per_image, dir_repeats, dirs_per_repeat)
    self.centres = [c.to(self.device) for c in draws['centres']]
    self.dirs = [d.to(self.device) for d in draws['dirs']]
    D = 3 * nhood_size * nhood_size
    rows = self.num_images * self.nhoods
    self.desc = {k: [torch.empty((rows, D), device=self.device) for _ in self.resolutions] for k in KINDS}
    self.count = {k: 0 for k in KINDS}

  def _st(self):
    return torch.cuda.current_stream(self.device).cuda_stream

  def feed(self, kind: str, batch: torch.Tensor) -> None:
    """Builds the Laplacian pyramid of `batch` ([b, R, R, 3], fp32; moved to the device if needed) and stores its
    descriptors as the next b images of set `kind` ('real' or 'fake')."""
    if kind not in KINDS:
      raise ValueError("kind must be 'real' or 'fake', got %r" % (kind,))
    R = self.resolution
    if batch.dim() != 4 or tuple(batch.shape[1:]) != (R, R, 3) or batch.shape[0] < 1:
      raise ValueError('expected a [b, %d, %d, 3] image batch, got %s' % (R, R, tuple(batch.shape)))
    b, start = int(batch.shape[0]), self.count[kind]
    if start + b > self.num_images:
      raise ValueError('%s set: %d images fed, %d more exceed num_images=%d' % (kind, start, b, self.num_images))
    x = batch.to(self.device, torch.float32).contiguous()
    if not bool(torch.isfinite(x).all()):
      raise ValueError('%s batch holds NaN or infinite values' % kind)
    L = lib()
    st = self._st()
    pyr = torch.empty(sum(b * r * r * 3 for r in self.resolutions), device=self.device)
    L.call('twg_swd_pyramid', x.data_ptr(), pyr.data_ptr(), b, R, len(self.resolutions), st)
    off = 0
    for l, r in enumerate(self.resolutions):
      dst = self.desc[kind][l][start * self.nhoods:(start + b) * self.nhoods]
      cen = self.centres[l][start:start + b]
      L.call('twg_swd_gather', pyr[off:].data_ptr(), cen.data_ptr(), dst.data_ptr(), b, r, self.nhoods,
             self.nhood_size, st)
      off += b * r * r * 3
    self.count[kind] = start + b

  def _distance(self, a: torch.Tensor, b: torch.Tensor, dirs: torch.Tensor, buf) -> torch.Tensor:
    """mean over the repeats of mean |sort(a' dirs) - sort(b' dirs)|, a' and b' each normalised per channel: an fp64
    device scalar."""
    L, st = lib(), self._st()
    rows, nd = a.shape[0], self.dirs_per_repeat
    stats = torch.empty((2, 6), device=self.device)
    L.call('twg_swd_stats', a.data_ptr(), stats[0].data_ptr(), rows, self.nhood_size, st)
    L.call('twg_swd_stats', b.data_ptr(), stats[1].data_ptr(), rows, self.nhood_size, st)
    sums = torch.empty(self.dir_repeats, device=self.device, dtype=torch.float64)
    pa, pb, ws = buf
    for r in range(self.dir_repeats):
      for desc, s, proj in ((a, stats[0], pa), (b, stats[1], pb)):
        L.call('twg_swd_project', desc.data_ptr(), s.data_ptr(), dirs[r].data_ptr(), proj.data_ptr(), rows,
               self.nhood_size, nd, st)
        L.call('twg_swd_sort', proj.data_ptr(), ws.data_ptr(), nd, rows, st)
      L.call('twg_swd_sorted_l1', pa.data_ptr(), pb.data_ptr(), sums[r:].data_ptr(), rows * nd, st)
    return sums.mean() / (rows * nd)

  def result(self) -> Dict[str, float]:
    for k in KINDS:
      if self.count[k] != self.num_images:
        raise RuntimeError('%s set: %d of %d images fed' % (k, self.count[k], self.num_images))
    rows, nd = self.num_images * self.nhoods, self.dirs_per_repeat
    ws_bytes = int(lib().cdll.twg_swd_sort_workspace(nd, rows))
    if ws_bytes < 0:
      raise ValueError(lib().last_error())
    buf = (torch.empty(nd * rows, device=self.device), torch.empty(nd * rows, device=self.device),
           torch.empty(ws_bytes, device=self.device, dtype=torch.uint8))
    fake, real = [], []
    for l in range(len(self.resolutions)):
      a, b = self.desc['real'][l], self.desc['fake'][l]
      fake.append(self._distance(a, b, self.dirs[l], buf))
      if self.real_floor:
        half = rows // 2
        real.append(self._distance(a[:half], a[half:], self.dirs[l], buf))
    out: Dict[str, float] = {}
    for prefix, vals in (('', fake), ('real_', real)):
      if not vals:
        continue
      vals = (torch.stack(vals) * 1e3).tolist()
      for r, v in zip(self.resolutions, vals):
        out['%sSWDx1e3_%d' % (prefix, r)] = v
      out['%sSWDx1e3_avg' % prefix] = sum(vals) / len(vals)
    return out


# -- translation quality (image_generation.py:868-927 with twingan.py:762-763) ----------------------------------------
def _draw_indices(ds, n: int, gen: torch.Generator, what: str) -> List[int]:
  if len(ds) < n:
    raise ValueError('%s dataset has %d images, fewer than the %d SWD needs' % (what, len(ds), n))
  return torch.randperm(len(ds), generator=gen)[:n].tolist()


def evaluate_translation(model, source_ds, target_ds, num_images: int, seed: int = 0, batch_size: int = 64,
                         real_floor: bool = True) -> Dict[str, float]:
  """SWD between target-domain images (real) and `model.infer` of source-domain images (fake), both `num_images` drawn
  without replacement with `seed` and preprocessed for evaluation (image_only.preprocess_image, is_training=False) at the
  model's resolution.  model.infer is the reference's t_prime_output in eval mode (twingan.py:762-763); the fakes are fed
  as floats, neither clipped nor quantised, as the reference feeds them.  Datasets give len() and image(i) -> uint8 HWC."""
  from .image_only import preprocess_image
  R = int(model.flags.train_image_size)
  check_resolution(R)
  gen = torch.Generator().manual_seed(int(seed))
  src = _draw_indices(source_ds, num_images, gen, 'source')
  tgt = _draw_indices(target_ds, num_images, gen, 'target')
  swd = SlicedWasserstein(R, num_images, model.device, seed, real_floor=real_floor)
  for i in range(0, num_images, batch_size):
    load = lambda ds, idx: torch.stack([preprocess_image(ds.image(j), R, is_training=False) for j in idx]).to(model.device)
    swd.feed('real', load(target_ds, tgt[i:i + batch_size]))
    swd.feed('fake', model.infer(load(source_ds, src[i:i + batch_size])))
  return swd.result()


def result_path(eval_dir: str, step: int, num_images: int, is_training: bool) -> str:
  """image_generation.py:882-883."""
  return os.path.join(eval_dir, 'swd_%s_step_%d_%d_images.txt' % ('train' if is_training else 'eval', step, num_images))


def write_result(eval_dir: str, step: int, num_images: int, result: Dict[str, float], is_training: bool) -> str:
  """The reference's result file (image_generation.py:918-924): a header line, `res real fake` rows from the finest level
  down, and the `Average` row; `real` is the real-vs-real floor.  Returns its path."""
  res = sorted((int(k[len('SWDx1e3_'):]) for k in result if k.startswith('SWDx1e3_') and k != 'SWDx1e3_avg'),
               reverse=True)
  if any('real_SWDx1e3_%d' % r not in result for r in res):
    raise ValueError('the result has no real-vs-real floor (evaluate with real_floor=True)')
  os.makedirs(eval_dir, exist_ok=True)
  path = result_path(eval_dir, step, num_images, is_training)
  with open(path, 'w') as f:
    f.write('swd sliced wasserstein score evaluated on %d images.\n' % num_images)
    f.write('res\treal\tfake\n')
    for r in res:
      f.write('%d\t%f\t%f\n' % (r, result['real_SWDx1e3_%d' % r], result['SWDx1e3_%d' % r]))
    f.write('Average\t%f\t%f\n' % (result['real_SWDx1e3_avg'], result['SWDx1e3_avg']))
  return path


def make_eval_fn(source_ds, target_ds, num_images: int, eval_dir: str, seed: int = 0, batch_size: int = 64):
  """The callable `pggan_runner.run_stage(eval_fn=...)` calls every `eval_every_n_iter_in_training` steps
  (twingan.py:679-680): eval_fn(model, step) writes swd_train_step_<step>_<n>_images.txt and returns the result, or skips
  (returns None) when that file already exists (image_generation.py:884-886).  It draws from its own generator and only
  runs the model in evaluation mode, so training continues exactly as without it."""
  def eval_fn(model, step: int) -> Optional[Dict[str, float]]:
    if os.path.exists(result_path(eval_dir, step, num_images, True)):
      return None
    res = evaluate_translation(model, source_ds, target_ds, num_images, seed, batch_size)
    write_result(eval_dir, step, num_images, res, is_training=True)
    return res
  return eval_fn
