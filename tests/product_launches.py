"""Every library launch of the product's training step and inference, recorded once per test session, and the recorder
the stage tests launch through.

The conv, normaliser and elementwise audits (test_gpu_conv_conformance.py, test_gpu_norm_conformance.py,
test_gpu_elementwise_conformance.py) each filter this one harvest, so the steps run once and there is one copy of the
recorder."""
import contextlib
import time

import torch

DEV = 'cuda:0'
_LAUNCHES = None
_CONFIGS = None          # [config label] beside each launch
HARVEST_SECONDS = None

_VARIANTS = (('instance_norm', False), ('batch_renorm', False), ('batch_norm', False), ('instance_norm', True))
# the optional flags of the step, each at 16 pairs
_FLAG_VARIANTS = (
    ('gan', {'loss_architecture': 'gan'}),
    ('wgan', {'loss_architecture': 'wgan'}),
    ('wgan+drift', {'loss_architecture': 'wgan', 'wgan_drift_loss_weight': 0.001}),
    ('wgan_gp', {'loss_architecture': 'wgan_gp'}),
    ('wgan_gp+drift', {'loss_architecture': 'wgan_gp', 'wgan_drift_loss_weight': 0.001}),
    ('hinge', {'loss_architecture': 'hinge'}),
    ('equalized_learning_rate', {'equalized_learning_rate': True}),
    ('pass_by_pass', {'batch_passes': False}),
)
_FLAG_STAGES = ((256, False), (64, True))          # one stable and one growing resolution, each with the cycle GAN loss
_INFER_BATCHES = (64, 1, 37)                       # the SWD evaluation's default batch, single images, a partial batch
_INFER_ALPHAS = (0.5, 1.0)                         # mid fade-in, and a growing stage's last step
_S_DIRECTION_GROWING_HW = 64                       # the growing stage that also runs the target -> source direction
_SWD_RESOLUTIONS = (16, 32, 64, 128, 256)
_SWD_IMAGES = 70                                   # one batch of 64 and a ragged one of 6; even, for the real floor


def inference_configs():
  """The evaluation-mode configurations of the harvest after the 256x256 one, in order: (label, hw, growing, alpha,
  target_domain, Flags keyword arguments).  GanModel.infer at every stage of pggan_runner.stage_plan(4, 256), as the SWD
  hook runs it during training and translate / swd_eval run it on a stage checkpoint: growing stages at alpha 0.5 and
  1.0, the four normaliser / residual variants, direction 't', and 's' at the 256x256 stable stage and one growing
  stage."""
  from twingan_b200 import pggan_runner as R
  out = []
  for s in R.stage_plan(4, 256):
    for norm, res in _VARIANTS:
      for alpha in (_INFER_ALPHAS if s.is_growing else (0.0,)):
        dirs = ('t', 's') if (s.hw == 256 and not s.is_growing) or (
            s.hw == _S_DIRECTION_GROWING_HW and s.is_growing and alpha == _INFER_ALPHAS[0]) else ('t',)
        for d in dirs:
          label = 'inference %s%s %s%s %s' % (s.name, ' alpha=%g' % alpha if s.is_growing else '', norm,
                                              ' res' if res else '', d)
          out.append((label, s.hw, s.is_growing, alpha, d, {'generator_norm_type': norm, 'use_res_block': res}))
  return out


def _harvest_inference(gen):
  """Launches GanModel.infer for every configuration of inference_configs() on _INFER_BATCHES; yields each label before
  its launches."""
  from twingan_b200 import twingan
  model, built = None, None
  for label, hw, growing, alpha, d, kw in inference_configs():
    if built != (hw, growing, tuple(sorted(kw.items()))):
      del model
      model = twingan.GanModel(twingan.Flags(train_image_size=hw, is_growing=growing, **kw), device=DEV)
      built = (hw, growing, tuple(sorted(kw.items())))
    model.flags.alpha_grow = alpha
    for n in _INFER_BATCHES:
      yield '%s batch %d' % (label, n)
      model.infer(torch.rand((n, hw, hw, 3), device=DEV, generator=gen), target_domain=d)
  del model


def _harvest_swd(gen):
  """The launches of the SWD hook (swd.evaluate_translation): one SlicedWasserstein per resolution, with the real-vs-real
  floor, fed in batches of 64 and a ragged last batch."""
  from twingan_b200 import swd
  for R in _SWD_RESOLUTIONS:
    yield 'swd %d images=%d' % (R, _SWD_IMAGES)
    sw = swd.SlicedWasserstein(R, _SWD_IMAGES, DEV, seed=R, real_floor=True)
    for i in range(0, _SWD_IMAGES, 64):
      n = min(64, _SWD_IMAGES - i)
      for kind in swd.KINDS:
        sw.feed(kind, torch.rand((n, R, R, 3), device=DEV, generator=gen))
    sw.result()


def _harvest_translate_front_end():
  """The uint8 front end and quantisation of `python -m twingan_b200.translate` on one small ragged batch."""
  import numpy as np
  from twingan_b200 import ops
  yield 'translate front end'
  rng = np.random.default_rng(0)
  images = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in ((37, 50), (32, 32), (5, 71))]
  payload, table = ops.pack_images(images)
  ops.batch_to_u8(ops.images_u8_to_batch(payload.to(DEV), table, 32))


def harvest_configs():
  """The training configurations of the harvest, in order: (label, hw, growing, pairs, Flags keyword arguments).
  The bench step at 16 pairs; every stage of the stage runner's two batch tables (pggan_runner.stage_plan from 4 to 256),
  each configuration once; the optional flags at 16 pairs.  Each with the four normaliser / residual variants, the
  optional flags with the default instance norm."""
  from twingan_b200 import pggan_runner as R
  out, done = [], set()

  def add(label, hw, growing, pairs, kw):
    sig = (hw, growing, pairs, tuple(sorted(kw.items())))
    if sig not in done:
      done.add(sig)
      out.append((label, hw, growing, pairs, kw))

  stages = [('bench', hw, growing, 16) for hw in (4, 8, 16, 32, 64, 128, 256)
            for growing in ((False, True) if hw >= 8 else (False,))]
  for table_name, table in (('DEFAULT_HW_TO_BATCH_SIZE', R.DEFAULT_HW_TO_BATCH_SIZE),
                            ('TWINGAN_HW_TO_BATCH_SIZE', R.TWINGAN_HW_TO_BATCH_SIZE)):
    stages += [(table_name, s.hw, s.is_growing, s.batch_size) for s in R.stage_plan(4, 256, hw_to_batch_size=table)]
  for source, hw, growing, pairs in stages:
    for norm, res in _VARIANTS:
      add('%s %d%s B=%d %s%s' % (source, hw, ' growing' if growing else '', pairs, norm, ' res' if res else ''),
          hw, growing, pairs, {'generator_norm_type': norm, 'use_res_block': res})
  for hw, growing in _FLAG_STAGES:
    for name, kw in _FLAG_VARIANTS:
      add('%s %d%s B=16' % (name, hw, ' growing' if growing else ''), hw, growing, 16, kw)
  return out


def harvest_product_launches():
  """(entry point, args) of every L.call, in order, of one eager training step per configuration of harvest_configs()
  (growing at alpha 0.5), each followed by its EMA pushes and its optimiser apply, and of inference at 256x256 on batches of
  64, 1 and 37 images (instance norm, batch renorm, batch norm); then of inference at every stage
  (inference_configs()), of the SWD evaluation at every resolution from 16 to 256 and of the translate front end.
  Cached for the session; launch_configs() names the configuration of each launch."""
  global _LAUNCHES, _CONFIGS, HARVEST_SECONDS
  if _LAUNCHES is not None:
    return _LAUNCHES
  from twingan_b200 import ops, twingan
  from twingan_b200._lib import lib
  L = lib()
  seen, configs = [], []
  label = [None]
  call = L.call

  def spy(name, *args):
    seen.append((name, args))
    configs.append(label[0])
    return call(name, *args)

  t0 = time.perf_counter()
  L.call = spy
  try:
    gen = torch.Generator(device=DEV).manual_seed(0)
    ops.set_precision(1)
    for label[0], hw, growing, B, kw in harvest_configs():
      flags = twingan.Flags(train_image_size=hw, is_growing=growing, alpha_grow=0.5 if growing else 0.0, **kw)
      model = twingan.GanModel(flags, device=DEV)
      s = torch.rand((B, hw, hw, 3), device=DEV, generator=gen)
      t = torch.rand((B, hw, hw, 3), device=DEV, generator=gen)
      _, _, _, stats = model.compute_gradients(s, t, twingan.make_dragan_rand(B, hw, DEV, gen))
      model.apply_stat_updates(stats)
      model.apply_gradients()
      del model
    for norm in ('instance_norm', 'batch_renorm', 'batch_norm'):
      model = twingan.GanModel(twingan.Flags(train_image_size=256, generator_norm_type=norm), device=DEV)
      for n in _INFER_BATCHES:
        label[0] = 'inference 256 %s batch %d' % (norm, n)
        model.infer(torch.rand((n, 256, 256, 3), device=DEV, generator=gen))
      del model
    for part in (_harvest_inference(gen), _harvest_swd(gen), _harvest_translate_front_end()):
      for label[0] in part:      # each part yields a label, then launches under it when resumed
        pass
    torch.cuda.synchronize()
  finally:
    del L.call
  HARVEST_SECONDS = time.perf_counter() - t0
  _LAUNCHES, _CONFIGS = seen, configs
  return seen


def launch_configs():
  """The configuration label of each launch of harvest_product_launches(), in the same order."""
  harvest_product_launches()
  return _CONFIGS


def key_configs(keys_of):
  """{key: label of the first configuration whose launches give it} for an audit's `keys_of` (launches -> set of keys),
  applied to each configuration's launches on their own."""
  launches, configs = harvest_product_launches(), launch_configs()
  out, start = {}, 0
  for i in range(1, len(launches) + 1):
    if i == len(launches) or configs[i] != configs[start]:
      for k in keys_of(launches[start:i]):
        out.setdefault(k, configs[start])
      start = i
  return out


class Recorder:
  """L.call that also keeps (entry, args): a stage test asserts that it launched the key it stands for, `keys` mapping
  the recorded launches to the keys of its audit.  Inside spying(), launches the library's Python layer (ops) makes are
  recorded too."""

  def __init__(self, L, keys):
    self.L, self.call, self.launches, self._keys = L, L.call, [], keys

  def __call__(self, name, *args):
    self.launches.append((name, args))
    self.call(name, *args)

  @contextlib.contextmanager
  def spying(self):
    self.L.call = self
    try:
      yield self
    finally:
      del self.L.call

  def keys(self):
    return self._keys(self.launches)
