"""Every library launch of the product's training step and inference, recorded once per test session, and the recorder
the stage tests launch through.

The conv, normaliser and elementwise audits (test_gpu_conv_conformance.py, test_gpu_norm_conformance.py,
test_gpu_elementwise_conformance.py) each filter this one harvest, so the step runs once and there is one copy of the
recorder."""
import contextlib

import torch

DEV = 'cuda:0'
_LAUNCHES = None


def harvest_product_launches():
  """(entry point, args) of every L.call, in order, of one eager training step per image size (4..256, 16 pairs; growing
  at alpha 0.5 from 8 up; instance norm, batch renorm, batch norm, instance norm with residual blocks) followed by its EMA
  pushes and its optimiser apply, and of inference on 64 images (instance norm, batch renorm, batch norm).  Cached for the session."""
  global _LAUNCHES
  if _LAUNCHES is not None:
    return _LAUNCHES
  from twingan_b200 import ops, twingan
  from twingan_b200._lib import lib
  L = lib()
  seen = []
  call = L.call

  def spy(name, *args):
    seen.append((name, args))
    return call(name, *args)

  L.call = spy
  try:
    gen = torch.Generator(device=DEV).manual_seed(0)
    ops.set_precision(1)
    for hw in (4, 8, 16, 32, 64, 128, 256):
      for growing in ((False, True) if hw >= 8 else (False,)):
        for norm, res in (('instance_norm', False), ('batch_renorm', False), ('batch_norm', False), ('instance_norm', True)):
          flags = twingan.Flags(train_image_size=hw, is_growing=growing, alpha_grow=0.5 if growing else 0.0,
                                generator_norm_type=norm, use_res_block=res)
          model = twingan.GanModel(flags, device=DEV)
          s = torch.rand((16, hw, hw, 3), device=DEV, generator=gen)
          t = torch.rand((16, hw, hw, 3), device=DEV, generator=gen)
          _, _, _, stats = model.compute_gradients(s, t, twingan.make_dragan_rand(16, hw, DEV, gen))
          model.apply_stat_updates(stats)
          model.apply_gradients()
          del model
    for norm in ('instance_norm', 'batch_renorm', 'batch_norm'):
      model = twingan.GanModel(twingan.Flags(train_image_size=256, generator_norm_type=norm), device=DEV)
      model.infer(torch.rand((64, 256, 256, 3), device=DEV, generator=gen))
      del model
    torch.cuda.synchronize()
  finally:
    del L.call
  _LAUNCHES = seen
  return seen


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
