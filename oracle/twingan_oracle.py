"""CPU oracle for the TwinGAN G+D step (TEST INFRASTRUCTURE ONLY).

This file is a restatement, in plain PyTorch-CPU autograd (fp64 by default), of
the arithmetic the reference builds as a TF-1.8 graph.  It is the *checker* for
the CUDA path: only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s
``cpu_baseline`` / ``--impl reference`` legs may import it.  The product package
``twingan_b200`` never imports anything under ``oracle/``.

PINNING (what this restatement has been held to, and what it has not).  The reference (
jerryli27/TwinGAN @4e55934) is Python-2 + tensorflow==1.8, cannot be run as shipped in this container, and ships no
test or golden vector for nets/pggan.py, nets/pggan_utils.py, libs/*, twingan.py or image_generation.py
(SURVEY.md section 4, 8c).  What is pinned, by tests/test_cpu_reference_golden.py against
tests/golden/reference_pggan_*.npz: the reference's OWN code -- nets/pggan.py, nets/pggan_utils.py, libs/batch_norm.py,
libs/instance_norm.py, util_misc.fp16_friendly_leaky_relu, and the method sources of twingan.GanModel._clone_fn /
add_loss, image_generation.GanModel.add_gan_loss / _add_dragan_loss / get_perturbed_batch / get_growing_image and
deployment/model_deploy.py (two clones) --
was executed in this container under a torch-backed stand-in for the TensorFlow-1.8 API
(tests/golden/tf18_shim.py, driver tests/golden/make_reference_golden.py); this file reproduces its variable names
and shapes (also at the 256x256 / 256-channel recipe size), every forward tensor, all named losses, both gradient
sets (incl. the double backward through the gradient penalty) and the moving-average pushes to 1e-9 (1e-5 where the
fixture stores float32).  Two restatement errors were found and fixed that way (plain batch_norm creates no renorm_*
variables, and its moving averages use decay 0.999, not 0.99).
PARITY UNPINNED for TensorFlow's own kernels: conv2d, avg_pool, resize_nearest_neighbor, nn.moments,
nn.batch_normalization, the tf.losses reductions, slim's conv2d / fully_connected wrappers and AdamOptimizer are
restated (here and in the stand-in) from the TF-1.8 documented semantics listed in SURVEY.md section 8a.4; no TF
binary was available to check them.  tests/golden/oracle_golden.npz (tests/golden/make_golden.py) is produced by THIS
file and only guards against regressions.

All tensors are NHWC like the reference (libs/batch_norm.py:409).  Every
function cites the reference file:line it follows.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, Optional, Tuple

import torch
import torch.nn.functional as F

Tensor = torch.Tensor

# nets/pggan_utils.py:32-47
DEFAULT_KERNEL_SIZE = 3
LEAKY_ALPHA = 0.2  # util_misc.py:68
BATCH_NORM_TYPE = 'batch_norm'
INSTANCE_NORM_TYPE = 'instance_norm'
BATCH_RENORM_TYPE = 'batch_renorm'
NO_NORM_TYPE = 'none'
BATCH_RENORM_BOUNDARIES = [10000, 20000, 30000]
BATCH_RENORM_RMAX_VALUES = [1.1, 1.5, 2.0, 4.0]
BATCH_RENORM_RMIN_VALUES = [0.9, 0.66, 0.5, 0.25]
BATCH_RENORM_DMAX_VALUES = [0.1, 0.3, 0.5, 1.0]


@dataclass
class Config:
  """Flag values that reach the hot path (defaults = docs/training.md:10-37 recipe)."""
  hw: int = 4                                   # train_image_size
  is_growing: bool = False                      # pggan_runner.py:93-98
  alpha_grow: float = 0.0                       # twingan.py:834-835
  max_num_channels: int = 256                   # nets/pggan.py:51-53
  generator_norm_type: str = INSTANCE_NORM_TYPE  # nets/pggan.py:25 (recipe: batch_renorm)
  do_pixel_norm: bool = True                    # nets/pggan.py:34
  use_unet: bool = True                         # twingan.py:52
  loss_architecture: str = 'dragan'             # image_generation.py:62
  gradient_penalty_lambda: float = 0.25         # image_generation.py:92 (recipe value)
  gan_weight: float = 1.0
  l_cyc_weight: float = 1.0                     # twingan.py:70
  do_l_cyc_gan: bool = True                     # twingan.py:75
  l_content_weight: float = 0.1                 # twingan.py:78
  learning_rate: float = 1e-4                   # docs/training.md:25
  adam_beta1: float = 0.5                       # model/model_inheritor.py:135-143
  adam_beta2: float = 0.99
  adam_eps: float = 1e-8
  global_step: int = 0                          # drives renorm clipping (pggan_utils.py:207-223)
  num_clones: int = 1                           # deployment/model_deploy.py:265-267
  # optional flags, off in the recipe (SURVEY 8f-4)
  equalized_learning_rate: bool = False         # nets/pggan.py:39-41, nets/pggan_utils.py:236-254
  wgan_drift_loss_weight: float = 0.0           # image_generation.py:96-98
  use_res_block: bool = False                   # nets/pggan.py:43-45, nets/pggan_utils.py:257-264, 334-342


def get_num_channels(stage: int, max_num_channels: int = 256) -> int:
  """nets/pggan_utils.py:369-372 (python-2 integer division)."""
  return min(1024 // (2 ** stage), max_num_channels)


def renorm_clipping(global_step: int) -> Dict[str, float]:
  """nets/pggan_utils.py:207-223: tf.train.piecewise_constant (x <= boundary -> that value)."""
  idx = 0
  for b in BATCH_RENORM_BOUNDARIES:
    if global_step > b:
      idx += 1
  return {'rmax': BATCH_RENORM_RMAX_VALUES[idx], 'rmin': BATCH_RENORM_RMIN_VALUES[idx],
          'dmax': BATCH_RENORM_DMAX_VALUES[idx]}


# ---------------------------------------------------------------------------------------------
# TF-1.8 primitive semantics (SURVEY 8a.4)
# ---------------------------------------------------------------------------------------------

def conv2d_nhwc(x: Tensor, w_hwio: Tensor, padding: str) -> Tensor:
  """tf.contrib.layers.conv2d stride 1 (nets/pggan_utils.py:316-320): cross-correlation, HWIO weights."""
  k = w_hwio.shape[0]
  pad = (k - 1) // 2 if padding == 'SAME' else 0
  y = F.conv2d(x.permute(0, 3, 1, 2), w_hwio.permute(3, 2, 0, 1), padding=pad)
  return y.permute(0, 2, 3, 1)


# ---- kink handling -------------------------------------------------------------------------------------
# leaky-ReLU and |a-b| have kinks: the GRADIENT of the step is discontinuous where a pre-activation (or a
# pixel difference) crosses zero, and an element within rounding noise of the kink takes either slope in
# any finite-precision evaluation (TF-CPU vs TF-GPU differ there too).  So gradient parity is defined
# modulo the sub-gradient choice AT the kink: when ACTIVE_SET is given, the oracle evaluates with the
# implementation's active set (one bool mask per leaky_relu call / one sign tensor per L1 call, in program
# order) and verifies that it departs from its own only on elements within KINK_AMBIGUITY (relative to the
# tensor's rms) of the kink -- anything else raises.
KINK_AMBIGUITY = 1e-3   # = the forward parity tolerance: a pre-activation the two sides may legitimately place on either side
ACTIVE_SET = None   # {'lrelu': iterator of bool tensors, 'l1': iterator of sign tensors, 'flips': [count, total]}


def _checked_override(x: Tensor, mine: Tensor, theirs: Tensor, what: str) -> None:
  diff = mine != theirs
  n = int(diff.sum())
  if n:
    rms = x.detach().pow(2).mean().sqrt().clamp_min(1e-30)
    worst = float((x.detach().abs()[diff] / rms).max())
    if worst > KINK_AMBIGUITY:
      raise AssertionError('%s: active set differs on an element %.3g rms away from the kink (> %g): not a '
                           'rounding-level difference' % (what, worst, KINK_AMBIGUITY))
  ACTIVE_SET['flips'][0] += n
  ACTIVE_SET['flips'][1] += diff.numel()


def leaky_relu(x: Tensor) -> Tensor:
  """util_misc.py:68-86: tf.maximum(alpha*x, x)."""
  if ACTIVE_SET is not None:
    m = next(ACTIVE_SET['lrelu']).to(x.device)
    _checked_override(x, x.detach() > 0, m, 'leaky_relu')
    return torch.where(m, x, LEAKY_ALPHA * x)
  return torch.maximum(LEAKY_ALPHA * x, x)


def pixel_norm(x: Tensor, eps: float = 1e-6) -> Tensor:
  """nets/pggan_utils.py:330-331."""
  return x / torch.sqrt(torch.mean(x * x, dim=3, keepdim=True) + eps)


def avg_pool2(x: Tensor) -> Tensor:
  """tf.nn.avg_pool 2x2/2 VALID (nets/pggan.py:274,306,436,468)."""
  n, h, w, c = x.shape
  return x.reshape(n, h // 2, 2, w // 2, 2, c).mean(dim=(2, 4))


def resize_twice_as_big(x: Tensor) -> Tensor:
  """nets/pggan_utils.py:349-350: nearest, out[i,j]=in[i//2,j//2]."""
  return x.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)


def minibatch_state_concat(x: Tensor) -> Tensor:
  """nets/pggan_utils.py:353-366 (hard-codes the 4x4 tile)."""
  mean = x.mean(dim=0, keepdim=True)
  std = torch.sqrt(((x - mean) ** 2).mean(dim=0, keepdim=True) + 1e-8)
  vals = std.mean().reshape(1, 1, 1, 1).expand(x.shape[0], 4, 4, 1)
  return torch.cat([x, vals], dim=3)


def sigmoid_cross_entropy(labels_value: float, logits: Tensor, weight: float) -> Tensor:
  """tf.losses.sigmoid_cross_entropy, scalar weight, SUM_BY_NONZERO_WEIGHTS => weight*mean (8a.4-3)."""
  z = torch.full_like(logits, labels_value)
  loss = torch.clamp(logits, min=0) - logits * z + torch.log1p(torch.exp(-logits.abs()))
  return weight * loss.mean()


def absolute_difference(labels: Tensor, predictions: Tensor, weight: float) -> Tensor:
  """tf.losses.absolute_difference => weight*mean|a-b|."""
  d = predictions - labels
  if ACTIVE_SET is not None:
    sgn = next(ACTIVE_SET['l1']).to(d.device).to(d.dtype)
    _checked_override(d, torch.sign(d.detach()), sgn, 'absolute_difference')
    return weight * (sgn * d).mean()
  return weight * d.abs().mean()


# ---------------------------------------------------------------------------------------------
# Normalizers (libs/batch_norm.py, libs/instance_norm.py)
# ---------------------------------------------------------------------------------------------

def instance_norm(x: Tensor, gamma: Tensor, beta: Tensor, eps: float = 1e-6) -> Tensor:
  """libs/instance_norm.py:31-138: moments over (H,W) per (n,c); tf.nn.batch_normalization."""
  mean = x.mean(dim=(1, 2), keepdim=True)
  var = ((x - mean) ** 2).mean(dim=(1, 2), keepdim=True)
  inv = torch.rsqrt(var + eps) * gamma
  return x * inv + (beta - mean * inv)


def batch_norm_train(x: Tensor, gamma: Tensor, beta: Tensor, stats: Optional[Dict[str, Tensor]],
                     renorm: bool, clip: Optional[Dict[str, float]], eps: float = 1e-3,
                     updates: Optional[Dict[str, Tensor]] = None) -> Tensor:
  """libs/batch_norm.py:396-470 (_batch_norm_aux, is_training=True) with :329-393 renorm correction.

  `stats` holds the PRE-update moving statistics (renorm_mean, renorm_stddev, *_weight); r and d are
  stop-gradient (:456-457).  `updates` (optional dict) receives the per-pass new moments that the
  reference would push into the EMAs (:371-393, :295-319)."""
  mean = x.mean(dim=(0, 1, 2))
  var = ((x - mean) ** 2).mean(dim=(0, 1, 2))
  scale, offset = gamma, beta
  if renorm:
    stddev = torch.sqrt(var + eps)
    mixed_mean = stats['renorm_mean'] + (1. - stats['renorm_mean_weight']) * mean
    mixed_std = stats['renorm_stddev'] + (1. - stats['renorm_stddev_weight']) * stddev
    r = (stddev / mixed_std).clamp(min=clip['rmin'], max=clip['rmax']).detach()
    d = ((mean - mixed_mean) / mixed_std).clamp(min=-clip['dmax'], max=clip['dmax']).detach()
    scale, offset = r * gamma, d * gamma + beta
    if updates is not None:
      updates['mean'] = mean.detach()
      updates['stddev'] = stddev.detach()
  elif updates is not None:
    updates['mean'] = mean.detach()
    updates['variance'] = var.detach()
  inv = torch.rsqrt(var + eps) * scale
  return x * inv + (offset - mean * inv)


def batch_norm_eval(x: Tensor, gamma: Tensor, beta: Tensor, moving_mean: Tensor, moving_var: Tensor,
                    eps: float = 1e-3) -> Tensor:
  """libs/batch_norm.py:266-278, 461-462: moving stats, r=1, d=0."""
  inv = torch.rsqrt(moving_var + eps) * gamma
  return x * inv + (beta - moving_mean * inv)


# ---------------------------------------------------------------------------------------------
# Parameters
# ---------------------------------------------------------------------------------------------

def _norm_scope(norm_type: str) -> str:
  # default scope names libs/batch_norm.py:79-80, libs/instance_norm.py:65-66
  return 'InstanceNorm' if norm_type == INSTANCE_NORM_TYPE else 'BatchNorm'


def layer_table(cfg: Config):
  """Enumerate every conv/fc layer of E, G, D for cfg as (scope-relative name, k, cin, cout, kind).

  kind: 'gen' = no bias + per-domain norm (generator/encoder arg scope, nets/pggan_utils.py:101-113),
        'dis' = bias, no norm (:116-127), 'fc' = fully connected with bias (nets/pggan.py:363-370)."""
  mc = cfg.max_num_channels
  max_stage = int(math.log2(cfg.hw)) - 2
  enc, gen, dis = [], [], []
  # encoder (nets/pggan.py:403-479) -- discriminator body has the same topology (:242-335)
  for lst, kind in ((enc, 'gen'), (dis, 'dis')):
    if cfg.is_growing:
      lst.append(('from_rgb_%dx%d/Conv' % (cfg.hw // 2, cfg.hw // 2), 1, 3, get_num_channels(max_stage - 1, mc), kind))
    lst.append(('from_rgb_%dx%d/Conv' % (cfg.hw, cfg.hw), 1, 3, get_num_channels(max_stage, mc), kind))
    if cfg.use_res_block:   # residual shortcuts: a 1x1 conv + bias, no normaliser / activation, where the channel counts differ
      if cfg.is_growing:
        lst.append(('from_rgb_%dx%d/shortcut' % (cfg.hw // 2, cfg.hw // 2), 1, 3, get_num_channels(max_stage - 1, mc), 'short'))
      lst.append(('from_rgb_%dx%d/shortcut' % (cfg.hw, cfg.hw), 1, 3, get_num_channels(max_stage, mc), 'short'))
    cin = get_num_channels(max_stage, mc)
    for stage in range(max_stage, 0, -1):
      nc = get_num_channels(stage - 1, mc)
      hw = cfg.hw // (2 ** (max_stage - stage))
      scope = 'encoder_block_%dx%dx%d' % (hw, hw, nc)
      lst.append((scope + '/Conv', 3, cin, cin, kind))
      lst.append((scope + '/Conv_1', 3, cin, nc, kind))
      if cfg.use_res_block and cin != nc:
        lst.append((scope + '/shortcut', 1, cin, nc, 'short'))
      cin = nc
  dis.append(('before_fc_1x1x%d/Conv' % mc, 3, cin + 1, mc, 'dis'))
  dis.append(('before_fc_1x1x%d/Conv_1' % mc, 4, mc, mc, 'dis'))
  dis.append(('prediction/fully_connected', 0, mc, 1, 'fc'))
  # generator (nets/pggan.py:93-211), source = 4x4 code
  code_c = get_num_channels(0, mc)
  c0 = get_num_channels(0, mc)
  gen.append(('block_4x4x%d/Conv' % c0, 3, code_c, c0, 'gen'))
  gen.append(('block_4x4x%d/Conv_1' % c0, 3, c0, c0, 'gen'))
  cin = c0
  for stage in range(1, max_stage + 1):
    hw = 2 ** (stage + 2)
    oc = get_num_channels(stage, mc)
    if stage == max_stage and cfg.is_growing:
      gen.append(('generator_to_rgb_%dx%d/Conv' % (hw // 2, hw // 2), 1, cin, 3, 'gen'))
    skip_c = get_num_channels(stage - 1, mc) if cfg.use_unet else 0
    scope = 'block_%dx%dx%d' % (hw, hw, oc)
    gen.append((scope + '/Conv', 3, cin + skip_c, oc, 'gen'))
    gen.append((scope + '/Conv_1', 3, oc, oc, 'gen'))
    if cfg.use_res_block and cin + skip_c != oc:
      gen.append((scope + '/shortcut', 1, cin + skip_c, oc, 'short'))
    cin = oc
  gen.append(('generator_to_rgb_%dx%d/Conv' % (cfg.hw, cfg.hw), 1, cin, 3, 'gen'))
  return {'encoder_content': enc, 'generator': gen, 'discriminator': dis}


def init_params(cfg: Config, seed: int = 1234, dtype=torch.float64, randomize_affine: bool = False
                ) -> Dict[str, Tensor]:
  """Variables with the reference's names (SURVEY 8a.4-11) and initialisers:
  weights N(0, 0.02) (nets/pggan_utils.py:56,93), biases 0, gamma 1, beta 0.
  `randomize_affine` perturbs gamma/beta/biases so parity tests exercise them."""
  g = torch.Generator().manual_seed(seed)
  tbl = layer_table(cfg)
  p: Dict[str, Tensor] = {}
  ns = _norm_scope(cfg.generator_norm_type)

  def normal(shape, std):
    return (torch.randn(shape, generator=g, dtype=torch.float64) * std).to(dtype)

  for scope in ('encoder_content', 'generator'):
    for name, k, cin, cout, kind in tbl[scope]:
      p['%s/%s/weights' % (scope, name)] = normal((k, k, cin, cout), 0.02)
      if kind == 'short':     # normalizer_fn=None: slim's conv2d adds a bias (nets/pggan_utils.py:339-341)
        p['%s/%s/biases' % (scope, name)] = normal((cout,), 0.1) if randomize_affine else torch.zeros(cout, dtype=dtype)
      elif cfg.generator_norm_type != NO_NORM_TYPE:
        for d in ('_s', '_t'):
          gam = torch.ones(cout, dtype=dtype)
          bet = torch.zeros(cout, dtype=dtype)
          if randomize_affine:
            gam = gam + normal((cout,), 0.2)
            bet = bet + normal((cout,), 0.1)
          p['%s/%s/%s/gamma%s' % (scope, name, ns, d)] = gam
          p['%s/%s/%s/beta%s' % (scope, name, ns, d)] = bet
      else:
        p['%s/%s/biases' % (scope, name)] = normal((cout,), 0.1) if randomize_affine else torch.zeros(cout, dtype=dtype)
  for dscope in ('discriminator_s', 'discriminator_t'):
    for name, k, cin, cout, kind in tbl['discriminator']:
      shape = (cin, cout) if kind == 'fc' else (k, k, cin, cout)
      p['%s/%s/weights' % (dscope, name)] = normal(shape, 0.02)
      p['%s/%s/biases' % (dscope, name)] = normal((cout,), 0.1) if randomize_affine else torch.zeros(cout, dtype=dtype)
  return p


def init_norm_state(cfg: Config, dtype=torch.float64, seed: Optional[int] = None) -> Dict[str, Tensor]:
  """Non-trainable normaliser state (libs/batch_norm.py:184-246): moving_mean 0, moving_variance 1,
  renorm_* 0 (so step-0 renorm has r=1, d=0, SURVEY 8a.4-7).  `seed` randomises them (tests)."""
  st: Dict[str, Tensor] = {}
  if cfg.generator_norm_type not in (BATCH_NORM_TYPE, BATCH_RENORM_TYPE):
    return st
  g = torch.Generator().manual_seed(seed) if seed is not None else None
  renorm = cfg.generator_norm_type == BATCH_RENORM_TYPE   # plain batch_norm creates no renorm_* variables (:214)
  tbl = layer_table(cfg)
  for scope in ('encoder_content', 'generator'):
    for name, k, cin, cout, kind in tbl[scope]:
      if kind == 'short':
        continue
      for d in ('_s', '_t'):
        base = '%s/%s/BatchNorm/' % (scope, name)
        if g is None:
          st[base + 'moving_mean' + d] = torch.zeros(cout, dtype=dtype)
          st[base + 'moving_variance' + d] = torch.ones(cout, dtype=dtype)
          if renorm:
            st[base + 'renorm_mean' + d] = torch.zeros(cout, dtype=dtype)
            st[base + 'renorm_stddev' + d] = torch.zeros(cout, dtype=dtype)
            st[base + 'renorm_mean_weight' + d] = torch.zeros((), dtype=dtype)
            st[base + 'renorm_stddev_weight' + d] = torch.zeros((), dtype=dtype)
        else:
          w = 0.6
          st[base + 'moving_mean' + d] = (torch.randn(cout, generator=g, dtype=torch.float64) * 0.1).to(dtype)
          st[base + 'moving_variance' + d] = (0.5 + torch.rand(cout, generator=g, dtype=torch.float64)).to(dtype)
          rm = (w * torch.randn(cout, generator=g, dtype=torch.float64) * 0.02).to(dtype)
          rs = (w * (0.05 + 0.1 * torch.rand(cout, generator=g, dtype=torch.float64))).to(dtype)
          if renorm:
            st[base + 'renorm_mean' + d] = rm
            st[base + 'renorm_stddev' + d] = rs
            st[base + 'renorm_mean_weight' + d] = torch.tensor(w, dtype=dtype)
            st[base + 'renorm_stddev_weight' + d] = torch.tensor(w, dtype=dtype)
  return st


# ---------------------------------------------------------------------------------------------
# One conv "layer" (SURVEY 3.3)
# ---------------------------------------------------------------------------------------------

class Nets:
  """The three network functions of nets/pggan.py bound to a parameter dict."""

  def __init__(self, cfg: Config, params: Dict[str, Tensor], norm_state: Optional[Dict[str, Tensor]] = None):
    self.cfg = cfg
    self.p = params
    self.st = norm_state or {}
    self.stat_updates = []  # (variable base name + domain, dict) in program order

  # -- generator/encoder arg-scope conv: conv -> normalizer -> activation (-> pixel norm) ------
  def gen_conv(self, x: Tensor, name: str, domain: str, padding: str = 'SAME', activation: bool = True,
               pixnorm: bool = True, is_training: bool = True) -> Tensor:
    """maybe_pixel_norm(maybe_equalized_conv2d(x, C)) under pggan_generator_arg_scope
    (nets/pggan.py:78-81, nets/pggan_utils.py:86-98): no bias when a normalizer is set."""
    cfg = self.cfg
    y = conv2d_nhwc(self._equalized(x, self.p[name + '/weights']), self.p[name + '/weights'], padding)
    nt = cfg.generator_norm_type
    if nt == INSTANCE_NORM_TYPE:
      y = instance_norm(y, self.p[name + '/InstanceNorm/gamma' + domain], self.p[name + '/InstanceNorm/beta' + domain])
    elif nt in (BATCH_NORM_TYPE, BATCH_RENORM_TYPE):
      base = name + '/BatchNorm/'
      gamma, beta = self.p[base + 'gamma' + domain], self.p[base + 'beta' + domain]
      if is_training:
        stats = {k: self.st[base + k + domain] for k in
                 ('renorm_mean', 'renorm_stddev', 'renorm_mean_weight', 'renorm_stddev_weight')} \
            if nt == BATCH_RENORM_TYPE else None
        upd: Dict[str, Tensor] = {}
        y = batch_norm_train(y, gamma, beta, stats, nt == BATCH_RENORM_TYPE,
                             renorm_clipping(cfg.global_step) if nt == BATCH_RENORM_TYPE else None, updates=upd)
        self.stat_updates.append((base, domain, upd))
      else:
        y = batch_norm_eval(y, gamma, beta, self.st[base + 'moving_mean' + domain],
                            self.st[base + 'moving_variance' + domain])
    elif nt == NO_NORM_TYPE:
      y = y + self.p[name + '/biases']
    else:
      raise NotImplementedError(nt)
    if activation:
      y = leaky_relu(y)
    if pixnorm and cfg.do_pixel_norm:
      y = pixel_norm(y)
    return y

  def _equalized(self, x: Tensor, w: Tensor) -> Tensor:
    """maybe_equalized_conv2d / maybe_equalized_fc (nets/pggan_utils.py:236-254): with --equalized_learning_rate the
    layer INPUT is scaled by sqrt(2 / fan_in), fan_in = in_ch * k^2 (conv, HWIO weights) or in_ch (fc, [in, out])."""
    if not self.cfg.equalized_learning_rate:
      return x
    fan_in = w.shape[0] * w.shape[1] * w.shape[2] if w.dim() == 4 else w.shape[0]
    return math.sqrt(2.0 / fan_in) * x

  def resblock(self, input_layer: Tensor, conv2d_out: Tensor, block_scope: str) -> Tensor:
    """maybe_resblock (nets/pggan_utils.py:257-264): with --use_res_block the block output is shortcut + conv2d_out, the
    shortcut being the block input, or (channel counts differ) a 1x1 conv of it with bias and neither normaliser nor
    activation in scope 'shortcut' (:334-342)."""
    if not self.cfg.use_res_block:
      return conv2d_out
    if input_layer.shape[-1] == conv2d_out.shape[-1]:
      return input_layer + conv2d_out
    w = self.p[block_scope + '/shortcut/weights']
    return conv2d_nhwc(self._equalized(input_layer, w), w, 'SAME') + self.p[block_scope + '/shortcut/biases'] + conv2d_out

  def dis_conv(self, x: Tensor, name: str, padding: str = 'SAME') -> Tensor:
    """pggan_discriminator_arg_scope (nets/pggan_utils.py:116-127): conv + bias -> leaky-ReLU."""
    w = self.p[name + '/weights']
    return leaky_relu(conv2d_nhwc(self._equalized(x, w), w, padding) + self.p[name + '/biases'])

  # -- encoder (nets/pggan.py:403-479) ------------------------------------------------------------
  def encoder(self, source: Tensor, domain: str, scope: str = 'encoder_content', is_training: bool = True
              ) -> Tuple[Tensor, Dict[str, Tensor]]:
    cfg = self.cfg
    mc = cfg.max_num_channels
    hw = source.shape[1]
    max_stage = int(math.log2(hw)) - 2
    ep: Dict[str, Tensor] = {'source': source}
    shrunk = None
    if cfg.is_growing:
      shrunk = avg_pool2(source)
      sn = 'from_rgb_%dx%d' % (hw // 2, hw // 2)
      pooled = shrunk
      shrunk = self.gen_conv(shrunk, '%s/%s/Conv' % (scope, sn), domain, is_training=is_training)
      shrunk = self.resblock(pooled, shrunk, '%s/%s' % (scope, sn))           # encoder_from_rgb_block, nets/pggan.py:395-399
      ep[sn] = shrunk
    sn = 'from_rgb_%dx%d' % (hw, hw)
    net = self.gen_conv(source, '%s/%s/Conv' % (scope, sn), domain, is_training=is_training)
    net = self.resblock(source, net, '%s/%s' % (scope, sn))
    ep[sn] = net
    for stage in range(max_stage, 0, -1):
      nc = get_num_channels(stage - 1, mc)
      cur = hw // (2 ** (max_stage - stage))
      sn = 'encoder_block_%dx%dx%d' % (cur, cur, nc)
      block_in = net
      net = self.gen_conv(net, '%s/%s/Conv' % (scope, sn), domain, is_training=is_training)
      net = self.gen_conv(net, '%s/%s/Conv_1' % (scope, sn), domain, is_training=is_training)
      net = self.resblock(block_in, net, '%s/%s' % (scope, sn))               # encoder_two_layer_block, :382-393
      ep[sn] = net
      cur //= 2
      net = avg_pool2(net)
      ep['downsample_to_%dx%dx%d' % (cur, cur, nc)] = net
      if stage == max_stage and cfg.is_growing:
        net = net * cfg.alpha_grow + (1 - cfg.alpha_grow) * shrunk
        ep['encoder_block_interpolated_%dx%dx%d' % (cur, cur, nc)] = net
    ep['before_classification'] = net
    return net, ep

  # -- generator (nets/pggan.py:93-211) ------------------------------------------------------------
  def generator(self, source: Tensor, domain: str, unet_end_points: Optional[Dict[str, Tensor]],
                scope: str = 'generator', is_training: bool = True) -> Tuple[Tensor, Dict[str, Tensor]]:
    cfg = self.cfg
    mc = cfg.max_num_channels
    max_stage = int(math.log2(cfg.hw)) - 2
    ep: Dict[str, Tensor] = {'source': source}
    assert source.shape[1] == 4 and source.shape[2] == 4  # nets/pggan.py:157
    net = source
    before_growth = None
    hw = 4
    for stage in range(0, max_stage + 1):
      hw = 2 ** (stage + 2)
      oc = get_num_channels(stage, mc)
      sn = 'block_%dx%dx%d' % (hw, hw, oc)
      if hw == 4:
        net = self.gen_conv(net, '%s/%s/Conv' % (scope, sn), domain, is_training=is_training)
        net = self.gen_conv(net, '%s/%s/Conv_1' % (scope, sn), domain, is_training=is_training)
      else:
        if stage == max_stage and cfg.is_growing:
          rn = 'generator_to_rgb_%dx%d' % (hw // 2, hw // 2)
          before_growth = self.gen_conv(net, '%s/%s/Conv' % (scope, rn), domain, activation=False, pixnorm=False,
                                        is_training=is_training)
          before_growth = resize_twice_as_big(before_growth)
          ep[rn] = before_growth
        net = resize_twice_as_big(net)
        net = self._concat_unet(net, unet_end_points)
        block_in = net
        net = self.gen_conv(net, '%s/%s/Conv' % (scope, sn), domain, is_training=is_training)
        net = self.gen_conv(net, '%s/%s/Conv_1' % (scope, sn), domain, is_training=is_training)
        net = self.resblock(block_in, net, '%s/%s' % (scope, sn))             # generator_three_layer_block, :69-83
      ep[sn] = net
    rn = 'generator_to_rgb_%dx%d' % (hw, hw)
    to_rgb = self.gen_conv(net, '%s/%s/Conv' % (scope, rn), domain, activation=False, pixnorm=False,
                           is_training=is_training)
    if not cfg.is_growing:
      out = to_rgb
    else:
      out = to_rgb * cfg.alpha_grow + (1 - cfg.alpha_grow) * before_growth
    ep['output'] = out
    return out, ep

  def _concat_unet(self, layer: Tensor, unet_end_points: Optional[Dict[str, Tensor]]) -> Tensor:
    """nets/pggan_utils.py:281-298."""
    if unet_end_points is None:
      return layer
    hw = layer.shape[1]
    nc = get_num_channels(int(math.log2(hw)) - 2 - 1, self.cfg.max_num_channels)
    name = 'encoder_block_interpolated_%dx%dx%d' % (hw, hw, nc)
    if name not in unet_end_points:
      name = 'encoder_block_%dx%dx%d' % (hw, hw, nc)
    if name not in unet_end_points:
      raise ValueError('%s not in unet_end_points' % name)
    return torch.cat((layer, unet_end_points[name]), dim=-1)

  # -- discriminator (nets/pggan.py:242-376) --------------------------------------------------------
  def discriminator(self, source: Tensor, scope: str) -> Tuple[Tensor, Dict[str, Tensor]]:
    cfg = self.cfg
    mc = cfg.max_num_channels
    hw = source.shape[1]
    max_stage = int(math.log2(hw)) - 2
    ep: Dict[str, Tensor] = {}
    shrunk = None
    if cfg.is_growing:
      shrunk = avg_pool2(source)
      sn = 'from_rgb_%dx%d' % (hw // 2, hw // 2)
      pooled = shrunk
      shrunk = self.dis_conv(shrunk, '%s/%s/Conv' % (scope, sn))
      shrunk = self.resblock(pooled, shrunk, '%s/%s' % (scope, sn))           # discriminator_from_rgb_block, :233-240
      ep[sn] = shrunk
    sn = 'from_rgb_%dx%d' % (hw, hw)
    net = self.dis_conv(source, '%s/%s/Conv' % (scope, sn))
    net = self.resblock(source, net, '%s/%s' % (scope, sn))
    ep[sn] = net
    for stage in range(max_stage, 0, -1):
      nc = get_num_channels(stage - 1, mc)
      cur = hw // (2 ** (max_stage - stage))
      sn = 'encoder_block_%dx%dx%d' % (cur, cur, nc)
      block_in = net
      net = self.dis_conv(net, '%s/%s/Conv' % (scope, sn))
      net = self.dis_conv(net, '%s/%s/Conv_1' % (scope, sn))
      net = self.resblock(block_in, net, '%s/%s' % (scope, sn))               # discriminator_two_layer_block, :221-231
      ep[sn] = net
      cur //= 2
      net = avg_pool2(net)
      ep['downsample_to_%dx%dx%d' % (cur, cur, nc)] = net
      if stage == max_stage and cfg.is_growing:
        net = net * cfg.alpha_grow + (1 - cfg.alpha_grow) * shrunk
        ep['encoder_block_interpolated_%dx%dx%d' % (cur, cur, nc)] = net
    sn = 'before_fc_1x1x%d' % mc
    net = minibatch_state_concat(net)
    net = self.dis_conv(net, '%s/%s/Conv' % (scope, sn), 'SAME')
    net = self.dis_conv(net, '%s/%s/Conv_1' % (scope, sn), 'VALID')
    ep['before_fc'] = net
    fcw = self.p['%s/prediction/fully_connected/weights' % scope]
    logits = self._equalized(net.reshape(net.shape[0], -1), fcw) @ fcw \
        + self.p['%s/prediction/fully_connected/biases' % scope]
    ep['prediction'] = logits
    return logits, ep


# ---------------------------------------------------------------------------------------------
# TwinGAN wiring + losses (twingan.py:146-521, image_generation.py:317-476)
# ---------------------------------------------------------------------------------------------

def get_growing_image(image: Tensor, alpha: float) -> Tensor:
  """image_generation.py:1001-1006."""
  low = resize_twice_as_big(avg_pool2(image))
  return alpha * image + (1 - alpha) * low


def dragan_interpolates(real: Tensor, alpha: Tensor, noise: Tensor) -> Tensor:
  """image_generation.py:441-460.  `alpha` ~U[0,1] shape [B,1,1,1] and `noise` ~U[-1,1] (full shape) are
  explicit inputs so both sides see the same randomness.  NB the reference scales by the VARIANCE
  (tf.nn.moments(...)[1]) although it calls it std (SURVEY 8a.4-10)."""
  var = ((real - real.mean()) ** 2).mean()
  perturbed = real + 0.5 * var * noise
  return real + alpha * (perturbed - real)


def twingan_losses(cfg: Config, params: Dict[str, Tensor], norm_state: Dict[str, Tensor], sources: Tensor,
                   targets: Tensor, dragan_rand: Dict[str, Tensor]):
  """Forward of GanModel._clone_fn + add_loss.  Returns (g_loss, d_loss, named losses, end_points, nets)."""
  nets = Nets(cfg, params, norm_state)
  if cfg.is_growing:  # twingan.py:827-839
    sources = get_growing_image(sources, cfg.alpha_grow)
    targets = get_growing_image(targets, cfg.alpha_grow)
  enc_s, ep_s = nets.encoder(sources, '_s')                      # twingan.py:198-200
  enc_t, ep_t = nets.encoder(targets, '_t')                      # :215-217
  unet = cfg.use_unet
  s_prime, _ = nets.generator(enc_t, '_s', ep_t if unet else None)   # :242-247
  s_cycle, _ = nets.generator(enc_s, '_s', ep_s if unet else None)   # :250-255
  t_prime, _ = nets.generator(enc_s, '_t', ep_s if unet else None)   # :258-262
  t_cycle, _ = nets.generator(enc_t, '_t', ep_t if unet else None)   # :265-269
  enc_t_prime, _ = nets.encoder(t_prime, '_t')                   # :275-277
  enc_s_prime, _ = nets.encoder(s_prime, '_s')                   # :281-284
  preds = {
      'real_s': nets.discriminator(sources, 'discriminator_s')[0],   # :370-381
      's_prime': nets.discriminator(s_prime, 'discriminator_s')[0],
      's_cycle': nets.discriminator(s_cycle, 'discriminator_s')[0],
      'real_t': nets.discriminator(targets, 'discriminator_t')[0],
      't_prime': nets.discriminator(t_prime, 'discriminator_t')[0],
      't_cycle': nets.discriminator(t_cycle, 'discriminator_t')[0],
  }
  ends = {'sources': sources, 'targets': targets, 's_prime': s_prime, 's_cycle': s_cycle, 't_prime': t_prime,
          't_cycle': t_cycle, 'enc_s': enc_s, 'enc_t': enc_t, 'enc_s_prime': enc_s_prime,
          'enc_t_prime': enc_t_prime}
  ends.update({'pred_' + k: v for k, v in preds.items()})
  gl: Dict[str, Tensor] = {}
  dl: Dict[str, Tensor] = {}
  gw = cfg.gan_weight
  for dom in ('s', 't'):                                          # twingan.py:451-521
    opp = 't' if dom == 's' else 's'
    original = sources if dom == 's' else targets
    gl['l_cyc_' + dom] = absolute_difference(original, ends[dom + '_cycle'], cfg.l_cyc_weight)   # :464
    real_pred = preds['real_' + dom]
    posts = []
    if cfg.hw >= 64 and cfg.do_l_cyc_gan:                         # :466-474
      posts.append('cycle')
    posts.append('prime')                                         # :477-482
    for post in posts:
      fake_pred = preds['%s_%s' % (dom, post)]
      arch = cfg.loss_architecture
      only_real_fake = post == 'cycle'                            # twingan.py:473
      if arch in ('wgan', 'wgan_gp', 'hinge'):                    # image_generation.py:330-336
        gl['generator_fool_loss_%s_%s' % (post, dom)] = gw * (-fake_pred.mean())
      elif arch in ('gan', 'dragan'):                             # :338-344
        gl['generator_fool_loss_%s_%s' % (post, dom)] = sigmoid_cross_entropy(1.0, fake_pred, gw)
      else:
        raise NotImplementedError('unsupported loss architecture: %s' % arch)   # :401
      if arch in ('wgan', 'wgan_gp'):                             # :348-379
        dl['discriminator_loss_%s_%s' % (post, dom)] = gw * (fake_pred.mean() - real_pred.mean())
        if only_real_fake:
          continue
        if cfg.wgan_drift_loss_weight:                            # :359-367
          dl['discriminator_drift_loss_%s_%s' % (post, dom)] = cfg.wgan_drift_loss_weight * (real_pred ** 2).mean()
        if arch == 'wgan_gp':                                     # :372-379, 414-439
          # interpolates between the real and the GENERATED image, alpha ~U[0,1] [B,1,1,1] an explicit input; the loss
          # sits in the discriminator collection, so only discriminator variables see its gradient
          fake_img = ends['%s_%s' % (dom, post)]
          xhat = (original + dragan_rand['alpha_' + dom] * (fake_img - original)).detach().requires_grad_(True)
          pred_hat, _ = nets.discriminator(xhat, 'discriminator_' + dom)
          grad = torch.autograd.grad(pred_hat.sum(), xhat, create_graph=True)[0]
          slopes = torch.sqrt((grad * grad).sum(dim=(1, 2, 3)))
          dl['discriminator_gradient_penalty_%s_%s' % (post, dom)] = \
              cfg.gradient_penalty_lambda * ((slopes - 1.0) ** 2).mean()
          ends['gp_grad_' + dom] = grad
      elif arch == 'hinge':                                       # :381-389
        dl['discriminator_loss_%s_%s' % (post, dom)] = gw * (torch.relu(1 + fake_pred).mean() + torch.relu(1 - real_pred).mean())
      else:                                                       # gan / dragan, :390-413
        dl['discriminator_fake_loss_%s_%s' % (post, dom)] = sigmoid_cross_entropy(0.0, fake_pred, gw)
        dl['discriminator_real_loss_%s_%s' % (post, dom)] = sigmoid_cross_entropy(1.0, real_pred, gw)
        if not only_real_fake and arch == 'dragan':
          xhat = dragan_interpolates(original.detach(), dragan_rand['alpha_' + dom], dragan_rand['noise_' + dom])
          xhat = xhat.requires_grad_(True)
          pred_hat, _ = nets.discriminator(xhat, 'discriminator_' + dom)
          grad = torch.autograd.grad(pred_hat.sum(), xhat, create_graph=True)[0]     # image_generation.py:466
          slopes = torch.sqrt((grad * grad).sum(dim=(1, 2, 3)))
          dl['discriminator_gradient_penalty_prime_' + dom] = cfg.gradient_penalty_lambda * ((slopes - 1.0) ** 2).mean()
          ends['gp_grad_' + dom] = grad
    if cfg.l_content_weight:                                      # twingan.py:485-505
      original_code = ends['enc_' + dom]
      prime_code = ends['enc_%s_prime' % opp]
      gl['l_content_' + dom] = absolute_difference(original_code, prime_code, cfg.l_content_weight)
  g_loss = sum(gl.values()) / cfg.num_clones                      # deployment/model_deploy.py:265-267
  d_loss = sum(dl.values()) / cfg.num_clones
  named = {}
  named.update(gl)
  named.update(dl)
  return g_loss, d_loss, named, ends, nets


def generator_variable_names(params):  # twingan.py:526-527
  return [k for k in params if k.startswith('encoder_content/') or k.startswith('generator/')]


def discriminator_variable_names(params):  # image_generation.py:484-485
  return [k for k in params if k.startswith('discriminator')]


def step_gradients(cfg: Config, params: Dict[str, Tensor], norm_state: Dict[str, Tensor], sources: Tensor,
                   targets: Tensor, dragan_rand: Dict[str, Tensor]):
  """Everything one reference session.run(train_tensor) computes except the variable update:
  both gradient sets (image_generation.py:599-610)."""
  leaf = {k: v.detach().clone().requires_grad_(True) for k, v in params.items()}
  g_loss, d_loss, named, ends, nets = twingan_losses(cfg, leaf, norm_state, sources, targets, dragan_rand)
  gnames = generator_variable_names(leaf)
  dnames = discriminator_variable_names(leaf)
  ggrads = torch.autograd.grad(g_loss, [leaf[k] for k in gnames], retain_graph=True, allow_unused=True)
  dgrads = torch.autograd.grad(d_loss, [leaf[k] for k in dnames], allow_unused=True)
  grads = {}
  for k, g in list(zip(gnames, ggrads)) + list(zip(dnames, dgrads)):
    grads[k] = torch.zeros_like(leaf[k]) if g is None else g.detach()
  named = {k: v.detach() for k, v in named.items()}
  ends = {k: v.detach() for k, v in ends.items()}
  return g_loss.detach(), d_loss.detach(), named, grads, ends, nets


def adam_apply(cfg: Config, param: Tensor, grad: Tensor, m: Tensor, v: Tensor, t: int):
  """tf.train.AdamOptimizer (SURVEY 8a.4-5): lr_t = lr*sqrt(1-b2^t)/(1-b1^t); p -= lr_t*m/(sqrt(v)+eps)."""
  b1, b2 = cfg.adam_beta1, cfg.adam_beta2
  m = b1 * m + (1 - b1) * grad
  v = b2 * v + (1 - b2) * grad * grad
  lr_t = cfg.learning_rate * math.sqrt(1 - b2 ** t) / (1 - b1 ** t)
  return param - lr_t * m / (torch.sqrt(v) + cfg.adam_eps), m, v


def apply_stat_updates(cfg: Config, norm_state: Dict[str, Tensor], nets: Nets) -> None:
  """EMA pushes of libs/batch_norm.py:295-319 (decay 0.99 for batch_renorm, 0.999 for batch_norm) and :359-393
  (renorm_momentum 0.99), applied sequentially in program order (the reference leaves the order of
  the 2-3 passes that share one `_s`/`_t` variable undefined; SURVEY 8a.4-7)."""
  for base, d, upd in nets.stat_updates:
    # batch_renorm passes decay=0.99 (nets/pggan_utils.py:165); plain batch_norm passes none and gets
    # conditional_batch_norm's default 0.999 (libs/batch_norm.py:44) -- pinned by tests/golden/reference_pggan_*.npz
    decay = 0.99 if 'stddev' in upd else 0.999
    if 'stddev' in upd:
      for var, wname, val in (('renorm_mean', 'renorm_mean_weight', upd['mean']),
                              ('renorm_stddev', 'renorm_stddev_weight', upd['stddev'])):
        norm_state[base + var + d] = norm_state[base + var + d] * decay + val * (1 - decay)
      new_mean_w = norm_state[base + 'renorm_mean_weight' + d] * decay + (1 - decay)
      new_std_w = norm_state[base + 'renorm_stddev_weight' + d] * decay + (1 - decay)
      new_mean = norm_state[base + 'renorm_mean' + d] / new_mean_w
      new_std = norm_state[base + 'renorm_stddev' + d] / new_std_w
      norm_state[base + 'renorm_mean_weight' + d] = new_mean_w
      norm_state[base + 'renorm_stddev_weight' + d] = new_std_w
      mm, mv = new_mean, new_std * new_std - 1e-3
    else:
      mm, mv = upd['mean'], upd['variance']
    norm_state[base + 'moving_mean' + d] = norm_state[base + 'moving_mean' + d] * decay + mm * (1 - decay)
    norm_state[base + 'moving_variance' + d] = norm_state[base + 'moving_variance' + d] * decay + mv * (1 - decay)


def train_step(cfg: Config, params, adam_m, adam_v, norm_state, sources, targets, dragan_rand, adam_t: int):
  """One 'simultaneous' step (SURVEY 8d mode B): both gradient sets on one batch, then BOTH Adam applies
  (G first: image_generation.py:640; one optimizer => shared beta powers, t advances per apply)."""
  g_loss, d_loss, named, grads, ends, nets = step_gradients(cfg, params, norm_state, sources, targets, dragan_rand)
  t = adam_t
  for names in (generator_variable_names(params), discriminator_variable_names(params)):
    t += 1
    for k in names:
      params[k], adam_m[k], adam_v[k] = adam_apply(cfg, params[k], grads[k], adam_m[k], adam_v[k], t)
  apply_stat_updates(cfg, norm_state, nets)
  return g_loss, d_loss, named, grads, t


def inference(cfg: Config, params, norm_state, sources: Tensor) -> Tensor:
  """inference/image_translation_infer.py:46-99 compute: G(E(x;'_s',eval);'_t',eval, skips) (twingan.py:310-365)."""
  nets = Nets(cfg, params, norm_state)
  code, ep = nets.encoder(sources, '_s', is_training=False)
  out, _ = nets.generator(code, '_t', ep if cfg.use_unet else None, is_training=False)
  return out


def make_inputs(cfg: Config, batch: int, seed: int = 0, dtype=torch.float64, kind: str = 'uniform'):
  """Synthetic paired-domain batch + DRAGAN randomness.  kind='truncnorm' follows
  model/model_inheritor.py:785-799 (truncated normal sigma 0.1, resample outside 2 sigma)."""
  g = torch.Generator().manual_seed(seed)
  shape = (batch, cfg.hw, cfg.hw, 3)

  def img():
    if kind == 'uniform':
      return torch.rand(shape, generator=g, dtype=torch.float64).to(dtype)
    x = torch.randn(shape, generator=g, dtype=torch.float64)
    bad = x.abs() > 2
    while bad.any():
      x = torch.where(bad, torch.randn(shape, generator=g, dtype=torch.float64), x)
      bad = x.abs() > 2
    return (0.1 * x).to(dtype)

  sources, targets = img(), img()
  rand = {}
  for d in ('s', 't'):
    rand['alpha_' + d] = torch.rand((batch, 1, 1, 1), generator=g, dtype=torch.float64).to(dtype)
    rand['noise_' + d] = (torch.rand(shape, generator=g, dtype=torch.float64) * 2 - 1).to(dtype)
  return sources, targets, rand
