"""Operator layer: thin torch.autograd.Function wrappers over the C-ABI kernels of libtwg.so.

This mirrors the reference's *operator plug-in* level (SURVEY 8b-2): `tf.contrib.layers.conv2d`
(nets/pggan_utils.py:316-320), the arg-scope `normalizer_fn`/`activation_fn` hooks
(nets/pggan_utils.py:86-98 -> libs/batch_norm.py:41, libs/instance_norm.py:31, util_misc.py:68),
`_pixel_norm` (:330), `minibatch_state_concat` (:353), `resize_twice_as_big` (:349), `tf.nn.avg_pool`,
`tf.losses.*` and `tf.gradients`.  PyTorch is used for device memory, streams and the autograd tape
only: every tensor-sized computation is a kernel of this repository.  Discriminator-side operators are
twice differentiable (their backward is itself built from Functions) because the DRAGAN penalty
(image_generation.py:451-476) differentiates d D(x)/dx again.

All activations are NHWC fp32 contiguous CUDA tensors; weights are HWIO.
"""
from __future__ import annotations

import contextlib
import math
import weakref
from typing import Optional, Sequence, Tuple

import torch
from torch.autograd import Function

from ._lib import lib, TwgError

FLAG_LRELU = 1
FLAG_PIXNORM = 2
NORM_NONE, NORM_INSTANCE, NORM_BATCH, NORM_RENORM = 0, 1, 2, 3

# 1 = wgmma tensor-core convs where the library covers the shape, 0 = exact fp32 CUDA cores everywhere
_PREC = 1
_SKIP_PARAM_GRADS = set()   # parameter groups whose wgrad / bias-grad is not wanted in the running backward


def set_precision(prec: int) -> None:
  global _PREC
  _PREC = int(prec)


def get_precision() -> int:
  return _PREC


@contextlib.contextmanager
def skip_param_grads(*groups: str):
  """Inside this context, backward passes do not compute parameter gradients of `groups`
  (the reference gets the same effect from `var_list` in optimizer.compute_gradients,
  deployment/model_deploy.py:285-315)."""
  added = [g for g in groups if g not in _SKIP_PARAM_GRADS]
  _SKIP_PARAM_GRADS.update(added)
  try:
    yield
  finally:
    for g in added:
      _SKIP_PARAM_GRADS.discard(g)


def _check(t: torch.Tensor) -> torch.Tensor:
  if not t.is_cuda:
    raise TwgError('twingan_b200 ops need CUDA tensors (no CPU fallback)')
  if t.dtype != torch.float32:
    raise TwgError('twingan_b200 ops are fp32 (got %s)' % t.dtype)
  return t if t.is_contiguous() else t.contiguous()


def _p(t: Optional[torch.Tensor]):
  return None if t is None else t.data_ptr()


def _st():
  return torch.cuda.current_stream().cuda_stream


_DOMAIN_STREAMS = {}   # device index -> the stream the second discriminator domain runs on


def domain_stream(device) -> torch.cuda.Stream:
  """The stream of the training step's second discriminator domain on `device`: one per device for the process, bound to a
  partial-sum region of its own in the library, so that its reductions never share scratch with the other domain's."""
  idx = torch.device(device).index
  idx = torch.cuda.current_device() if idx is None else idx
  st = _DOMAIN_STREAMS.get(idx)
  if st is None:
    st = torch.cuda.Stream(device=idx)
    with torch.cuda.device(idx):        # the library keys the binding on the current device
      if lib().try_call('twg_partials_bind', st.cuda_stream, 1) != 0:     # binds, launches nothing
        raise TwgError('twg_partials_bind: ' + lib().last_error())
    _DOMAIN_STREAMS[idx] = st
  return st


# ------------------------------------------------------------------------------------------------
# convolution (bilinear => closed under differentiation)
# ------------------------------------------------------------------------------------------------

# test hook: when a dict {'lrelu': [], 'l1': []}, forward passes append the active set (sign masks) of every
# leaky-ReLU / L1 call in program order so the parity harness can evaluate the oracle on the same side of
# each kink (tests/parity.py).  Never set in production.
ACTIVE_SET_TRACE = None
TRACE_TAG = None      # which (batched) network pass is being recorded; entries are (tag, tensor)


@contextlib.contextmanager
def trace_tag(tag):
  global TRACE_TAG
  prev, TRACE_TAG = TRACE_TAG, tag
  try:
    yield
  finally:
    TRACE_TAG = prev


def _trace(kind: str, t: torch.Tensor) -> None:
  ACTIVE_SET_TRACE[kind].append((TRACE_TAG, t.cpu()))


_CONV_TIMING = None   # list of (family, flops, bytes, start event, end event) while bench.py's roofline pass runs


def enable_conv_timing(on: bool) -> None:
  global _CONV_TIMING
  _CONV_TIMING = [] if on else None


def collect_conv_timing():
  """{family: {'launches', 'ms', 'flops', 'bytes', 'tflops', 'algorithmic_gbs'}} -- CUDA-event time of every conv launch
  since enable, by kernel family ('tc_fwd', 'tc_wgrad', 'tc_ws', 'fp32_cuda_core')."""
  out = {}
  for fam, fl, nb, e0, e1 in (_CONV_TIMING or []):
    d = out.setdefault(fam, {'launches': 0, 'ms': 0.0, 'flops': 0.0, 'bytes': 0.0})
    d['launches'] += 1
    d['ms'] += e0.elapsed_time(e1)
    d['flops'] += fl
    d['bytes'] += nb
  for d in out.values():
    d['ms'] = round(d['ms'], 4)
    d['tflops'] = round(d['flops'] / max(d['ms'], 1e-9) / 1e9, 3)
    d['algorithmic_gbs'] = round(d['bytes'] / max(d['ms'], 1e-9) / 1e6, 1)
  return out


def conv_fwd_raw(x, w, k, pad):
  """y = conv2d(x, w) outside autograd: the tensor-core kernel where tc_eligible(), else the exact-fp32 one."""
  return _conv_fwd(_check(x), _check(w), k, pad)[0]


def conv_dgrad_raw(gy, w, x_shape, k, pad):
  return _conv_dgrad(_check(gy), _check(w), tuple(x_shape), k, pad)[0]


def conv_wgrad_raw(x, gy, k, pad):
  return _conv_wgrad(_check(x), _check(gy), k, pad)


# ---- split-bf16 planes: split an activation ONCE (forward + wgrad), a gradient ONCE (dgrad + wgrad) and a
# ---- registered weight once per optimiser step ----------------------------------------------------------------

_WEIGHT_TABLES = {}      # data_ptr of a registered conv weight -> weak reference to its WeightPlaneTable
_LIVE_TABLES = weakref.WeakSet()


class WeightPlaneTable:
  """Split-bf16 planes (forward and dgrad layout) of EVERY tensor-core-eligible conv weight of a VariableStore, rebuilt by
  ONE kernel launch after the variables change (Adam apply, load, init) instead of one k_split_weights per weight and
  layout inside every step."""

  def __init__(self, store):
    import struct
    self.flat = store.flat
    self.index = {}
    rows, off, self.max_elems = [], 0, 1
    for name, t in store.vars.items():
      if not name.endswith('/weights') or t.dim() != 4:
        continue
      k, _, cin, cout = (int(v) for v in t.shape)
      if conv_path(1, 1, 1, cin, cout, k, (k - 1) // 2) != CONV_TC:    # (the path does not depend on N, H, W)
        continue
      n = k * k * cin * cout
      for dgrad in (0, 1):
        rows.append(struct.pack('<qqiiii', store.offsets[name][0], off, k * k, cin, cout, dgrad))
        self.index[(t.data_ptr(), bool(dgrad))] = (off, n)
        off += 2 * n
      self.max_elems = max(self.max_elems, n)
    self.rows = len(rows)
    dev = store.flat.device
    self.planes = torch.empty(max(off, 8), device=dev, dtype=torch.bfloat16)
    self.table = torch.frombuffer(bytearray(b''.join(rows) or bytes(32)), dtype=torch.uint8).to(dev)
    self.dirty = True
    for (ptr, _dg) in self.index:
      _WEIGHT_TABLES[ptr] = weakref.ref(self)
    _LIVE_TABLES.add(self)

  def refresh(self) -> None:
    if self.rows:
      lib().call('twg_split_weights_table', _p(self.flat), _p(self.planes), _p(self.table), self.rows, self.max_elems, _st())
    self.dirty = False

  def get(self, ptr: int, dgrad: bool) -> torch.Tensor:
    if self.dirty:
      self.refresh()
    off, n = self.index[(ptr, bool(dgrad))]
    return self.planes[off:off + 2 * n].view(2, n)


def invalidate_weight_cache() -> None:
  """Must be called whenever registered variables change outside the optimiser apply (load_dict, init, tests poking the
  flat buffer): the planes are rebuilt lazily by the next conv that needs them."""
  for t in list(_LIVE_TABLES):
    t.dirty = True


CONV_SIMT, CONV_PW, CONV_TC = 0, 1, 2     # kernel families of twg_conv_path
_CONV_PATHS = {}


def conv_path(N, H, W, Cin, Cout, k, pad) -> int:
  """Which kernel family the library has for this conv shape: CONV_SIMT, CONV_PW (exact fp32) or CONV_TC (tensor cores)."""
  key = (N, H, W, Cin, Cout, k, pad)
  v = _CONV_PATHS.get(key)
  if v is None:
    v = _CONV_PATHS[key] = int(lib().cdll.twg_conv_path(N, H, W, Cin, Cout, k, pad))
  return v


def tc_eligible(N, H, W, Cin, Cout, k, pad) -> bool:
  return _PREC == 1 and conv_path(N, H, W, Cin, Cout, k, pad) == CONV_TC


def _epilogue_slots(N, H, W, Cin, Cout, k, pad) -> int:
  """Statistics records per image of the forward conv's fused epilogue; 0: this conv has no fused epilogue (no statistics,
  sign mask or evaluation-mode affine)."""
  if not tc_eligible(N, H, W, Cin, Cout, k, pad):
    return 0
  return int(lib().cdll.twg_conv_epilogue_slots(N, H, W, Cin, Cout, k, pad))


def split_act(x: torch.Tensor) -> torch.Tensor:
  """fp32 [N,H,W,C] -> bf16 planes [2,N,H,W,C] (hi, lo) with x = hi + lo to ~2^-17 relative."""
  x = _check(x)
  planes = torch.empty((2,) + tuple(x.shape), device=x.device, dtype=torch.bfloat16)
  lib().call('twg_split_act', _p(x), _p(planes), x.numel(), _st())
  return planes


# Producer kernels (normaliser/activation, pooling, UNet join) can write their result directly as split-bf16 planes
# for the tensor-core conv that consumes it.  The planes travel beside the autograd tensor in this side table keyed by
# the tensor OBJECT (validated through a weak reference); a "planes-only" tensor has the right shape/dtype for autograd
# but its fp32 payload is never written -- it may only feed tensor-core convs (the emitter checks eligibility).
_PLANES = {}


def _put_planes(t: torch.Tensor, planes: torch.Tensor) -> None:
  _PLANES[id(t)] = (weakref.ref(t), planes)


def _take_planes(t: torch.Tensor):
  e = _PLANES.pop(id(t), None)
  if e is None or e[0]() is not t:
    return None
  return e[1]


# sign masks of discriminator activations (ConvBiasActFn): z (by object) -> uint8 mask, for the stand-alone activation
# backward of the twice-differentiable path (LreluBwdFn)
_MASKS = {}


def _mask_of(t: torch.Tensor):
  e = _MASKS.get(id(t))
  return e[1] if (e is not None and e[0]() is t) else None


def begin_step() -> None:
  _PLANES.clear()
  _MASKS.clear()


def planes_of(t: torch.Tensor) -> torch.Tensor:
  """The split planes of `t`: taken from the producer if it emitted them, else computed now."""
  p = _take_planes(t)
  return p if p is not None else split_act(t)


def _new_planes(shape, device) -> torch.Tensor:
  return torch.empty((2,) + tuple(shape), device=device, dtype=torch.bfloat16)


def weight_planes(w: torch.Tensor, dgrad: bool) -> torch.Tensor:
  w = _check(w)
  ref = _WEIGHT_TABLES.get(w.data_ptr())
  table = ref() if ref is not None else None
  if table is not None and (w.data_ptr(), bool(dgrad)) in table.index and table.flat.device == w.device:
    return table.get(w.data_ptr(), dgrad)
  k, _, Cin, Cout = w.shape
  planes = torch.empty((2, k * k * Cin * Cout), device=w.device, dtype=torch.bfloat16)
  lib().call('twg_split_weights', _p(w), _p(planes), k, Cin, Cout, int(dgrad), _st())
  return planes


EPILOGUE_STATS = True    # A/B switch: instance-norm statistics from the conv epilogue instead of a twg_moments pass
ACT_SIGN_MASK = True     # A/B switch: discriminator conv epilogues write z's sign mask; the activation backward reads it, not z


# ---- conv dispatch: every conv launch goes through _conv_fwd / _conv_dgrad / _conv_wgrad.  Each takes its activation
# ---- operands as fp32 and / or split planes, runs the tensor-core kernel on planes when tc_eligible() and the exact-fp32
# ---- kernel on fp32 otherwise, and records the launch while conv timing is on.

def _nhwc(t, planes):
  return tuple(int(d) for d in (t.shape if t is not None else planes.shape[1:]))


def _conv_launch(fam, shape, name, *args):
  """lib().call(name, *args) for a conv of `shape` = (N, H, W, Cin, Cout, k, pad), timed under `fam` while conv timing is
  on.  The tensor-core families also count the bytes of their fp32-sized input and output."""
  if _CONV_TIMING is None:
    lib().call(name, *args)
    return
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  lib().call(name, *args)
  e1.record()
  N, H, W, Cin, Cout, k, pad = shape
  Ho, Wo = H + 2 * pad - k + 1, W + 2 * pad - k + 1
  nbytes = 4.0 * N * H * W * (Cin + Cout) if fam in ('tc_fwd', 'tc_wgrad') else 0.0
  _CONV_TIMING.append((fam, 2.0 * N * Ho * Wo * Cin * Cout * k * k, nbytes, e0, e1))


def _exact_family(shape) -> str:
  # bench.py reports the pointwise fromRGB / toRGB kernels apart from the SIMT ones at precision 1 only
  return 'tc_ws' if (_PREC == 1 and conv_path(*shape) == CONV_PW) else 'fp32_cuda_core'


def _conv_fwd(x, w, k, pad, xp=None, bias=None, act=False, zp=None, mask=None, stats=None):
  """y = lrelu?(conv2d(x, w) + bias), x given as fp32 and / or its planes `xp` (taken from the producer or split here when
  missing).  The epilogue outputs -- y's planes `zp`, its sign `mask`, instance-norm `stats` (N x _epilogue_slots x Cout
  float4) -- need the tensor-core path.  Returns (y, x's planes on the tensor-core path, else None)."""
  N, H, W_, Cin = _nhwc(x, xp)
  Cout = int(w.shape[3])
  shape = (N, H, W_, Cin, Cout, k, pad)
  y = torch.empty((N, H + 2 * pad - k + 1, W_ + 2 * pad - k + 1, Cout), device=w.device, dtype=torch.float32)
  if not tc_eligible(*shape):
    if bias is not None or zp is not None or mask is not None or stats is not None:
      raise TwgError('fused conv epilogues need the tensor-core path')
    _conv_launch(_exact_family(shape), shape, 'twg_conv_fwd', _p(_check(x)), _p(_check(w)), _p(y), N, H, W_, Cin, Cout, k,
                 pad, _st())
    return y, None
  xp = xp if xp is not None else planes_of(x)
  _conv_launch('tc_fwd', shape, 'twg_conv_fwd_planes', _p(xp), _p(weight_planes(w, False)), _p(bias), int(act), _p(y),
               _p(zp), _p(mask), _p(stats), N, H, W_, Cin, Cout, k, pad, _st())
  return y, xp


def _conv_dgrad(gy, w, x_shape, k, pad, gp=None):
  """gx = conv2d_backprop_input(gy, w), gy given as fp32 and / or its planes `gp`.  Returns (gx, gy's planes on the
  tensor-core path, else None)."""
  N, H, W_, Cin = x_shape
  Cout = int(w.shape[3])
  shape = (N, H, W_, Cin, Cout, k, pad)
  gx = torch.empty(x_shape, device=w.device, dtype=torch.float32)
  if not tc_eligible(*shape):
    _conv_launch(_exact_family(shape), shape, 'twg_conv_dgrad', _p(_check(gy)), _p(_check(w)), _p(gx), N, H, W_, Cin, Cout,
                 k, pad, _st())
    return gx, None
  gp = gp if gp is not None else split_act(gy)
  _conv_launch('tc_fwd', shape, 'twg_conv_dgrad_planes', _p(gp), _p(weight_planes(w, True)), _p(gx), N, H, W_, Cin, Cout, k,
               pad, _st())
  return gx, gp


def _conv_wgrad(x, gy, k, pad, xp=None, gp=None, out=None):
  """gw = conv2d_backprop_filter(x, gy), each operand given as fp32 and / or planes.  `out`: add (+=) into this fp32
  buffer of k*k*Cin*Cout elements (a gradient sink) instead of returning a new tensor."""
  N, H, W_, Cin = _nhwc(x, xp)
  Cout = _nhwc(gy, gp)[3]
  shape = (N, H, W_, Cin, Cout, k, pad)
  acc = 1 if out is not None else 0
  gw = out if out is not None else torch.empty((k, k, Cin, Cout), device=(x if x is not None else xp).device,
                                               dtype=torch.float32)
  if not tc_eligible(*shape):
    _conv_launch(_exact_family(shape), shape, 'twg_conv_wgrad', _p(_check(x)), _p(_check(gy)), _p(gw), N, H, W_, Cin, Cout,
                 k, pad, acc, _st())
    return gw
  xp = xp if xp is not None else split_act(x)
  gp = gp if gp is not None else split_act(gy)
  _conv_launch('tc_wgrad', shape, 'twg_conv_wgrad_planes', _p(xp), _p(gp), _p(gw), N, H, W_, Cin, Cout, k, pad, acc, _st())
  return gw


# ---- gradient sinks: weight gradients accumulate straight into the flat gradient buffer (each use of a shared variable
# ---- adds its gradient there with accumulate=1, after the kernel has summed its own partials in a fixed order) instead
# ---- of autograd summing per-use tensors and a later packing
_GRAD_SINKS = {}     # weight data_ptr -> fp32 view of the flat gradient buffer


def register_grad_sinks(mapping) -> None:
  _GRAD_SINKS.clear()
  _GRAD_SINKS.update({int(k): v for k, v in mapping.items()})


# Autograd runs the ready nodes of a backward in an order it takes from per-thread node sequence numbers.  The nodes of a
# double backward (the DRAGAN / WGAN-GP input gradient, built with create_graph=True) are created on autograd's CUDA
# worker thread, the forward's on the main thread, and the two counters advance independently, so where both reach the
# same weight -- a residual block's diamond under --use_res_block -- the order in which their weight gradients are added
# into the sink depends on how many nodes the process created before.  Inside fixed_order_weight_grads(group) the conv
# weight gradients of `group` are recorded instead, and flush_weight_grads() adds them into their sinks in the order
# their conv nodes were created, which is the program's order and does not depend on that history.
_CONV_SERIAL = [0]          # creation counter of the conv nodes (forward order; the first-order backward's are in order)
_DEFER_GROUPS = set()
_DEFERRED = []              # (serial, operands of _conv_wgrad, sink, the stream the conv node's backward ran on)


def _next_serial() -> int:
  _CONV_SERIAL[0] += 1
  return _CONV_SERIAL[0]


@contextlib.contextmanager
def fixed_order_weight_grads(group: Optional[str]):
  """Record the conv weight gradients of `group` (None: none) in the running backward for flush_weight_grads()."""
  added = group is not None and group not in _DEFER_GROUPS
  if added:
    _DEFER_GROUPS.add(group)
  try:
    yield
  finally:
    if added:
      _DEFER_GROUPS.discard(group)


def flush_weight_grads() -> None:
  """Add the recorded weight gradients into their sinks, in the creation order of their conv nodes, each on the stream its
  node ran on (a discriminator domain's stream keeps that domain's adds in order after the operands it made)."""
  for _, (x, gy, k, pad, xp, gp), sink, stream in sorted(_DEFERRED, key=lambda e: e[0]):
    with torch.cuda.stream(stream):
      _conv_wgrad(x, gy, k, pad, xp, gp, out=sink)
  _DEFERRED.clear()


def drop_weight_grads() -> None:
  _DEFERRED.clear()


def _weight_grad(ctx, w, x, gy, xp=None, gp=None):
  """The weight gradient of the conv node `ctx` (inputs [x-like, w, ...]) from its operands: added into w's gradient sink
  when one is registered (or recorded for flush_weight_grads), else returned for autograd; None when not wanted or sunk."""
  if not (ctx.needs_input_grad[1] and ctx.group not in _SKIP_PARAM_GRADS):
    return None
  sink = _sink(w)
  if sink is not None:
    if ctx.group in _DEFER_GROUPS:
      _DEFERRED.append((ctx.serial, (x, gy, ctx.k, ctx.pad, xp, gp), sink, torch.cuda.current_stream()))
    else:
      _conv_wgrad(x, gy, ctx.k, ctx.pad, xp, gp, out=sink)
    return None
  return ConvWgradFn.apply(x, gy, ctx.k, ctx.pad, ctx.group, xp, gp)


class ConvFn(Function):
  """y = conv2d(x, w), stride 1 (tf.contrib.layers.conv2d without bias/normalizer/activation).
  On the tensor-core path the input is split once; the planes (not x) are kept for the weight gradient."""

  @staticmethod
  def forward(ctx, x, w, k, pad, group):
    ctx.k, ctx.pad, ctx.group, ctx.xshape = k, pad, group, tuple(x.shape)
    ctx.serial = _next_serial()
    y, xp = _conv_fwd(x, w, k, pad)
    ctx.save_for_backward(x if xp is None else None, xp, w)
    return y

  @staticmethod
  def backward(ctx, gy):
    x, xp, w = ctx.saved_tensors     # x on the exact path, its planes on the tensor-core path
    gp = planes_of(gy) if xp is not None else None
    gx = ConvDgradFn.apply(gy, w, ctx.xshape, ctx.k, ctx.pad, ctx.group, gp) if ctx.needs_input_grad[0] else None
    return gx, _weight_grad(ctx, w, x, gy, xp, gp), None, None, None


class ConvDgradFn(Function):
  """gx = conv2d_backprop_input(gy, w).  `gy_planes` (optional) = the already split gy."""

  @staticmethod
  def forward(ctx, gy, w, x_shape, k, pad, group, gy_planes=None):
    ctx.k, ctx.pad, ctx.group = k, pad, group
    ctx.serial = _next_serial()
    gx, gp = _conv_dgrad(gy, w, tuple(x_shape), k, pad, gy_planes)
    ctx.save_for_backward(gy if gp is None else None, gp, w)
    return gx

  @staticmethod
  def backward(ctx, ggx):
    gy, gp, w = ctx.saved_tensors    # gy on the exact path, its planes on the tensor-core path
    ggx_planes = None
    if gp is not None:
      # ggx feeds a conv (d_gy) and a weight gradient: split it ONCE and hand the planes to both
      ggx_planes = planes_of(ggx)
      _put_planes(ggx, ggx_planes)
    d_gy = ConvFn.apply(ggx, w, ctx.k, ctx.pad, ctx.group) if ctx.needs_input_grad[0] else None
    _take_planes(ggx)
    return d_gy, _weight_grad(ctx, w, ggx, gy, ggx_planes, gp), None, None, None, None, None


class ConvWgradFn(Function):
  """gw = conv2d_backprop_filter(x, gy).  Either operand may be given as fp32 (x / gy) and / or as split planes."""

  @staticmethod
  def forward(ctx, x, gy, k, pad, group, x_planes=None, gy_planes=None):
    ctx.k, ctx.pad, ctx.group, ctx.xshape = k, pad, group, _nhwc(x, x_planes)
    ctx.save_for_backward(x, gy)
    return _conv_wgrad(x, gy, k, pad, x_planes, gy_planes)

  @staticmethod
  def backward(ctx, ggw):
    # third-order term: never needed by the TwinGAN step (the penalty is differentiated once more, not twice)
    x, gy = ctx.saved_tensors
    if x is None or gy is None:
      raise TwgError('ConvWgradFn backward needs fp32 operands (no third-order path in the step)')
    d_x = d_gy = None
    if ctx.needs_input_grad[0]:
      d_x = ConvDgradFn.apply(gy, ggw, ctx.xshape, ctx.k, ctx.pad, ctx.group, None)
    if ctx.needs_input_grad[1]:
      d_gy = ConvFn.apply(x, ggw, ctx.k, ctx.pad, ctx.group)
    return d_x, d_gy, None, None, None, None, None


class ConvBiasActFn(Function):
  """z = lrelu?(conv2d(x, w) + bias): one discriminator layer (pggan_discriminator_arg_scope) with bias and
  activation fused into the tensor-core conv epilogue.  Twice differentiable like ConvFn + BiasActFn.

  `pool`: None, or 'fp32' / 'planes' -- also return avg_pool2(z); the first-order backward then reads the pooled
  tensor's gradient at half resolution inside the activation-backward kernel (no full-resolution pool gradient)."""

  @staticmethod
  def forward(ctx, x, w, bias, k, pad, act, group, emit_planes=False, pool=None):
    N, H, W_, Cin = x.shape
    Cout = w.shape[3]
    ctx.set_materialize_grads(False)
    ctx.k, ctx.pad, ctx.group, ctx.act = k, pad, group, act
    ctx.xshape = tuple(x.shape)
    ctx.serial = _next_serial()
    zp = _new_planes((N, H, W_, Cout), x.device) if emit_planes else None
    mask = None
    if act and ACT_SIGN_MASK and _epilogue_slots(N, H, W_, Cin, Cout, k, pad):
      # the epilogue also writes the sign bits of z (one byte per 4 channels): all the first-order backward needs of z
      mask = torch.empty(N * H * W_ * Cout // 4, device=x.device, dtype=torch.uint8)
    z, xp = _conv_fwd(x, w, k, pad, bias=_check(bias), act=act, zp=zp, mask=mask)
    ctx.mask = mask
    if mask is not None:
      _MASKS[id(z)] = (weakref.ref(z), mask)
    if zp is not None:
      _put_planes(z, zp)
    if ACTIVE_SET_TRACE is not None and act:
      _trace('lrelu', z > 0)
    ctx.save_for_backward(xp, w, z, bias)
    if pool is None:
      return z
    pooled = torch.empty((N, H // 2, W_ // 2, Cout), device=x.device, dtype=torch.float32)
    pp = _new_planes(pooled.shape, x.device) if pool == 'planes' else None
    lib().call('twg_pool2', _p(z), _p(pooled), _p(pp), N, H, W_, Cout, 0.25, _st())
    if pp is not None:
      _put_planes(pooled, pp)
    return z, pooled

  @staticmethod
  def backward(ctx, gz, gpool=None):
    xp, w, z, bias = ctx.saved_tensors
    if gz is None and gpool is None:
      return (None,) * 9
    want_p = ctx.group not in _SKIP_PARAM_GRADS
    gb = None
    pooled_only = gz is None
    if torch.is_grad_enabled() or not pooled_only:
      # differentiable composition (DRAGAN's double backward), or a layer output with a second consumer
      if gpool is not None:
        up = Upsample2Fn.apply(gpool, 0.25)
        gz = up if gz is None else gz + up
    if not torch.is_grad_enabled():
      # first-order backward: ONE pass over the incoming gradient produces the bias gradient and gy directly as split
      # planes (gy is consumed by dgrad and wgrad only, so its fp32 form is never materialised).  Also used when the
      # discriminator's parameter gradients are skipped (generator-loss backward): the column sums are discarded.
      src = _check(gpool if pooled_only else gz)
      C = z.shape[-1]
      gy = None
      gp = _new_planes(z.shape, z.device)
      bsink = _sink(bias) if (want_p and ctx.needs_input_grad[2]) else None
      gb = bsink if bsink is not None else torch.empty(C, device=z.device, dtype=torch.float32)
      H, W_ = int(z.shape[1]), int(z.shape[2])
      lib().call('twg_lrelu_bwd_colsum', _p(src), _p(z), _p(ctx.mask), None, _p(gp), _p(gb), z.numel() // C, C,
                 int(ctx.act), H if pooled_only else 0, W_ if pooled_only else 0, 1 if bsink is not None else 0, _st())
      if bsink is not None or not (want_p and ctx.needs_input_grad[2]):
        gb = None
    else:
      gy = LreluBwdFn.apply(gz, z, True, ctx.mask) if ctx.act else gz
      if want_p and ctx.needs_input_grad[2]:
        gb = ColsumFn.apply(gy)
      gp = planes_of(gy)           # written by LreluBwdFn's own pass when it ran
    gx = ConvDgradFn.apply(gy, w, ctx.xshape, ctx.k, ctx.pad, ctx.group, gp) if ctx.needs_input_grad[0] else None
    return gx, _weight_grad(ctx, w, None, gy, xp, gp), gb, None, None, None, None, None, None


def vec_ok(C: int) -> bool:
  """Channel counts the vectorised elementwise kernels cover (mirrors vec_geom in csrc/twg_common.cuh)."""
  if C % 4:
    return False
  q = C // 4
  return (q & (q - 1)) == 0 if q <= 32 else (q % 32 == 0 and q // 32 in (2, 4))


def conv_bias_act(x, w, bias, pad, act=True, group='D', emit_planes=False, pool=None):
  """Discriminator conv layer; uses the fused tensor-core epilogue when the shape is covered.  With `pool` ('fp32' or
  'planes') returns (z, avg_pool2(z))."""
  k = int(w.shape[0])
  N, H, W_, Cin = x.shape
  Cout = int(w.shape[3])
  # Below 16384 output pixels the layer runs as conv + a separate bias / activation pass, which is then over a small
  # tensor.  The bound dates from kernels that split K on those layers; it stays because moving it changes which kernels
  # run, and its effect on the step time has not been measured since.
  if tc_eligible(N, H, W_, Cin, Cout, k, int(pad)) and N * H * W_ >= 16384:
    if pool is not None and vec_ok(Cout) and H % 2 == 0 and W_ % 2 == 0:
      return ConvBiasActFn.apply(x, w, bias, k, int(pad), bool(act), group, bool(emit_planes), pool)
    z = ConvBiasActFn.apply(x, w, bias, k, int(pad), bool(act), group, bool(emit_planes))
  else:
    z = bias_act(conv2d(x, w, pad, group), bias, act, group, emit_planes)
  if pool is None:
    return z
  return z, avg_pool2(z, emit_planes=(pool == 'planes'))


def conv2d(x, w, pad, group='G'):
  k = int(w.shape[0])
  if int(pad) == 0 and k > 1 and int(x.shape[1]) == k and int(x.shape[2]) == k and x.is_contiguous():
    # A VALID k x k conv over a k x k input (the discriminator's 4x4 head, nets/pggan.py:330) IS a 1x1 conv over the
    # flattened input: HWIO weights [k,k,Cin,Cout] are [(h,w,ci), co] in memory.  As a k x k conv its input gradient
    # went through the generic padded form, which multiplies 15 zero taps out of 16 per output pixel.
    N = int(x.shape[0])
    return ConvFn.apply(x.view(N, 1, 1, k * k * int(x.shape[3])), w.view(1, 1, k * k * int(w.shape[2]), int(w.shape[3])), 1, 0,
                        group)
  return ConvFn.apply(x, w, k, int(pad), group)


# ------------------------------------------------------------------------------------------------
# normaliser + leaky-ReLU + pixel-norm (generator / encoder arg scope); first-order
# ------------------------------------------------------------------------------------------------

_REQUIRE_SINKS = False


def require_sinks(on: bool) -> None:
  """While on, a parameter gradient that has no registered sink is an error instead of being handed back to autograd
  (GanModel.compute_gradients asks autograd for no parameter gradient at all)."""
  global _REQUIRE_SINKS
  _REQUIRE_SINKS = bool(on)


def _sink(t: Optional[torch.Tensor]):
  if t is None:
    return None
  s = _GRAD_SINKS.get(t.data_ptr())
  if s is None:
    padded = _PADDED_SINKS.get(t.data_ptr())
    if padded is not None:
      return padded[1]
  if s is None and _REQUIRE_SINKS:
    raise TwgError('no gradient sink registered for a parameter of shape %s' % (tuple(t.shape),))
  return s


def _norm_forward(L, y, gamma0, beta0, gamma1, beta1, kind, eps, clip_dev, snap0, snap1, stats_out, gs, dom_mask,
                  epi_stats=None, epi_slots=0):
  """moments -> finalize for y [N,H,W,C]; returns (buf [4,N,C] = a, b, mean, rstd ; rd [groups,2,C] | None).
  `epi_stats`: the conv epilogue's statistics records (instance norm): no pass over y at all."""
  N, H, W_, C = y.shape
  HW = H * W_
  dev = y.device
  buf = torch.empty((4, N, C), device=dev, dtype=torch.float32)
  if epi_stats is not None and kind == NORM_INSTANCE:
    L.call('twg_norm_finalize_partials', _p(epi_stats), int(epi_slots), _p(gamma0), _p(beta0), _p(gamma1), _p(beta1),
           int(dom_mask), gs, float(eps), _p(buf[0]), _p(buf[1]), _p(buf[2]), _p(buf[3]), N, C, _st())
    return buf, None
  sums = None
  if kind != NORM_NONE:
    sums = torch.empty((N, C, 2), device=dev, dtype=torch.float32)
    L.call('twg_moments', _p(y), _p(sums), N, HW, C, 1 if kind == NORM_INSTANCE else gs, _st())
  rd = torch.empty((N // gs, 2, C), device=dev, dtype=torch.float32) if kind == NORM_RENORM else None
  rn0 = rn1 = None
  if kind == NORM_RENORM:
    rn0 = snap0.data_ptr() + 2 * C * 4
    rn1 = snap1.data_ptr() + 2 * C * 4 if snap1 is not None else None
  L.call('twg_norm_finalize', _p(sums), _p(y), _p(gamma0), _p(beta0), _p(gamma1), _p(beta1), int(dom_mask), gs, rn0, rn1, kind,
         float(eps), _p(clip_dev), _p(buf[0]), _p(buf[1]), _p(buf[2]), _p(buf[3]), _p(rd), _p(stats_out), N, HW, C, _st())
  return buf, rd


def _norm_param_grads(C, dev, want_p, gamma0, beta0, gamma1, beta1):
  """Where the normaliser's parameter gradients go: straight into the flat gradient buffer (+=) when every parameter of
  the layer has a registered sink, else into fresh tensors handed back to autograd.  Returns (pointers [gg0, gb0, gg1,
  gb1], accumulate, tensors to return [gg0, gb0, gg1, gb1])."""
  params = (gamma0, beta0, gamma1, beta1)
  if not want_p:
    return [None] * 4, 0, [None] * 4
  sinks = [_sink(t) for t in params]
  if all(s is not None for s, t in zip(sinks, params) if t is not None):
    return [(_p(s) if t is not None else None) for s, t in zip(sinks, params)], 1, [None] * 4
  fresh = [torch.empty(C, device=dev, dtype=torch.float32) if t is not None else None for t in params]
  return [_p(t) for t in fresh], 0, fresh


class NormActFn(Function):
  """z = pixel_norm?(lrelu?(normalizer(y))) in training mode (single domain; the fused layer op is GenLayerFn).

  `state_snapshot`: flat fp32 view [4C+2] = {moving_mean, moving_var, renorm_mean, renorm_stddev,
  renorm_mean_weight, renorm_stddev_weight} holding PRE-update values (libs/batch_norm.py:341-344);
  `batch_stats_out` [2,C] receives the batch moments for the EMA push; `clip`: device tensor {rmin, rmax, dmax}."""

  @staticmethod
  def forward(ctx, y, gamma, beta, kind, flags, eps, clip, state_snapshot, batch_stats_out, group):
    y = _check(y)
    N, H, W_, C = y.shape
    L = lib()
    if clip is not None and not isinstance(clip, torch.Tensor):
      clip = torch.tensor([float(v) for v in clip], device=y.device, dtype=torch.float32)
    buf, rd = _norm_forward(L, y, gamma, beta, None, None, kind, eps, clip, state_snapshot, None, batch_stats_out, N, 0)
    z = torch.empty_like(y)
    L.call('twg_norm_act_fwd', _p(y), _p(buf[0]), _p(buf[1]), _p(z), None, N, H * W_, C, flags, _st())
    if ACTIVE_SET_TRACE is not None and (flags & FLAG_LRELU):
      _trace('lrelu', z > 0)
    ctx.save_for_backward(y, buf, rd)
    ctx.kind, ctx.flags, ctx.group = kind, flags, group
    ctx.has_gamma = gamma is not None
    return z

  @staticmethod
  def backward(ctx, gz):
    y, buf, rd = ctx.saved_tensors
    gz = _check(gz)
    N, H, W_, C = y.shape
    HW = H * W_
    L = lib()
    a, b, mean, rstd = buf[0], buf[1], buf[2], buf[3]
    gu = torch.empty_like(y)
    red = torch.empty((N, C, 2), device=y.device, dtype=torch.float32)
    L.call('twg_norm_act_bwd_reduce', _p(y), _p(a), _p(b), _p(mean), _p(rstd), _p(gz), None, 0, _p(gu), _p(red), N, HW, C,
           ctx.flags, _st())
    want_p = ctx.group not in _SKIP_PARAM_GRADS
    ggamma = torch.empty(C, device=y.device, dtype=torch.float32) if (ctx.has_gamma and want_p) else None
    gbeta = torch.empty(C, device=y.device, dtype=torch.float32) if want_p else None
    gy = torch.empty_like(y) if ctx.kind != NORM_NONE else gu
    if ctx.kind != NORM_NONE:
      L.call('twg_norm_act_bwd_apply', _p(y), _p(a), _p(mean), _p(rstd), _p(gu), _p(red), _p(rd), _p(gy), None,
             _p(ggamma), _p(gbeta), None, None, 0, 0, N, ctx.kind, N, HW, C, _st())
    elif want_p:
      L.call('twg_colsum', _p(gu), _p(gbeta), N * HW, C, 0, _st())
    return gy, ggamma, gbeta, None, None, None, None, None, None, None


class GenLayerFn(Function):
  """One generator/encoder layer as a single autograd node (first order only; E and G are never differentiated
  twice): conv -> normaliser (+ per-domain gamma/beta) -> leaky-ReLU -> pixel-norm, forward and backward.

  The batch may hold several network passes that share the conv weights (twingan.py:196-284 runs E twice and G four
  times on different inputs / domains): `group_size` samples per pass, bit g of `dom_mask` = domain of pass g, whose
  normaliser variables are (gamma0, beta0) or (gamma1, beta1) (`snap0`/`snap1`: the domains' state snapshots,
  `stats_out` [passes, 2, C]: batch moments per pass for the EMA pushes).

  Merging conv and epilogue lets the backward hand gy to dgrad/wgrad as split planes written by the normaliser's
  backward kernel (no fp32 gy, no split pass), and lets the forward emit z as planes for the next tensor-core conv.
  `emit`: 'fp32' | 'planes' (planes only: the fp32 payload of the returned tensor is NOT written) | 'both'."""

  @staticmethod
  def forward(ctx, x, w, gamma0, beta0, gamma1, beta1, k, pad, kind, flags, eps, clip_dev, snap0, snap1, stats_out,
              group_size, dom_mask, group, emit, pool=None):
    """`pool`: None, or 'fp32' / 'planes' -- also return avg_pool2(z) (optionally with split planes).  The backward then
    takes the pooled tensor's gradient at half resolution and folds its 2x2 broadcast (and the sum with a UNet-skip
    gradient of z) into the normaliser's backward-reduce kernel."""
    N, H, W_, Cin = x.shape
    Cout = int(w.shape[3])
    L = lib()
    gs = int(group_size) if group_size else N
    ctx.set_materialize_grads(False)
    epi_slots = _epilogue_slots(N, H, W_, Cin, Cout, k, pad) if (kind == NORM_INSTANCE and EPILOGUE_STATS) else 0
    epi_stats = torch.empty((N, epi_slots, Cout, 4), device=x.device, dtype=torch.float32) if epi_slots else None
    y, xp = _conv_fwd(x, w, k, pad, stats=epi_stats)
    Ho, Wo = int(y.shape[1]), int(y.shape[2])
    HW = Ho * Wo
    dev = y.device
    buf, rd = _norm_forward(L, y, gamma0, beta0, gamma1, beta1, kind, eps, clip_dev, snap0, snap1, stats_out, gs, dom_mask,
                            epi_stats, epi_slots)
    z = torch.empty_like(y)
    tracing = ACTIVE_SET_TRACE is not None and bool(flags & FLAG_LRELU)
    want_planes = emit in ('planes', 'both') and Cout % 4 == 0
    want_fp32 = (emit != 'planes') or (not want_planes) or tracing or pool is not None
    zp = _new_planes(y.shape, dev) if want_planes else None
    L.call('twg_norm_act_fwd', _p(y), _p(buf[0]), _p(buf[1]), _p(z) if want_fp32 else None, _p(zp), N, HW, Cout, flags,
           _st())
    if zp is not None:
      _put_planes(z, zp)
    if tracing:
      _trace('lrelu', z > 0)
    ctx.save_for_backward(x if xp is None else None, xp, w, y, buf, rd, gamma0, beta0, gamma1, beta1)
    ctx.k, ctx.pad, ctx.kind, ctx.flags, ctx.group = k, pad, kind, flags, group
    ctx.gs, ctx.dom_mask = gs, int(dom_mask)
    ctx.xshape = (N, H, W_, Cin)
    ctx.serial = _next_serial()
    ctx.pool = pool is not None
    if pool is None:
      return z
    pooled = torch.empty((N, Ho // 2, Wo // 2, Cout), device=dev, dtype=torch.float32)
    pp = _new_planes(pooled.shape, dev) if pool == 'planes' else None
    L.call('twg_pool2', _p(z), _p(pooled), _p(pp), N, Ho, Wo, Cout, 0.25, _st())
    if pp is not None:
      _put_planes(pooled, pp)
    return z, pooled

  @staticmethod
  def backward(ctx, gz, gpool=None):
    # x on the exact path, its planes on the tensor-core path
    x, xp, w, y, buf, rd, gamma0, beta0, gamma1, beta1 = ctx.saved_tensors
    gz = _check(gz) if gz is not None else None
    gpool = _check(gpool) if gpool is not None else None
    N, Ho, Wo, C = y.shape
    if gz is None and gpool is None:
      return (None,) * 20
    HW = Ho * Wo
    L = lib()
    a, b, mean, rstd = buf[0], buf[1], buf[2], buf[3]
    gu = torch.empty_like(y)
    red = torch.empty((N, C, 2), device=y.device, dtype=torch.float32)
    L.call('twg_norm_act_bwd_reduce', _p(y), _p(a), _p(b), _p(mean), _p(rstd), _p(gz), _p(gpool), Wo, _p(gu), _p(red),
           N, HW, C, ctx.flags, _st())
    want_p = ctx.group not in _SKIP_PARAM_GRADS
    ptrs, acc, ret = _norm_param_grads(C, y.device, want_p, gamma0, beta0, gamma1, beta1)
    gy = gp = None
    if ctx.kind != NORM_NONE:
      if xp is not None:
        gp = _new_planes(y.shape, y.device)        # gy exists only as the split planes dgrad/wgrad consume
      else:
        gy = torch.empty_like(y)
      L.call('twg_norm_act_bwd_apply', _p(y), _p(a), _p(mean), _p(rstd), _p(gu), _p(red), _p(rd), _p(gy), _p(gp),
             ptrs[0], ptrs[1], ptrs[2], ptrs[3], acc, ctx.dom_mask, ctx.gs, ctx.kind, N, HW, C, _st())
    else:
      gy = gu
      if want_p:
        L.call('twg_colsum', _p(gu), ptrs[1], N * HW, C, acc, _st())
      if xp is not None:
        gp = split_act(gu)
    gx = _conv_dgrad(gy, w, ctx.xshape, ctx.k, ctx.pad, gp)[0] if ctx.needs_input_grad[0] else None
    gw = _weight_grad(ctx, w, x, gy, xp, gp)
    return (gx, gw, ret[0], ret[1], ret[2], ret[3]) + (None,) * 14


def norm_act_eval(y, gamma, beta, kind, flags, eps, moving_mean=None, moving_var=None, emit='fp32'):
  """Inference-mode normaliser (libs/batch_norm.py:266-278: moving stats, r=1, d=0).  No autograd.  `emit='planes'`
  also writes z as split-bf16 planes for the tensor-core conv that consumes it."""
  y = _check(y)
  N, H, W_, C = y.shape
  L = lib()
  if kind in (NORM_BATCH, NORM_RENORM):
    buf = torch.empty((4, N, C), device=y.device, dtype=torch.float32)
    L.call('twg_norm_eval_affine', _p(gamma), _p(beta), _p(moving_mean), _p(moving_var), float(eps), _p(buf[0]),
           _p(buf[1]), N, C, _st())
  else:
    buf, _ = _norm_forward(L, y, gamma, beta, None, None, kind, eps, None, None, None, None, N, 0)
  z = torch.empty_like(y)
  zp = _new_planes(y.shape, y.device) if (emit == 'planes' and vec_ok(C)) else None
  L.call('twg_norm_act_fwd', _p(y), _p(buf[0]), _p(buf[1]), _p(z), _p(zp), N, H * W_, C, flags, _st())
  if zp is not None:
    _put_planes(z, zp)
  return z


def affine_epilogue_ok(N, H, W, Cin, Cout, k, pad) -> bool:
  """Whether conv_affine_act_eval covers this shape (one output-channel block: all Cout channels of a pixel are in one CTA)."""
  return _epilogue_slots(N, H, W, Cin, Cout, k, pad) > 0


def conv_affine_act_eval(x, w, gamma, beta, moving_mean, moving_var, flags, eps, emit='fp32'):
  """Inference-mode generator / encoder layer in one kernel: the normaliser with moving statistics is a per-channel affine
  known before the conv (libs/batch_norm.py:266-278), so conv -> affine -> leaky-ReLU -> pixel norm all happen in the conv
  epilogue and the pre-normalisation tensor never exists.  `emit='planes'`: only the split planes are written."""
  N, H, W_, Cin = x.shape
  Cout = int(w.shape[3])
  L = lib()
  ab = torch.empty((2, Cout), device=x.device, dtype=torch.float32)
  L.call('twg_norm_eval_affine', _p(gamma), _p(beta), _p(moving_mean), _p(moving_var), float(eps), _p(ab[0]), _p(ab[1]), 1, Cout,
         _st())
  xp = planes_of(x)
  z = torch.empty((N, H, W_, Cout), device=x.device, dtype=torch.float32)
  planes_only = emit == 'planes'
  zp = _new_planes(z.shape, x.device) if emit in ('planes', 'both') else None
  _conv_launch('tc_fwd', (N, H, W_, Cin, Cout, 3, 1), 'twg_conv_affine_act_fwd_planes', _p(xp), _p(weight_planes(w, False)),
               _p(ab[0]), _p(ab[1]), int(flags), None if planes_only else _p(z), _p(zp), N, H, W_, Cin, Cout, 3, 1, _st())
  if zp is not None:
    _put_planes(z, zp)
  return z


def norm_update_stats(state_live, batch_stats, kind, C, decay=0.99, eps=1e-3):
  lib().call('twg_norm_update_stats', _p(state_live), _p(batch_stats), kind, float(decay), float(eps), C, _st())


# ------------------------------------------------------------------------------------------------
# discriminator arg scope: bias + leaky-ReLU, twice differentiable
# ------------------------------------------------------------------------------------------------

_DUMMY_COLSUM = {}   # (device, stream) -> discarded column sums; per stream, so that a buffer outgrown and freed on
                     # one stream is never one another stream is still writing into


def _dummy_colsum(device, C):
  key = (device, torch.cuda.current_stream(device).cuda_stream)
  t = _DUMMY_COLSUM.get(key)
  if t is None or t.numel() < C:
    t = torch.zeros(max(C, 1024), device=device, dtype=torch.float32)
    _DUMMY_COLSUM[key] = t
  return t


class LreluBwdFn(Function):
  """out = g * slope(ref) -- the gradient of tf.maximum(0.2x, x); linear in g.  `emit_planes`: the caller consumes the
  result as split-bf16 planes right away (the differentiable backward of ConvBiasActFn, a tensor-core layer), so the same
  pass writes them too (side table, see planes_of) instead of a later split pass.  (Emitting them unconditionally was measured slower: the
  other consumers receive the tensor through the autograd engine, where the side table cannot follow it.)"""

  @staticmethod
  def forward(ctx, g, ref, emit_planes=False, mask=None):
    """`mask`: the sign bytes of `ref` written by the conv epilogue that produced it (ConvBiasActFn) -- read instead of ref."""
    g, ref = _check(g), _check(ref)
    ctx.save_for_backward(ref)
    out = torch.empty_like(g)
    C = int(g.shape[-1]) if g.dim() == 4 else 0
    if mask is None and C and vec_ok(C):
      mask = _mask_of(ref)
    if not (C and vec_ok(C)):
      mask = None
    ctx.mask = mask
    if emit_planes and C and g.numel() >= (1 << 16):
      planes = _new_planes(g.shape, g.device)
      lib().call('twg_lrelu_bwd_colsum', _p(g), _p(ref), _p(mask), _p(out), _p(planes),
                 _p(_dummy_colsum(g.device, C)), g.numel() // C, C, 1, 0, 0, 1, _st())
      _put_planes(out, planes)
    elif mask is not None:
      lib().call('twg_lrelu_bwd_colsum', _p(g), _p(ref), _p(mask), _p(out), None,
                 _p(_dummy_colsum(g.device, C)), g.numel() // C, C, 1, 0, 0, 1, _st())
    else:
      lib().call('twg_lrelu_bwd', _p(g), _p(ref), _p(out), g.numel(), _st())
    return out

  @staticmethod
  def backward(ctx, gout):
    (ref,) = ctx.saved_tensors
    return LreluBwdFn.apply(gout, ref, False, ctx.mask), None, None, None


class ColsumFn(Function):
  @staticmethod
  def forward(ctx, g):
    g = _check(g)
    C = g.shape[-1]
    out = torch.empty(C, device=g.device, dtype=torch.float32)
    lib().call('twg_colsum', _p(g), _p(out), g.numel() // C, C, 0, _st())
    return out

  @staticmethod
  def backward(ctx, gout):
    raise TwgError('ColsumFn is not differentiable (bias gradients never feed the DRAGAN penalty)')


class BiasActFn(Function):
  """z = lrelu?(y + bias)  (pggan_discriminator_arg_scope: bias because no normalizer).  `emit_planes`: z also feeds a
  tensor-core conv (the caller has checked tc_eligible for it), so the same pass writes its split planes."""

  @staticmethod
  def forward(ctx, y, bias, act, group, emit_planes=False):
    y = _check(y)
    C = y.shape[-1]
    z = torch.empty_like(y)
    vec = y.dim() == 4 and vec_ok(C) and y.numel() >= (1 << 16)
    planes = _new_planes(y.shape, y.device) if (emit_planes and vec) else None
    mask = torch.empty(y.numel() // 4, device=y.device, dtype=torch.uint8) if (act and vec and ACT_SIGN_MASK) else None
    lib().call('twg_bias_lrelu_fwd', _p(y), _p(bias), _p(z), _p(planes), _p(mask), y.numel() // C, C, int(act), _st())
    if planes is not None:
      _put_planes(z, planes)
    if ACTIVE_SET_TRACE is not None and act:
      _trace('lrelu', z > 0)
    ctx.act, ctx.group, ctx.mask = act, group, mask
    ctx.save_for_backward(z, bias)
    return z

  @staticmethod
  def backward(ctx, gz):
    z, bias = ctx.saved_tensors
    want_b = ctx.needs_input_grad[1] and ctx.group not in _SKIP_PARAM_GRADS
    if want_b and not torch.is_grad_enabled():
      # plain first-order backward: one fused pass produces gy and the bias gradient (+= into its sink when registered)
      gz = _check(gz)
      C = gz.shape[-1]
      gy = torch.empty_like(gz) if ctx.act else gz
      bsink = _sink(bias)
      gb = bsink if bsink is not None else torch.empty(C, device=gz.device, dtype=torch.float32)
      lib().call('twg_lrelu_bwd_colsum', _p(gz), _p(z), _p(ctx.mask), _p(gy) if ctx.act else None, None, _p(gb),
                 gz.numel() // C, C, int(ctx.act), 0, 0, 1 if bsink is not None else 0, _st())
      return gy, (None if bsink is not None else gb), None, None, None
    gy = LreluBwdFn.apply(gz, z, False, ctx.mask) if ctx.act else gz
    gb = ColsumFn.apply(gy) if want_b else None
    return gy, gb, None, None, None


def bias_act(y, bias, act=True, group='D', emit_planes=False):
  return BiasActFn.apply(y, bias, bool(act), group, bool(emit_planes))


# ------------------------------------------------------------------------------------------------
# resampling / joins (linear; pool and upsample are each other's adjoint)
# ------------------------------------------------------------------------------------------------

class Pool2Fn(Function):
  @staticmethod
  def forward(ctx, x, scale, emit_planes=False):
    x = _check(x)
    N, H, W_, C = x.shape
    ctx.scale = scale
    out = torch.empty((N, H // 2, W_ // 2, C), device=x.device, dtype=torch.float32)
    planes = _new_planes(out.shape, x.device) if (emit_planes and C % 4 == 0) else None
    lib().call('twg_pool2', _p(x), _p(out), _p(planes), N, H, W_, C, float(scale), _st())
    if planes is not None:
      _put_planes(out, planes)
    return out

  @staticmethod
  def backward(ctx, g):
    return Upsample2Fn.apply(g, ctx.scale), None, None


class Upsample2Fn(Function):
  @staticmethod
  def forward(ctx, x, scale):
    x = _check(x)
    N, H, W_, C = x.shape
    ctx.scale = scale
    out = torch.empty((N, 2 * H, 2 * W_, C), device=x.device, dtype=torch.float32)
    lib().call('twg_upsample2', _p(x), _p(out), N, H, W_, C, float(scale), _st())
    return out

  @staticmethod
  def backward(ctx, g):
    return Pool2Fn.apply(g, ctx.scale), None


def avg_pool2(x, emit_planes=False):
  """tf.nn.avg_pool(x, 2x2, stride 2, VALID) (nets/pggan.py:274,306,436,468).  `emit_planes`: also write the
  result as split-bf16 planes for the tensor-core conv that consumes it."""
  return Pool2Fn.apply(x, 0.25, bool(emit_planes))


def resize_twice_as_big(x):
  """nets/pggan_utils.py:349-350."""
  return Upsample2Fn.apply(x, 1.0)


class UpsampleConcatFn(Function):
  """concat(nearest2(a), b) along C: generator block input with the UNet skip (nets/pggan.py:72-76).  `b` may hold fewer
  samples than `a` (b.shape[0] divides a.shape[0]): sample n reads b[n % Nb] -- several generator passes that share one
  encoder pass run as one batch, and the skip's gradient is the sum over its uses."""

  @staticmethod
  def forward(ctx, a, b, planes_only=False):
    a, b = _check(a), _check(b)
    N, H, W_, Ca = a.shape
    Nb, Cb = int(b.shape[0]), int(b.shape[3])
    out = torch.empty((N, 2 * H, 2 * W_, Ca + Cb), device=a.device, dtype=torch.float32)
    if planes_only and Ca % 4 == 0 and Cb % 4 == 0:
      # the joined tensor only feeds the block's first (tensor-core) conv: write it as split planes, never as fp32
      planes = _new_planes(out.shape, a.device)
      lib().call('twg_upsample_concat', _p(a), _p(b), None, _p(planes), N, H, W_, Ca, Cb, Nb, _st())
      _put_planes(out, planes)
    else:
      lib().call('twg_upsample_concat', _p(a), _p(b), _p(out), None, N, H, W_, Ca, Cb, Nb, _st())
    ctx.dims = (N, H, W_, Ca, Cb, Nb)
    return out

  @staticmethod
  def backward(ctx, g):
    g = _check(g)
    N, H, W_, Ca, Cb, Nb = ctx.dims
    ga = torch.empty((N, H, W_, Ca), device=g.device, dtype=torch.float32)
    gb = torch.empty((Nb, 2 * H, 2 * W_, Cb), device=g.device, dtype=torch.float32)
    lib().call('twg_upsample_concat_bwd', _p(g), _p(ga), _p(gb), N, H, W_, Ca, Cb, Nb, _st())
    return ga, gb, None


def _copy_into(dst: torch.Tensor, src: torch.Tensor) -> None:
  lib().call('twg_axpby', _p(src), None, _p(dst), 1.0, 0.0, src.numel(), _st())


def cat_batch(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
  """[a ; b] along the batch axis (input data, no gradient)."""
  a, b = _check(a), _check(b)
  out = torch.empty((a.shape[0] + b.shape[0],) + tuple(a.shape[1:]), device=a.device, dtype=torch.float32)
  _copy_into(out[:a.shape[0]], a)
  _copy_into(out[a.shape[0]:], b)
  return out


class RepeatBatchFn(Function):
  """[x ; x]: the encoder codes feed two generator passes each (twingan.py:242-269)."""

  @staticmethod
  def forward(ctx, x):
    x = _check(x)
    N = x.shape[0]
    out = torch.empty((2 * N,) + tuple(x.shape[1:]), device=x.device, dtype=torch.float32)
    _copy_into(out[:N], x)
    _copy_into(out[N:], x)
    return out

  @staticmethod
  def backward(ctx, g):
    g = _check(g)
    N = g.shape[0] // 2
    out = torch.empty((N,) + tuple(g.shape[1:]), device=g.device, dtype=torch.float32)
    lib().call('twg_axpby', _p(g[:N]), _p(g[N:]), _p(out), 1.0, 1.0, out.numel(), _st())
    return out


def repeat_batch(x):
  return RepeatBatchFn.apply(x)


class AxpbyFn(Function):
  """out = alpha*x + beta*y; fade-in lerp (nets/pggan.py:205,314,475)."""

  @staticmethod
  def forward(ctx, x, y, alpha, beta):
    x = _check(x)
    y = _check(y) if y is not None else None
    ctx.alpha, ctx.beta, ctx.has_y = alpha, beta, y is not None
    out = torch.empty_like(x)
    lib().call('twg_axpby', _p(x), _p(y), _p(out), float(alpha), float(beta), x.numel(), _st())
    return out

  @staticmethod
  def backward(ctx, g):
    gx = AxpbyFn.apply(g, None, ctx.alpha, 0.0) if ctx.needs_input_grad[0] else None
    gy = AxpbyFn.apply(g, None, ctx.beta, 0.0) if (ctx.has_y and ctx.needs_input_grad[1]) else None
    return gx, gy, None, None


def lerp(hi, lo, alpha):
  """alpha*hi + (1-alpha)*lo."""
  return AxpbyFn.apply(hi, lo, float(alpha), 1.0 - float(alpha))


# ------------------------------------------------------------------------------------------------
# minibatch stddev (nets/pggan_utils.py:353-366) with explicit double backward
# ------------------------------------------------------------------------------------------------

class MbstdFn(Function):
  """`groups`: the batch is that many independent minibatches (one per original discriminator pass).  `ct` >= C+1 output
  channels: [x | statistic | zeros] (zero channels pad the next conv's input to a tensor-core channel count)."""

  @staticmethod
  def forward(ctx, x, groups=1, ct=None):
    x = _check(x)
    N, H, W_, C = x.shape
    ct = C + 1 if ct is None else int(ct)
    out = torch.empty((N, H, W_, ct), device=x.device, dtype=torch.float32)
    lib().call('twg_mbstd_fwd', _p(x), _p(out), None, N, H * W_, C, ct, int(groups), _st())
    ctx.save_for_backward(x)
    ctx.groups = int(groups)
    return out

  @staticmethod
  def backward(ctx, gout):
    (x,) = ctx.saved_tensors
    return MbstdBwdFn.apply(x, gout, ctx.groups), None, None


class MbstdBwdFn(Function):
  @staticmethod
  def forward(ctx, x, gout, groups=1):
    x, gout = _check(x), _check(gout)
    N, H, W_, C = x.shape
    gx = torch.empty_like(x)
    lib().call('twg_mbstd_bwd', _p(x), _p(gout), _p(gx), N, H * W_, C, int(gout.shape[3]), int(groups), _st())
    ctx.save_for_backward(x, gout)
    ctx.groups = int(groups)
    return gx

  @staticmethod
  def backward(ctx, ggx):
    x, gout = ctx.saved_tensors
    ggx = _check(ggx)
    N, H, W_, C = x.shape
    dgout = torch.empty_like(gout)
    dx = torch.empty_like(x)
    lib().call('twg_mbstd_bwd2', _p(x), _p(gout), _p(ggx), _p(dgout), _p(dx), N, H * W_, C, int(gout.shape[3]),
               ctx.groups, _st())
    return dx, dgout, None


def minibatch_state_concat(x, groups=1, ct=None):
  return MbstdFn.apply(x, int(groups), ct)


def tc_channel_pad(c: int) -> int:
  """Smallest channel count >= c the tensor-core conv kernels take (16, 32, 64 or a multiple of 128)."""
  for v in (16, 32, 64):
    if c <= v:
      return v
  return (c + 127) // 128 * 128


# Weights padded with zero input-channel rows (the conv after minibatch_state_concat: C+1 -> a tensor-core channel
# count).  The padded tensor is a per-step temporary, so its weight gradient goes to a temporary sink of the padded
# shape; flush_padded_sinks() adds the real rows into the variable's own sink.
# The same mechanism serves weights scaled by the equalized-learning-rate constant (ScaleWeightFn): scratch * scale is
# added to the variable's sink.  A padded scaled weight chains: its sink is the scaled weight's scratch.  Each entry
# also keeps the variable's own sink at the end of the chain, so that one gradient set can be flushed on its own.
_PADDED_SINKS = {}   # temporary weight data_ptr -> (temporary (kept alive), scratch gradient, target sink, scale, variable sink)


def _sink_target(w):
  """(sink the gradient of `w` goes to, the variable's own sink at the end of the chain), or (None, None)."""
  s = _GRAD_SINKS.get(w.data_ptr())
  if s is not None:
    return s, s
  if w.data_ptr() in _PADDED_SINKS:
    e = _PADDED_SINKS[w.data_ptr()]
    return e[1], e[4]
  return None, None


class PadCinFn(Function):
  @staticmethod
  def forward(ctx, w, cpad):
    w = _check(w)
    k, _, cin, cout = w.shape
    out = torch.zeros((k, k, int(cpad), cout), device=w.device, dtype=torch.float32)
    lib().call('twg_copy_cols', _p(w), _p(out), k * k, cin * cout, 0, int(cpad) * cout, 0, cin * cout, _st())
    ctx.wshape = tuple(w.shape)
    sink, root = _sink_target(w)
    if sink is not None:
      _PADDED_SINKS[out.data_ptr()] = (out, torch.zeros_like(out), sink, 1.0, root)
    return out

  @staticmethod
  def backward(ctx, g):
    k, _, cin, cout = ctx.wshape
    g = _check(g)
    gw = torch.empty(ctx.wshape, device=g.device, dtype=torch.float32)
    lib().call('twg_copy_cols', _p(g), _p(gw), k * k, int(g.shape[2]) * cout, 0, cin * cout, 0, cin * cout, _st())
    return gw, None


def pad_cin(w, cpad):
  return PadCinFn.apply(w, int(cpad))


def flush_padded_sinks(within: Optional[torch.Tensor] = None) -> None:
  """Add the scratch gradients into their sinks and forget them.  `within`: only the entries whose variable's sink lies in
  this slice of the gradient buffer (one gradient set); the others stay for a later call."""
  keys = list(_PADDED_SINKS)
  if within is not None:
    lo = within.data_ptr()
    hi = lo + within.numel() * within.element_size()
    keys = [k for k in keys if lo <= _PADDED_SINKS[k][4].data_ptr() < hi]
  for key in reversed(keys):                    # a padded scaled weight flushes first
    out, scratch, sink, scale, _ = _PADDED_SINKS.pop(key)
    if out.numel() == sink.numel():             # a scaled weight (the fc weight is a [1,1,C,1] view of its [C,1] variable)
      tmp = scratch
    else:
      k, _, cpad, cout = out.shape
      cin = int(sink.shape[2])
      tmp = torch.empty_like(sink)
      lib().call('twg_copy_cols', _p(scratch), _p(tmp), k * k, cpad * cout, 0, cin * cout, 0, cin * cout, _st())
    lib().call('twg_axpby', _p(tmp), _p(sink), _p(sink), float(scale), 1.0, sink.numel(), _st())


class ScaleWeightFn(Function):
  """w * c for the equalized learning rate (nets/pggan_utils.py:236-254 scales the layer INPUT by c = sqrt(2 / fan_in);
  conv and matmul are linear, so scaling the few KB of weights instead gives the same function and the same gradients
  without a pass over the activations).  Twice differentiable; gradients the kernels accumulate into sinks go to a
  scratch buffer that flush_padded_sinks() adds, times c, to the variable's own sink."""

  @staticmethod
  def forward(ctx, w, c):
    w = _check(w)
    ctx.c = float(c)
    out = torch.empty_like(w)
    lib().call('twg_axpby', _p(w), None, _p(out), float(c), 0.0, w.numel(), _st())
    sink, root = _sink_target(w)
    if sink is not None:
      _PADDED_SINKS[out.data_ptr()] = (out, torch.zeros_like(out), sink, float(c), root)
    return out

  @staticmethod
  def backward(ctx, g):
    return AxpbyFn.apply(g, None, ctx.c, 0.0), None


def equalized(w):
  """The weight scaled by the reference's equalized-learning-rate constant: HWIO conv weights sqrt(2 / (Cin k^2)), [in, out]
  fully connected weights sqrt(2 / in) (nets/pggan_utils.py:236-254)."""
  fan_in = int(w.shape[0]) * int(w.shape[1]) * int(w.shape[2]) if w.dim() == 4 else int(w.shape[0])
  return ScaleWeightFn.apply(w, math.sqrt(2.0 / fan_in))


def drop_padded_sinks() -> None:
  _PADDED_SINKS.clear()


# ------------------------------------------------------------------------------------------------
# losses
# ------------------------------------------------------------------------------------------------

class SigmoidCEFn(Function):
  """weight * mean(sigmoid_cross_entropy(label, logits))  (tf.losses.sigmoid_cross_entropy)."""

  @staticmethod
  def forward(ctx, logits, label, weight):
    logits = _check(logits)
    loss = torch.empty(1, device=logits.device, dtype=torch.float32)
    grad = torch.empty_like(logits)
    lib().call('twg_sigmoid_ce', _p(logits), float(label), float(weight), _p(loss), _p(grad), logits.numel(), 0, _st())
    ctx.save_for_backward(grad)
    return loss

  @staticmethod
  def backward(ctx, gl):
    (grad,) = ctx.saved_tensors
    out = torch.empty_like(grad)
    lib().call('twg_scale_by_dev', _p(grad), _p(_check(gl)), _p(out), 1.0, grad.numel(), _st())
    return out, None, None


class LogitMeanFn(Function):
  """weight * mean_i f(sign * x_i + margin), f = identity (0), relu (1) or square (2): the WGAN / hinge terms of
  image_generation.py:330-389 -- generator fool loss -mean(D(G)), critic loss mean(D(G)) - mean(D(x)), drift
  c * mean(D(x)^2), hinge mean(relu(1 + D(G))) + mean(relu(1 - D(x))) -- through tf.losses.compute_weighted_loss."""

  @staticmethod
  def forward(ctx, x, sign, margin, kind, weight):
    x = _check(x)
    out = torch.empty((), device=x.device, dtype=torch.float32)
    lib().call('twg_logit_mean', _p(x), _p(out), x.numel(), float(sign), float(margin), int(kind), float(weight), _st())
    ctx.save_for_backward(x)
    ctx.args = (float(sign), float(margin), int(kind), float(weight))
    return out

  @staticmethod
  def backward(ctx, gl):
    (x,) = ctx.saved_tensors
    sign, margin, kind, weight = ctx.args
    gx = torch.empty_like(x)
    lib().call('twg_logit_mean_bwd', _p(x), _p(_check(gl)), _p(gx), x.numel(), sign, margin, kind, weight, _st())
    return gx, None, None, None, None


def logit_mean(x, sign=1.0, margin=0.0, kind=0, weight=1.0):
  return LogitMeanFn.apply(x, sign, margin, kind, weight)


class L1Fn(Function):
  """weight * mean|a - b|  (tf.losses.absolute_difference)."""

  @staticmethod
  def forward(ctx, a, b, weight):
    a, b = _check(a), _check(b)
    loss = torch.empty(1, device=a.device, dtype=torch.float32)
    grad = torch.empty_like(a)
    lib().call('twg_l1', _p(a), _p(b), float(weight), _p(loss), _p(grad), a.numel(), 0, _st())
    if ACTIVE_SET_TRACE is not None:
      _trace('l1', torch.sign(grad))
    ctx.save_for_backward(grad)
    return loss

  @staticmethod
  def backward(ctx, gl):
    (grad,) = ctx.saved_tensors
    gl = _check(gl)
    ga = gb = None
    if ctx.needs_input_grad[0]:
      ga = torch.empty_like(grad)
      lib().call('twg_scale_by_dev', _p(grad), _p(gl), _p(ga), 1.0, grad.numel(), _st())
    if ctx.needs_input_grad[1]:
      gb = torch.empty_like(grad)
      lib().call('twg_scale_by_dev', _p(grad), _p(gl), _p(gb), -1.0, grad.numel(), _st())
    return ga, gb, None


class GradPenaltyFn(Function):
  """lambda * mean_n (||g_n||_2 - 1)^2  (image_generation.py:467-475)."""

  @staticmethod
  def forward(ctx, g, lam):
    g = _check(g)
    N = g.shape[0]
    loss = torch.empty(1, device=g.device, dtype=torch.float32)
    coef = torch.empty(N, device=g.device, dtype=torch.float32)
    lib().call('twg_grad_penalty', _p(g), float(lam), _p(loss), _p(coef), N, g.numel() // N, 0, _st())
    ctx.save_for_backward(g, coef)
    return loss

  @staticmethod
  def backward(ctx, gl):
    g, coef = ctx.saved_tensors
    out = torch.empty_like(g)
    N = g.shape[0]
    lib().call('twg_scale_rows', _p(g), _p(coef), _p(_check(gl)), _p(out), N, g.numel() // N, _st())
    return out, None


_ONES = {}


def _one(device) -> torch.Tensor:
  t = _ONES.get(device)
  if t is None:
    t = torch.ones(1, device=device, dtype=torch.float32)
    _ONES[device] = t
  return t


class SumScalarsFn(Function):
  """scale * sum of up to 16 one-element device tensors in one launch: generator_loss / discriminator_loss = sum of their
  named losses / num_clones (deployment/model_deploy.py:265-267)."""

  @staticmethod
  def forward(ctx, scale, *losses):
    import ctypes
    dev = losses[0].device
    out = torch.empty(1, device=dev, dtype=torch.float32)
    arr = (ctypes.c_void_p * len(losses))(*[t.data_ptr() for t in losses])
    lib().call('twg_sum_scalars', arr, len(losses), float(scale), _p(out), _st())
    ctx.scale, ctx.n = float(scale), len(losses)
    return out

  @staticmethod
  def backward(ctx, g):
    g = _check(g)
    s = torch.empty(1, device=g.device, dtype=torch.float32)
    lib().call('twg_scale_by_dev', _p(g), _p(_one(g.device)), _p(s), ctx.scale, 1, _st())
    return (None,) + (s,) * ctx.n


def sum_scalars(losses, scale=1.0):
  return SumScalarsFn.apply(float(scale), *losses)


class FanoutFn(Function):
  """The wiring between the batched generator pass and its consumers (twingan.py:242-284, 370-381, 464): from
  gout = [s_cycle | t_cycle | t_prime | s_prime] and x = [sources | targets] build, in one pass, the discriminator
  batches ds = [sources | s_cycle | s_prime], dt = [targets | t_cycle | t_prime], the second encoder batch
  e2 = [t_prime | s_prime] and the cycle losses (l_cyc_s, l_cyc_t).  gout then has ONE consumer, so its gradient is
  assembled by one kernel instead of autograd summing five zero-padded slices."""

  @staticmethod
  def forward(ctx, gout, x, weight):
    gout, x = _check(gout), _check(x)
    B = x.shape[0] // 2
    per = gout[0].numel()
    shape = tuple(gout.shape[1:])
    dev = gout.device
    ds = torch.empty((3 * B,) + shape, device=dev, dtype=torch.float32)
    dt = torch.empty((3 * B,) + shape, device=dev, dtype=torch.float32)
    e2 = torch.empty((2 * B,) + shape, device=dev, dtype=torch.float32)
    sgn = torch.empty_like(x)
    loss = torch.empty(2, device=dev, dtype=torch.float32)
    lib().call('twg_fanout_fwd', _p(gout), _p(x), _p(ds), _p(dt), _p(e2), _p(sgn), _p(loss), float(weight), B, per, _st())
    if ACTIVE_SET_TRACE is not None:
      _trace('l1', torch.sign(sgn))
    ctx.set_materialize_grads(False)
    ctx.save_for_backward(sgn)
    ctx.B, ctx.per = B, per
    return ds, dt, e2, loss[0:1], loss[1:2]

  @staticmethod
  def backward(ctx, gds, gdt, ge2, gl_s, gl_t):
    (sgn,) = ctx.saved_tensors
    if gds is None and gdt is None and ge2 is None and gl_s is None and gl_t is None:
      return None, None, None
    c = lambda t: _check(t) if t is not None else None
    gg = torch.empty((4 * ctx.B,) + tuple(sgn.shape[1:]), device=sgn.device, dtype=torch.float32)
    lib().call('twg_fanout_bwd', _p(c(gds)), _p(c(gdt)), _p(c(ge2)), _p(sgn), _p(c(gl_s)), _p(c(gl_t)), _p(gg), ctx.B, ctx.per,
               _st())
    return gg, None, None


class L1GroupsFn(Function):
  """(weight * mean|pred_g - label_g|) for two equal row blocks g: l_content_{s,t} (twingan.py:485-505); both arguments
  receive gradients like tf.losses.absolute_difference."""

  @staticmethod
  def forward(ctx, pred, label, weight):
    pred, label = _check(pred), _check(label)
    grad = torch.empty_like(pred)
    loss = torch.empty(2, device=pred.device, dtype=torch.float32)
    lib().call('twg_l1_groups', _p(pred), _p(label), float(weight), _p(loss), _p(grad), 2, pred.numel() // 2, _st())
    if ACTIVE_SET_TRACE is not None:
      _trace('l1', torch.sign(grad))
    ctx.set_materialize_grads(False)
    ctx.save_for_backward(grad)
    return loss[0:1], loss[1:2]

  @staticmethod
  def backward(ctx, g0, g1):
    (grad,) = ctx.saved_tensors
    if g0 is None and g1 is None:
      return None, None, None
    c = lambda t: _check(t) if t is not None else None
    out = [None, None]
    for i, sign in ((0, 1.0), (1, -1.0)):
      if ctx.needs_input_grad[i]:
        out[i] = torch.empty_like(grad)
        lib().call('twg_scale_groups2', _p(grad), _p(c(g0)), _p(c(g1)), sign, _p(out[i]), grad.numel() // 2, _st())
    return out[0], out[1], None


class GanLossesFn(Function):
  """The six sigmoid-cross-entropy terms of one discriminator batch [real | cycle | prime] (image_generation.py:341-344,
  392-401): (generator_fool_cycle, generator_fool_prime, discriminator_fake_cycle, discriminator_real [cycle term],
  discriminator_fake_prime, discriminator_real [prime term])."""

  @staticmethod
  def forward(ctx, logits, weight):
    logits = _check(logits)
    B = logits.numel() // 3
    sig = torch.empty_like(logits)
    loss = torch.empty(6, device=logits.device, dtype=torch.float32)
    lib().call('twg_gan_losses', _p(logits), float(weight), _p(loss), _p(sig), B, _st())
    ctx.set_materialize_grads(False)
    ctx.save_for_backward(sig)
    ctx.weight, ctx.B = float(weight), B
    return tuple(loss[i:i + 1] for i in range(6))

  @staticmethod
  def backward(ctx, *gs):
    (sig,) = ctx.saved_tensors
    if all(g is None for g in gs):
      return None, None
    ptrs = [_p(_check(g)) if g is not None else None for g in gs]
    grad = torch.empty_like(sig)
    lib().call('twg_gan_losses_bwd', _p(sig), ctx.weight, *ptrs, _p(grad), ctx.B, _st())
    return grad, None


def sigmoid_cross_entropy(label, logits, weight=1.0):
  return SigmoidCEFn.apply(logits, float(label), float(weight))


def absolute_difference(labels, predictions, weight=1.0):
  return L1Fn.apply(predictions, labels, float(weight))


def gradient_penalty(g, lam):
  return GradPenaltyFn.apply(g, float(lam))


def dragan_xhat(x, alpha, noise):
  """image_generation.py:441-460 with explicit randomness."""
  x, alpha, noise = _check(x), _check(alpha), _check(noise)
  N = x.shape[0]
  out = torch.empty_like(x)
  scratch = torch.empty(4, device=x.device, dtype=torch.float64)
  lib().call('twg_dragan_xhat', _p(x), _p(alpha), _p(noise), _p(out), _p(scratch), N, x.numel() // N, _st())
  return out


def growing_image(x, alpha):
  """image_generation.py:1001-1006 (input data, no gradient)."""
  with torch.no_grad():
    low = resize_twice_as_big(avg_pool2(x))
    return lerp(x, low, alpha)


# ------------------------------------------------------------------------------------------------
# image translation front and back end (inference/image_translation_infer.py:54-58, util_io.imsave)
# ------------------------------------------------------------------------------------------------

def pack_images(images) -> Tuple[torch.Tensor, torch.Tensor]:
  """Decoded uint8 [H, W, 3] RGB arrays (numpy or CPU tensors) -> (payload, table) host tensors for images_u8_to_batch:
  payload uint8 [sum of H*W*3], the images back to back; table int64 [B, 3] of {byte offset, H, W}."""
  import numpy as np
  arrs = []
  for i, im in enumerate(images):
    a = im.numpy() if isinstance(im, torch.Tensor) else np.asarray(im)
    if a.dtype != np.uint8 or a.ndim != 3 or a.shape[2] != 3:
      raise ValueError('image %d: want a uint8 [H, W, 3] array, got %s %s' % (i, a.dtype, tuple(a.shape)))
    if a.shape[0] < 1 or a.shape[1] < 1:
      raise ValueError('image %d is empty (%d x %d)' % (i, a.shape[0], a.shape[1]))
    arrs.append(np.ascontiguousarray(a))
  if not arrs:
    raise ValueError('pack_images: no images')
  table = np.zeros((len(arrs), 3), np.int64)
  off = 0
  for i, a in enumerate(arrs):
    table[i] = (off, a.shape[0], a.shape[1])
    off += a.size
  payload = torch.from_numpy(np.concatenate([a.reshape(-1) for a in arrs]))
  table = torch.from_numpy(table)
  check_table(table, payload.numel())
  return payload, table


def check_table(table: torch.Tensor, payload_bytes: int) -> None:
  """Every row {offset, H, W} of a host table must describe a non-empty image inside a payload of `payload_bytes` bytes
  (the kernel reads the table on the device and cannot check it)."""
  if table.device.type != 'cpu' or table.dtype != torch.int64 or table.dim() != 2 or table.shape[1] != 3 \
      or table.shape[0] < 1:
    raise ValueError('image table: want a host int64 [B, 3] tensor, got %s %s on %s'
                     % (table.dtype, tuple(table.shape), table.device))
  for i, (off, h, w) in enumerate(table.tolist()):
    if h < 1 or w < 1 or off < 0 or off + h * w * 3 > payload_bytes:
      raise ValueError('image table row %d {offset %d, H %d, W %d} does not fit a payload of %d bytes'
                       % (i, off, h, w, payload_bytes))


def images_u8_to_batch(payload: torch.Tensor, table: torch.Tensor, hw: int, out: Optional[torch.Tensor] = None
                       ) -> torch.Tensor:
  """Ragged uint8 images -> the model's fp32 [B, hw, hw, 3] input in one launch (convert_image_dtype + TF-1 bilinear
  resize, twg_images_u8_to_batch).  `payload`: uint8 CUDA tensor; `table`: int64 [B, 3] -- a host table is checked
  against the payload and uploaded; a device table must come from pack_images (through a copy of it)."""
  if not payload.is_cuda or payload.dtype != torch.uint8:
    raise TwgError('images_u8_to_batch: payload must be a uint8 CUDA tensor (no CPU fallback)')
  if table.device.type == 'cpu':
    check_table(table, payload.numel())
    table = table.to(payload.device, non_blocking=False)
  elif table.dtype != torch.int64 or table.dim() != 2 or table.shape[1] != 3:
    raise ValueError('image table: want int64 [B, 3], got %s %s' % (table.dtype, tuple(table.shape)))
  B = int(table.shape[0])
  if out is None:
    out = torch.empty((B, hw, hw, 3), device=payload.device, dtype=torch.float32)
  lib().call('twg_images_u8_to_batch', payload.data_ptr(), table.contiguous().data_ptr(), _p(out), B, int(hw), _st())
  return out


JPEG_STAGES = ('twgjpeg_entropy', 'twgjpeg_idct', 'twgjpeg_color')


def jpeg_decode(payload: torch.Tensor, data: torch.Tensor, segs: torch.Tensor, comps: torch.Tensor, images: torch.Tensor,
                qt: torch.Tensor, huff: torch.Tensor, blocks: int, plane_bytes: int, pixels: int, stage_hook=None
                ) -> torch.Tensor:
  """Decode the JPEG scans of one batch into their regions of a uint8 CUDA payload (twgjpeg_entropy, twgjpeg_idct,
  twgjpeg_color): the descriptors are a jpeg.Batch on the device, `blocks`, `plane_bytes` and `pixels` its host sizes.
  Returns the int32 [images] device status without waiting for it: 0 for an image decoded bit for bit as libjpeg-turbo,
  else the TWG_JPEG_* bits of what made the device stop (jpeg.STATUS_*); such an image's region is undefined.
  `stage_hook(name)`, when given, is called after each stage is enqueued (timing)."""
  if not payload.is_cuda or payload.dtype != torch.uint8:
    raise TwgError('jpeg_decode: payload must be a uint8 CUDA tensor (no CPU fallback)')
  dev = payload.device
  n = int(images.shape[0])
  status = torch.empty(n, device=dev, dtype=torch.int32)
  coefs = torch.empty(blocks * 64, device=dev, dtype=torch.int16)
  L = lib()
  L.call('twgjpeg_entropy', data.data_ptr(), segs.data_ptr(), int(segs.shape[0]), images.data_ptr(), n,
         comps.data_ptr(), huff.data_ptr(), coefs.data_ptr(), status.data_ptr(), _st())
  if stage_hook:
    stage_hook(JPEG_STAGES[0])
  _jpeg_pixels(payload, coefs, comps, images, qt, blocks, plane_bytes, pixels, status, stage_hook)
  return status


def _jpeg_pixels(payload, coefs, comps, images, qt, blocks: int, plane_bytes: int, pixels: int, status, stage_hook):
  """The stages after entropy decoding, shared by baseline and progressive files: dequantisation and inverse DCT into
  sample planes (twgjpeg_idct), then upsampling and colour conversion into the payload (twgjpeg_color)."""
  planes = torch.empty(plane_bytes, device=payload.device, dtype=torch.uint8)
  L = lib()
  L.call('twgjpeg_idct', coefs.data_ptr(), comps.data_ptr(), int(comps.shape[0]), blocks, qt.data_ptr(),
         planes.data_ptr(), status.data_ptr(), _st())
  if stage_hook:
    stage_hook(JPEG_STAGES[1])
  L.call('twgjpeg_color', planes.data_ptr(), images.data_ptr(), int(images.shape[0]), comps.data_ptr(), pixels,
         payload.data_ptr(), _st())
  if stage_hook:
    stage_hook(JPEG_STAGES[2])


JPEGP_STAGES = ('twgjpegp_reset', 'twgjpegp_entropy') + JPEG_STAGES[1:]


def jpeg_progressive_decode(payload: torch.Tensor, data: torch.Tensor, segs: torch.Tensor, scans: torch.Tensor,
                            comps: torch.Tensor, images: torch.Tensor, qt: torch.Tensor, huff: torch.Tensor,
                            blocks: int, plane_bytes: int, pixels: int, levels: Sequence[int], stage_hook=None
                            ) -> torch.Tensor:
  """Decode the progressive JPEG files of one batch into their regions of a uint8 CUDA payload: zero the coefficients
  (twgjpegp_reset), decode the scans one level at a time in stream order (twgjpegp_entropy: segment rows
  [levels[l], levels[l + 1]) are level l's), then the baseline inverse DCT and colour conversion (twgjpeg_idct,
  twgjpeg_color).  The descriptors are a jpeg_progressive.Batch on the device, `blocks`, `plane_bytes`, `pixels` and
  `levels` its host sizes.  Returns the int32 [images] device status without waiting for it: 0 for an image decoded bit
  for bit as libjpeg-turbo, else the TWG_JPEG_* / TWG_JPEGP_* bits of what made the device stop
  (jpeg.STATUS_*, jpeg_progressive.STATUS_*); such an image's region is undefined.  The scratch comes from the caching
  allocator on the current stream, so calls on several streams may run at once.  `stage_hook(name)`, when given, is
  called after each stage is enqueued, with 'twgjpegp_entropy:<level>' for each level (timing)."""
  if not payload.is_cuda or payload.dtype != torch.uint8:
    raise TwgError('jpeg_progressive_decode: payload must be a uint8 CUDA tensor (no CPU fallback)')
  dev = payload.device
  n = int(images.shape[0])
  status = torch.empty(n, device=dev, dtype=torch.int32)
  coefs = torch.empty(blocks * 64, device=dev, dtype=torch.int16)
  L = lib()
  L.call('twgjpegp_reset', coefs.data_ptr(), blocks, status.data_ptr(), n, _st())
  if stage_hook:
    stage_hook(JPEGP_STAGES[0])
  for l in range(len(levels) - 1):
    a, e = int(levels[l]), int(levels[l + 1])
    if e > a:
      L.call('twgjpegp_entropy', data.data_ptr(), segs[a:].data_ptr(), e - a, scans.data_ptr(), comps.data_ptr(),
             huff.data_ptr(), coefs.data_ptr(), status.data_ptr(), _st())
    if stage_hook:
      stage_hook('%s:%d' % (JPEGP_STAGES[1], l))
  _jpeg_pixels(payload, coefs, comps, images, qt, blocks, plane_bytes, pixels, status, stage_hook)
  return status


PNG_STAGES = ('twgpng_inflate', 'twgpng_unfilter', 'twgpng_rgb')


def png_decode(payload: torch.Tensor, data: torch.Tensor, images: torch.Tensor, palettes: torch.Tensor, raw_bytes: int,
               pixels: int, stage_hook=None) -> torch.Tensor:
  """Decode the PNG streams of one batch into their regions of a uint8 CUDA payload (twgpng_inflate, twgpng_unfilter,
  twgpng_rgb): the descriptors are a png.Batch on the device, `raw_bytes` and `pixels` its host sizes.  Returns the
  int32 [images] device status without waiting for it: 0 for an image decoded exactly (PIL's pixels), else the TWG_PNG_*
  bits of what made the device stop (png.STATUS_*); such an image's region is undefined.  The inflated scratch comes
  from the caching allocator on the current stream, so calls on several streams may run at once and, after warm-up,
  none reaches cudaMalloc.  `stage_hook(name)`, when given, is called after each stage is enqueued (timing)."""
  if not payload.is_cuda or payload.dtype != torch.uint8:
    raise TwgError('png_decode: payload must be a uint8 CUDA tensor (no CPU fallback)')
  dev = payload.device
  n = int(images.shape[0])
  if data.numel() < 1 or raw_bytes < 1:
    raise ValueError('png_decode: an empty stream or image (png.parse declines them)')
  raw = torch.empty(raw_bytes, device=dev, dtype=torch.uint8)
  status = torch.empty(n, device=dev, dtype=torch.int32)
  L = lib()
  L.call('twgpng_inflate', data.data_ptr(), images.data_ptr(), n, raw.data_ptr(), status.data_ptr(), _st())
  if stage_hook:
    stage_hook(PNG_STAGES[0])
  L.call('twgpng_unfilter', raw.data_ptr(), images.data_ptr(), n, status.data_ptr(), _st())
  if stage_hook:
    stage_hook(PNG_STAGES[1])
  L.call('twgpng_rgb', raw.data_ptr(), images.data_ptr(), n, palettes.data_ptr(), pixels, status.data_ptr(),
         payload.data_ptr(), _st())
  if stage_hook:
    stage_hook(PNG_STAGES[2])
  return status


_JENC_QT = {}


def jpeg_encode(rgb: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
  """The entropy-coded scans of uint8 [n, h, w, 3] RGB CUDA images, byte for byte what PIL writes between
  jpeg.encoder_header(h, w) and EOI for Image.fromarray(rgb[i]).save(f, 'JPEG') (twgjenc_dct, twgjenc_bits,
  twgjenc_pack).  Returns (uint8 device buffer, int64 [n + 1] device offsets) without waiting: image i's scan is
  buffer[offsets[i]:offsets[i + 1]]."""
  from . import jpeg
  if not rgb.is_cuda or rgb.dtype != torch.uint8 or rgb.dim() != 4 or rgb.shape[3] != 3:
    raise TwgError('jpeg_encode: want a uint8 [n, h, w, 3] CUDA tensor (no CPU fallback), got %s %s %s'
                   % (rgb.device, rgb.dtype, tuple(rgb.shape)))
  rgb = rgb.contiguous()
  n, h, w = (int(s) for s in rgb.shape[:3])
  dev = rgb.device
  if dev not in _JENC_QT:
    _JENC_QT[dev] = torch.from_numpy(jpeg.encoder_qt()).to(dev)
  qt = _JENC_QT[dev]
  L = lib()
  ws, cap = L.cdll.twgjenc_workspace_bytes(n, h, w), L.cdll.twgjenc_scan_capacity(n, h, w)
  if ws < 0 or cap < 0:
    raise TwgError('jpeg_encode: %s' % L.last_error())
  blocks = 6 * ((h + 15) // 16) * ((w + 15) // 16)
  coefs = torch.empty(n * blocks * 64, device=dev, dtype=torch.int16)
  bitpos = torch.empty(n * (blocks + 1), device=dev, dtype=torch.int32)
  work = torch.empty(ws, device=dev, dtype=torch.uint8)
  out = torch.empty(cap, device=dev, dtype=torch.uint8)
  offsets = torch.empty(n + 1, device=dev, dtype=torch.int64)
  L.call('twgjenc_dct', rgb.data_ptr(), n, h, w, qt.data_ptr(), coefs.data_ptr(), _st())
  L.call('twgjenc_bits', coefs.data_ptr(), n, h, w, bitpos.data_ptr(), _st())
  L.call('twgjenc_pack', coefs.data_ptr(), bitpos.data_ptr(), n, h, w, work.data_ptr(), out.data_ptr(),
         offsets.data_ptr(), _st())
  return out, offsets


def batch_to_u8(x: torch.Tensor) -> torch.Tensor:
  """uint8 image of the model output, clip(x * 255, 0, 255) truncated (util_io.imsave; twg_batch_to_u8)."""
  x = _check(x)
  out = torch.empty(x.shape, device=x.device, dtype=torch.uint8)
  lib().call('twg_batch_to_u8', _p(x), out.data_ptr(), x.numel(), _st())
  return out


def adam_(p, g, m, v, lr_t, beta1, beta2, eps):
  """lr_t: python float, or a 1-element device tensor (graph-replayable)."""
  if isinstance(lr_t, torch.Tensor):
    lib().call('twg_adam_dev_lr', _p(p), _p(g), _p(m), _p(v), p.numel(), _p(lr_t), float(beta1), float(beta2),
               float(eps), _st())
  else:
    lib().call('twg_adam', _p(p), _p(g), _p(m), _p(v), p.numel(), float(lr_t), float(beta1), float(beta2), float(eps), _st())
