"""Conformance of the kernels of twg_elementwise.cu -- discriminator bias + leaky-ReLU and its fused backward with the
bias-gradient column sums, resampling and the UNet join, minibatch stddev, the losses and the wiring of the batched passes,
the DRAGAN perturbation, the gradient penalty and Adam -- as the training step launches them.

  * coverage: every launch of these kernels in the product (entry point and whatever selects its route or changes its
    arithmetic: sizes, flags, which optional pointers were passed, accumulate) is a key of PRODUCT_ELEMENTWISE, and each
    key is a case of the stage test below, which runs it at the product's own sizes;
  * copies, power-of-two scales, the leaky-ReLU and fixed-order sums of at most four terms bit for bit against torch fp32
    arithmetic in the kernel's order; every other output per element against fp64 on the kernel's own fp32 inputs, within
    c * S (S: the same operation on absolute values), c from the reduction's structure (tests/parity.py; the bounds of
    the column sums, loss sums, penalty, DRAGAN variance and minibatch stddev are calibrated against fp32 emulations in
    test_cpu_reduction_error_model.py, those of the few-rounding elementwise outputs count their roundings);
  * run-to-run reproducibility of every output;
  * one audit that gives every entry point of the harvest exactly one owning suite."""
import pytest
import torch

from tests.parity import (MB_THREADS, U32, _log_result, conv_error_ratio, dragan_var_rel_bound, grid_sum_c,
                          mbstd_bwd2_ref, mbstd_fwd_ref, mbstd_sig_rel, mbstd_stats, norm_sum_c, penalty_c_ss, penalty_ref)
from tests.product_elementwise import (EXTRA_ELEMENTWISE, PRODUCT_ELEMENTWISE_KEYS, colsum_geom, colsum_plain_geom,
                                       grid_for, penalty_geom, pool_rows_route, vec_geom)
from tests import product_launches
from tests.product_launches import Recorder, harvest_product_launches, key_configs
from tests.test_gpu_conv_conformance import _GEOM_AT, _bits, _split_ref

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
LEAK = float(torch.tensor(0.2, dtype=torch.float32))


# ---------------------------------------------------------------------------------------------------------------------
# launch keys
# ---------------------------------------------------------------------------------------------------------------------
def _opts(args, ptrs):
  return '+'.join(n for n, i in ptrs if args[i])


def _f(v):
  """A float argument as a key field: the fp32 value the kernel sees, to 6 significant digits (a stable literal)."""
  return float('%.6g' % float(torch.tensor(float(v), dtype=torch.float32)))


def elementwise_keys(launches):
  """The keys of the launches of twg_elementwise.cu's entry points among (entry, args); layouts in
  tests/product_elementwise.py."""
  keys = set()
  for name, a in launches:
    if name == 'twg_bias_lrelu_fwd':
      keys.add((name, a[5], a[6], a[7], _opts(a, (('bias', 1), ('planes', 3), ('mask', 4)))))
    elif name == 'twg_lrelu_bwd':
      keys.add((name, a[3]))
    elif name == 'twg_lrelu_bwd_colsum':
      keys.add((name, a[6], a[7], a[8], a[9], a[10], a[11], _opts(a, (('ref', 1), ('mask', 2), ('out', 3), ('planes', 4)))))
    elif name == 'twg_colsum':
      keys.add((name, a[2], a[3], a[4]))
    elif name == 'twg_pool2':
      keys.add((name, a[3], a[4], a[5], a[6], _f(a[7]), _opts(a, (('out', 1), ('planes', 2)))))
    elif name == 'twg_upsample2':
      keys.add((name, a[2], a[3], a[4], a[5], _f(a[6])))
    elif name == 'twg_upsample_concat':
      keys.add((name, a[4], a[5], a[6], a[7], a[8], a[9], _opts(a, (('out', 2), ('planes', 3)))))
    elif name == 'twg_upsample_concat_bwd':
      keys.add((name,) + tuple(a[3:9]))
    elif name == 'twg_axpby':
      keys.add((name, a[5], _opts(a, (('y', 1),)), _f(a[3]), _f(a[4])))
    elif name == 'twg_scale_by_dev':
      keys.add((name, a[4], _f(a[3])))
    elif name == 'twg_copy_cols':
      keys.add((name,) + tuple(a[2:8]))
    elif name in ('twg_mbstd_fwd', 'twg_mbstd_bwd'):
      keys.add((name,) + tuple(a[3:8]) + ((_opts(a, (('s_out', 2),)),) if name == 'twg_mbstd_fwd' else ()))
    elif name == 'twg_mbstd_bwd2':
      keys.add((name,) + tuple(a[5:10]))
    elif name == 'twg_sigmoid_ce':
      keys.add((name, a[5], _f(a[1]), a[6], _opts(a, (('grad', 4),))))
    elif name in ('twg_logit_mean', 'twg_logit_mean_bwd'):
      i = 2 if name == 'twg_logit_mean' else 3
      keys.add((name, a[i], _f(a[i + 1]), _f(a[i + 2]), a[i + 3]))
    elif name == 'twg_l1':
      keys.add((name, a[5], a[6], _opts(a, (('grad', 4),))))
    elif name == 'twg_dragan_xhat':
      keys.add((name, a[5], a[6]))
    elif name == 'twg_grad_penalty':
      keys.add((name, a[4], a[5], a[6]))
    elif name == 'twg_scale_rows':
      keys.add((name, a[4], a[5], _opts(a, (('scalar', 2),))))
    elif name == 'twg_fanout_fwd':
      keys.add((name, a[8], a[9]))
    elif name == 'twg_fanout_bwd':
      keys.add((name, a[7], a[8], _opts(a, (('gds', 0), ('gdt', 1), ('ge2', 2), ('gl_s', 4), ('gl_t', 5)))))
    elif name == 'twg_l1_groups':
      keys.add((name, a[5], a[6]))
    elif name == 'twg_scale_groups2':
      keys.add((name, a[5], _f(a[3]), _opts(a, (('gl0', 1), ('gl1', 2)))))
    elif name == 'twg_gan_losses':
      keys.add((name, a[4]))
    elif name == 'twg_gan_losses_bwd':
      keys.add((name, a[9], _opts(a, tuple(('g%d' % k, 2 + k) for k in range(6)))))
    elif name == 'twg_sum_scalars':
      keys.add((name, a[1], _f(a[2])))
    elif name in ('twg_adam', 'twg_adam_dev_lr'):
      keys.add((name, a[4], _f(a[6]), _f(a[7]), _f(a[8])))
  return keys


def _Rec(L):
  return Recorder(L, elementwise_keys)


def _p(t):
  return None if t is None else t.data_ptr()


def _st():
  from twingan_b200 import ops
  return ops._st()


def _cdiv(a, b):
  return -(-a // b)


# ---------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------
def _gen(seed):
  return torch.Generator(device=DEV).manual_seed(seed)


def _rn(shape, seed, scale=1.0, offset=0.0):
  return torch.randn(shape, device=DEV, generator=_gen(seed)) * scale + offset


def _grad(shape, seed):
  """Gradients of mixed sign (column sums cancel), every fourth channel from 2 at mean 3 (an error in a sum shows)."""
  g = _rn(shape, seed)
  C = shape[-1]
  if C > 2:
    g[..., 2::4] += 3.0
  return g


def _ratio(dev, ref, bound):
  return float(((dev.double() - ref).abs() / (bound + 1e-30)).max())


def _mask_of(z):
  """The sign mask of z [..., C]: one byte per 4 channels, bit j = z[4i + j] > 0."""
  pos = (z.reshape(-1, 4) > 0).to(torch.int32)
  return (pos * torch.tensor([1, 2, 4, 8], device=DEV, dtype=torch.int32)).sum(1).to(torch.uint8)


def _slope(z):
  return torch.where(z > 0, torch.ones_like(z), torch.full_like(z, LEAK))


def _same(a, b):
  assert a is None or torch.equal(a, b)


def _check_colsum(cs, t, before, c):
  """cs [C] against the fp64 column sums of the kernel's own fp32 terms t [rows, C] (+ before)."""
  t64 = t.double()
  ref, S = t64.sum(0), t64.abs().sum(0)
  if before is not None:
    ref, S = ref + before.double(), S + before.double().abs()
  return conv_error_ratio(cs, ref, S, c)


# ---------------------------------------------------------------------------------------------------------------------
# discriminator activation and column sums
# ---------------------------------------------------------------------------------------------------------------------
def _run_bias_lrelu(key, rec):
  _, rows, C, act, opts = key
  o = set(opts.split('+'))
  y = _rn((rows, C), 601)
  bias = _rn(C, 602, 0.3) if 'bias' in o else None
  outs = []
  for _ in range(2):
    z = torch.empty_like(y)
    planes = torch.empty((2, rows * C), device=DEV, dtype=torch.bfloat16) if 'planes' in o else None
    mask = torch.empty(rows * C // 4, device=DEV, dtype=torch.uint8) if 'mask' in o else None
    rec('twg_bias_lrelu_fwd', _p(y), _p(bias), _p(z), _p(planes), _p(mask), rows, C, act, _st())
    outs.append((z, planes, mask))
  torch.cuda.synchronize()
  for a, b in zip(*outs):
    _same(a, b)
  z, planes, mask = outs[0]
  t = y + bias if bias is not None else y
  want = torch.maximum(LEAK * t, t) if act else t
  assert torch.equal(z, want)
  if planes is not None:
    assert torch.equal(_bits(planes), _bits(_split_ref(want.reshape(-1))))
  if mask is not None:
    assert torch.equal(mask, _mask_of(want))
  return {}


def _run_lrelu_bwd(key, rec):
  _, n = key
  g, ref = _rn(n, 611), _rn(n, 612)
  outs = [torch.empty_like(g) for _ in range(2)]
  for o in outs:
    rec('twg_lrelu_bwd', _p(g), _p(ref), _p(o), n, _st())
  torch.cuda.synchronize()
  assert torch.equal(outs[0], outs[1])
  assert torch.equal(outs[0], g * _slope(ref))
  return {}


def _run_lrelu_bwd_colsum(key, rec):
  _, rows, C, act, poolH, poolW, acc, opts = key
  o = set(opts.split('+'))
  z = _rn((rows, C), 621)
  if poolW:
    n_img = rows // (poolH * poolW)
    g = _grad((n_img, poolH // 2, poolW // 2, C), 622)
    g_full = g.repeat_interleave(2, 1).repeat_interleave(2, 2).reshape(rows, C)
  else:
    g = g_full = _grad((rows, C), 622)
  mask = _mask_of(z) if 'mask' in o else None
  before = _rn(C, 623) if acc else None
  outs = []
  for _ in range(2):
    out = torch.empty_like(z) if 'out' in o else None
    planes = torch.empty((2, rows * C), device=DEV, dtype=torch.bfloat16) if 'planes' in o else None
    cs = before.clone() if acc else torch.full((C,), float('nan'), device=DEV)
    rec('twg_lrelu_bwd_colsum', _p(g), _p(z) if 'ref' in o else None, _p(mask), _p(out), _p(planes), _p(cs), rows, C, act,
        poolH, poolW, acc, _st())
    outs.append((out, planes, cs))
  torch.cuda.synchronize()
  for a, b in zip(*outs):
    _same(a, b)
  out, planes, cs = outs[0]
  rows_route = pool_rows_route(C, act, poolW, 'out' in o, 'planes' in o)
  if poolW:
    flat = (0.25 * g_full) * _slope(z) if act else 0.25 * g_full
    if act:       # the pool-rows route's g * (0.25 * slope): the same bits for normal numbers
      assert torch.equal(g_full * (0.25 * _slope(z)), flat)
    t = flat
  else:
    t = g_full * _slope(z) if act else g_full
  if out is not None:
    assert torch.equal(out, t)
  if planes is not None:
    assert torch.equal(_bits(planes), _bits(_split_ref(t.reshape(-1))))
  R, nb = colsum_geom(rows, C, poolW, rows_route)
  return {'colsum': _check_colsum(cs, t, before, norm_sum_c(R, samples=nb))}


def _run_colsum(key, rec):
  _, rows, C, acc = key
  g = _grad((rows, C), 631)
  before = _rn(C, 632) if acc else None
  outs = []
  for _ in range(2):
    cs = before.clone() if acc else torch.full((C,), float('nan'), device=DEV)
    rec('twg_colsum', _p(g), _p(cs), rows, C, acc, _st())
    outs.append(cs)
  torch.cuda.synchronize()
  assert torch.equal(outs[0], outs[1])
  R, nb = colsum_plain_geom(rows, C)
  return {'colsum': _check_colsum(outs[0], g, before, norm_sum_c(R, samples=nb))}


# ---------------------------------------------------------------------------------------------------------------------
# resampling and the UNet join
# ---------------------------------------------------------------------------------------------------------------------
def _quad(x):
  """The 2x2 cells of x [N, H, W, C]: (top-left, top-right, bottom-left, bottom-right), each [N, H/2, W/2, C]."""
  return x[:, 0::2, 0::2], x[:, 0::2, 1::2], x[:, 1::2, 0::2], x[:, 1::2, 1::2]


def _up(x):
  return x.repeat_interleave(2, 1).repeat_interleave(2, 2)


def _run_pool2(key, rec):
  _, N, H, W, C, scale, opts = key
  o = set(opts.split('+'))
  x = _rn((N, H, W, C), 641)
  outs = []
  for _ in range(2):
    out = torch.empty((N, H // 2, W // 2, C), device=DEV) if 'out' in o else None
    planes = torch.empty((2, N * H * W * C // 4), device=DEV, dtype=torch.bfloat16) if 'planes' in o else None
    rec('twg_pool2', _p(x), _p(out), _p(planes), N, H, W, C, scale, _st())
    outs.append((out, planes))
  torch.cuda.synchronize()
  for a, b in zip(*outs):
    _same(a, b)
  a, b, c, d = _quad(x)
  want = scale * (((a + b) + c) + d)
  out, planes = outs[0]
  if out is not None:
    assert torch.equal(out, want)
  if planes is not None:
    assert torch.equal(_bits(planes), _bits(_split_ref(want.reshape(-1))))
  return {}


def _run_upsample2(key, rec):
  _, N, H, W, C, scale = key
  x = _rn((N, H, W, C), 651)
  outs = [torch.empty((N, 2 * H, 2 * W, C), device=DEV) for _ in range(2)]
  for out in outs:
    rec('twg_upsample2', _p(x), _p(out), N, H, W, C, scale, _st())
  torch.cuda.synchronize()
  assert torch.equal(outs[0], outs[1])
  assert torch.equal(outs[0], scale * _up(x))
  return {}


def _run_upsample_concat(key, rec):
  _, N, H, W, Ca, Cb, Nb, opts = key
  o = set(opts.split('+'))
  a, b = _rn((N, H, W, Ca), 661), _rn((Nb, 2 * H, 2 * W, Cb), 662)
  outs = []
  for _ in range(2):
    out = torch.empty((N, 2 * H, 2 * W, Ca + Cb), device=DEV) if 'out' in o else None
    planes = torch.empty((2, N * 4 * H * W * (Ca + Cb)), device=DEV, dtype=torch.bfloat16) if 'planes' in o else None
    rec('twg_upsample_concat', _p(a), _p(b), _p(out), _p(planes), N, H, W, Ca, Cb, Nb, _st())
    outs.append((out, planes))
  torch.cuda.synchronize()
  for x, y in zip(*outs):
    _same(x, y)
  want = torch.cat([_up(a), b.repeat(N // Nb, 1, 1, 1)], -1)     # sample n reads skip sample n % Nb
  out, planes = outs[0]
  if out is not None:
    assert torch.equal(out, want)
  if planes is not None:
    assert torch.equal(_bits(planes), _bits(_split_ref(want.reshape(-1))))
  return {}


def _run_upsample_concat_bwd(key, rec):
  _, N, H, W, Ca, Cb, Nb = key
  gout = _grad((N, 2 * H, 2 * W, Ca + Cb), 671)
  outs = []
  for _ in range(2):
    ga, gb = torch.empty((N, H, W, Ca), device=DEV), torch.empty((Nb, 2 * H, 2 * W, Cb), device=DEV)
    rec('twg_upsample_concat_bwd', _p(gout), _p(ga), _p(gb), N, H, W, Ca, Cb, Nb, _st())
    outs.append((ga, gb))
  torch.cuda.synchronize()
  for x, y in zip(*outs):
    assert torch.equal(x, y)
  ga, gb = outs[0]
  a, b, c, d = _quad(gout[..., :Ca])
  assert torch.equal(ga, ((a + b) + c) + d)
  uses = gout[..., Ca:].double().reshape(N // Nb, Nb, 2 * H, 2 * W, Cb)   # use j of skip sample m is sample m + j Nb
  reps = N // Nb
  return {'gb': conv_error_ratio(gb, uses.sum(0), uses.abs().sum(0), 2 * reps * U32)}


# ---------------------------------------------------------------------------------------------------------------------
# lerp, scaling and copies
# ---------------------------------------------------------------------------------------------------------------------
def _run_axpby(key, rec):
  _, n, opts, alpha, beta = key
  x = _rn(n, 681)
  y = _rn(n, 682) if opts == 'y' else None
  outs = [torch.empty_like(x) for _ in range(2)]
  for out in outs:
    rec('twg_axpby', _p(x), _p(y), _p(out), alpha, beta, n, _st())
  torch.cuda.synchronize()
  assert torch.equal(outs[0], outs[1])
  al, be = _f32(alpha), _f32(beta)
  ref, S = al * x.double(), abs(al) * x.double().abs()
  if y is not None:
    ref, S = ref + be * y.double(), S + abs(be) * y.double().abs()
  return {'axpby': conv_error_ratio(outs[0], ref, S, 3 * U32)}      # two products and a sum, or an fma and a product


def _f32(v):
  return float(torch.tensor(float(v), dtype=torch.float32))


def _run_scale_by_dev(key, rec):
  _, n, alpha = key
  x, s = _rn(n, 691), _rn(1, 692)
  outs = [torch.empty_like(x) for _ in range(2)]
  for out in outs:
    rec('twg_scale_by_dev', _p(x), _p(s), _p(out), alpha, n, _st())
  torch.cuda.synchronize()
  assert torch.equal(outs[0], outs[1])
  assert torch.equal(outs[0], x * (torch.tensor(alpha, device=DEV, dtype=torch.float32) * s))
  return {}


def _run_copy_cols(key, rec):
  _, rows, Cs, so, Cd, do, nc = key
  src = _rn((rows, Cs), 701)
  fill = _rn((rows, Cd), 702)
  outs = [fill.clone() for _ in range(2)]
  for dst in outs:
    rec('twg_copy_cols', _p(src), _p(dst), rows, Cs, so, Cd, do, nc, _st())
  torch.cuda.synchronize()
  assert torch.equal(outs[0], outs[1])
  want = fill.clone()
  want[:, do:do + nc] = src[:, so:so + nc]
  assert torch.equal(outs[0], want)
  return {}


# ---------------------------------------------------------------------------------------------------------------------
# minibatch stddev
# ---------------------------------------------------------------------------------------------------------------------
def _mb_x(N, P, C, seed):
  """[N, P, C]: N(0.2, 1), every fourth channel from 1 at mean 10, std 0.05 (|mean| >> spread)."""
  x = _rn((N, P, C), seed, 1.0, 0.2)
  x[..., 1::4] = _rn((N, P, len(range(1, C, 4))), seed + 1, 0.05, 10.0)
  return x


def _run_mbstd_fwd(key, rec):
  _, N, P, C, Ct, groups, opts = key
  x = _mb_x(N, P, C, 711)
  outs = []
  for _ in range(2):
    out = torch.full((N, P, Ct), float('nan'), device=DEV)
    s = torch.empty(groups, device=DEV) if 's_out' in opts else None
    rec('twg_mbstd_fwd', _p(x), _p(out), _p(s), N, P, C, Ct, groups, _st())
    outs.append((out, s))
  torch.cuda.synchronize()
  for a, b in zip(*outs):
    _same(a, b)
  out = outs[0][0]
  assert torch.equal(out[..., :C], x)
  assert bool((out[..., C + 1:] == 0).all())
  Ng = N // groups
  s_ref, bound = mbstd_fwd_ref(x, groups)
  s_dev = out[..., C].reshape(groups, Ng * P)
  assert bool((s_dev == s_dev[:, :1]).all())
  return {'s': _ratio(s_dev[:, 0], s_ref, bound)}


def _run_mbstd_bwd(key, rec):
  _, N, P, C, Ct, groups = key
  x = _mb_x(N, P, C, 721)
  gout = _rn((N, P, Ct), 722)
  gout[..., C] += 0.5                        # a statistic gradient that does not cancel
  outs = [torch.empty((N, P, C), device=DEV) for _ in range(2)]
  for gx in outs:
    rec('twg_mbstd_bwd', _p(x), _p(gout), _p(gx), N, P, C, Ct, groups, _st())
  torch.cuda.synchronize()
  assert torch.equal(outs[0], outs[1])
  Ng, F = N // groups, P * C
  d, var, sig, A = mbstd_stats(x, groups)
  gs = gout[..., C].double().reshape(groups, Ng * P)
  G, SG = gs.sum(1)[:, None, None], gs.abs().sum(1)[:, None, None]
  cG = norm_sum_c(_cdiv(Ng * P, MB_THREADS), 16)
  coef = G / (Ng * F * sig)
  g0 = gout[..., :C].double().reshape(groups, Ng, F)
  ref = g0 + coef * d
  bound = (2 * U32 * g0.abs() + cG * SG / (Ng * F * sig) * d.abs()
           + coef.abs() * ((mbstd_sig_rel(Ng, A, var) + 6 * U32) * d.abs() + (Ng + 2) * U32 * A))
  return {'gx': _ratio(outs[0].reshape(groups, Ng, F), ref, bound)}


def _run_mbstd_bwd2(key, rec):
  _, N, P, C, Ct, groups = key
  x = _mb_x(N, P, C, 731)
  gout = _rn((N, P, Ct), 732)
  gout[..., C] += 0.5
  ggx = _rn((N, P, C), 733, 1.0, 0.3)         # a non-zero mean over the samples: the gm term matters
  outs = []
  for _ in range(2):
    dgout, dx = torch.full((N, P, Ct), float('nan'), device=DEV), torch.empty((N, P, C), device=DEV)
    rec('twg_mbstd_bwd2', _p(x), _p(gout), _p(ggx), _p(dgout), _p(dx), N, P, C, Ct, groups, _st())
    outs.append((dgout, dx))
  torch.cuda.synchronize()
  for a, b in zip(*outs):
    assert torch.equal(a, b)
  dgout, dx = outs[0]
  assert torch.equal(dgout[..., :C], ggx)
  assert bool((dgout[..., C + 1:] == 0).all())
  Ng, F = N // groups, P * C
  dG_ref, dG_b, dx_ref, dx_b = mbstd_bwd2_ref(x, ggx, gout[..., C], groups)
  dG_dev = dgout[..., C].reshape(groups, Ng * P)
  assert bool((dG_dev == dG_dev[:, :1]).all())
  res = {'dgout': _ratio(dG_dev[:, 0], dG_ref, dG_b)}
  res['dx'] = _ratio(dx.reshape(groups, Ng, F), dx_ref, dx_b)
  return res


# ---------------------------------------------------------------------------------------------------------------------
# losses and the wiring of the batched passes
# ---------------------------------------------------------------------------------------------------------------------
def _sign_grad(d, wn):
  return torch.where(d > 0, wn, torch.where(d < 0, -wn, torch.zeros_like(wn)))


def _run_fanout_fwd(key, rec):
  _, B, per = key
  n = B * per
  gout, x = _rn((4, n), 741), _rn((2, n), 742)
  gout[:2, ::5] = x[:, ::5]                  # exact zeros of x - cycle: sign 0
  weight = 1.0
  outs = []
  for _ in range(2):
    ds, dt, e2 = (torch.empty((k, n), device=DEV) for k in (3, 3, 2))
    sgn, loss = torch.empty((2, n), device=DEV), torch.full((2,), float('nan'), device=DEV)
    rec('twg_fanout_fwd', _p(gout), _p(x), _p(ds), _p(dt), _p(e2), _p(sgn), _p(loss), weight, B, per, _st())
    outs.append((ds, dt, e2, sgn, loss))
  torch.cuda.synchronize()
  for a, b in zip(*outs):
    assert torch.equal(a, b)
  ds, dt, e2, sgn, loss = outs[0]
  assert torch.equal(ds, torch.stack([x[0], gout[0], gout[3]]))
  assert torch.equal(dt, torch.stack([x[1], gout[1], gout[2]]))
  assert torch.equal(e2, gout[2:])
  wn = torch.tensor(weight, device=DEV) / torch.tensor(float(n), device=DEV)
  d = gout[:2] - x
  assert torch.equal(sgn, _sign_grad(d, wn))
  nb = grid_for(n, 2)
  R = 4 * _cdiv(n // 4, nb * 256)
  ad = d.double().abs()
  return {'loss': conv_error_ratio(loss, ad.sum(1) * float(wn), ad.sum(1) * float(wn), grid_sum_c(R, nb))}


def _run_fanout_bwd(key, rec):
  _, B, per, opts = key
  o = set(opts.split('+'))
  n = B * per
  gds, gdt = (_rn((3, n), 751 + i) if nm in o else None for i, nm in enumerate(('gds', 'gdt')))
  ge2 = _rn((2, n), 753) if 'ge2' in o else None
  sgn = _sign_grad(_rn((2, n), 754), torch.tensor(1e-3, device=DEV))
  gl = {nm: _rn(1, 755 + i) if nm in o else None for i, nm in enumerate(('gl_s', 'gl_t'))}
  outs = [torch.empty((4, n), device=DEV) for _ in range(2)]
  for gg in outs:
    rec('twg_fanout_bwd', _p(gds), _p(gdt), _p(ge2), _p(sgn), _p(gl['gl_s']), _p(gl['gl_t']), _p(gg), B, per, _st())
  torch.cuda.synchronize()
  assert torch.equal(outs[0], outs[1])
  z = torch.zeros(n, device=DEV, dtype=torch.float64)
  v = lambda t, i: t[i].double() if t is not None else z
  ls = [float(gl[k]) if gl[k] is not None else 0.0 for k in ('gl_s', 'gl_t')]
  terms = [[v(gds, 1), ls[0] * sgn[0].double()], [v(gdt, 1), ls[1] * sgn[1].double()],
           [v(gdt, 2), v(ge2, 0)], [v(gds, 2), v(ge2, 1)]]
  ref = torch.stack([a + b for a, b in terms])
  S = torch.stack([a.abs() + b.abs() for a, b in terms])
  return {'ggout': conv_error_ratio(outs[0], ref, S, 2 * U32)}


def _run_l1_groups(key, rec):
  _, groups, per = key
  a, b = _rn((groups, per), 761), _rn((groups, per), 762)
  b[:, ::7] = a[:, ::7]
  weight = 0.1
  outs = []
  for _ in range(2):
    loss, grad = torch.full((groups,), float('nan'), device=DEV), torch.empty_like(a)
    rec('twg_l1_groups', _p(a), _p(b), weight, _p(loss), _p(grad), groups, per, _st())
    outs.append((loss, grad))
  torch.cuda.synchronize()
  for x, y in zip(*outs):
    assert torch.equal(x, y)
  loss, grad = outs[0]
  wn = torch.tensor(weight, device=DEV) / torch.tensor(float(per), device=DEV)
  d = a - b
  assert torch.equal(grad, _sign_grad(d, wn))
  nb = grid_for(per, 8)
  ad = d.double().abs().sum(1) * float(wn)
  return {'loss': conv_error_ratio(loss, ad, ad, grid_sum_c(_cdiv(per, nb * 256), nb))}


def _run_l1(key, rec):
  _, n, acc, opts = key
  a, b = _rn(n, 765), _rn(n, 766)
  b[::7] = a[::7]
  weight = 10.0
  before = _rn(1, 767)
  outs = []
  for _ in range(2):
    loss = before.clone() if acc else torch.full((1,), float('nan'), device=DEV)
    grad = torch.empty_like(a) if opts == 'grad' else None
    rec('twg_l1', _p(a), _p(b), weight, _p(loss), _p(grad), n, acc, _st())
    outs.append((loss, grad))
  torch.cuda.synchronize()
  for x, y in zip(*outs):
    _same(x, y)
  loss, grad = outs[0]
  wn = torch.tensor(weight, device=DEV) / torch.tensor(float(n), device=DEV)
  d = a - b
  if grad is not None:
    assert torch.equal(grad, _sign_grad(d, wn))
  nb = grid_for(n, 8)
  ad = d.double().abs().sum() * float(wn)
  ref, S = ad, ad
  if acc:
    ref, S = ref + float(before), S + abs(float(before))
  return {'loss': conv_error_ratio(loss, ref.reshape(1), S.reshape(1), grid_sum_c(_cdiv(n, nb * 256), nb))}


def _run_sigmoid_ce(key, rec):
  _, n, label, acc, opts = key
  x = _rn(n, 768, 2.0)
  weight = 1.0
  before = _rn(1, 769)
  outs = []
  for _ in range(2):
    loss = before.clone() if acc else torch.full((1,), float('nan'), device=DEV)
    grad = torch.empty_like(x) if opts == 'grad' else None
    rec('twg_sigmoid_ce', _p(x), label, weight, _p(loss), _p(grad), n, acc, _st())
    outs.append((loss, grad))
  torch.cuda.synchronize()
  for a, b in zip(*outs):
    _same(a, b)
  loss, grad = outs[0]
  wn = weight / n
  ref = _ce64(x, label).sum() * wn
  S = (x.double().abs() * (1 + abs(label)) + torch.log1p(torch.exp(-x.double().abs()))).sum() * wn
  if acc:
    ref, S = ref + float(before), S + abs(float(before))
  # one block: each thread adds cdiv(n, 256) terms of a few roundings each (expf, log1pf), then block_sum
  res = {'loss': conv_error_ratio(loss, ref.reshape(1), S.reshape(1), norm_sum_c(_cdiv(n, 256), 256) + 16 * U32)}
  if grad is not None:
    sig = torch.sigmoid(x.double())
    res['grad'] = conv_error_ratio(grad, wn * (sig - label), wn * (sig + abs(label)), 8 * U32)
  return res


def _run_scale_groups2(key, rec):
  _, per, sign, opts = key
  o = set(opts.split('+'))
  grad = _rn((2, per), 771)
  gl = [_rn(1, 772 + i) if 'gl%d' % i in o else None for i in range(2)]
  outs = [torch.empty_like(grad) for _ in range(2)]
  for out in outs:
    rec('twg_scale_groups2', _p(grad), _p(gl[0]), _p(gl[1]), sign, _p(out), per, _st())
  torch.cuda.synchronize()
  assert torch.equal(outs[0], outs[1])
  f = torch.stack([sign * g[0] if g is not None else torch.zeros((), device=DEV) for g in gl])
  assert torch.equal(outs[0], grad * f[:, None])
  return {}


def _ce64(v, label):
  v = v.double()
  return torch.clamp(v, min=0) - v * label + torch.log1p(torch.exp(-v.abs()))


def _run_gan_losses(key, rec):
  _, B = key
  x = _rn(3 * B, 781, 2.0)
  weight = 1.0
  outs = []
  for _ in range(2):
    loss, sig = torch.full((6,), float('nan'), device=DEV), torch.empty_like(x)
    rec('twg_gan_losses', _p(x), weight, _p(loss), _p(sig), B, _st())
    outs.append((loss, sig))
  torch.cuda.synchronize()
  for a, b in zip(*outs):
    assert torch.equal(a, b)
  loss, sig = outs[0]
  real, cyc, prime = x[:B], x[B:2 * B], x[2 * B:]
  parts = [(cyc, 1.0), (prime, 1.0), (cyc, 0.0), (real, 1.0), (prime, 0.0), (real, 1.0)]
  ref = torch.stack([_ce64(v, l).sum() for v, l in parts]) * weight / B
  S = torch.stack([(v.double().abs() * (1 + l) + torch.log1p(torch.exp(-v.double().abs()))).sum() for v, l in parts]) * weight / B
  sig_ref = torch.sigmoid(x.double())
  return {'loss': conv_error_ratio(loss, ref, S, 16 * U32), 'sig': conv_error_ratio(sig, sig_ref, sig_ref, 8 * U32)}


def _run_gan_losses_bwd(key, rec):
  _, B, opts = key
  o = set(opts.split('+'))
  sig = torch.sigmoid(_rn(3 * B, 791, 2.0))
  g = [_rn(1, 792 + k) if 'g%d' % k in o else None for k in range(6)]
  weight = 1.0
  outs = [torch.empty_like(sig) for _ in range(2)]
  for grad in outs:
    rec('twg_gan_losses_bwd', _p(sig), weight, *[_p(t) for t in g], _p(grad), B, _st())
  torch.cuda.synchronize()
  assert torch.equal(outs[0], outs[1])
  u = [float(t) if t is not None else 0.0 for t in g]
  s = sig.double()
  blk = torch.arange(3 * B, device=DEV) // B
  wn = weight / B
  a = torch.where(blk == 0, (u[3] + u[5]) * (s - 1), torch.where(blk == 1, u[0] * (s - 1), u[1] * (s - 1)))
  b = torch.where(blk == 1, u[2] * s, torch.where(blk == 2, u[4] * s, torch.zeros_like(s)))
  S = wn * (a.abs() + b.abs() + abs(u[3]) * (s - 1).abs() * (blk == 0))
  return {'grad': conv_error_ratio(outs[0], wn * (a + b), S, 6 * U32)}


def _run_sum_scalars(key, rec):
  import ctypes
  _, n, scale = key
  vals = _rn(n, 801)
  ptrs = (ctypes.c_void_p * n)(*[vals.data_ptr() + 4 * i for i in range(n)])
  outs = [torch.empty(1, device=DEV) for _ in range(2)]
  for out in outs:
    rec('twg_sum_scalars', ptrs, n, scale, _p(out), _st())
  torch.cuda.synchronize()
  assert torch.equal(outs[0], outs[1])
  v = vals.double()
  return {'sum': conv_error_ratio(outs[0], v.sum() * scale, v.abs().sum() * abs(scale), (n + 1) * U32)}


def _run_logit_mean(key, rec):
  name, n, sign, margin, kind = key
  x = _rn(n, 811, 1.5)
  u32 = sign * x + margin                         # fmaf(sign, x, margin) with sign = +-1: one rounding, as here
  u = u32.double()
  f = torch.clamp(u, min=0) if kind == 1 else (u * u if kind == 2 else u)
  weight = 0.5
  if name == 'twg_logit_mean':
    outs = [torch.empty(1, device=DEV) for _ in range(2)]
    for out in outs:
      rec(name, _p(x), _p(out), n, sign, margin, kind, weight, _st())
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1])
    A = x.double().abs() + abs(margin)
    S = (A * A if kind == 2 else A).sum() * weight / n
    return {'loss': conv_error_ratio(outs[0], f.sum() * weight / n, S, norm_sum_c(_cdiv(n, 256), 256) + 4 * U32)}
  gl = _rn(1, 812)
  outs = [torch.empty_like(x) for _ in range(2)]
  for out in outs:
    rec(name, _p(x), _p(gl), _p(out), n, sign, margin, kind, weight, _st())
  torch.cuda.synchronize()
  assert torch.equal(outs[0], outs[1])
  dfu = (u32 > 0).double() if kind == 1 else (2 * u if kind == 2 else torch.ones_like(u))
  ref = float(gl) * weight / n * sign * dfu
  return {'grad': conv_error_ratio(outs[0], ref, ref.abs(), 6 * U32)}


# ---------------------------------------------------------------------------------------------------------------------
# DRAGAN perturbation and gradient penalty
# ---------------------------------------------------------------------------------------------------------------------
def _run_dragan_xhat(key, rec):
  _, N, per = key
  g = _gen(821)
  x = torch.rand((N, per), device=DEV, generator=g)        # real images in [0, 1], as the product draws them
  x[:, 0::3] = x[:, 0::3] * 0.1 + 0.8                     # one channel with |mean| >> spread
  alpha = torch.rand(N, device=DEV, generator=g)
  noise = torch.rand((N, per), device=DEV, generator=g) * 2 - 1
  outs = []
  for _ in range(2):
    xhat, scratch = torch.empty_like(x), torch.empty(4, device=DEV)
    rec('twg_dragan_xhat', _p(x), _p(alpha), _p(noise), _p(xhat), _p(scratch), N, per, _st())
    outs.append(xhat)
  torch.cuda.synchronize()
  assert torch.equal(outs[0], outs[1])
  x64 = x.double()
  m = x64.mean()
  var = ((x64 - m) ** 2).mean()
  kappa = 1 + m * m / var
  R = _cdiv(N * per, 256)                                  # one block: each thread adds every 256th element
  pert = alpha.double()[:, None] * (0.5 * var * noise.double())
  ref = x64 + pert
  bound = (dragan_var_rel_bound(R, kappa) + 4 * U32) * pert.abs() + 2 * U32 * ref.abs()
  return {'xhat': _ratio(outs[0], ref, bound)}


def _penalty_g(N, per, seed):
  """[N, per] gradients whose per-sample norms spread over 0.4 .. 1.6, none within 1 % of 1."""
  s = torch.linspace(0.4, 1.6, N, device=DEV, dtype=torch.float64)
  s = torch.where((s - 1).abs() < 0.01, s + 0.05, s)
  g = _rn((N, per), seed)
  return (g.double() / g.double().norm(dim=1, keepdim=True) * s[:, None]).float()


def _run_grad_penalty(key, rec):
  _, N, per, acc = key
  g = _penalty_g(N, per, 831)
  lam = 0.25
  before = _rn(1, 832)
  outs = []
  for _ in range(2):
    loss = before.clone() if acc else torch.full((1,), float('nan'), device=DEV)
    coef = torch.full((N,), float('nan'), device=DEV)
    rec('twg_grad_penalty', _p(g), lam, _p(loss), _p(coef), N, per, acc, _st())
    outs.append((loss, coef))
  torch.cuda.synchronize()
  for a, b in zip(*outs):
    assert torch.equal(a, b)
  loss, coef = outs[0]
  chunk, nb = penalty_geom(per)
  coef_ref, coef_b, loss_ref, loss_b = penalty_ref((g.double() ** 2).sum(1), penalty_c_ss(chunk, nb), lam, N)
  if acc:
    loss_ref, loss_b = loss_ref + float(before), loss_b + 2 * U32 * (abs(float(before)) + loss_ref)
  return {'coef': _ratio(coef, coef_ref, coef_b), 'loss': _ratio(loss, loss_ref.reshape(1), loss_b.reshape(1))}


def _run_scale_rows(key, rec):
  _, N, per, opts = key
  x, coef = _rn((N, per), 841), _rn(N, 842)
  s = _rn(1, 843) if opts == 'scalar' else None
  outs = [torch.empty_like(x) for _ in range(2)]
  for out in outs:
    rec('twg_scale_rows', _p(x), _p(coef), _p(s), _p(out), N, per, _st())
  torch.cuda.synchronize()
  assert torch.equal(outs[0], outs[1])
  want = x * coef[:, None]
  assert torch.equal(outs[0], want * s if s is not None else want)     # (x * coef) * scalar: two roundings in this order
  return {}


# ---------------------------------------------------------------------------------------------------------------------
# Adam
# ---------------------------------------------------------------------------------------------------------------------
def _run_adam(key, rec, applies=5):
  name, n, b1, b2, eps = key
  p, m, v = _rn(n, 851, 0.05), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
  b1f, b2f, epsf, lr = _f32(b1), _f32(b2), _f32(eps), _f32(2e-4)
  lr_dev = torch.tensor([lr], device=DEV)
  p64, m64, v64 = p.double(), m.double(), v.double()
  Ma, pe = torch.zeros_like(m64), torch.zeros_like(p64)
  again = (p.clone(), m.clone(), v.clone())
  for t in range(applies):
    g = _rn(n, 860 + t, 1e-2)
    g[t::7] = 0.0                             # g = 0, on some elements with m = v = 0
    for st in ((p, m, v), again):
      if name == 'twg_adam':
        rec(name, _p(st[0]), _p(g), _p(st[1]), _p(st[2]), n, lr, b1, b2, eps, _st())
      else:
        rec(name, _p(st[0]), _p(g), _p(st[1]), _p(st[2]), n, _p(lr_dev), b1, b2, eps, _st())
    g64 = g.double()
    m64 = b1f * m64 + (1 - b1f) * g64
    v64 = b2f * v64 + (1 - b2f) * g64 * g64
    Ma = b1f * Ma + (1 - b1f) * g64.abs()
    c = (4 * t + 4) * U32                     # a few roundings per apply, added up over the applies
    den = v64.sqrt() + epsf
    upd = lr * m64 / den
    # m within c * Ma, v within c * v (no cancellation), sqrt halves that; then the quotient, the product and p's rounding
    pe = pe + lr * (c * Ma / den + m64.abs() / den * (0.5 * c + 4 * U32)) + 2 * U32 * (p64 - upd).abs()
    p64 = p64 - upd
  torch.cuda.synchronize()
  for a, b in zip((p, m, v), again):
    assert torch.equal(a, b)
  c = (4 * applies + 4) * U32
  return {'m': conv_error_ratio(m, m64, Ma, c), 'v': conv_error_ratio(v, v64, v64, c), 'p': _ratio(p, p64, pe)}


# ---------------------------------------------------------------------------------------------------------------------
# the product's launches, the cases beside them, and the audit
# ---------------------------------------------------------------------------------------------------------------------
_RUNNERS = {'twg_bias_lrelu_fwd': _run_bias_lrelu, 'twg_lrelu_bwd': _run_lrelu_bwd,
            'twg_lrelu_bwd_colsum': _run_lrelu_bwd_colsum, 'twg_colsum': _run_colsum, 'twg_pool2': _run_pool2,
            'twg_upsample2': _run_upsample2, 'twg_upsample_concat': _run_upsample_concat,
            'twg_upsample_concat_bwd': _run_upsample_concat_bwd, 'twg_axpby': _run_axpby,
            'twg_scale_by_dev': _run_scale_by_dev, 'twg_copy_cols': _run_copy_cols, 'twg_mbstd_fwd': _run_mbstd_fwd,
            'twg_mbstd_bwd': _run_mbstd_bwd, 'twg_mbstd_bwd2': _run_mbstd_bwd2, 'twg_fanout_fwd': _run_fanout_fwd,
            'twg_fanout_bwd': _run_fanout_bwd, 'twg_l1_groups': _run_l1_groups, 'twg_l1': _run_l1,
            'twg_sigmoid_ce': _run_sigmoid_ce, 'twg_scale_groups2': _run_scale_groups2,
            'twg_gan_losses': _run_gan_losses, 'twg_gan_losses_bwd': _run_gan_losses_bwd,
            'twg_sum_scalars': _run_sum_scalars, 'twg_logit_mean': _run_logit_mean, 'twg_logit_mean_bwd': _run_logit_mean,
            'twg_dragan_xhat': _run_dragan_xhat, 'twg_grad_penalty': _run_grad_penalty, 'twg_scale_rows': _run_scale_rows,
            'twg_adam': _run_adam, 'twg_adam_dev_lr': _run_adam}
_STAGE = {'twg_bias_lrelu_fwd': 'activation', 'twg_lrelu_bwd': 'activation', 'twg_lrelu_bwd_colsum': 'colsum',
          'twg_colsum': 'colsum', 'twg_pool2': 'resampling', 'twg_upsample2': 'resampling',
          'twg_upsample_concat': 'resampling', 'twg_upsample_concat_bwd': 'resampling', 'twg_axpby': 'lerp',
          'twg_scale_by_dev': 'lerp', 'twg_copy_cols': 'lerp', 'twg_mbstd_fwd': 'mbstd', 'twg_mbstd_bwd': 'mbstd',
          'twg_mbstd_bwd2': 'mbstd', 'twg_fanout_fwd': 'losses', 'twg_fanout_bwd': 'losses', 'twg_l1_groups': 'losses',
          'twg_l1': 'losses', 'twg_sigmoid_ce': 'losses',
          'twg_scale_groups2': 'losses', 'twg_gan_losses': 'losses', 'twg_gan_losses_bwd': 'losses',
          'twg_sum_scalars': 'losses', 'twg_logit_mean': 'losses', 'twg_logit_mean_bwd': 'losses',
          'twg_dragan_xhat': 'penalty', 'twg_grad_penalty': 'penalty', 'twg_scale_rows': 'penalty', 'twg_adam': 'adam',
          'twg_adam_dev_lr': 'adam'}

SUITE_ELEMENTWISE_KEYS = PRODUCT_ELEMENTWISE_KEYS | EXTRA_ELEMENTWISE


def _key_id(k):
  return '-'.join(str(v) for v in k).replace('twg_', '')


@pytest.mark.parametrize('key', sorted(SUITE_ELEMENTWISE_KEYS, key=str), ids=_key_id)
def test_elementwise_stage_against_fp64(built_lib, key):
  rec = _Rec(built_lib)
  res = _RUNNERS[key[0]](key, rec)
  assert key in rec.keys(), (key, sorted(rec.keys(), key=str))
  _log_result({'test': 'elementwise_stage', 'stage': _STAGE[key[0]], 'key': list(key), 'ratios': res})
  bad = {k: v for k, v in res.items() if not v <= 1.0}
  assert not bad, (key, res)


def _owners():
  """{suite: the entry points it checks}: the conv suite (every conv entry, and the split kernels it checks bit for bit),
  the normaliser suite, this file, the trajectory suite that holds the step counters and the lr_t / renorm clipping
  derived from them to the reference's after every step of a run, the SWD stage suite, and the translate tests that hold the uint8 front end to the fp64 restatement and the quantisation bit
  for bit."""
  from tests.test_gpu_norm_conformance import _RUNNERS as NORM_RUNNERS
  from tests.test_gpu_swd_conformance import _RUNNERS as SWD_RUNNERS
  return {'test_gpu_conv_conformance': set(_GEOM_AT) | {'twg_split_act', 'twg_split_weights', 'twg_split_weights_table'},
          'test_gpu_norm_conformance': set(NORM_RUNNERS),
          'test_gpu_elementwise_conformance': set(_RUNNERS),
          'test_gpu_trajectory': {'twg_step_schedule', 'twg_step_advance'},
          'test_gpu_swd_conformance': set(SWD_RUNNERS),
          'test_gpu_translate': {'twg_images_u8_to_batch', 'twg_batch_to_u8'}}


def test_every_product_launch_belongs_to_one_audit(built_lib):
  launches = harvest_product_launches()
  owners = _owners()
  names = sorted({n for n, _ in launches})
  claims = {n: [o for o, entries in owners.items() if n in entries] for n in names}
  unowned = [n for n, c in claims.items() if not c]
  shared = {n: c for n, c in claims.items() if len(c) > 1}
  seen = elementwise_keys(launches)
  where = key_configs(elementwise_keys)
  _log_result({'test': 'elementwise_coverage', 'harvested': len(seen), 'entries': len(names),
               'harvest_s': product_launches.HARVEST_SECONDS, 'keys': sorted(seen, key=str)})
  assert not unowned and not shared, ('unowned', unowned, 'shared', shared)
  assert seen == PRODUCT_ELEMENTWISE_KEYS, ('new', sorted(((k, where[k]) for k in seen - PRODUCT_ELEMENTWISE_KEYS), key=str),
                                            'gone', sorted(PRODUCT_ELEMENTWISE_KEYS - seen, key=str))
  missing = sorted(((k, where[k]) for k in seen if k not in SUITE_ELEMENTWISE_KEYS or k[0] not in _RUNNERS), key=str)
  assert not missing, missing
