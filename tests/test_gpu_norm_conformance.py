"""Conformance of the generator / encoder normaliser layer (normaliser + leaky-ReLU + pixel norm, training and evaluation
mode) as the training step and inference launch it.

  * coverage: every launch of the normaliser kernels in the product (entry point, batch N, group size, domain mask,
    geometry, channels, kind, flags, which optional pointers were passed, accumulate) is a key of PRODUCT_NORMS, and each
    key is a case of the stage tests below, which run at the product's own N;
  * each stage against fp64 evaluated on the device's own fp32 inputs to that kernel, per element, with bounds from
    tests/parity.py (calibrated in test_cpu_norm_error_model.py): statistics (twg_moments + twg_norm_finalize, epilogue
    records + twg_norm_finalize_partials, batch renorm's r / d with every clipping regime), forward apply and its output
    modes, backward reduce (incl. the pool-gradient fold), backward apply (gy, its planes, per-domain gamma / beta
    gradients, accumulate), evaluation-mode affine and the EMA pushes;
  * run-to-run reproducibility of every output, and batch invariance of instance norm;
  * the fused layer (ops.GenLayerFn) end to end against the oracle's fp64 chain once per product backward key, at the
    product's N, groups, domains, gy route, pool fold and accumulate, with the device's active set transferred; and the
    single-domain 8x8 layer (NormActFn) for all four kinds, incl. the 3-channel scalar and 256-channel routes."""
import contextlib

import pytest
import torch

from tests.parity import (REL_TOL, U32, _log_result, conv_error_ratio, ema_c, exact_elem_c, mean_bound, norm_sum_c, rel_err,
                          rstd_rel_bound, serial_run)
from tests.product_launches import harvest_product_launches
from tests.product_norms import PRODUCT_NORM_KEYS
from tests.test_gpu_conv_conformance import _bits, _split_ref

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
INSTANCE, BATCH, RENORM = 1, 2, 3          # TWG_NORM_*
LRELU, PIXNORM = 1, 2                      # TWG_FLAG_*
EPS = {INSTANCE: 1e-6, BATCH: 1e-3, RENORM: 1e-3}
CLIP = (0.9, 1.1, 0.1)                     # {rmin, rmax, dmax} of the renorm schedule's first stage
LEAK = float(torch.tensor(0.2, dtype=torch.float32))

# ---------------------------------------------------------------------------------------------------------------------
# launch keys
# ---------------------------------------------------------------------------------------------------------------------
_FIN_PTRS = (('gamma0', 2), ('beta0', 3), ('gamma1', 4), ('beta1', 5), ('renorm0', 8), ('renorm1', 9), ('clip', 12),
             ('rd', 17), ('batch_stats', 18))
_PART_PTRS = (('gamma0', 2), ('beta0', 3), ('gamma1', 4), ('beta1', 5))
_APPLY_PTRS = (('rd', 6), ('gy', 7), ('gy_planes', 8), ('ggamma0', 9), ('gbeta0', 10), ('ggamma1', 11), ('gbeta1', 12))


def _opts(args, ptrs):
  return '+'.join(n for n, i in ptrs if args[i])


def norm_keys(launches):
  """The keys of the normaliser launches among (entry, args) in launch order.  twg_norm_finalize_partials is keyed with the
  geometry of the conv whose epilogue wrote its records (the twg_conv_fwd_planes launch before it)."""
  keys = set()
  conv = None
  for name, a in launches:
    if name == 'twg_conv_fwd_planes':
      conv = a
    elif name == 'twg_moments':
      keys.add((name, a[2], a[3], a[4], a[5]))                                     # N, HW, C, pivot group
    elif name == 'twg_norm_finalize':                                              # kind, N, gs, dom, HW, C
      keys.add((name, a[10], a[19], a[7], a[6], a[20], a[21], _opts(a, _FIN_PTRS)))
    elif name == 'twg_norm_finalize_partials':                                     # N, gs, dom, H, W, Cin, C, slots
      keys.add((name, a[13], a[7], a[6], conv[9], conv[10], conv[11], a[14], a[1], _opts(a, _PART_PTRS)))
    elif name == 'twg_norm_eval_affine':                                           # N, C
      keys.add((name, a[7], a[8]))
    elif name == 'twg_norm_act_fwd':                                               # N, HW, C, flags
      keys.add((name, a[5], a[6], a[7], a[8], _opts(a, (('z', 3), ('planes', 4)))))
    elif name == 'twg_norm_act_bwd_reduce':                                        # N, HW, W (pool fold), C, flags
      keys.add((name, a[10], a[11], a[7] if a[6] else 0, a[12], a[13], _opts(a, (('gz', 5), ('gpool', 6)))))
    elif name == 'twg_norm_act_bwd_apply':                                         # kind, N, gs, dom, HW, C
      keys.add((name, a[16], a[17], a[15], a[14], a[18], a[19],
                '+'.join(filter(None, (_opts(a, _APPLY_PTRS), 'accumulate' if a[13] else '')))))
    elif name == 'twg_norm_update_stats':                                          # kind, C, decay
      keys.add((name, a[2], a[5], round(float(a[3]), 6)))
    elif name == 'twg_colsum':
      keys.add((name, a[2], a[3], a[4]))
  return keys


class _Recorder:
  """L.call that also keeps (entry, args): a stage test asserts that it launched the key it stands for.  Inside spying(),
  launches the library's Python layer (ops) makes are recorded too."""

  def __init__(self, L):
    self.L, self.call, self.launches = L, L.call, []

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
    return norm_keys(self.launches)


def _p(t):
  return None if t is None else t.data_ptr()


def _st():
  from twingan_b200 import ops
  return ops._st()


# ---------------------------------------------------------------------------------------------------------------------
# inputs and fp64 references
# ---------------------------------------------------------------------------------------------------------------------
def _gen(seed):
  return torch.Generator(device=DEV).manual_seed(seed)


def _y(N, HW, C, seed):
  """[N, HW, C] fp32: N(0.3, 0.7), every fourth channel from 1 at mean 10, std 0.05 (|mean| >> std)."""
  g = _gen(seed)
  y = torch.randn((N, HW, C), device=DEV, generator=g) * 0.7 + 0.3
  if C > 1:
    y[..., 1::4] = torch.randn((N, HW, len(range(1, C, 4))), device=DEV, generator=g) * 0.05 + 10.0
  return y


def _vec(C, seed, scale, offset=0.0):
  return torch.randn(C, device=DEV, generator=_gen(seed)) * scale + offset


def _params(C, seed):
  """gamma0, beta0, gamma1, beta1: the two domains' variables, far enough apart that a wrong domain shows."""
  return [_vec(C, seed, 0.2, 1.0), _vec(C, seed + 1, 0.1), _vec(C, seed + 2, 0.2, -0.7), _vec(C, seed + 3, 0.1, 0.5)]


def _dom(dom_mask, N, gs):
  """[N] domain of each sample."""
  return torch.tensor([(dom_mask >> (n // gs)) & 1 for n in range(N)], device=DEV)


def _per_sample(dom, p0, p1):
  """[N, C]: each sample's row of a per-domain [C] variable (p0 for domain 0, p1 for domain 1), in fp64."""
  return torch.where(dom[:, None].bool(), p1.double()[None], p0.double()[None])


def _group_view(t, gs):
  """[N, HW, C] -> [groups, gs * HW, C]."""
  N, HW, C = t.shape
  return t.reshape(N // gs, gs * HW, C)


def _ab(y, seed):
  """A plausible fp32 affine (a, b) [N, C] of the normaliser from fp64 statistics of y, plus (mean, rstd) [N, C]."""
  N, HW, C = y.shape
  y64 = y.double()
  mean = y64.mean(1)
  rstd = 1.0 / (((y64 - mean[:, None]) ** 2).mean(1) + 1e-6).sqrt()
  g, be = _vec(C, seed, 0.2, 1.0).double(), _vec(C, seed + 1, 0.1).double()
  a = g * rstd
  b = be - mean * a
  return a.float(), b.float(), mean.float(), rstd.float()


def _act_ref(y, a, b, flags):
  """fp64 t = a y + b, v = lrelu?(t), rinv (1 without pixel norm), z = v * rinv on fp32 inputs [N, HW, C] / [N, C]."""
  t = a.double()[:, None] * y.double() + b.double()[:, None]
  v = torch.where(t > 0, t, LEAK * t) if flags & LRELU else t
  if flags & PIXNORM:
    rinv = 1.0 / ((v * v).mean(-1, keepdim=True) + float(torch.tensor(1e-6, dtype=torch.float32))).sqrt()
  else:
    rinv = torch.ones_like(v[..., :1])
  return t, v, rinv, v * rinv


def _ratio(dev, ref, bound):
  return float(((dev.double() - ref).abs() / (bound + 1e-30)).max())


def _pool_bcast(gp, H, W):
  """[N, H/2, W/2, C] -> the 2x2 broadcast [N, H * W, C]."""
  N, C = gp.shape[0], gp.shape[-1]
  return gp.repeat_interleave(2, 1).repeat_interleave(2, 2).reshape(N, H * W, C)


# ---------------------------------------------------------------------------------------------------------------------
# statistics
# ---------------------------------------------------------------------------------------------------------------------
def _check_moments(sums, y, pg):
  N, HW, C = y.shape
  y64 = y.double()
  piv = y64[torch.arange(N, device=DEV) // pg * pg, 0]
  d = y64 - piv[:, None]
  c = norm_sum_c(serial_run(HW, C))
  r1 = conv_error_ratio(sums[..., 0], d.sum(1), d.abs().sum(1), c)
  r2 = conv_error_ratio(sums[..., 1], (d * d).sum(1), (d * d).sum(1), c)
  return max(r1, r2)


def _renorm_state(y, gs, dom_mask, C):
  """{renorm_mean, renorm_stddev, mean weight, stddev weight} per domain, set from the first group of that domain so that
  r is clipped at rmin, at rmax or interior, and d at -dmax, +dmax or interior, each on some channels."""
  N = y.shape[0]
  yg = _group_view(y.double(), gs)
  m, sd = yg.mean(1), (yg.var(1, unbiased=False) + 1e-3).sqrt()
  c = torch.arange(C, device=DEV)
  r_t = torch.tensor([0.5, 2.0, 1.0, 1.02], device=DEV, dtype=torch.float64)[(c // 2) % 4]
  d_t = torch.tensor([-1.0, 1.0, 0.0, 0.03], device=DEV, dtype=torch.float64)[(c // 3) % 4]
  w = 0.6
  out = []
  for dom in (0, 1):
    grp = next((g for g in range(N // gs) if (dom_mask >> g) & 1 == dom), 0)
    ms = sd[grp] / r_t                               # mixed_std = renorm_stddev + (1 - w) * std
    rsd = ms - (1 - w) * sd[grp]
    rm = w * m[grp] - d_t * ms                       # mixed_mean = renorm_mean + (1 - w) * mean
    out.append(torch.cat([rm, rsd, torch.tensor([w, w], device=DEV, dtype=torch.float64)]).float())
  return out


def _run_statistics(key, rec):
  """Runs the statistics launch of `key` and checks it; returns the worst ratio of each check."""
  from twingan_b200 import ops
  name = key[0]
  res = {}
  if name == 'twg_moments':
    _, N, HW, C, pg = key
    y = _y(N, HW, C, 401)
    sums = torch.empty((N, C, 2), device=DEV)
    rec(name, _p(y), _p(sums), N, HW, C, pg, _st())
    again = torch.empty_like(sums)
    rec(name, _p(y), _p(again), N, HW, C, pg, _st())
    torch.cuda.synchronize()
    assert torch.equal(sums, again)
    res['moments'] = _check_moments(sums, y, pg)
    return res
  gam = _params(key[-3] if name == 'twg_norm_finalize_partials' else key[6], 411)
  if name == 'twg_norm_finalize_partials':
    _, N, gs, dom_mask, H, W, Cin, C, slots, opts = key
    HW, kind = H * W, INSTANCE
    x = torch.randn((N, H, W, Cin), device=DEV, generator=_gen(402)) * 0.5 + 2.0
    w = torch.randn((3, 3, Cin, C), device=DEV, generator=_gen(403)) * 0.05 + 0.02
    assert ops._epilogue_slots(N, H, W, Cin, C, 3, 1) == slots
    stats = torch.empty((N, slots, C, 4), device=DEV)
    xp = ops.split_act(x)
    with rec.spying():                                               # the conv whose epilogue writes the records
      y4, _ = ops._conv_fwd(None, w, 3, 1, xp=xp, stats=stats)
    y = y4.reshape(N, HW, C)
    ptr = dict(zip(('gamma0', 'beta0', 'gamma1', 'beta1'), gam))
    outs = [torch.empty((4, N, C), device=DEV) for _ in range(2)]
    for buf in outs:
      rec(name, _p(stats), slots, *[_p(ptr[k]) if k in opts.split('+') else None for k in ('gamma0', 'beta0', 'gamma1', 'beta1')],
          dom_mask, gs, EPS[INSTANCE], _p(buf[0]), _p(buf[1]), _p(buf[2]), _p(buf[3]), N, C, _st())
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1])
    a, b, mean, rstd = outs[0]
    pivot = stats[:, 0, :, 1].double()                               # the first record's pivot
    rd = bs = None
  else:
    _, kind, N, gs, dom_mask, HW, C, opts = key
    o = set(opts.split('+'))
    y = _y(N, HW, C, 404)
    pg = 1 if kind == INSTANCE else gs
    sums = torch.empty((N, C, 2), device=DEV)
    rec('twg_moments', _p(y), _p(sums), N, HW, C, pg, _st())
    rn = _renorm_state(y, gs, dom_mask, C) if kind == RENORM else [None, None]
    clip = torch.tensor(CLIP, device=DEV)
    ptr = dict(zip(('gamma0', 'beta0', 'gamma1', 'beta1'), gam), renorm0=rn[0], renorm1=rn[1], clip=clip)
    groups = N // gs
    outs = []
    for _ in range(2):
      buf = torch.empty((4, N, C), device=DEV)
      rd = torch.empty((groups, 2, C), device=DEV) if 'rd' in o else None
      bs = torch.empty((groups, 2, C), device=DEV) if 'batch_stats' in o else None
      args = [_p(ptr[k]) if k in o else None for k in ('gamma0', 'beta0', 'gamma1', 'beta1')]
      rec(name, _p(sums), _p(y), *args, dom_mask, gs, _p(ptr['renorm0']) if 'renorm0' in o else None,
          _p(ptr['renorm1']) if 'renorm1' in o else None, kind, EPS[kind], _p(clip) if 'clip' in o else None,
          _p(buf[0]), _p(buf[1]), _p(buf[2]), _p(buf[3]), _p(rd), _p(bs), N, HW, C, _st())
      outs.append((buf, rd, bs))
    torch.cuda.synchronize()
    for t0, t1 in zip(outs[0], outs[1]):
      assert t0 is None or torch.equal(t0, t1)
    res['moments'] = _check_moments(sums, y, pg)
    (buf, rd, bs) = outs[0]
    a, b, mean, rstd = buf
    y64 = y.double()
    pivot = y64[torch.arange(N, device=DEV) // pg * pg, 0]
  # mean and rstd against two-pass fp64 moments of y over the reduction domain
  eps = EPS[kind]
  red_gs = 1 if kind == INSTANCE else gs
  yg = _group_view(y.double(), red_gs)
  L = HW / slots if name == 'twg_norm_finalize_partials' else serial_run(HW, C)    # serial run of each sample's sums
  m_ref = yg.mean(1)
  var = ((yg - m_ref[:, None]) ** 2).mean(1)
  piv_g = pivot.reshape(-1, red_gs, C)[:, 0]
  kappa = 1.0 + (m_ref - piv_g) ** 2 / var
  A1 = (yg - piv_g[:, None]).abs().mean(1)
  expand = lambda t: t.repeat_interleave(red_gs, 0)
  res['mean'] = _ratio(mean, expand(m_ref), expand(mean_bound(L, A1, m_ref, red_gs)))
  rs_ref = 1.0 / (var + eps).sqrt()
  res['rstd'] = _ratio(rstd, expand(rs_ref), expand(rs_ref * rstd_rel_bound(L, kappa, var, eps, red_gs)))
  # a, b from the device's own mean, rstd (and r, d) with the group's domain variables
  dom = _dom(dom_mask, N, gs)
  o = set(opts.split('+'))
  g_ = _per_sample(dom, gam[0] if 'gamma0' in o else torch.ones(C, device=DEV), gam[2] if 'gamma1' in o else torch.ones(C, device=DEV))
  be = _per_sample(dom, gam[1] if 'beta0' in o else torch.zeros(C, device=DEV), gam[3] if 'beta1' in o else torch.zeros(C, device=DEV))
  r = d = None
  if kind == RENORM:
    std = bs[:, 1].double()
    mg = bs[:, 0].double()
    st_dom = torch.stack([rn[int(_dom(dom_mask, N, gs)[g * gs])] for g in range(N // gs)]).double()
    rm, rsd, rmw, rsw = st_dom[:, :C], st_dom[:, C:2 * C], st_dom[:, 2 * C:2 * C + 1], st_dom[:, 2 * C + 1:]
    mixed_m, mixed_s = rm + (1 - rmw) * mg, rsd + (1 - rsw) * std
    r_ref = (std / mixed_s).clamp(CLIP[0], CLIP[1])
    d_raw = (mg - mixed_m) / mixed_s
    d_ref = d_raw.clamp(-CLIP[2], CLIP[2])
    res['rd'] = max(_ratio(rd[:, 0], r_ref, 8 * U32 * r_ref.abs()),
                    _ratio(rd[:, 1], d_ref, 8 * U32 * ((mg.abs() + rm.abs() + mixed_m.abs()) / mixed_s + d_raw.abs())))
    # every clipping regime is exercised
    if C >= 16:
      r0, d0 = rd[:, 0], rd[:, 1]
      f32 = lambda v: float(torch.tensor(v, dtype=torch.float32))
      assert bool((r0 == f32(CLIP[0])).any()) and bool((r0 == f32(CLIP[1])).any())
      assert bool(((r0 > f32(CLIP[0])) & (r0 < f32(CLIP[1]))).any())
      assert bool((d0 == f32(CLIP[2])).any()) and bool((d0 == -f32(CLIP[2])).any()) and bool((d0.abs() < f32(CLIP[2])).any())
    r, d = expand(rd[:, 0].double()), expand(rd[:, 1].double())
    res['batch_stats'] = _ratio(std, (var + eps).sqrt(), (var + eps).sqrt() * rstd_rel_bound(L, kappa, var, eps, red_gs))
    assert torch.equal(bs[:, 0], mean[::gs])
  elif kind == BATCH and bs is not None:
    res['batch_stats'] = _ratio(bs[:, 1], var, 2 * var * rstd_rel_bound(L, kappa, var, 0.0, red_gs))
    assert torch.equal(bs[:, 0], mean[::gs])
  if r is None:
    r, d = torch.ones_like(g_), torch.zeros_like(g_)
  a_ref = g_ * r * rstd.double()
  b_ref = d * g_ + be - mean.double() * a.double()
  res['a'] = _ratio(a, a_ref, 4 * U32 * a_ref.abs())
  res['b'] = _ratio(b, b_ref, 4 * U32 * ((d * g_).abs() + be.abs() + (mean.double() * a.double()).abs()))
  if kind == INSTANCE and name == 'twg_norm_finalize':
    # batch invariance: the last sample alone gives the same bits
    n = N - 1
    s1 = torch.empty((1, C, 2), device=DEV)
    rec('twg_moments', _p(y[n:]), _p(s1), 1, HW, C, 1, _st())
    one = torch.empty((4, 1, C), device=DEV)
    g0 = gam[2] if int(dom[n]) else gam[0]
    b0 = gam[3] if int(dom[n]) else gam[1]
    rec(name, _p(s1), _p(y[n:]), _p(g0) if 'gamma0' in o else None, _p(b0) if 'beta0' in o else None, None, None, 0, 1, None,
        None, kind, eps, None, _p(one[0]), _p(one[1]), _p(one[2]), _p(one[3]), None, None, 1, HW, C, _st())
    torch.cuda.synchronize()
    assert torch.equal(s1[0], sums[n])
    assert torch.equal(one[:, 0], torch.stack([a[n], b[n], mean[n], rstd[n]]))
  return res


# ---------------------------------------------------------------------------------------------------------------------
# forward apply
# ---------------------------------------------------------------------------------------------------------------------
def _run_forward(key, rec):
  _, N, HW, C, flags, opts = key
  y = _y(N, HW, C, 421)
  a, b, _, _ = _ab(y, 422)
  t, v, rinv, z_ref = _act_ref(y, a, b, flags)
  vec = C % 4 == 0 and (C // 4 <= 32 and (C // 4) & (C // 4 - 1) == 0 or C // 4 % 32 == 0 and C // 128 in (1, 2, 4))
  z_only, z_both = torch.empty_like(y), torch.empty_like(y)
  rec('twg_norm_act_fwd', _p(y), _p(a), _p(b), _p(z_only), None, N, HW, C, flags, _st())
  if vec:
    zp_both, zp_only = (torch.empty((2, N, HW, C), device=DEV, dtype=torch.bfloat16) for _ in range(2))
    rec('twg_norm_act_fwd', _p(y), _p(a), _p(b), _p(z_both), _p(zp_both), N, HW, C, flags, _st())
    rec('twg_norm_act_fwd', _p(y), _p(a), _p(b), None, _p(zp_only), N, HW, C, flags, _st())
  again = torch.empty_like(y)
  rec('twg_norm_act_fwd', _p(y), _p(a), _p(b), _p(again), None, N, HW, C, flags, _st())
  torch.cuda.synchronize()
  assert torch.equal(again, z_only)
  if vec:
    assert torch.equal(z_both, z_only)
    assert torch.equal(_bits(zp_both), _bits(_split_ref(z_only)))
    assert torch.equal(_bits(zp_only), _bits(zp_both))
  # one rounding of a y + b, the leaky-ReLU product, and the pixel norm's sum of C squares, rsqrt and product
  c_pix = (0.5 * exact_elem_c(C) + 4 * U32) if flags & PIXNORM else 0.0
  bound = 3 * U32 * t.abs() * rinv + c_pix * z_ref.abs()
  return {'forward': _ratio(z_only, z_ref, bound)}


# ---------------------------------------------------------------------------------------------------------------------
# backward reduce
# ---------------------------------------------------------------------------------------------------------------------
def _gu_ref(y, a, b, flags, g):
  """fp64 gradient w.r.t. u = a y + b of sum(g * pixel_norm?(lrelu?(u))) and its per-element scale S."""
  t, v, rinv, z = _act_ref(y, a, b, flags)
  C = y.shape[-1]
  if flags & PIXNORM:
    dot = (g * z).mean(-1, keepdim=True)
    gu = rinv * (g - z * dot)
    S = rinv * (g.abs() + z.abs() * (g * z).abs().mean(-1, keepdim=True))
  else:
    gu, S = g.clone(), g.abs()
  if flags & LRELU:
    slope = torch.where(t > 0, 1.0, LEAK)     # the device's slope: the sign of fmaf(a, y, b) = the sign of the exact t
    gu, S = gu * slope, S * slope
  return gu, S


def _run_reduce(key, rec):
  _, N, HW, W, C, flags, opts = key
  o = set(opts.split('+'))
  y = _y(N, HW, C, 431)
  a, b, mean, rstd = _ab(y, 432)
  H = HW // W if W else 0
  gz = torch.randn((N, HW, C), device=DEV, generator=_gen(433)) if 'gz' in o else None
  gp = torch.randn((N, H // 2, W // 2, C), device=DEV, generator=_gen(434)) if 'gpool' in o else None
  outs = []
  for _ in range(2):
    gu, red = torch.empty_like(y), torch.empty((N, C, 2), device=DEV)
    rec('twg_norm_act_bwd_reduce', _p(y), _p(a), _p(b), _p(mean), _p(rstd), _p(gz), _p(gp), W, _p(gu), _p(red), N, HW, C,
        flags, _st())
    outs.append((gu, red))
  torch.cuda.synchronize()
  (gu, red), (gu2, red2) = outs
  assert torch.equal(gu, gu2) and torch.equal(red, red2)
  g = torch.zeros((N, HW, C), device=DEV, dtype=torch.float64)
  if gz is not None:
    g += gz.double()
  if gp is not None:
    g += 0.25 * _pool_bcast(gp.double(), H, W)
  gu_ref, S = _gu_ref(y, a, b, flags, g)
  res = {'gu': conv_error_ratio(gu, gu_ref, S, exact_elem_c(C))}
  # red = {sum gu, sum gu * yhat} per (n, c) against fp64 sums of the device's own gu
  gu64 = gu.double()
  yhat = (y.double() - mean.double()[:, None]) * rstd.double()[:, None]
  c = norm_sum_c(serial_run(HW, C)) + 4 * U32      # + the roundings of each term gu * (y - mean) * rstd
  res['reduce'] = max(conv_error_ratio(red[..., 0], gu64.sum(1), gu64.abs().sum(1), c),
                      conv_error_ratio(red[..., 1], (gu64 * yhat).sum(1), (gu64 * yhat).abs().sum(1), c))
  # batch invariance: the last sample alone
  n = N - 1
  gu1, red1 = torch.empty_like(y[n:]), torch.empty((1, C, 2), device=DEV)
  rec('twg_norm_act_bwd_reduce', _p(y[n:]), _p(a[n:]), _p(b[n:]), _p(mean[n:]), _p(rstd[n:]),
      _p(gz[n:]) if gz is not None else None, _p(gp[n:]) if gp is not None else None, W, _p(gu1), _p(red1), 1, HW, C, flags,
      _st())
  torch.cuda.synchronize()
  assert torch.equal(gu1[0], gu[n]) and torch.equal(red1[0], red[n])
  return res


# ---------------------------------------------------------------------------------------------------------------------
# backward apply
# ---------------------------------------------------------------------------------------------------------------------
def _run_apply(key, rec):
  _, kind, N, gs, dom_mask, HW, C, opts = key
  o = set(opts.split('+'))
  y = _y(N, HW, C, 441)
  a, _, mean, rstd = _ab(y, 442)
  gu = torch.randn((N, HW, C), device=DEV, generator=_gen(443)) * 0.3 + 0.05
  yhat = (y.double() - mean.double()[:, None]) * rstd.double()[:, None]
  red = torch.stack([gu.double().sum(1), (gu.double() * yhat).sum(1)], -1).float()     # what the reduce pass hands over
  groups = N // gs
  rd = None
  if 'rd' in o:
    rd = torch.stack([_vec(groups * C, 444, 0.05, 1.0).reshape(groups, C), _vec(groups * C, 445, 0.05).reshape(groups, C)], 1)
  params = {k: k in o for k in ('ggamma0', 'gbeta0', 'ggamma1', 'gbeta1')}
  vec = C % 4 == 0

  def run(gy_on, planes_on, acc, before=None):
    gy = torch.empty_like(y) if gy_on else None
    gp = torch.empty((2, N, HW, C), device=DEV, dtype=torch.bfloat16) if planes_on else None
    pg = {k: (before[k].clone() if before is not None else torch.full((C,), float('nan'), device=DEV)) if on else None
          for k, on in params.items()}
    r = red.clone()
    rec('twg_norm_act_bwd_apply', _p(y), _p(a), _p(mean), _p(rstd), _p(gu), _p(r), _p(rd), _p(gy), _p(gp),
        _p(pg['ggamma0']), _p(pg['gbeta0']), _p(pg['ggamma1']), _p(pg['gbeta1']), acc, dom_mask, gs, kind, N, HW, C, _st())
    return gy, gp, pg

  gy, _, pg = run(True, False, 0)
  gy2, _, pg2 = run(True, False, 0)
  runs = []
  if vec:
    runs = [run(True, True, 0), run(False, True, 0)]
  before = {k: _vec(C, 446 + i, 1.0) for i, k in enumerate(params)}
  _, _, pg_acc = run('gy' in o or not vec, 'gy_planes' in o, 1, before)
  torch.cuda.synchronize()
  assert torch.equal(gy, gy2)
  for k in params:
    assert pg[k] is None or torch.equal(pg[k], pg2[k])
  if vec:
    (gy_b, gp_b, _), (_, gp_only, _) = runs
    assert torch.equal(gy_b, gy)
    assert torch.equal(_bits(gp_b), _bits(_split_ref(gy)))
    assert torch.equal(_bits(gp_only), _bits(gp_b))
  # gy against fp64 on the same inputs
  red64 = red.double()
  M = HW if kind == INSTANCE else HW * gs
  if kind == INSTANCE:
    t1, t2 = red64[..., 0], red64[..., 1]
    A1, A2 = t1.abs(), t2.abs()
  else:
    t1 = red64[..., 0].reshape(groups, gs, C).sum(1).repeat_interleave(gs, 0)
    t2 = red64[..., 1].reshape(groups, gs, C).sum(1).repeat_interleave(gs, 0)
    A1 = red64[..., 0].abs().reshape(groups, gs, C).sum(1).repeat_interleave(gs, 0)
    A2 = red64[..., 1].abs().reshape(groups, gs, C).sum(1).repeat_interleave(gs, 0)
  k1, k2 = (t1 / M)[:, None], (t2 / M)[:, None]
  a64 = a.double()[:, None]
  gy_ref = a64 * (gu.double() - k1 - yhat * k2)
  S = a64.abs() * (gu.double().abs() + k1.abs() + (yhat * k2).abs() + (A1 / M)[:, None] + yhat.abs() * (A2 / M)[:, None])
  res = {'apply': conv_error_ratio(gy, gy_ref, S, exact_elem_c(gs if kind != INSTANCE else 1))}
  # gamma / beta gradients of each domain over its groups
  dom = _dom(dom_mask, N, gs)
  if rd is not None:
    r_n, d_n = rd[:, 0].double().repeat_interleave(gs, 0), rd[:, 1].double().repeat_interleave(gs, 0)
  else:
    r_n, d_n = torch.ones((N, C), device=DEV, dtype=torch.float64), torch.zeros((N, C), device=DEV, dtype=torch.float64)
  tg, tb = red64[..., 1] * r_n + red64[..., 0] * d_n, red64[..., 0]
  Sg, Sb = (red64[..., 1] * r_n).abs() + (red64[..., 0] * d_n).abs(), red64[..., 0].abs()
  c = exact_elem_c(N)
  worst = 0.0
  for k, (ref_t, S_t, dm) in {'ggamma0': (tg, Sg, 0), 'gbeta0': (tb, Sb, 0), 'ggamma1': (tg, Sg, 1),
                              'gbeta1': (tb, Sb, 1)}.items():
    if pg[k] is None:
      continue
    sel = (dom == dm)[:, None]
    ref = (ref_t * sel).sum(0)
    S_k = (S_t * sel).sum(0)
    worst = max(worst, conv_error_ratio(pg[k], ref, S_k, c))
    # accumulate = 1 onto a non-zero buffer
    if kind == INSTANCE:    # each sample's term is added onto the buffer in turn
      worst = max(worst, conv_error_ratio(pg_acc[k], before[k].double() + ref, S_k + before[k].double().abs(), c))
    else:                   # the total is added once
      assert torch.equal(pg_acc[k], before[k] + pg[k]), k
  res['gamma_beta'] = worst
  if kind == INSTANCE:
    # batch invariance: the last sample alone, although the grid of the apply kernel depends on N
    n = N - 1
    gy1 = torch.empty_like(y[n:])
    r1 = red[n:].clone()
    rec('twg_norm_act_bwd_apply', _p(y[n:]), _p(a[n:]), _p(mean[n:]), _p(rstd[n:]), _p(gu[n:]), _p(r1), None, _p(gy1), None,
        None, None, None, None, 0, 0, 1, kind, 1, HW, C, _st())
    torch.cuda.synchronize()
    assert torch.equal(gy1[0], gy[n])
  return res


# ---------------------------------------------------------------------------------------------------------------------
# evaluation mode and EMA
# ---------------------------------------------------------------------------------------------------------------------
def _run_eval_affine(key, rec):
  _, N, C = key
  g, be, mm = _vec(C, 451, 0.2, 1.0), _vec(C, 452, 0.1), _vec(C, 453, 3.0)
  mv = _vec(C, 454, 0.5).abs() + 1e-3
  ab = [torch.empty((N, C), device=DEV) for _ in range(4)]
  for i in (0, 2):
    rec('twg_norm_eval_affine', _p(g), _p(be), _p(mm), _p(mv), 1e-3, _p(ab[i]), _p(ab[i + 1]), N, C, _st())
  torch.cuda.synchronize()
  assert torch.equal(ab[0], ab[2]) and torch.equal(ab[1], ab[3])
  a_ref = g.double() / (mv.double() + float(torch.tensor(1e-3, dtype=torch.float32))).sqrt()
  b_ref = be.double() - mm.double() * ab[0][0].double()
  return {'eval_affine': max(_ratio(ab[0], a_ref[None], 5 * U32 * a_ref.abs()[None]),
                             _ratio(ab[1], b_ref[None], 3 * U32 * (be.double().abs() + (mm.double() * a_ref).abs())[None]))}


def _run_update_stats(key, rec, pushes=5):
  _, kind, C, decay = key
  eps = 1e-3
  st = torch.cat([_vec(C, 461, 1.0), _vec(C, 462, 0.3).abs() + 0.2, _vec(C, 463, 1.0), _vec(C, 464, 0.3).abs() + 0.2,
                  torch.tensor([0.7, 0.8], device=DEV)])
  s64 = st.double()
  S = s64.abs()
  d = float(torch.tensor(decay, dtype=torch.float32))
  om = 1.0 - d
  for i in range(pushes):
    bs = torch.cat([_vec(C, 470 + i, 1.0, 0.5), _vec(C, 480 + i, 0.3).abs() + 0.1])
    rec('twg_norm_update_stats', _p(st), _p(bs), kind, decay, eps, C, _st())
    b64 = bs.double()
    n = s64.clone()
    if kind == RENORM:
      n[2 * C:3 * C] = s64[2 * C:3 * C] * d + b64[:C] * om
      n[3 * C:4 * C] = s64[3 * C:4 * C] * d + b64[C:] * om
      n[4 * C:] = s64[4 * C:] * d + om
      new_mean, new_std = n[2 * C:3 * C] / n[4 * C], n[3 * C:4 * C] / n[4 * C + 1]
      n[:C] = s64[:C] * d + new_mean * om
      n[C:2 * C] = s64[C:2 * C] * d + (new_std * new_std - float(torch.tensor(eps, dtype=torch.float32))) * om
      Sb = torch.cat([b64.abs(), b64[C:] ** 2, b64[C:] ** 2, torch.ones(2, device=DEV, dtype=torch.float64)])
    else:
      n[:2 * C] = s64[:2 * C] * d + b64 * om
      Sb = torch.cat([b64.abs(), b64[C:].abs(), b64[C:].abs(), torch.ones(2, device=DEV, dtype=torch.float64)])
    s64 = n
    S = torch.maximum(S, torch.maximum(n.abs(), Sb))
  torch.cuda.synchronize()
  # each push rounds a handful of fp32 operations (renorm: a quotient and its square); errors add over the pushes
  return {'ema': conv_error_ratio(st, s64, S, ema_c(pushes))}


# ---------------------------------------------------------------------------------------------------------------------
# the product's launches, and the cases beside them
# ---------------------------------------------------------------------------------------------------------------------

# cases beside the product's: the scalar route (3 channels, no float4) and the 256-channel V = 2 route at 8x8, 4 samples
EXTRA_NORMS = set()
for _C, _flags in ((3, LRELU), (256, LRELU | PIXNORM), (64, LRELU | PIXNORM)):
  EXTRA_NORMS |= {('twg_moments', 4, 64, _C, 1), ('twg_moments', 4, 64, _C, 4),
                  ('twg_norm_act_fwd', 4, 64, _C, _flags, 'z'), ('twg_norm_act_bwd_reduce', 4, 64, 0, _C, _flags, 'gz'),
                  ('twg_norm_finalize', INSTANCE, 4, 4, 0, 64, _C, 'gamma0+beta0'),
                  ('twg_norm_finalize', BATCH, 4, 4, 0, 64, _C, 'gamma0+beta0+batch_stats'),
                  ('twg_norm_finalize', RENORM, 4, 4, 0, 64, _C, 'gamma0+beta0+renorm0+clip+rd+batch_stats')}
  for _kind in (INSTANCE, BATCH):
    EXTRA_NORMS.add(('twg_norm_act_bwd_apply', _kind, 4, 4, 0, 64, _C, 'gy+ggamma0+gbeta0'))
  EXTRA_NORMS.add(('twg_norm_act_bwd_apply', RENORM, 4, 4, 0, 64, _C, 'rd+gy+ggamma0+gbeta0'))

SUITE_NORM_KEYS = PRODUCT_NORM_KEYS | EXTRA_NORMS
_RUNNERS = {'twg_moments': _run_statistics, 'twg_norm_finalize': _run_statistics,
            'twg_norm_finalize_partials': _run_statistics, 'twg_norm_act_fwd': _run_forward,
            'twg_norm_act_bwd_reduce': _run_reduce, 'twg_norm_act_bwd_apply': _run_apply,
            'twg_norm_eval_affine': _run_eval_affine, 'twg_norm_update_stats': _run_update_stats}
_STAGE = {'twg_moments': 'statistics', 'twg_norm_finalize': 'statistics', 'twg_norm_finalize_partials': 'statistics',
          'twg_norm_act_fwd': 'forward', 'twg_norm_act_bwd_reduce': 'reduce', 'twg_norm_act_bwd_apply': 'apply',
          'twg_norm_eval_affine': 'evaluation', 'twg_norm_update_stats': 'ema'}


def _key_id(k):
  return '-'.join(str(v) for v in k).replace('twg_', '')


@pytest.mark.parametrize('key', sorted(SUITE_NORM_KEYS, key=str), ids=_key_id)
def test_normaliser_stage_against_fp64(built_lib, key):
  rec = _Recorder(built_lib)
  res = _RUNNERS[key[0]](key, rec)
  assert key in rec.keys(), (key, sorted(rec.keys()))
  _log_result({'test': 'norm_stage', 'stage': _STAGE[key[0]], 'key': list(key), 'ratios': res})
  bad = {k: v for k, v in res.items() if not v <= 1.0}
  assert not bad, (key, res)


def test_every_product_normaliser_launch_is_a_suite_case(built_lib):
  seen = norm_keys(harvest_product_launches())
  _log_result({'test': 'norm_coverage', 'harvested': len(seen), 'keys': sorted(seen, key=str)})
  assert seen == PRODUCT_NORM_KEYS, ('new', sorted(seen - PRODUCT_NORM_KEYS, key=str),
                                     'gone', sorted(PRODUCT_NORM_KEYS - seen, key=str))
  missing = sorted((k for k in seen if k not in SUITE_NORM_KEYS or k[0] not in _RUNNERS), key=str)
  assert not missing, missing


# ---------------------------------------------------------------------------------------------------------------------
# end to end: the fused layer against the oracle's fp64 chain
# ---------------------------------------------------------------------------------------------------------------------
def _layer_cases():
  """One case per pair of a product backward-apply key and a backward-reduce key of the same layer (N, HW, C): the
  normaliser layer at the product's N, group size, domain mask, gy route (fp32 / planes), accumulate, flags and pool
  fold."""
  applies = sorted((k for k in PRODUCT_NORM_KEYS if k[0] == 'twg_norm_act_bwd_apply'), key=str)
  reduces = sorted((k for k in PRODUCT_NORM_KEYS if k[0] == 'twg_norm_act_bwd_reduce'), key=str)
  return [(a, r) for a in applies for r in reduces if (r[1], r[2], r[4]) == (a[2], a[5], a[6])]


LAYER_CASES = _layer_cases()


@pytest.mark.parametrize('case', LAYER_CASES, ids=lambda c: _key_id(c[0][1:]) + '-' + _key_id(c[1][3:]))
def test_gen_layer_against_the_fp64_chain_at_every_product_key(built_lib, case):
  """ops.GenLayerFn (conv -> normaliser with per-domain gamma / beta -> leaky-ReLU -> pixel norm, optional 2x2 pool fold)
  forward and backward, as the step runs it, against the oracle's fp64 chain (O.instance_norm / O.batch_norm_train ->
  O.leaky_relu -> O.pixel_norm -> O.avg_pool2) evaluated per group from the device's own fp32 conv output y, with the
  device's active set passed through O.ACTIVE_SET; the conv gradients from the fp64 gy.  The parameter gradients go into
  gradient sinks that already hold a value (accumulate = 1) when the key says so.  Tolerances of the 8x8 test below."""
  from oracle import twingan_oracle as O
  from twingan_b200 import ops
  (_, kind, N, gs, dom_mask, HW, C, aopts), (_, _, _, Wp, _, flags, gin) = case
  ao, gin = set(aopts.split('+')), set(gin.split('+'))
  H = W = int(round(HW ** 0.5))
  assert H * W == HW and (not Wp or Wp == W)
  # the conv in front: a tensor-core 3x3 when gy goes to the next kernels as planes, an exact-fp32 1x1 otherwise
  Cin, k, pad = (C, 3, 1) if 'gy_planes' in ao else (3, 1, 0)
  assert ops.tc_eligible(N, H, W, Cin, C, k, pad) == ('gy_planes' in ao)
  x = torch.randn((N, H, W, Cin), device=DEV, generator=_gen(501))
  w = torch.randn((k, k, Cin, C), device=DEV, generator=_gen(502)) * (1.0 / (k * k * Cin) ** 0.5)
  gam = _params(C, 503)
  two = 'ggamma1' in ao
  params = gam if two else gam[:2]
  groups = N // gs
  y = ops._conv_fwd(x, w, k, pad)[0]
  yg = y.double().reshape(groups, gs, H, W, C)
  sd = yg.std(dim=(1, 2, 3), unbiased=False)
  snaps, clip, stats_out, ostats = [None, None], None, None, [None, None]
  if kind == RENORM:
    clip = torch.tensor(CLIP, device=DEV)
    stats_out = torch.empty((groups, 2, C), device=DEV)
    for d in (0, 1):
      ref_sd = sd[0] * 0.6
      rm = _vec(C, 510 + d, 0.02) * 0.6
      rsd = (ref_sd * (1 + 0.3 * _vec(C, 512 + d, 1.0).abs())).float()
      snaps[d] = torch.cat([torch.zeros(2 * C, device=DEV), rm, rsd, torch.tensor([0.6, 0.6], device=DEV)])
      ostats[d] = {'renorm_mean': rm.double(), 'renorm_stddev': rsd.double(),
                   'renorm_mean_weight': torch.tensor(0.6, dtype=torch.float64, device=DEV),
                   'renorm_stddev_weight': torch.tensor(0.6, dtype=torch.float64, device=DEV)}
  elif kind == BATCH:
    stats_out = torch.empty((groups, 2, C), device=DEV)
  acc = 'accumulate' in ao
  before = [_vec(C, 520 + i, 0.5) for i in range(len(params))]
  sinks = [b.clone() for b in before]
  saved = dict(ops._GRAD_SINKS)
  xd = x.clone().requires_grad_(True)
  wd = w.clone().requires_grad_(True)
  pd = [t.clone().requires_grad_(True) for t in params]
  if acc:
    ops.register_grad_sinks({p.data_ptr(): s_ for p, s_ in zip(pd, sinks)})
  pool = 'fp32' if 'gpool' in gin else None
  gz = torch.randn((N, H, W, C), device=DEV, generator=_gen(530)) if 'gz' in gin else None
  gp = torch.randn((N, H // 2, W // 2, C), device=DEV, generator=_gen(531)) if pool else None
  rec = _Recorder(built_lib)
  ops.ACTIVE_SET_TRACE = {'lrelu': [], 'l1': []}
  try:
    with rec.spying():
      ops.begin_step()
      out = ops.GenLayerFn.apply(xd, wd, pd[0], pd[1], pd[2] if two else None, pd[3] if two else None, k, pad, kind, flags,
                                 EPS[kind], clip, snaps[0], snaps[1] if two else None, stats_out, gs, dom_mask, 'G',
                                 'fp32', pool)
      z_d, pooled_d = out if pool else (out, None)
      outs = [o for o, g in ((z_d, gz), (pooled_d, gp)) if g is not None]
      grads_out = [g for g in (gz, gp) if g is not None]
      wrt = [xd, wd] + ([] if acc else pd)
      grads = torch.autograd.grad(outs, wrt, grads_out)
      torch.cuda.synchronize()
    trace = ops.ACTIVE_SET_TRACE
  finally:
    ops.ACTIVE_SET_TRACE = None
    ops._GRAD_SINKS.clear()
    ops._GRAD_SINKS.update(saved)
  launched = rec.keys()
  assert case[0] in launched and case[1] in launched, '%r\n%r' % (case, sorted(launched, key=str))
  # the fp64 chain on the device's y, per group with that group's domain variables
  y64 = y.double().requires_grad_(True)
  p64 = [t.double().requires_grad_(True) for t in params]
  us = []
  for g in range(groups):
    d = (dom_mask >> g) & 1
    ga, be = (p64[2], p64[3]) if d else (p64[0], p64[1])
    yg_ = y64[g * gs:(g + 1) * gs]
    if kind == INSTANCE:
      us.append(O.instance_norm(yg_, ga, be, EPS[kind]))
    else:
      us.append(O.batch_norm_train(yg_, ga, be, ostats[d], kind == RENORM,
                                   dict(zip(('rmin', 'rmax', 'dmax'), CLIP)), eps=EPS[kind]))
  z = torch.cat(us)
  O.ACTIVE_SET = {'lrelu': iter([t for _, t in trace['lrelu']]), 'l1': iter([]), 'flips': [0, 0]}
  try:
    if flags & LRELU:
      z = O.leaky_relu(z)
    assert next(O.ACTIVE_SET['lrelu'], None) is None
  finally:
    O.ACTIVE_SET = None
  if flags & PIXNORM:
    z = O.pixel_norm(z)
  refs, gouts = [z], [gz]
  if pool:
    refs.append(O.avg_pool2(z))
    gouts.append(gp)
  pairs = [(r, g.double()) for r, g in zip(refs, gouts) if g is not None]
  gy_ref, *gp_ref = torch.autograd.grad([r for r, _ in pairs], [y64] + p64, [g for _, g in pairs])
  x64 = x.double().requires_grad_(True)
  w64 = w.double().requires_grad_(True)
  gx_ref, gw_ref = torch.autograd.grad(O.conv2d_nhwc(x64, w64, 'SAME' if pad else 'VALID'), (x64, w64), gy_ref)
  torch.cuda.synchronize()
  res = {'z': rel_err(z_d, z), 'gx': rel_err(grads[0], gx_ref), 'gw': rel_err(grads[1], gw_ref)}
  if pool:
    res['pooled'] = rel_err(pooled_d, refs[1])
  got = [s_ - b for s_, b in zip(sinks, before)] if acc else grads[2:]
  for i, (gd, gr) in enumerate(zip(got, gp_ref)):
    res['param%d' % i] = rel_err(gd, gr)
  _log_result({'test': 'norm_layer_e2e', 'case': [list(case[0]), list(case[1])], 'rel_err': res})
  assert res['z'] < REL_TOL * 0.1 and res.get('pooled', 0.0) < REL_TOL * 0.1, res
  assert max(v for n, v in res.items() if n not in ('z', 'pooled')) < REL_TOL * 0.2, res


@pytest.mark.parametrize('kind', ['instance_norm', 'batch_norm', 'batch_renorm', 'none'])
@pytest.mark.parametrize('C,pix', [(16, True), (64, True), (256, True), (3, False), (32, False)])
def test_norm_act_layer_against_the_fp64_chain(built_lib, kind, C, pix):
  """normaliser + leaky-ReLU + pixel-norm, forward and backward through NormActFn, against the oracle's fp64 chain
  (4 samples at 8x8; the 3-channel scalar route and the 256-channel V = 2 route included)."""
  from oracle import twingan_oracle as O
  from twingan_b200 import ops
  from twingan_b200 import pggan_utils as pu
  from tests.test_gpu_kernels import _dev, _rand
  N, H, W = 4, 8, 8
  y = (_rand((N, H, W, C), 5) * 0.7 + 0.3).requires_grad_(True)
  gamma = (1 + _rand((C,), 6, 0.2)).requires_grad_(True)
  beta = _rand((C,), 7, 0.1).requires_grad_(True)
  gz = _rand((N, H, W, C), 8)
  clip = {'rmin': 0.9, 'rmax': 1.1, 'dmax': 0.1}
  stats = {'renorm_mean': _rand((C,), 9, 0.02) * 0.6, 'renorm_stddev': (0.3 + 0.1 * _rand((C,), 10).abs()) * 0.6,
           'renorm_mean_weight': torch.tensor(0.6, dtype=torch.float64),
           'renorm_stddev_weight': torch.tensor(0.6, dtype=torch.float64)}
  if kind == 'instance_norm':
    u = O.instance_norm(y, gamma, beta)
  elif kind == 'batch_norm':
    u = O.batch_norm_train(y, gamma, beta, None, False, None)
  elif kind == 'batch_renorm':
    u = O.batch_norm_train(y, gamma, beta, stats, True, clip)
  else:
    u = y + beta
  z = O.leaky_relu(u)
  if pix:
    z = O.pixel_norm(z)
  gy_ref, gg_ref, gb_ref = torch.autograd.grad(z, (y, gamma, beta), gz, allow_unused=True)

  yd = _dev(y.detach()).requires_grad_(True)
  gd = _dev(gamma.detach()).requires_grad_(True)
  bd = _dev(beta.detach()).requires_grad_(True)
  kid = pu._KIND[kind]
  flags = ops.FLAG_LRELU | (ops.FLAG_PIXNORM if pix else 0)
  snap = torch.zeros(4 * C + 2, device=DEV)
  snap[2 * C:3 * C] = _dev(stats['renorm_mean'])
  snap[3 * C:4 * C] = _dev(stats['renorm_stddev'])
  snap[4 * C] = 0.6
  snap[4 * C + 1] = 0.6
  bs = torch.empty((2, C), device=DEV)
  zd = ops.NormActFn.apply(yd, gd if kid != ops.NORM_NONE else None, bd, kid, flags, pu._EPS[kid], (0.9, 1.1, 0.1),
                           snap, bs if kid in (ops.NORM_BATCH, ops.NORM_RENORM) else None, 'G')
  grads = torch.autograd.grad(zd, (yd, gd, bd) if kid != ops.NORM_NONE else (yd, bd), _dev(gz))
  torch.cuda.synchronize()
  assert rel_err(zd, z) < REL_TOL * 0.1
  assert rel_err(grads[0], gy_ref) < REL_TOL * 0.2
  if kid != ops.NORM_NONE:
    assert rel_err(grads[1], gg_ref) < REL_TOL * 0.2
  assert rel_err(grads[-1], gb_ref) < REL_TOL * 0.2
