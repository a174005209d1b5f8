"""Parity harness: run the CUDA path (through the C-ABI) and the CPU oracle on identical seeded inputs and
compare.  Used by tests/test_gpu_*.py and __graft_entry__.smoke().  The oracle is the checker only."""
from __future__ import annotations

import math
import os
import sys
from dataclasses import dataclass, replace

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
  sys.path.insert(0, ROOT)

from oracle import twingan_oracle as O  # noqa: E402

# north_star: "outputs match the reference ... within 1e-3 relative fp32"
REL_TOL = 1e-3


def rel_err(a: torch.Tensor, b: torch.Tensor) -> float:
  """||a-b||_inf / ||b||_inf (SURVEY 8d config 2)."""
  a = a.detach().double().cpu()
  b = b.detach().double().cpu()
  denom = b.abs().max().item()
  if denom == 0.0:
    return (a - b).abs().max().item()
  return (a - b).abs().max().item() / denom


def conv_error_ratio(dev: torch.Tensor, ref: torch.Tensor, S: torch.Tensor, c, tiny: float = 1e-30) -> float:
  """max over elements of |dev - ref| / (c * S + tiny): the check |dev - ref| <= c * S + tiny holds iff this is <= 1.

  S is the operation applied to the operands' absolute values (conv(|x|, |w|) for a forward), i.e. the sum of |products|
  each output element adds up.  Rounding errors of a sum are bounded relative to S, not to the output itself or to the
  largest output, so this holds every element to its own condition: border pixels, taps that read only padding (S = 0
  demands an exact 0) and small weight-gradient entries.  `c`: a number or a per-element tensor (tc_elem_c,
  exact_elem_c).  Compared in fp64 on `ref`'s device."""
  ref = ref.detach().double()
  dev = dev.detach().to(ref.device, torch.float64)
  S = S.detach().to(ref.device, torch.float64)
  if torch.is_tensor(c):
    c = c.detach().to(ref.device, torch.float64)
  return float(((dev - ref).abs() / (c * S + tiny)).max())


# Per-element bound c of conv_error_ratio on the tensor-core path, for an output that adds K >= 256 products.  Split-bf16
# operands (a = hi + lo, three MMAs per product) leave each product off by at most 3 * 2^-16 ~ 4.6e-5 relative, typically
# ~2^-18 and of either sign, so a long sum stays within ~5e-6 of S; a kernel that drops a cross term is off by > 1e-4 of S.
TC_ELEM_C = 2e-5


def tc_elem_c(K: torch.Tensor) -> torch.Tensor:
  """Per-element c of the tensor-core path for outputs that each add K products (K = the operation on all-ones operands).
  A short sum averages its products' rounding less: c grows like 1/sqrt(K) below K = 256, to 16 * TC_ELEM_C = 3.2e-4 at
  K = 1, 7x the worst split-bf16 error of a single product."""
  return TC_ELEM_C * torch.sqrt(256.0 / K.clamp(min=1.0)).clamp(min=1.0)


def exact_elem_c(K) -> torch.Tensor:
  """Per-element c of an exact-fp32 conv for outputs that each add K products: 4x the 2 u of rounding the fp64 operands to
  fp32, and 4x the sqrt(K) u statistical growth of K rounded additions, u = 2^-24."""
  return (8.0 + 4.0 * torch.as_tensor(K, dtype=torch.float64).sqrt()) * 2.0 ** -24


U32 = 2.0 ** -24   # unit roundoff of fp32


def serial_run(L, C) -> float:
  """Terms one thread of the normaliser's statistics / reduce kernels adds serially in a sum of L terms over C channels:
  256 threads per block, G = min(C / 4, 32) of them share a pixel (vec_geom), one thread per pixel on the scalar route
  (C % 4 != 0)."""
  G = min(C // 4, 32) if C % 4 == 0 else 1
  return max(1.0, L * G / 256.0)


def norm_sum_c(R, samples=1) -> float:
  """c of conv_error_ratio for an fp32 reduction whose threads each add R terms serially (serial_run), followed by a tree,
  and for the batch kinds by a serial sum of the `samples` per-sample sums of a group.  A serial run of same-sign terms is
  off by ~sqrt(R) u / 2 of its S at worst over the channels (the emulation in tests/test_cpu_norm_error_model.py);
  c = (16 + 2 sqrt(R) + 2 sqrt(samples)) u keeps that 4x inside at every audited geometry, while a pixel left out of a
  sum of 65536 terms (~1/65536 of S, more in the channel where that pixel is large) exceeds it 4x."""
  return (16.0 + 2.0 * math.sqrt(R) + 2.0 * math.sqrt(samples)) * U32


def dragan_var_rel_bound(R, kappa):
  """Bound on |var_dev - var| / var for the DRAGAN perturbation's variance over all pixels, taken as E[x^2] - m^2 from
  unshifted fp32 sums whose threads each add R terms (norm_sum_c(R) of their S each): the difference loses accuracy with
  the condition kappa = 1 + m^2 / var, E[x^2] + 2 m^2 = var (1 + 3 m^2 / var) <= 3 kappa var."""
  return 3.0 * (norm_sum_c(R) + U32) * kappa + 4.0 * U32


def unit_distance_bound(c_ss, s):
  """Bound on |(s_dev - 1) - (s - 1)| for s = sqrt(ss) of an fp32 sum of squares ss with c of conv_error_ratio `c_ss`:
  sqrt halves the relative error of ss and adds its own rounding, and the subtraction of 1 is exact or adds one more.
  Relative to |s - 1| this is ill-conditioned by s / |s - 1| (the gradient penalty's (||g|| - 1))."""
  return s * (0.5 * c_ss + 2.0 * U32)


def grid_sum_c(R, nb):
  """c of a grid-stride loss sum (k_l1, k_l1_groups, k_fanout_fwd): each thread adds R terms serially, block_sum over 256
  threads, one product by w / n per block, then add_partials adds the nb block partials in block order."""
  return norm_sum_c(R, nb) + 2 * U32


def penalty_c_ss(chunk, nb):
  """c of the per-sample sum of squares of twg_grad_penalty: k_row_sumsq's threads each add cdiv(chunk, 256) squares
  (one rounding each, the fma), a block_sum over 256 threads, then add_partials adds the nb blocks of a sample."""
  return norm_sum_c(-(-chunk // 256), nb * 256) + U32


def penalty_ref(ss, c_ss, lam, N):
  """fp64 coefficients lam 2 (s - 1) / (N s) and loss lam mean (s - 1)^2 of k_grad_penalty_finalize from the exact sums
  of squares ss [N], with their bounds when the device's sums carry c_ss (unit_distance_bound for s - 1; the quotient,
  products and the 64-thread block sum add a few roundings)."""
  s = ss.sqrt()
  e = unit_distance_bound(c_ss, s)
  coef = lam * 2 * (s - 1) / (N * s)
  coef_b = lam * 2 / (N * s) * (e + (s - 1).abs() * (0.5 * c_ss + 6 * U32))
  loss = lam * ((s - 1) ** 2).sum() / N
  loss_b = lam * (2 * (s - 1).abs() * e + 16 * U32 * (s - 1) ** 2).sum() / N
  return coef, coef_b, loss, loss_b


MB_CLUSTER, MB_THREADS = 8, 512   # k_mbstd_*: one cluster of 8 CTAs of 512 threads per group


def mbstd_stats(x, groups):
  """Per group and feature of x [N, P, C] (any device), fp64: d = x - mean over the group's samples, var (population),
  sigma = sqrt(var + 1e-8), and A = mean |x| (the scale of the fp32 mean's error), each [groups, Ng, F] or [groups, 1, F]."""
  N = x.shape[0]
  x64 = x.double().reshape(groups, N // groups, -1)
  m = x64.mean(1, keepdim=True)
  d = x64 - m
  var = (d * d).mean(1, keepdim=True)
  return d, var, (var + 1e-8).sqrt(), x64.abs().mean(1, keepdim=True)


def mbstd_sig_rel(Ng, A, var):
  """Relative bound on the fp32 sigma of one feature: the two-pass variance of Ng samples around an fp32 mean m + e
  (|e| <= Ng u A) adds sum (x - m - e)^2 = var Ng + Ng e^2 -- no first-order term -- plus Ng + 4 roundings; sqrt halves it."""
  return (Ng + 8) * U32 + 2 * (Ng * U32 * A) ** 2 / var


def mbstd_feature_sum_c(F):
  """c of a sum over the F features of one group: each thread of the cluster adds cdiv(F, 8 * 512) features serially,
  then a block_sum over 512 threads and the 8 CTAs' sums in rank order."""
  return norm_sum_c(-(-F // (MB_CLUSTER * MB_THREADS)), MB_CLUSTER * 32)


def mbstd_fwd_ref(x, groups):
  """fp64 statistic s [groups] of twg_mbstd_fwd on x [N, P, C] and its bound."""
  N, P, C = x.shape
  _, var, sig, A = mbstd_stats(x, groups)
  s = sig.mean(-1).reshape(groups)
  return s, (sig * mbstd_sig_rel(N // groups, A, var)).mean(-1).reshape(groups) + mbstd_feature_sum_c(P * C) * s


def mbstd_bwd2_ref(x, ggx, gstat, groups):
  """fp64 outputs of twg_mbstd_bwd2 on x, ggx [N, P, C] and the statistic channel's gradient gstat [N, P], with bounds:
  (dG [groups], its bound, dx [groups, Ng, F], its bound).  G = sum gstat is a block sum of Ng P terms; each feature's
  gd = sum ggx d reads d = x - (m + e) and so carries e sum ggx; dx = G k (ggx - gm - d gd / (Ng sigma^2)).  The
  last term is d/dx of 1 / sigma, sigma^2 = var + 1e-8: with few samples per group a feature's var can come near the 1e-8."""
  N, P, C = x.shape
  Ng, F = N // groups, P * C
  d, var, sig, A = mbstd_stats(x, groups)
  gg = ggx.double().reshape(groups, Ng, F)
  Agg = gg.abs().sum(1, keepdim=True)
  gs = gstat.double().reshape(groups, Ng * P)
  G, SG = gs.sum(1)[:, None, None], gs.abs().sum(1)[:, None, None]
  cG = norm_sum_c(-(-(Ng * P) // MB_THREADS), 16)
  k = 1.0 / (Ng * F * sig)
  gd = (gg * d).sum(1, keepdim=True)
  gm = gg.mean(1, keepdim=True)
  sr = mbstd_sig_rel(Ng, A, var)
  # e, the fp32 mean's error: a serial sum of Ng samples and a quotient, at worst (Ng + 3) / 2 u A.  With 3 .. 8 samples a
  # group (the stage runner's batches) the data reach that worst case on some feature, so the bound takes 4x it, the
  # margin exact_elem_c keeps over its worst case
  e_b = 2 * (Ng + 3) * U32 * A
  gd_err = (Ng + 4) * U32 * (gg * d).abs().sum(1, keepdim=True) + e_b * Agg
  dG = (gd * k).sum(-1).reshape(groups)
  dG_S = (gd.abs() * k).sum(-1).reshape(groups)
  dG_b = ((gd_err + (sr + 4 * U32) * gd.abs()) * k).sum(-1).reshape(groups) + mbstd_feature_sum_c(F) * dG_S
  sig2 = sig * sig
  inner = gg - gm - d * gd / (Ng * sig2)
  t3 = (d * gd / (Ng * sig2)).abs()
  inner_err = (4 * U32 * (gg.abs() + gm.abs() + t3) + U32 * Agg + e_b * gd.abs() / (Ng * sig2)
               + d.abs() * gd_err / (Ng * sig2) + t3 * (2 * sr + 6 * U32))
  dx_b = (G * k).abs() * inner_err + (cG * SG * k + (G * k).abs() * (sr + 6 * U32)) * inner.abs()
  return dG, dG_b, G * k * inner, dx_b


def mean_bound(R, abs_dev_mean, mean, samples=1):
  """Per-element bound on |mean_dev - mean_ref| for a mean taken from shifted sums with serial runs of R terms: the sum's
  bound on E|y - pivot| (`abs_dev_mean`), plus 4x the final rounding of pivot + E[y - pivot] (<= u |mean|)."""
  return norm_sum_c(R, samples) * abs_dev_mean + 4.0 * U32 * abs(mean)


def rstd_rel_bound(R, kappa, var, eps, samples=1):
  """Per-element bound on |rstd_dev - rstd_ref| / rstd_ref, rstd = 1 / sqrt(var + eps), var from shifted sums with serial
  runs of R terms (over `samples` samples).  The variance E[(y - p)^2] - E[y - p]^2 loses accuracy with the condition
  kappa = 1 + (mean - p)^2 / var of the pivot p: relative error <= 3 (norm_sum_c + u) kappa; rsqrt halves it and adds
  its own few ulp.  The single-pass unshifted form (p = 0) has kappa = 1 + mean^2 / var, 4e4 at mean 10, std 0.05, and
  breaks this bound; a pivot drawn from the data keeps kappa = O(1)."""
  return 1.5 * (norm_sum_c(R, samples) + U32) * kappa * var / (var + eps) + 4.0 * U32


def ema_c(pushes) -> float:
  """c of the EMA state after `pushes` pushes of k_norm_update_stats, relative to the running magnitudes of the state and
  the pushed statistics: each push rounds a handful of fp32 operations (renorm: a quotient and its square, ~8 u), and the
  errors add over the pushes; 16 u per push."""
  return 16.0 * U32 * pushes


def _log_result(rec):
  try:
    import json
    os.makedirs(os.path.join(ROOT, 'gpurun_out'), exist_ok=True)
    with open(os.path.join(ROOT, 'gpurun_out', 'parity_results.jsonl'), 'a') as f:
      f.write(json.dumps(rec) + '\n')
  except Exception:
    pass


def oracle_config(hw, is_growing, alpha, mc, norm, num_clones=1, global_step=0, **kw):
  return O.Config(hw=hw, is_growing=is_growing, alpha_grow=alpha, max_num_channels=mc, generator_norm_type=norm,
                  num_clones=num_clones, global_step=global_step, **kw)


@dataclass
class RefCounters:
  """The reference's counters, kept by its rules and never read back from the model: Adam's t advances per apply
  (model/model_inheritor.py:537-542), n_critic_counter per mode-A run (image_generation.py:622, 641-645), global_step per
  mode-B step and per mode-A generator turn (:648-651)."""
  adam_t: int = 0
  global_step: int = 0
  n_critic_counter: int = 0


def _by_name(v, flat):
  return {n: flat[o:o + math.prod(s)].view(s).detach().cpu().double() for n, (o, s) in v.offsets.items()}


def entry_state(model, renorm=True):
  """What a step starts from, read off the device in fp64: parameters, Adam slots and normaliser state under the
  reference's names (`renorm`: with the renorm_* entries, which only batch_renorm has), and the device step counters."""
  v = model.variables
  return {'params': _by_name(v, v.flat), 'adam_m': _by_name(v, v.adam_m), 'adam_v': _by_name(v, v.adam_v),
          'state': {k: t.detach().cpu().double() for k, t in v.state_to_dict(renorm).items()},
          'counters': model._counters.tolist()}


def _f32(x):
  return float(torch.tensor(float(x), dtype=torch.float32))


# c of the Adam kernel's m and v: a few roundings each, relative to the magnitudes of their two terms
ADAM_C = 8 * U32
# twg_step_schedule's lr_t (fp64 arithmetic on the fp32 flags, rounded to fp32) against lr_t of the exact flags
LR_REL = 1e-6


def adam_ref(cfg, p, g, m0, v0, t):
  """One apply of the fp32 Adam kernel at time t from the fp32 entry values p, m0, v0 and the gradient g (fp64 tensors):
  O.adam_apply on the flags as the kernel receives them (fp32), and bounds in the way of the Adam stage test's, for one
  apply from nonzero slots: m within ADAM_C of Ma = |b1 m0| + |(1 - b1) g|, v within ADAM_C of v (no cancellation), sqrt
  halves that; the quotient and the product add a few roundings, p's rounding one of |p'|, lr_t's rounding to fp32 one of
  the update.  Returns (update p' - p, m', v', bound on the update, Ma)."""
  c32 = replace(cfg, learning_rate=_f32(cfg.learning_rate), adam_beta1=_f32(cfg.adam_beta1),
                adam_beta2=_f32(cfg.adam_beta2), adam_eps=_f32(cfg.adam_eps))
  p1, m1, v1 = O.adam_apply(c32, p, g, m0, v0, t)
  b1, b2 = c32.adam_beta1, c32.adam_beta2
  lr_t = c32.learning_rate * math.sqrt(1 - b2 ** t) / (1 - b1 ** t)
  Ma = b1 * m0.abs() + (1 - b1) * g.abs()
  den = v1.sqrt() + c32.adam_eps
  upd = (p1 - p).abs()
  pe = lr_t * (ADAM_C * Ma / den + m1.abs() / den * (0.5 * ADAM_C + 4 * U32)) + 2 * U32 * (p1.abs() + upd)
  return p1 - p, m1, v1, pe, Ma


def lr_t(cfg, t):
  return cfg.learning_rate * math.sqrt(1 - cfg.adam_beta2 ** t) / (1 - cfg.adam_beta1 ** t)


class _Captured(object):
  """Runs `run()` with ops.ACTIVE_SET_TRACE on, keeping what the model's compute_gradients returned (the forward end points
  the entry points do not return)."""

  def __init__(self, model, run):
    from twingan_b200 import ops
    self.calls = []
    orig = model.compute_gradients

    def spy(*a, **k):
      out = orig(*a, **k)
      self.calls.append(out)
      return out
    model.compute_gradients = spy                # instance attribute: train_step's self.compute_gradients finds it
    ops.ACTIVE_SET_TRACE = {'lrelu': [], 'l1': []}
    try:
      self.result = run()
      torch.cuda.synchronize()
      self.trace = ops.ACTIVE_SET_TRACE
    finally:
      ops.ACTIVE_SET_TRACE = None
      del model.compute_gradients
    assert len(self.calls) == 1, 'the step computed its gradients %d times' % len(self.calls)


def check_step(model, run, cfg, sources, targets, rand, ref, alternating=False, n_critic=2, tol=REL_TOL, grad_floor=0.0,
               loose=None):
  """Run one real training step of `model` (`run()`: train_step, train_step_alternating, or whatever calls one of them)
  and hold it to the fp64 oracle evaluated once from the device's own entry state (teacher forcing: errors do not
  compound over steps, and any state the device carries from step to step and gets wrong shows on that step).

  `cfg`: the oracle configuration of the step, its global_step and alpha_grow those of the reference's counters `ref`
  (RefCounters at entry), which this advances by the reference's rules: a mode-B step applies the generator set at t + 1,
  the discriminator set at t + 2, global_step + 1; a mode-A run (`alternating`) applies the set of its turn
  (n_critic_counter % n_critic) at t + 1, n_critic_counter + 1, global_step + 1 on generator turns.

  Gradients of a leaky-ReLU / L1 network are discontinuous where a pre-activation (pixel difference) crosses
  zero, and an element within rounding noise of the kink takes either slope in ANY finite-precision evaluation.
  Parity is therefore defined modulo the sub-gradient choice at the kink: the device run exports its active set
  (sign masks, test hook ops.ACTIVE_SET_TRACE) and the oracle is evaluated on the same side of every kink, after
  verifying that the two active sets differ only on elements within O.KINK_AMBIGUITY (1e-3 rms, the forward tolerance) of
  the kink.  Every forward value, loss and gradient tensor must then agree within `tol` (1e-3, north_star), and so must
  the normaliser state after the EMA pushes.  Adam is compared on the device's own gradients (m / (sqrt(v) + eps) is
  sign-like on a fresh slot, so each side's own gradient would turn 1e-7 noise into +-lr_t differences): the update
  p' - p, m and v of each applying group against adam_ref's bounds; a group that does not apply keeps p, m and v bit for
  bit.  Counters: the device's {adam_t, global_step} equal the reference's after the step, lr_t of the step's applies
  matches the reference's t within LR_REL, and the renorm clipping is that of the reference's global_step.
  Returns {'ok', 'worst', 'bad', 'details', 'kink_flips', 'turn', 'result': what run() returned}."""
  from twingan_b200 import twingan
  renorm = cfg.generator_norm_type == O.BATCH_RENORM_TYPE
  entry = entry_state(model, renorm)
  cap = _Captured(model, run)
  _, _, ends_d, _ = cap.calls[0]
  B = int(sources.shape[0])
  d64 = lambda t: t.detach().cpu().double()
  src, tgt, rnd = d64(sources), d64(targets), {k: d64(t) for k, t in rand.items()}
  trace = twingan.GanModel.trace_in_reference_order(cap.trace, B)
  O.ACTIVE_SET = {'lrelu': iter(trace['lrelu']), 'l1': iter(trace['l1']), 'flips': [0, 0]}
  try:
    g_loss, d_loss, named, grads, ends, nets = O.step_gradients(cfg, entry['params'], entry['state'], src, tgt, rnd)
    flips = tuple(O.ACTIVE_SET['flips'])
    assert next(O.ACTIVE_SET['lrelu'], None) is None and next(O.ACTIVE_SET['l1'], None) is None, 'call-order mismatch'
  finally:
    O.ACTIVE_SET = None

  details, bounds, exact = {}, {}, []
  worst = 0.0

  def add(name, e):
    nonlocal worst
    details[name] = e
    worst = max(worst, e)

  # losses, forward end points, both gradient sets
  for k, ref_loss in (('generator_loss', g_loss), ('discriminator_loss', d_loss)):
    add(k, abs(model.last_losses[k].item() - ref_loss.item()) / abs(ref_loss.item()))
  for k, val in named.items():
    add('loss/' + k, abs(model.last_losses[k].item() - val.item()) / max(abs(val.item()), 1e-12))
  for k in ('s_prime', 't_prime', 's_cycle', 't_cycle', 'enc_s', 'enc_t_prime', 'pred_real_s', 'pred_t_prime'):
    add('fwd/' + k, rel_err(ends_d[k], ends[k]))
  v = model.variables
  gdev = _by_name(v, model.flat_grad)
  group_of = lambda name: 'D' if name.startswith('discriminator') else 'G'
  # `grad_floor` > 0: a gradient tensor is compared on the scale max(its own max, grad_floor * the largest gradient of
  # its optimiser group).  Needed where a gradient is an (almost) exact cancellation -- e.g. the critic loss
  # mean D(G) - mean D(x) w.r.t. a bias, or a residual shortcut's bias in front of a normalised toRGB (exactly zero) --
  # so that fp32 rounding residue of the cancelling sums is not divided by ~0.
  gmax = {}
  for name in v.offsets:
    gmax[group_of(name)] = max(gmax.get(group_of(name), 0.0), float(grads[name].abs().max()))
  for name in v.offsets:
    got, want = gdev[name], grads[name]
    floor = grad_floor * gmax[group_of(name)]
    if grad_floor > 0.0 and float(want.abs().max()) < floor:
      add('grad/' + name, float((got - want).abs().max()) / floor)
    else:
      add('grad/' + name, rel_err(got, want))

  # Adam, on the device's gradients from the device's entry slots, at the reference's t of each apply
  t0 = ref.adam_t
  if alternating:
    turn = O.alternating_turn(ref.n_critic_counter, n_critic)
    applies = {turn: t0 + 1}
    ref.adam_t, ref.n_critic_counter = t0 + 1, ref.n_critic_counter + 1
    ref.global_step += 1 if turn == 'G' else 0
    if isinstance(cap.result, tuple) and len(cap.result) == 3 and cap.result[2] != turn:
      exact.append('turn: the device applied %s, the reference %s' % (cap.result[2], turn))
  else:
    turn = None
    applies = {'G': t0 + 1, 'D': t0 + 2}
    ref.adam_t, ref.global_step = t0 + 2, ref.global_step + 1
  after = {'params': _by_name(v, v.flat), 'adam_m': _by_name(v, v.adam_m), 'adam_v': _by_name(v, v.adam_v)}
  for name in v.offsets:
    p0, m0, v0 = entry['params'][name], entry['adam_m'][name], entry['adam_v'][name]
    p1, m1, v1 = after['params'][name], after['adam_m'][name], after['adam_v'][name]
    grp = group_of(name)
    if grp not in applies:
      if not (torch.equal(p0, p1) and torch.equal(m0, m1) and torch.equal(v0, v1)):
        exact.append('%s moved on a %s turn' % (name, turn))
      continue
    dp, m_ref, v_ref, pe, Ma = adam_ref(cfg, p0, gdev[name], m0, v0, applies[grp])
    for k, r in (('adam/update/' + grp, conv_error_ratio(p1 - p0, dp, pe, 1.0)),
                 ('adam/m/' + grp, conv_error_ratio(m1, m_ref, Ma, ADAM_C)),
                 ('adam/v/' + grp, conv_error_ratio(v1, v_ref, v_ref, ADAM_C))):
      bounds[k] = max(bounds.get(k, 0.0), r)

  # normaliser state after the EMA pushes
  state_ref = dict(entry['state'])
  O.apply_stat_updates(cfg, state_ref, nets)
  got_state = v.state_to_dict(renorm)
  for k, val in state_ref.items():
    add('state/' + k, rel_err(got_state[k], val))

  # counters
  counters = model._counters.tolist()
  if counters != [ref.adam_t, ref.global_step]:
    exact.append('device counters %s, reference (adam_t, global_step) %s' % (counters, [ref.adam_t, ref.global_step]))
  if alternating and model.n_critic_counter != ref.n_critic_counter:
    exact.append('n_critic_counter %d, reference %d' % (model.n_critic_counter, ref.n_critic_counter))
  for i, lr_dev in enumerate(model._lr_dev.tolist()):
    want = lr_t(cfg, t0 + 1 + i)
    bounds['lr_t/%d' % i] = abs(lr_dev - want) / (LR_REL * want)
  clip = O.renorm_clipping(cfg.global_step)
  want_clip = [_f32(clip['rmin']), _f32(clip['rmax']), _f32(clip['dmax'])]
  if model._clip_dev.tolist() != want_clip:
    exact.append('renorm clipping %s, reference %s at global_step %d' % (model._clip_dev.tolist(), want_clip,
                                                                          cfg.global_step))

  def tol_for(k):
    # `loose`: {substring of a detail name: tolerance} for entries known to be ill-conditioned in fp32 (documented at the caller)
    for sub, t in (loose or {}).items():
      if sub in k:
        return max(t, tol)
    return tol
  bad = {k: e for k, e in details.items() if not (e <= tol_for(k))}
  bad.update({k: r for k, r in bounds.items() if not (r <= 1.0)})
  bad.update({'exact/%d' % i: msg for i, msg in enumerate(exact)})
  details.update(bounds)
  return {'ok': not bad, 'worst': worst, 'bad': bad, 'details': details, 'kink_flips': flips, 'turn': turn,
          'result': cap.result}


def run_step_parity(hw=8, batch=4, max_num_channels=32, norm='instance_norm', is_growing=False, alpha=0.5, seed=0,
                    prec=None, verbose=False, tol=REL_TOL, global_step=0, batch_passes=True, extra_flags=None,
                    weight_scale=1.0, grad_floor=0.0, loose=None):
  """One TwinGAN G+D step (GanModel.train_step) on the device from seeded parameters and normaliser state vs the fp64
  oracle on identical seeded inputs: check_step's comparison of losses, forward values, gradients, Adam applies,
  normaliser state and counters."""
  from twingan_b200 import ops, twingan
  if prec is not None:
    ops.set_precision(prec)
  # `extra_flags`: optional reference flags (SURVEY 8f-4) under the names both Flags and the oracle's Config use;
  # `weight_scale` multiplies the N(0, 0.02) conv / fc weights (equalized lr expects N(0, 1) weights)
  extra_flags = dict(extra_flags or {})
  cfg = oracle_config(hw, is_growing, alpha, max_num_channels, norm, global_step=global_step, **extra_flags)
  model, (src, tgt, rand) = seeded_model(cfg, batch, seed, weight_scale, batch_passes=batch_passes)
  res = check_step(model, lambda: model.train_step(src, tgt, rand), cfg, src, tgt, rand,
                   RefCounters(global_step=global_step), tol=tol, grad_floor=grad_floor, loose=loose)
  worst, details, flips = res['worst'], res['details'], res['kink_flips']
  _log_result(dict(hw=hw, batch=batch, mc=max_num_channels, norm=norm, growing=is_growing, prec=ops.get_precision(),
                   batched=batch_passes, worst=worst, flips=flips, top=sorted(details.items(), key=lambda kv: -kv[1])[:5]))
  if verbose:
    top = sorted(details.items(), key=lambda kv: -kv[1])[:8]
    print('[parity] hw=%d B=%d mc=%d norm=%s growing=%s prec=%d seed=%d kink_flips=%d/%d worst=%.3e' %
          (hw, batch, max_num_channels, norm, is_growing, ops.get_precision(), seed, flips[0], flips[1], worst))
    for k, e in top:
      print('   %-70s %.3e' % (k, e))
  res['seed'] = seed
  return res


def seeded_model(cfg, batch, seed=0, weight_scale=1.0, **flags):
  """A GanModel of `cfg` on cuda:0 loaded with seeded parameters (gamma / beta / biases randomised too) and normaliser
  state, and a seeded batch with its DRAGAN draws on the device.  `flags`: further twingan.Flags fields."""
  from twingan_b200 import twingan
  params = O.init_params(cfg, seed=1234 + seed, randomize_affine=True)
  if weight_scale != 1.0:
    params = {k: (v * weight_scale if k.endswith('/weights') else v) for k, v in params.items()}
  state = O.init_norm_state(cfg, seed=77 + seed)
  src, tgt, rand = O.make_inputs(cfg, batch, seed=seed)
  opt = {k: getattr(cfg, k) for k in ('equalized_learning_rate', 'wgan_drift_loss_weight', 'use_res_block',
                                      'loss_architecture', 'gradient_penalty_lambda', 'gan_weight', 'l_cyc_weight',
                                      'do_l_cyc_gan', 'l_content_weight', 'learning_rate', 'adam_beta1', 'adam_beta2')}
  f = twingan.Flags(train_image_size=cfg.hw, is_growing=cfg.is_growing, alpha_grow=cfg.alpha_grow,
                    pggan_max_num_channels=cfg.max_num_channels, generator_norm_type=cfg.generator_norm_type,
                    global_step=cfg.global_step, opt_epsilon=cfg.adam_eps, **opt, **flags)
  model = twingan.GanModel(f, device='cuda:0')
  model.variables.load_dict(params, state if state else None)
  f32 = lambda t: t.to(device=model.device, dtype=torch.float32).contiguous()
  return model, (f32(src), f32(tgt), {k: f32(v) for k, v in rand.items()})
