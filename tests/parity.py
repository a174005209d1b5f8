"""Parity harness: run the CUDA path (through the C-ABI) and the CPU oracle on identical seeded inputs and
compare.  Used by tests/test_gpu_*.py and __graft_entry__.smoke().  The oracle is the checker only."""
from __future__ import annotations

import math
import os
import sys

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


def run_step_parity(hw=8, batch=4, max_num_channels=32, norm='instance_norm', is_growing=False, alpha=0.5, seed=0,
                    prec=None, check_adam=True, verbose=False, tol=REL_TOL, global_step=0, batch_passes=True,
                    extra_flags=None, weight_scale=1.0, grad_floor=0.0, loose=None):
  """One TwinGAN G+D step on the device vs the fp64 oracle on identical seeded inputs.

  Gradients of a leaky-ReLU / L1 network are discontinuous where a pre-activation (pixel difference) crosses
  zero, and an element within rounding noise of the kink takes either slope in ANY finite-precision evaluation.
  Parity is therefore defined modulo the sub-gradient choice at the kink: the device run exports its active set
  (sign masks, test hook ops.ACTIVE_SET_TRACE) and the oracle is evaluated on the same side of every kink, after
  verifying that the two active sets differ only on elements within O.KINK_AMBIGUITY (1e-3 rms, the forward tolerance) of the kink.
  Every forward value, loss and gradient tensor must then agree within `tol` (1e-3, north_star)."""
  from twingan_b200 import ops, twingan
  if prec is not None:
    ops.set_precision(prec)
  # `extra_flags`: optional reference flags (SURVEY 8f-4) under the names both Flags and the oracle's Config use;
  # `weight_scale` multiplies the N(0, 0.02) conv / fc weights (equalized lr expects N(0, 1) weights)
  extra_flags = dict(extra_flags or {})
  cfg = oracle_config(hw, is_growing, alpha, max_num_channels, norm, global_step=global_step, **extra_flags)
  params = O.init_params(cfg, seed=1234 + seed, randomize_affine=True)
  if weight_scale != 1.0:
    params = {k: (v * weight_scale if k.endswith('/weights') else v) for k, v in params.items()}
  state = O.init_norm_state(cfg, seed=77 + seed)
  src, tgt, rand = O.make_inputs(cfg, batch, seed=seed)

  flags = twingan.Flags(train_image_size=hw, is_growing=is_growing, alpha_grow=alpha,
                        pggan_max_num_channels=max_num_channels, generator_norm_type=norm, global_step=global_step,
                        batch_passes=batch_passes, **extra_flags)
  model = twingan.GanModel(flags, device='cuda:0')
  model.variables.load_dict(params, state if state else None)
  dev = model.device
  f32 = lambda t: t.to(device=dev, dtype=torch.float32).contiguous()
  rand_d = {k: f32(v) for k, v in rand.items()}
  ops.ACTIVE_SET_TRACE = {'lrelu': [], 'l1': []}
  try:
    gl, dl, ends_d, stats = model.compute_gradients(f32(src), f32(tgt), rand_d)
    torch.cuda.synchronize()
    trace = ops.ACTIVE_SET_TRACE
  finally:
    ops.ACTIVE_SET_TRACE = None
  trace = twingan.GanModel.trace_in_reference_order(trace, batch)
  O.ACTIVE_SET = {'lrelu': iter(trace['lrelu']), 'l1': iter(trace['l1']), 'flips': [0, 0]}
  try:
    g_loss, d_loss, named, grads, ends, nets = O.step_gradients(cfg, params, state, src, tgt, rand)
    flips = tuple(O.ACTIVE_SET['flips'])
    assert next(O.ACTIVE_SET['lrelu'], None) is None and next(O.ACTIVE_SET['l1'], None) is None, 'call-order mismatch'
  finally:
    O.ACTIVE_SET = None

  details = {}
  worst = 0.0

  def add(name, e):
    nonlocal worst
    details[name] = e
    worst = max(worst, e)

  add('generator_loss', abs(gl.item() - g_loss.item()) / abs(g_loss.item()))
  add('discriminator_loss', abs(dl.item() - d_loss.item()) / abs(d_loss.item()))
  for k, v in named.items():
    add('loss/' + k, abs(model.last_losses[k].item() - v.item()) / max(abs(v.item()), 1e-12))
  for k in ('s_prime', 't_prime', 's_cycle', 't_cycle', 'enc_s', 'enc_t_prime', 'pred_real_s', 'pred_t_prime'):
    add('fwd/' + k, rel_err(ends_d[k], ends[k]))
  v = model.variables
  # `grad_floor` > 0: a gradient tensor is compared on the scale max(its own max, grad_floor * the largest gradient of
  # its optimiser group).  Needed where a gradient is an (almost) exact cancellation -- e.g. the critic loss
  # mean D(G) - mean D(x) w.r.t. a bias, or a residual shortcut's bias in front of a normalised toRGB (exactly zero) --
  # so that fp32 rounding residue of the cancelling sums is not divided by ~0.
  gmax = {}
  for name in v.offsets:
    grp = 'D' if name.startswith('discriminator') else 'G'
    gmax[grp] = max(gmax.get(grp, 0.0), float(grads[name].abs().max()))
  for name, (o, shape) in v.offsets.items():
    n = 1
    for s in shape:
      n *= s
    got = model.flat_grad[o:o + n].view(shape)
    ref = grads[name]
    floor = grad_floor * gmax['D' if name.startswith('discriminator') else 'G']
    if grad_floor > 0.0 and float(ref.abs().max()) < floor:
      add('grad/' + name, float((got.detach().double().cpu() - ref.double()).abs().max()) / floor)
    else:
      add('grad/' + name, rel_err(got, ref))
  if check_adam:
    # Adam kernel parity on IDENTICAL gradients (the device's own): m/(sqrt(v)+eps) is sign-like at step 1, so
    # feeding each side its own gradient would turn 1e-7 gradient noise into +-lr parameter differences.
    gdev = {}
    for name, (o, shape) in v.offsets.items():
      n = 1
      for s_ in shape:
        n *= s_
      gdev[name] = model.flat_grad[o:o + n].view(shape).detach().cpu().double()
    m = {k: torch.zeros_like(p) for k, p in params.items()}
    vv = {k: torch.zeros_like(p) for k, p in params.items()}
    t = 0
    p2 = {k: p.float().double() for k, p in params.items()}
    for names in (O.generator_variable_names(params), O.discriminator_variable_names(params)):
      t += 1
      for k in names:
        p2[k], m[k], vv[k] = O.adam_apply(cfg, p2[k], gdev[k], m[k], vv[k], t)
    model.apply_gradients()
    got = model.variables.to_dict()
    upd_err = 0.0
    for k in p2:
      upd_err = max(upd_err, rel_err(got[k], p2[k]))
    add('adam/params', upd_err)
    if state:
      O.apply_stat_updates(cfg, state, nets)
      model.apply_stat_updates(stats)
      got_state = model.variables.state_to_dict()
      for k, val in state.items():
        add('state/' + k, rel_err(got_state[k], val))
  torch.cuda.synchronize()
  # `loose`: {substring of a detail name: tolerance} for entries known to be ill-conditioned in fp32 (documented at the caller)
  def tol_for(k):
    for sub, t in (loose or {}).items():
      if sub in k:
        return max(t, tol)
    return tol
  bad = {k: e for k, e in details.items() if not (e <= tol_for(k))}
  _log_result(dict(hw=hw, batch=batch, mc=max_num_channels, norm=norm, growing=is_growing, prec=ops.get_precision(),
                   batched=batch_passes, worst=worst, flips=flips, top=sorted(details.items(), key=lambda kv: -kv[1])[:5]))
  if verbose:
    top = sorted(details.items(), key=lambda kv: -kv[1])[:8]
    print('[parity] hw=%d B=%d mc=%d norm=%s growing=%s prec=%d seed=%d kink_flips=%d/%d worst=%.3e' %
          (hw, batch, max_num_channels, norm, is_growing, ops.get_precision(), seed, flips[0], flips[1], worst))
    for k, e in top:
      print('   %-70s %.3e' % (k, e))
  return {'ok': not bad, 'worst': worst, 'bad': bad, 'details': details, 'seed': seed, 'kink_flips': flips}
