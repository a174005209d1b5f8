"""Calibration of the normaliser bounds (tests/parity.py norm_sum_c, mean_bound, rstd_rel_bound) on the CPU.

The statistics kernels add in a fixed order: within one block per sample, the thread of pixel group `grp` adds the pixels
grp, grp + 256/G, grp + 2 * 256/G, ... serially in fp32 (G = lanes per pixel, vec_geom(C) in twg_common.cuh), the
squares with one rounding (fma); a shared-memory tree then halves the 256/G partials.  The batch kinds add the per-sample
sums serially over the group; the conv-epilogue route merges per-warp records {count, pivot, sum (y - pivot),
sum (y - pivot)^2} as k_norm_finalize_inst_partials does, 32 lanes each striding over the slots, then a butterfly.  This
file emulates that arithmetic in numpy float32 and shows, at every audited geometry, for random data and for mean 10 /
std 0.05, that it stays 4x inside the bounds the GPU suite holds the kernels to, and that a pixel dropped from a sum, the
pivot of the wrong sample, a skipped record, the single-pass unshifted variance and a pool gradient read from row h
instead of h >> 1 each exceed them by more than 4x.  The backward apply (gy, and the parameter gradients the serial sums
over samples and groups of k_norm_bwd_coeffs / k_norm_bwd_coeffs_inst form) and the EMA recurrence are emulated too, at
every audited apply geometry, against the bounds the GPU suite uses for them."""
import math

import numpy as np
import pytest
import torch

from tests.parity import (U32, conv_error_ratio, ema_c, exact_elem_c, mean_bound, norm_sum_c, rstd_rel_bound,
                          serial_run)
from tests.product_norms import PRODUCT_NORM_KEYS

MARGIN = 4.0
F32 = np.float32
EPS = {'instance': 1e-6, 'batch': 1e-3}


def lanes_per_pixel(C):
  """G of vec_geom(C): lanes that share one pixel's C / 4 float4s; 0 for the scalar route (C % 4 != 0)."""
  return min(C // 4, 32) if C % 4 == 0 else 0


def _butterfly(v):
  """warp_sum over axis 0 of v [32 * k, ...]: lane sums by xor shuffles 16 .. 1, within each warp."""
  w = v.reshape(-1, 32, *v.shape[1:])
  for off in (16, 8, 4, 2, 1):
    w = w + w[:, np.arange(32) ^ off]
  return w[:, 0]


def _audited(entry):
  return sorted({k for k in PRODUCT_NORM_KEYS if k[0] == entry})


# (HW, C, group size) of every statistics pass the product runs through twg_moments: pivot_group 1 is instance norm
MOMENT_GEOMS = sorted({(k[2], k[3], k[4]) for k in _audited('twg_moments')})
# (HW, C, slots) of every epilogue-record merge
RECORD_GEOMS = sorted({(k[4] * k[5], k[7], k[8]) for k in _audited('twg_norm_finalize_partials')})


def emu_sum(terms, G, square=False):
  """fp32 sum over the pixels (axis 0) of terms [HW, C] in the kernels' order; `square`: sum of terms^2, each added with
  one rounding (the fma of acc + d * d)."""
  HW, C = terms.shape
  gpb = 256 // G if G else 256      # scalar route: 256 threads stride over the pixels, then block_sum
  K = -(-HW // gpb)
  t = np.zeros((K * gpb, C), F32)
  t[:HW] = terms
  t = t.reshape(K, gpb, C)
  acc = np.zeros((gpb, C), F32)
  for k in range(K):
    if square:
      acc = (acc.astype(np.float64) + t[k].astype(np.float64) ** 2).astype(F32)
    else:
      acc = acc + t[k]
  if not G:
    warps = np.zeros((32, C), F32)
    warps[:8] = _butterfly(acc)
    return _butterfly(warps)[0]
  h = gpb // 2
  while h >= 1:
    acc = acc[:h] + acc[h:2 * h]
    h //= 2
  return acc[0]


def emu_moments(y, pivot, G, drop_last=False):
  """{sum (y - p), sum (y - p)^2} of one sample y [HW, C] (fp32) around the pivot p [C] as k_moments_vec adds them."""
  d = (y[:-1] if drop_last else y) - pivot
  return emu_sum(d, G), emu_sum(d, G, square=True)


def emu_finalize(s1, s2, pivot, count, eps):
  inv = F32(1.0 / count)
  d1 = F32(s1 * inv)
  var = np.maximum(F32(F32(s2 * inv) - F32(d1 * d1)), F32(0))
  mean = F32(pivot + d1)
  rstd = (1.0 / np.sqrt(var.astype(np.float64) + eps)).astype(F32)
  return mean, rstd


def emu_records(y, slots, skip=None):
  """The epilogue records of one sample (modelled as equal pixel ranges, pivot = the range's first pixel, serial fp32 sums)
  merged as k_norm_finalize_inst_partials merges them; `skip`: one record left out.  Returns (mean, rstd)."""
  HW, C = y.shape
  per = HW // slots
  recs = []
  for s in range(slots):
    ys = y[s * per:(s + 1) * per]
    p = ys[0]
    d = ys - p
    s1 = np.zeros(C, F32)
    s2 = np.zeros(C, F32)
    for row in d:
      s1 = s1 + row
      s2 = (s2.astype(np.float64) + row.astype(np.float64) ** 2).astype(F32)
    recs.append((F32(per), p, s1, s2))
  p0 = recs[0][1]
  cn, sm, q = (np.zeros((32, C), F32) for _ in range(3))
  for s, (n, p, s1, s2) in enumerate(recs):
    if s == skip:
      continue
    lane = s % 32
    d = F32(p - p0)
    cn[lane] = cn[lane] + n
    sm[lane] = sm[lane] + (d.astype(np.float64) * n + s1).astype(F32)
    t = (d.astype(np.float64) * n + F32(2) * s1).astype(F32)
    q[lane] = q[lane] + (s2 + d.astype(np.float64) * t).astype(F32)
  for off in (16, 8, 4, 2, 1):
    idx = np.arange(32) ^ off
    cn, sm, q = cn + cn[idx], sm + sm[idx], q + q[idx]
  inv = F32(1) / cn[0]
  dm = F32(sm[0] * inv)
  var = np.maximum(F32(F32(q[0] * inv) - F32(dm * dm)), F32(0))
  return F32(p0 + dm), (1.0 / np.sqrt(var.astype(np.float64) + EPS['instance'])).astype(F32)


def _data(HW, C, samples, seed, offset):
  """fp32 samples [samples, HW, C]: N(0.3, 0.7), or every other channel at mean 10, std 0.05 (|mean| >> std)."""
  g = np.random.default_rng(seed)
  y = g.standard_normal((samples, HW, C)) * 0.7 + 0.3
  if offset:
    y[..., 1::2] = g.standard_normal((samples, HW, C // 2)) * 0.05 + 10.0
  return y.astype(F32)


def _ref_stats(y64):
  """Two-pass fp64 moments over axis 0 (and over the samples of a group, axis 0 after reshaping)."""
  mean = y64.mean(0)
  return mean, ((y64 - mean) ** 2).mean(0)


def _stat_ratios(mean, rstd, y64, pivot, R, eps, samples=1):
  m_ref, var = _ref_stats(y64)
  rs_ref = 1.0 / np.sqrt(var + eps)
  kappa = 1.0 + (m_ref - pivot) ** 2 / var
  rm = np.abs(mean - m_ref) / mean_bound(R, np.abs(y64 - pivot).mean(0), m_ref, samples)
  rr = np.abs(rstd - rs_ref) / (rs_ref * rstd_rel_bound(R, kappa, var, eps, samples))
  return float(rm.max()), float(rr.max())


def _sum_ratio(s, y64, pivot, square, R):
  d = y64 - pivot
  ref = (d * d if square else d).sum(0)
  S = (d * d if square else np.abs(d)).sum(0)
  return conv_error_ratio(torch.from_numpy(np.asarray(s, np.float64)), torch.from_numpy(ref), torch.from_numpy(S),
                          norm_sum_c(R))


def test_the_audited_geometries_are_known():
  assert MOMENT_GEOMS and RECORD_GEOMS


@pytest.mark.parametrize('offset', [False, True])
@pytest.mark.parametrize('geom', MOMENT_GEOMS)
def test_moments_model_is_within_the_bound_and_kernel_bugs_are_not(geom, offset):
  HW, C, gs = geom
  G = lanes_per_pixel(C)
  samples = gs if gs > 1 else 4                  # a whole group of the batch kinds, or four instance-norm samples
  y = _data(HW, C, samples, 7 + HW + C, offset)
  y64 = y.astype(np.float64)
  eps = EPS['instance' if gs == 1 else 'batch']
  R = serial_run(HW, C)
  pivot = y[0, 0]
  sums = [emu_moments(y[n], pivot if gs > 1 else y[n, 0], G) for n in range(samples)]
  # each sample's sums, against fp64 around the same pivot
  model = max(_sum_ratio(sums[n][sq], y64[n], (pivot if gs > 1 else y[n, 0]).astype(np.float64), sq, R)
              for n in range(samples) for sq in (0, 1))
  assert model <= 1.0 / MARGIN, model
  # mean and rstd after the finalize (instance: per sample; batch: over the group, summed serially over its samples)
  if gs == 1:
    stats = [_stat_ratios(*emu_finalize(*sums[n], y[n, 0], HW, eps), y64[n], y64[n, 0], R, eps) for n in range(samples)]
  else:
    s1, s2 = sums[0]
    for n in range(1, samples):
      s1, s2 = s1 + sums[n][0], s2 + sums[n][1]
    m, rs = emu_finalize(s1, s2, pivot, HW * samples, eps)
    stats = [_stat_ratios(m, rs, y64.reshape(-1, C), y64[0, 0], R, eps, samples)]
  worst = max(max(s) for s in stats)
  assert worst <= 1.0 / MARGIN, (worst, stats)
  # the last pixel of each sample left out of its sums
  piv = [pivot if gs > 1 else y[n, 0] for n in range(samples)]
  s_drop = [emu_moments(y[n], piv[n], G, drop_last=True) for n in range(samples)]
  drop = max(_sum_ratio(s_drop[n][sq], y64[n], piv[n].astype(np.float64), sq, R) for n in range(samples) for sq in (0, 1))
  assert drop >= MARGIN, drop
  # the pivot of the next sample (the finalize still adds the right sample's pivot back)
  wrong = emu_finalize(*emu_moments(y[0], y[1, 0], G), y[0, 0], HW, eps)
  assert max(_stat_ratios(*wrong, y64[0], y64[0, 0], R, eps)) >= MARGIN
  if offset:
    # single-pass unshifted variance E[y^2] - E[y]^2 (pivot 0), judged with the condition of the pivot it should have used
    m0, rs0 = emu_finalize(*emu_moments(y[0], np.zeros(C, F32), G), F32(0), HW, eps)
    assert _stat_ratios(m0, rs0, y64[0], y64[0, 0], R, eps)[1] >= MARGIN


@pytest.mark.parametrize('offset', [False, True])
@pytest.mark.parametrize('geom', RECORD_GEOMS)
def test_epilogue_record_merge_is_within_the_bound_and_a_skipped_record_is_not(geom, offset):
  HW, C, slots = geom
  y = _data(HW, C, 1, 11 + HW + C, offset)[0]
  y64 = y.astype(np.float64)
  p0 = y64[0]
  R = HW / slots                         # the records' own serial runs
  model = _stat_ratios(*emu_records(y, slots), y64, p0, R, EPS['instance'])
  assert max(model) <= 1.0 / MARGIN, model
  skipped = _stat_ratios(*emu_records(y, slots, skip=slots // 2), y64, p0, R, EPS['instance'])
  assert max(skipped) >= MARGIN, skipped


@pytest.mark.parametrize('geom', [g for g in MOMENT_GEOMS if g[0] >= 16])
def test_pool_gradient_from_the_wrong_row_exceeds_the_gu_bound(geom):
  """gu = gz + 0.25 gpool[h >> 1][w >> 1] with one rounding per element is exact to u |gu|; row h (mod H/2) instead of
  h >> 1 is not."""
  HW, C, _ = geom
  H = W = int(math.isqrt(HW))
  g = np.random.default_rng(HW + C)
  gz = g.standard_normal((H, W, C)).astype(F32)
  gp = g.standard_normal((H // 2, W // 2, C)).astype(F32)
  h, w = np.arange(H)[:, None], np.arange(W)[None, :]
  ref = gz.astype(np.float64) + 0.25 * gp[h >> 1, w >> 1].astype(np.float64)
  S = np.abs(gz.astype(np.float64)) + 0.25 * np.abs(gp[h >> 1, w >> 1].astype(np.float64))
  c = exact_elem_c(C)
  model = (gz + F32(0.25) * gp[h >> 1, w >> 1]).astype(np.float64)
  assert float((np.abs(model - ref) / (c * S)).max()) <= 1.0 / MARGIN
  wrong = (gz + F32(0.25) * gp[h % (H // 2), w >> 1]).astype(np.float64)
  assert float((np.abs(wrong - ref) / (c * S)).max()) >= MARGIN
  assert c >= 8 * U32


# (kind, N, group size, domain mask, C) of every backward apply the product runs
APPLY_GEOMS = sorted({(k[1], k[2], k[3], k[4], k[6]) for k in _audited('twg_norm_act_bwd_apply')})


def _f(v):
  return np.asarray(v, F32)


@pytest.mark.parametrize('geom', APPLY_GEOMS)
def test_backward_apply_and_parameter_gradients_are_within_their_bounds(geom):
  """k_norm_bwd_coeffs(_inst) and k_norm_act_bwd_apply in fp32, in their order: per group t = serial sum of the samples'
  red, k = t / M; gamma += r t2 + d t1 and beta += t1 over the groups of each domain (instance norm: each sample's t2, t1
  added onto the buffer in turn); gy = a (gu - k1 - (y - mean) rstd k2) per element (on 256 pixels per sample: the
  arithmetic is per element)."""
  kind, N, gs, dom_mask, C = geom
  HW = 1024
  g = np.random.default_rng(N + C + kind)
  red = _f(g.standard_normal((N, 2, C)) * 20)
  rd = np.stack([_f(1 + 0.05 * g.standard_normal((N // gs, C))), _f(0.05 * g.standard_normal((N // gs, C)))], 1)
  if kind != 3:
    rd = np.stack([np.ones((N // gs, C), F32), np.zeros((N // gs, C), F32)], 1)
  before = _f(g.standard_normal((2, 2, C)))                      # [domain][gamma, beta]
  out = before.copy()
  r64, rd64 = red.astype(np.float64), rd.astype(np.float64)
  ref, S = before.astype(np.float64), np.abs(before.astype(np.float64))
  inv = F32(1.0 / (HW * (1 if kind == 1 else gs)))
  k = np.zeros_like(red)
  acc = np.zeros((2, 2, C), F32)
  for grp in range(N // gs):
    dom = (dom_mask >> grp) & 1
    ns = range(grp * gs, (grp + 1) * gs)
    if kind == 1:
      for n in ns:
        out[dom, 0] = out[dom, 0] + red[n, 1]
        out[dom, 1] = out[dom, 1] + red[n, 0]
        k[n] = red[n] * inv
    else:
      t = np.zeros((2, C), F32)
      for n in ns:
        t = t + red[n]
      acc[dom, 0] = acc[dom, 0] + _f(rd[grp, 0] * t[1] + _f(rd[grp, 1] * t[0]))
      acc[dom, 1] = acc[dom, 1] + t[0]
      for n in ns:
        k[n] = t * inv
    for n in ns:
      ref[dom, 0] += r64[n, 1] * rd64[grp, 0] + r64[n, 0] * rd64[grp, 1]
      ref[dom, 1] += r64[n, 0]
      S[dom, 0] += abs(r64[n, 1] * rd64[grp, 0]) + abs(r64[n, 0] * rd64[grp, 1])
      S[dom, 1] += abs(r64[n, 0])
  if kind != 1:
    out = before + acc
  c = exact_elem_c(N).item()
  assert float((np.abs(out - ref) / (c * S + 1e-30)).max()) <= 1.0 / MARGIN
  # gy on 256 pixels per sample, with k from the emulated coefficients
  P = 256
  y = _data(P, C, N, N + C, True)
  mean, rstd, a = _f(y.mean(1) + 0.01), _f(1.0 / y.std(1)), _f(g.standard_normal((N, C)))
  gu = _f(g.standard_normal((N, P, C)))
  yh = _f(_f(y - mean[:, None]) * rstd[:, None])
  gy = a[:, None] * _f(_f(gu - k[:, None, 0]) - _f(yh * k[:, None, 1]))
  if kind == 1:
    t1, t2, A1, A2 = r64[:, 0], r64[:, 1], np.abs(r64[:, 0]), np.abs(r64[:, 1])
  else:
    grp = lambda v: v.reshape(N // gs, gs, C).sum(1).repeat(gs, 0)
    t1, t2, A1, A2 = grp(r64[:, 0]), grp(r64[:, 1]), grp(np.abs(r64[:, 0])), grp(np.abs(r64[:, 1]))
  M = HW * (1 if kind == 1 else gs)
  k1, k2 = (t1 / M)[:, None], (t2 / M)[:, None]
  y64, a64 = y.astype(np.float64), a.astype(np.float64)[:, None]
  yh64 = (y64 - mean.astype(np.float64)[:, None]) * rstd.astype(np.float64)[:, None]
  ref = a64 * (gu - k1 - yh64 * k2)
  S = np.abs(a64) * (np.abs(gu) + np.abs(k1) + np.abs(yh64 * k2) + (A1 / M)[:, None] + np.abs(yh64) * (A2 / M)[:, None])
  c = exact_elem_c(gs if kind != 1 else 1).item()
  assert float((np.abs(gy - ref) / (c * S)).max()) <= 1.0 / MARGIN


@pytest.mark.parametrize('kind', [2, 3])
def test_ema_pushes_are_within_their_bound(kind):
  """k_norm_update_stats in fp32 over five pushes against the fp64 recurrence, bound ema_c(pushes) of the running
  magnitudes (the GPU suite's check)."""
  C, d, eps, pushes = 256, F32(0.99 if kind == 3 else 0.999), F32(1e-3), 5
  g = np.random.default_rng(kind)
  st = np.concatenate([_f(g.standard_normal(C)), _f(np.abs(g.standard_normal(C)) * 0.3 + 0.2), _f(g.standard_normal(C)),
                       _f(np.abs(g.standard_normal(C)) * 0.3 + 0.2), _f([0.7, 0.8])])
  s64 = st.astype(np.float64)
  S = np.abs(s64)
  om, om64 = F32(1) - d, 1.0 - float(d)
  for _ in range(pushes):
    bs = np.concatenate([_f(g.standard_normal(C) + 0.5), _f(np.abs(g.standard_normal(C)) * 0.3 + 0.1)])
    b64 = bs.astype(np.float64)
    n = s64.copy()
    if kind == 3:
      wm, ws = st[4 * C] * d + om, st[4 * C + 1] * d + om
      nrm, nrs = st[2 * C:3 * C] * d + bs[:C] * om, st[3 * C:4 * C] * d + bs[C:] * om
      mean, std = nrm / wm, nrs / ws
      st[:C], st[C:2 * C] = st[:C] * d + mean * om, st[C:2 * C] * d + (std * std - eps) * om
      st[2 * C:3 * C], st[3 * C:4 * C], st[4 * C], st[4 * C + 1] = nrm, nrs, wm, ws
      n[2 * C:3 * C] = s64[2 * C:3 * C] * float(d) + b64[:C] * om64
      n[3 * C:4 * C] = s64[3 * C:4 * C] * float(d) + b64[C:] * om64
      n[4 * C:] = s64[4 * C:] * float(d) + om64
      m64, sd64 = n[2 * C:3 * C] / n[4 * C], n[3 * C:4 * C] / n[4 * C + 1]
      n[:C] = s64[:C] * float(d) + m64 * om64
      n[C:2 * C] = s64[C:2 * C] * float(d) + (sd64 * sd64 - float(eps)) * om64
      Sb = np.concatenate([np.abs(b64), b64[C:] ** 2, b64[C:] ** 2, np.ones(2)])
    else:
      st[:2 * C] = st[:2 * C] * d + bs * om
      n[:2 * C] = s64[:2 * C] * float(d) + b64 * om64
      Sb = np.concatenate([np.abs(b64), np.abs(b64[C:]), np.abs(b64[C:]), np.ones(2)])
    s64 = n
    S = np.maximum(S, np.maximum(np.abs(n), Sb))
  assert float((np.abs(st - s64) / (ema_c(pushes) * S)).max()) <= 1.0 / MARGIN
