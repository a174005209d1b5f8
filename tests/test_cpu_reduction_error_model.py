"""Calibration of the reduction bounds of test_gpu_elementwise_conformance.py on the CPU.

k_lrelu_bwd_colsum_vec, k_lrelu_bwd_colsum_pool_rows and k_colsum add in a fixed order: block b owns a chunk of rows, the
thread of pixel group `grp` adds the rows r0 + grp, r0 + grp + gpb, ... serially in fp32 (gpb = 256 / G pixel groups per
block, G = lanes per pixel from vec_geom(C)), block_tree_sum halves the gpb partials, and add_partials adds the nb block
partials in block order onto the output.  The grid-stride loss sums (k_l1, k_l1_groups, k_fanout_fwd) add every
(nb * 256)-th term per thread, then block_sum (a warp butterfly and a sum over the 8 warps), then add_partials.  The
gradient penalty's k_row_sumsq adds squares over each sample's chunks, add_partials adds the chunks and
k_grad_penalty_finalize forms sqrt, the coefficients and the loss; the DRAGAN perturbation's k_sum_sq adds all pixels and
their squares in one block and takes E[x^2] - m^2 in fp64; the minibatch-stddev cluster kernels take per-feature
two-pass statistics and sum over the features through the block and the cluster.  This file emulates each in numpy
float32 at every audited geometry (the columns of a column sum are independent, so four columns stand for C) and shows
that it stays 4x inside the bound the GPU suite holds the kernel to, while a dropped last row of each chunk, a skipped
partial block, a V = 2 column sum written to lane slot lg instead of lg + 32, a join backward that sums one skip use too
few, a skipped thread of the DRAGAN sums and an mbstd_bwd2 without its gm term each exceed it by more than 4x.  (A pool
fold read from the wrong row is caught by the GPU suite's bit-exact comparison of the fused backward's outputs.)"""
import numpy as np
import pytest
import torch

from tests.parity import (U32, dragan_var_rel_bound, grid_sum_c, mbstd_bwd2_ref, mbstd_fwd_ref, norm_sum_c, penalty_c_ss,
                          penalty_ref)
from tests.product_elementwise import (EXTRA_ELEMENTWISE, PRODUCT_ELEMENTWISE_KEYS, cdiv, colsum_geom, colsum_plain_geom,
                                       grid_for, penalty_geom, pool_rows_route, vec_geom)

MARGIN = 4.0
F32 = np.float32
COLS = 4


def _keys(entry):
  return sorted(k for k in PRODUCT_ELEMENTWISE_KEYS | EXTRA_ELEMENTWISE if k[0] == entry)


def _colsum_cases():
  """(rows, C, poolW, route) of every audited column sum: the fused backward's routes and twg_colsum."""
  cases = set()
  for _, rows, C, act, poolH, poolW, acc, opts in _keys('twg_lrelu_bwd_colsum'):
    o = set(opts.split('+'))
    route = 'rows' if pool_rows_route(C, act, poolW, 'out' in o, 'planes' in o) else ('vec' if vec_geom(C) else 'plain')
    cases.add((rows, C, poolW, route))
  for _, rows, C, _ in _keys('twg_colsum'):
    cases.add((rows, C, 0, 'plain'))
  return sorted(cases)


def _gpb(C, route):
  if route == 'plain':
    Cw = 1
    while Cw < C and Cw < 256:
      Cw <<= 1
    return 256 // Cw
  return 256 // vec_geom(C)[0]


def _rows_per_block(rows, C, poolW, route):
  """Rows of each block's chunk, as the host code splits them."""
  R, nb = colsum_geom(rows, C, poolW, route == 'rows') if route != 'plain' else colsum_plain_geom(rows, C)
  if route == 'rows':
    rpb = max(1, -(-(rows // poolW) // (8 * 132)))
    return rpb * poolW, R, nb
  return -(-rows // nb), R, nb


def emu_colsum(t, C, poolW, route, drop_last=False, skip_block=None):
  """fp32 column sums of t [rows, COLS] in the kernels' order.  On the pool-rows route a thread walks the pixels w = grp,
  grp + gpb, ... of each image row of its block in turn, which for whole rows is the same serial order as the flat form's
  row stride (W is a multiple of gpb there)."""
  rows = t.shape[0]
  chunk, R, nb = _rows_per_block(rows, C, poolW, route)
  gpb = _gpb(C, route)
  parts = []
  for b in range(nb):
    blk = t[b * chunk:min(rows, (b + 1) * chunk)]
    if drop_last:
      blk = blk[:-1]
    K = -(-blk.shape[0] // gpb)
    pad = np.zeros((K * gpb, t.shape[1]), F32)
    pad[:blk.shape[0]] = blk
    pad = pad.reshape(K, gpb, -1)
    acc = np.zeros((gpb, t.shape[1]), F32)
    for k in range(K):
      acc = acc + pad[k]
    h = gpb // 2
    while h >= 1:
      acc = acc[:h] + acc[h:2 * h]
      h //= 2
    parts.append(acc[0])
  s = np.zeros(t.shape[1], F32)
  for b, p in enumerate(parts):
    if b != skip_block:
      s = s + p
  return s, R, nb


def _terms(rows, seed):
  """The fused backward's terms g * slope: mixed sign, one column at mean 3 (so a missing row shows)."""
  g = np.random.default_rng(seed)
  t = g.standard_normal((rows, COLS))
  t[:, 1] += 3.0
  slope = np.where(g.standard_normal((rows, COLS)) > 0, 1.0, 0.2)
  return (t.astype(F32) * slope.astype(F32)).astype(F32)


def _ratio(s, t, c):
  t64 = t.astype(np.float64)
  return float((np.abs(s.astype(np.float64) - t64.sum(0)) / (c * np.abs(t64).sum(0))).max())


@pytest.mark.parametrize('case', _colsum_cases(), ids=lambda c: '-'.join(map(str, c)))
def test_column_sum_model_is_within_the_bound_and_kernel_bugs_are_not(case):
  rows, C, poolW, route = case
  t = _terms(rows, rows + C)
  s, R, nb = emu_colsum(t, C, poolW, route)
  c = norm_sum_c(R, samples=nb)
  model = _ratio(s, t, c)
  print('colsum %s: R %d, nb %d, model %.3g' % (case, R, nb, model))
  assert model <= 1.0 / MARGIN, model
  if rows >= 2 * _gpb(C, route) * nb:          # chunks of at least two rows per thread group
    drop = _ratio(emu_colsum(t, C, poolW, route, drop_last=True)[0], t, c)
    print('   dropped last row of each chunk %.3g' % drop)
    assert drop >= MARGIN, drop
  if nb > 1:
    skip = _ratio(emu_colsum(t, C, poolW, route, skip_block=nb - 1)[0], t, c)
    print('   skipped last partial block %.3g' % skip)
    assert skip >= MARGIN, skip
  if route == 'vec' and vec_geom(C)[1] == 2:
    # V = 2: lane lg's second float4 (channels 4 (lg + 32) ..) written to slot lg: column 0 receives column 1's sum,
    # column 1's slot keeps the zeroed partial
    wrong = np.array([s[1], 0.0, s[2], s[3]], F32)
    lane = _ratio(wrong, t, c)
    print('   V = 2 sum in slot lg %.3g' % lane)
    assert lane >= MARGIN, lane


@pytest.mark.parametrize('key', _keys('twg_upsample_concat_bwd'), ids=lambda k: '-'.join(map(str, k[1:])))
def test_join_backward_missing_a_skip_use_exceeds_its_bound(key):
  """gb = the serial sum of the N / Nb uses of each skip pixel, held to 2 (N / Nb) u of its S; one use too few is not."""
  _, N, H, W, Ca, Cb, Nb = key
  reps = N // Nb
  g = np.random.default_rng(N + H + Ca)
  uses = g.standard_normal((reps, 64)).astype(F32)
  c = 2 * reps * U32
  S = np.abs(uses.astype(np.float64)).sum(0)
  acc = uses[0].copy()
  for j in range(1, reps):
    acc = acc + uses[j]
  assert float((np.abs(acc - uses.astype(np.float64).sum(0)) / (c * S)).max()) <= 1.0 / MARGIN
  short = uses[:-1].astype(np.float64).sum(0)
  assert float((np.abs(short - uses.astype(np.float64).sum(0)) / (c * S)).max()) >= MARGIN


# ---------------------------------------------------------------------------------------------------------------------
# grid-stride loss sums
# ---------------------------------------------------------------------------------------------------------------------
def _f(v):
  return np.asarray(v, F32)


def _fma(a, b, c):
  """fmaf: the exact a b + c rounded once (a b of two fp32 values is exact in fp64)."""
  return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(F32)


def block_sum(v):
  """block_sum over axis -1 of v [..., T] (T = 32 k threads): a butterfly in each warp, then the warp sums in warp 0."""
  w = v.reshape(*v.shape[:-1], -1, 32)
  for off in (16, 8, 4, 2, 1):
    w = w + w[..., np.arange(32) ^ off]
  r = np.zeros((*v.shape[:-1], 32), F32)
  r[..., :w.shape[-2]] = w[..., 0]
  for off in (16, 8, 4, 2, 1):
    r = r + r[..., np.arange(32) ^ off]
  return r[..., 0]


def emu_grid_sum(vals, nb, wn, offset=0, skip_block=None):
  """wn * sum of vals [n] as a grid-stride kernel of nb blocks of 256 threads adds the items i = offset .. offset + n - 1
  (thread i % 256 of block (i / 256) % nb, serially in i), block_sum, the product by wn per block, then add_partials."""
  stride = nb * 256
  K = cdiv(offset + vals.shape[0], stride)
  pad = np.zeros(K * stride, F32)
  pad[offset:offset + vals.shape[0]] = vals
  pad = pad.reshape(K, nb, 256)
  acc = np.zeros((nb, 256), F32)
  for k in range(K):
    acc = acc + pad[k]
  parts = block_sum(acc) * F32(wn)
  s = F32(0)
  for b in range(nb):
    if b != skip_block:
      s = F32(s + parts[b])
  return s


def _l1_cases():
  cases = {('l1', n, grid_for(n, 8), 1) for _, n, _, _ in _keys('twg_l1')}
  cases |= {('l1_groups', per, grid_for(per, 8), 1) for _, _, per in _keys('twg_l1_groups')}
  cases |= {('fanout_fwd', B * per, grid_for(B * per, 2), 4) for _, B, per in _keys('twg_fanout_fwd')}
  return sorted(cases)


@pytest.mark.parametrize('case', _l1_cases(), ids=lambda c: '-'.join(map(str, c)))
def test_loss_sum_model_is_within_the_bound_and_a_skipped_block_is_not(case):
  """k_l1 / k_l1_groups add |a - b| per element; k_fanout_fwd adds, per float4 item, ((|d0| + |d1|) + |d2|) + |d3| and
  holds R = 4 terms per item (the GPU suite's R)."""
  name, n, nb, per_item = case
  g = np.random.default_rng(n)
  d = _f(g.standard_normal(n))
  terms = np.abs(d)
  if per_item == 4:
    q = terms.reshape(-1, 4)
    items = ((q[:, 0] + q[:, 1]) + q[:, 2]) + q[:, 3]
  else:
    items = terms
  wn = F32(F32(0.1) / F32(n))
  R = per_item * cdiv(items.shape[0], nb * 256)
  c = grid_sum_c(R, nb)
  ref = float(wn) * terms.astype(np.float64).sum()
  offsets = (0, items.shape[0]) if name == 'fanout_fwd' else (0,)      # the source and the target half of the batch
  for off in offsets:
    model = abs(float(emu_grid_sum(items, nb, wn, off)) - ref) / (c * ref)
    print('%s offset %d: R %d, nb %d, model %.3g' % (case, off, R, nb, model))
    assert model <= 1.0 / MARGIN, model
  if nb > 1:
    # the last block holds items of the second half only when the batch is small (k_fanout_fwd's grid covers all four
    # row blocks of gout): the mutant shows in whichever half it touches
    skip = max(abs(float(emu_grid_sum(items, nb, wn, off, skip_block=nb - 1)) - ref) / (c * ref) for off in offsets)
    assert skip >= MARGIN, skip


# ---------------------------------------------------------------------------------------------------------------------
# gradient penalty
# ---------------------------------------------------------------------------------------------------------------------
def _penalty_g(N, per, seed):
  """[N, per] fp32 gradients whose per-sample norms spread over 0.4 .. 1.6 (the GPU suite's inputs)."""
  s = np.linspace(0.4, 1.6, N)
  s = np.where(np.abs(s - 1) < 0.01, s + 0.05, s)
  g = np.random.default_rng(seed).standard_normal((N, per))
  return _f(g / np.linalg.norm(g, axis=1, keepdims=True) * s[:, None])


def emu_penalty(g, lam, drop_last=False, skip_block=None):
  """k_row_sumsq over each sample's chunks (fma squares, block_sum), add_partials onto the zeroed coefficients, then
  k_grad_penalty_finalize (one 64-thread block).  Returns (coef [N], loss)."""
  N, per = g.shape
  chunk, nb = penalty_geom(per)
  parts = np.zeros((nb, N), F32)
  for b in range(nb):
    blk = g[:, b * chunk:min(per, (b + 1) * chunk)]
    if drop_last:
      blk = blk[:, :-1]
    K = cdiv(blk.shape[1], 256)
    pad = np.zeros((N, K * 256), F32)
    pad[:, :blk.shape[1]] = blk
    pad = pad.reshape(N, K, 256)
    acc = np.zeros((N, 256), F32)
    for k in range(K):
      acc = _fma(pad[:, k], pad[:, k], acc)
    parts[b] = block_sum(acc)
  ss = np.zeros(N, F32)
  for b in range(nb):
    if b != skip_block:
      ss = ss + parts[b]
  s = np.sqrt(ss)
  t = s - F32(1)
  acc = np.zeros(64, F32)
  acc[:N] = _fma(t, t, np.zeros(N, F32))
  lam32, N32 = F32(lam), F32(N)
  coef = (lam32 * F32(2) * t) / (N32 * np.maximum(s, F32(1e-20)))
  loss = (lam32 * block_sum(acc)) / N32
  return coef.astype(F32), F32(loss)


@pytest.mark.parametrize('key', _keys('twg_grad_penalty'), ids=lambda k: '-'.join(map(str, k[1:])))
def test_gradient_penalty_model_is_within_the_bound_and_kernel_bugs_are_not(key):
  _, N, per, _ = key
  g = _penalty_g(N, per, per)
  lam = 0.25
  chunk, nb = penalty_geom(per)
  ss = torch.from_numpy((g.astype(np.float64) ** 2).sum(1))
  coef_ref, coef_b, loss_ref, loss_b = penalty_ref(ss, penalty_c_ss(chunk, nb), lam, N)

  def ratio(coef, loss):
    return max(float(((torch.from_numpy(coef.astype(np.float64)) - coef_ref).abs() / coef_b).max()),
               abs(float(loss) - float(loss_ref)) / float(loss_b))
  model = ratio(*emu_penalty(g, lam))
  print('penalty %s: chunk %d, nb %d, model %.3g' % (key, chunk, nb, model))
  assert model <= 1.0 / MARGIN, model
  if chunk >= 2 * 256:
    drop = ratio(*emu_penalty(g, lam, drop_last=True))
    print('   dropped last element of each chunk %.3g' % drop)
    assert drop >= MARGIN, drop
  if nb > 1:
    skip = ratio(*emu_penalty(g, lam, skip_block=nb - 1))
    print('   skipped last partial block %.3g' % skip)
    assert skip >= MARGIN, skip


# ---------------------------------------------------------------------------------------------------------------------
# DRAGAN variance
# ---------------------------------------------------------------------------------------------------------------------
def emu_dragan_var(x, skip_thread=None):
  """k_sum_sq (one block: thread t adds x[t + 256 k] and its square, the square with one rounding) and k_dragan_xhat's
  var = max(E[x^2] - m^2, 0) in fp64 from the two fp32 block sums, rounded to fp32."""
  n = x.shape[0]
  K = cdiv(n, 256)
  pad = np.zeros(K * 256, F32)
  pad[:n] = x
  pad = pad.reshape(K, 256)
  a1, a2 = np.zeros(256, F32), np.zeros(256, F32)
  for k in range(K):
    a1 = a1 + pad[k]
    a2 = _fma(pad[k], pad[k], a2)
  if skip_thread is not None:
    a1[skip_thread] = a2[skip_thread] = 0
  s1, s2 = float(block_sum(a1)), float(block_sum(a2))
  m = s1 / n
  return F32(max(s2 / n - m * m, 0.0))


@pytest.mark.parametrize('key', _keys('twg_dragan_xhat'), ids=lambda k: '-'.join(map(str, k[1:])))
def test_dragan_variance_model_is_within_the_bound_and_a_skipped_thread_is_not(key):
  """Real images in [0, 1] with one channel at 0.8 .. 0.9 (|mean| >> spread), as the GPU suite draws them."""
  _, N, per = key
  g = np.random.default_rng(per)
  x = g.random((N, per))
  x[:, 0::3] = x[:, 0::3] * 0.1 + 0.8
  x = _f(x).reshape(-1)
  x64 = x.astype(np.float64)
  m = x64.mean()
  var = ((x64 - m) ** 2).mean()
  R = cdiv(x.shape[0], 256)
  b = dragan_var_rel_bound(R, 1 + m * m / var) * var
  model = abs(float(emu_dragan_var(x)) - var) / b
  print('dragan %s: R %d, kappa %.3g, model %.3g' % (key, R, 1 + m * m / var, model))
  assert model <= 1.0 / MARGIN, model
  skip = abs(float(emu_dragan_var(x, skip_thread=255)) - var) / b
  print('   skipped thread %.3g' % skip)
  assert skip >= MARGIN, skip


# ---------------------------------------------------------------------------------------------------------------------
# minibatch stddev
# ---------------------------------------------------------------------------------------------------------------------
def _mb_x(N, P, C, seed):
  """[N, P, C] fp32: N(0.2, 1), every fourth channel from 1 at mean 10, std 0.05 (the GPU suite's inputs)."""
  g = np.random.default_rng(seed)
  x = g.standard_normal((N, P, C)) + 0.2
  x[..., 1::4] = g.standard_normal((N, P, len(range(1, C, 4)))) * 0.05 + 10.0
  return _f(x)


def cluster_sum(per_thread):
  """Sum of one value per thread of an 8-CTA cluster of 512 threads (per_thread [8 * 512]): block_sum in each CTA, then
  the CTAs' sums in rank order."""
  b = block_sum(per_thread.reshape(8, 512))
  s = F32(0)
  for r in range(8):
    s = F32(s + b[r])
  return s


def emu_mbstd_features(x):
  """Per feature of one group x [Ng, F] as k_mbstd_* forms them: m, d = x - m, v = sum d^2 (fma), var = v / Ng + 1e-8."""
  Ng = x.shape[0]
  m = np.zeros(x.shape[1], F32)
  for n in range(Ng):
    m = m + x[n]
  m = m / F32(Ng)
  d = x - m
  v = np.zeros(x.shape[1], F32)
  for n in range(Ng):
    v = _fma(d[n], d[n], v)
  return m, d, v


def _per_thread(vals):
  """One feature per thread of the cluster (F = 8 * 512 at the audited geometry)."""
  assert vals.shape[0] == 8 * 512
  return vals


@pytest.mark.parametrize('key', _keys('twg_mbstd_fwd'), ids=lambda k: '-'.join(map(str, k[1:])))
def test_mbstd_statistic_model_is_within_the_bound(key):
  _, N, P, C, Ct, groups, _ = key
  x = _mb_x(N, P, C, N)
  s_ref, bound = mbstd_fwd_ref(torch.from_numpy(x), groups)
  Ng, F = N // groups, P * C
  worst = 0.0
  for grp in range(groups):
    _, _, v = emu_mbstd_features(x[grp * Ng:(grp + 1) * Ng].reshape(Ng, F))
    sig = np.sqrt(v / F32(Ng) + F32(1e-8))
    s = cluster_sum(_per_thread(sig)) / F32(F)
    worst = max(worst, abs(float(s) - float(s_ref[grp])) / float(bound[grp]))
  print('mbstd_fwd %s: model %.3g' % (key, worst))
  assert worst <= 1.0 / MARGIN, worst


def emu_mbstd_bwd2(x, ggx, gstat, with_gm=True):
  """k_mbstd_bwd2 for one group: x, ggx [Ng, F], gstat [Ng P] (the statistic channel's gradient).  Returns (dG, dx)."""
  Ng, F = x.shape
  acc = np.zeros(512, F32)
  acc[:gstat.shape[0]] = gstat
  G = block_sum(acc)
  m, d, v = emu_mbstd_features(x)
  gm = np.zeros(F, F32)
  gd = np.zeros(F, F32)
  for n in range(Ng):
    gm = gm + ggx[n]
  gm = gm / F32(Ng)
  for n in range(Ng):
    gd = _fma(ggx[n], d[n], gd)
  var = v / F32(Ng) + F32(1e-8)
  sig = np.sqrt(var)
  k = F32(1) / (F32(Ng) * F32(F) * sig)
  dG = cluster_sum(_per_thread(_fma(gd, k, np.zeros(F, F32))))
  q = (d * gd) / (F32(Ng) * var)
  inner = (ggx - gm) - q if with_gm else ggx - q
  dx = (G * k) * inner
  return dG, dx


@pytest.mark.parametrize('key', _keys('twg_mbstd_bwd2'), ids=lambda k: '-'.join(map(str, k[1:])))
def test_mbstd_double_backward_model_is_within_the_bound_and_a_missing_gm_is_not(key):
  _, N, P, C, Ct, groups = key
  g = np.random.default_rng(N + 1)
  x = _mb_x(N, P, C, N + 2)
  ggx = _f(g.standard_normal((N, P, C)) + 0.3)
  gstat = _f(g.standard_normal((N, P)) + 0.5)
  dG_ref, dG_b, dx_ref, dx_b = mbstd_bwd2_ref(torch.from_numpy(x), torch.from_numpy(ggx), torch.from_numpy(gstat), groups)
  Ng, F = N // groups, P * C

  def ratios(with_gm):
    rdG = rdx = 0.0
    for grp in range(groups):
      sl = slice(grp * Ng, (grp + 1) * Ng)
      dG, dx = emu_mbstd_bwd2(x[sl].reshape(Ng, F), ggx[sl].reshape(Ng, F), gstat[sl].reshape(-1), with_gm)
      rdG = max(rdG, abs(float(dG) - float(dG_ref[grp])) / float(dG_b[grp]))
      rdx = max(rdx, float(((torch.from_numpy(dx.astype(np.float64)) - dx_ref[grp]).abs() / dx_b[grp]).max()))
    return rdG, rdx
  model = ratios(True)
  print('mbstd_bwd2 %s: dG %.3g, dx %.3g' % (key, *model))
  assert max(model) <= 1.0 / MARGIN, model
  no_gm = ratios(False)[1]
  print('   without gm: dx %.3g' % no_gm)
  assert no_gm >= MARGIN, no_gm
