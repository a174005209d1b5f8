#!/usr/bin/env python
"""Where the time of the bench.py workload goes: one warmed-up eager model.train_step (256x256, 16 pairs, instance norm)
under torch.profiler with CUDA activities.

  python tools/profile_step.py --out DIR [--hw 256] [--batch 16]

Prints and writes to DIR:
  * kernels.json / the first table: every kernel name with its launches, total microseconds and share of the GPU time of
    the step (the sum of all kernel durations);
  * convs.json / the second table: every tensor-core conv launch of the step (entry point and geometry, recorded where
    twingan_b200.ops calls the library) matched to its kernel in the trace, with its time, FLOPs, algorithmic HBM bytes and
    the modelled L2 -> shared-memory operand bytes of the per-tap and the column-box kernels (conv_traffic);
  * fill.json / the third table: how much of the GPU each launch fills (its grid against one wave, 132 SMs times the CTAs
    one SM holds at the launch's registers, shared memory and block size), summed over the discriminator chains, which
    run one domain after the other on one stream: D_s / D_t ('Ds', 'Dt') and their DRAGAN penalty chains ('DRs', 'DRt'),
    forward and both backward passes (a backward node carries the chain of the forward call that made it).  For each
    chain: the time of the launches below one wave, the time of the last partial wave of the others, the idle share of
    the GPU over the chain's launches, and the upper bound of what running the two domains' chains side by side could
    save (launch i of D_s beside launch i of D_t: their two durations against the longer one and their summed work);
  * trace.json, the profiler's Chrome trace.
The card name and power limit are read in the same run.  TWG_LIB selects another build of the library.  Needs a GPU."""
from __future__ import annotations

import argparse
import collections
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
  sys.path.insert(0, ROOT)

_GEOM_AT = {'twg_conv_fwd_planes': 8, 'twg_conv_affine_act_fwd_planes': 7, 'twg_conv_dgrad_planes': 3,
            'twg_conv_wgrad_planes': 3}


# ---- the library's tile choices (twg_conv_tc.cu: pick_tile, chunk_for, the BN / BNW rules), restated for the model ----
def _pow2_le(v):
  p = 1
  while p * 2 <= v:
    p *= 2
  return p


def _tiles(N, H, W):
  TW = _pow2_le(min(W, 16))
  TH = _pow2_le(min(H, 128 // TW))
  TN = 128 // (TW * TH)
  return TW, TH, TN, -(-W // TW) * -(-H // TH) * -(-N // TN)


def _chunk(c):
  return 64 if c % 64 == 0 else (32 if c % 32 == 0 else 16)


def conv_traffic(entry, N, H, W, Cin, Cout, k, pad):
  """{'flops', 'hbm', 'l2_before', 'l2_after', 'cols'} of one tensor-core conv launch.
  flops: 2 MACs per product of the convolution (not the 3 split-bf16 MMAs).  hbm: algorithmic bytes, every operand read and
  every result written once (split planes 4 B per element, fp32 results 4 B).  l2_*: bytes the kernel's TMA loads move from
  L2 into shared memory, per CTA work item summed over the grid (resident weights: once per CTA), with the per-tap kernel
  (before) and the kernel the shape takes (after).  cols: the shape takes the column-box kernel."""
  TW, TH, TN, tiles = _tiles(N, H, W)
  taps, px = k * k, N * H * W
  flops = 2.0 * px * Cin * Cout * taps
  if entry == 'twg_conv_wgrad_planes':
    CN = _chunk(Cin)
    BNW = 64 if (Cout >= 64 and CN < 64) else (32 if Cout >= 32 else Cout)
    items = tiles * (Cout // BNW) * (Cin // CN)
    gy = 2 * 128 * BNW * 2                                       # gy tile, hi and lo planes
    before = items * (gy + taps * 2 * 128 * CN * 2)             # one x tile per tap
    cols = k == 3 and pad == 1 and TW == 16 and TH == 8 and TN == 1 and H >= 10
    after = items * (gy + 3 * 2 * 160 * CN * 2) if cols else before   # three {CN, 16, 10} column boxes per tile
    return {'flops': flops, 'hbm': 4.0 * px * (Cin + Cout) + 4.0 * taps * Cin * Cout, 'l2_before': float(before),
            'l2_after': float(after), 'cols': cols}
  K, Nc = (Cout, Cin) if entry == 'twg_conv_dgrad_planes' else (Cin, Cout)
  CC = _chunk(K)
  BN = min(Nc, 128)
  items = tiles * (Nc // BN)
  weights = taps * 2 * BN * K * 2                                 # one weight tile per (tap, chunk), hi and lo
  before = items * (taps * 2 * 128 * K * 2 + weights)            # one shifted 128-pixel A tile per (tap, chunk)
  cols = k == 3 and pad == 1 and K == CC and TW == 16 and TH == 8 and TN == 1 and H >= 10
  # the column-box keys with one small weight block (cols_resident) load it once per persistent CTA (one per SM)
  w_loads = min(items, 132) if cols and K <= 32 and BN <= 64 else items
  after = items * 3 * 2 * 160 * K * 2 + w_loads * weights if cols else before   # three {K, 16, 10} column boxes per tile
  return {'flops': flops, 'hbm': 4.0 * px * (K + Nc) + 4.0 * taps * K * Nc, 'l2_before': float(before),
          'l2_after': float(after), 'cols': cols}


# ---- launch fill: CTAs one SM of an H100 (sm_90) holds, from the launch's resources (the CUDA occupancy rules) ----
SMS = 132


def resident_ctas(threads, regs, smem):
  """CTAs of `threads` threads, `regs` registers per thread and `smem` bytes of shared memory one sm_90 SM holds."""
  warps = -(-threads // 32)
  by_warps = 64 // warps
  by_blocks = 32
  reg_warp = -(-max(regs, 1) * 32 // 256) * 256                # registers are allocated per warp in units of 256
  by_regs = (65536 // reg_warp) // warps
  by_smem = 233472 // (-(-(smem + 1024) // 128) * 128) if smem else by_blocks    # 1 KB per CTA is reserved
  return max(0, min(by_warps, by_blocks, by_regs, by_smem))


def launch_fill(grid, per_sm):
  """(waves, the launch's average share of the GPU's CTA slots, the share of its time spent in a last partial wave),
  every wave taken to last as long as the others."""
  wave = SMS * max(per_sm, 1)
  waves = -(-grid // wave)
  util = grid / float(waves * wave)
  tail = (1.0 / waves) if (grid % wave and waves > 1) else 0.0
  return waves, util, tail


def overlap_bound(a, b):
  """Upper bound of the time saved by running launch list `a` beside `b` (pairs in order, (us, util) each): a pair takes
  at least its longer launch and at least its summed work over the whole GPU."""
  saved = 0.0
  for (da, ua), (db, ub) in zip(a, b):
    saved += da + db - max(da, db, da * ua + db * ub)
  return saved


CHAINS = ('Ds', 'Dt', 'DRs', 'DRt')


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--out', required=True)
  ap.add_argument('--hw', type=int, default=256)
  ap.add_argument('--batch', type=int, default=16)
  ap.add_argument('--max-channels', type=int, default=256)
  ap.add_argument('--norm', default='instance_norm')
  ap.add_argument('--warmup', type=int, default=2)
  args = ap.parse_args()
  import torch
  from torch.profiler import ProfilerActivity, profile, record_function
  if not torch.cuda.is_available():
    raise SystemExit('profile_step.py needs a CUDA device')
  from bench import gpu_info
  from twingan_b200 import ops, twingan
  from twingan_b200._lib import lib, LIB_PATH
  ops.set_precision(1)
  dev = torch.device('cuda', 0)
  model = twingan.GanModel(twingan.Flags(train_image_size=args.hw, pggan_max_num_channels=args.max_channels,
                                         generator_norm_type=args.norm), device=dev, seed=1234)
  gen = torch.Generator(device=dev).manual_seed(100)
  s = torch.rand((args.batch, args.hw, args.hw, 3), device=dev, generator=gen)
  t = torch.rand((args.batch, args.hw, args.hw, 3), device=dev, generator=gen)
  r = twingan.make_dragan_rand(args.batch, args.hw, dev, gen)
  for _ in range(args.warmup):
    model.train_step(s, t, r)
  torch.cuda.synchronize()

  L = lib()
  calls = []
  call = L.call
  # the chain a launch belongs to: ops.trace_tag in the forward; in a backward, the tag its node was made under, which a
  # node made during that backward (create_graph) inherits
  chain = [None]

  def spy(name, *a):
    if name in _GEOM_AT:
      i = _GEOM_AT[name]
      calls.append((name,) + tuple(int(v) for v in a[i:i + 7]))
    with record_function('twg|%s|%s' % (chain[0] or ops.TRACE_TAG, name)):
      return call(name, *a)

  def tagged(fwd, bwd):
    def forward(ctx, *a, **k):
      ctx._twg_chain = chain[0] or ops.TRACE_TAG
      return fwd(ctx, *a, **k)

    def backward(ctx, *g):
      prev, chain[0] = chain[0], getattr(ctx, '_twg_chain', None)
      try:
        return bwd(ctx, *g)
      finally:
        chain[0] = prev
    return staticmethod(forward), staticmethod(backward)
  saved = {c: (vars(c)['forward'], vars(c)['backward']) for c in vars(ops).values()
           if isinstance(c, type) and issubclass(c, torch.autograd.Function) and 'forward' in vars(c)}
  for c in saved:
    c.forward, c.backward = tagged(c.forward, c.backward)
  L.call = spy
  try:
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
      model.train_step(s, t, r)
      torch.cuda.synchronize()
  finally:
    del L.call
    for c, (forward, backward) in saved.items():
      c.forward, c.backward = forward, backward
  os.makedirs(args.out, exist_ok=True)
  trace = os.path.join(args.out, 'trace.json')
  prof.export_chrome_trace(trace)
  events = json.load(open(trace))
  events = events['traceEvents'] if isinstance(events, dict) else events
  kernels = sorted((e for e in events if e.get('cat') == 'kernel' and e.get('ph') == 'X'), key=lambda e: e['ts'])
  gpu = gpu_info(0)

  def short(name):
    return name.replace('void ', '').split('(')[0]
  total = sum(e['dur'] for e in kernels)
  span = (kernels[-1]['ts'] + kernels[-1]['dur'] - kernels[0]['ts']) if kernels else 0.0
  per = collections.OrderedDict()
  for e in kernels:
    d = per.setdefault(short(e['name']), {'launches': 0, 'us': 0.0})
    d['launches'] += 1
    d['us'] += e['dur']
  table = sorted(({'kernel': n, 'launches': d['launches'], 'us': round(d['us'], 1), 'share': d['us'] / total}
                  for n, d in per.items()), key=lambda d: -d['us'])
  print('card: %s, power limit %s W; library %s' % (gpu['name'], gpu['power_limit_w'], LIB_PATH))
  print('one eager step: %d kernels, %.1f ms of kernel time, %.1f ms from first kernel start to last kernel end'
        % (len(kernels), total / 1e3, span / 1e3))
  print('%-64s %8s %11s %7s' % ('kernel', 'launches', 'total us', 'share'))
  for d in table:
    print('%-64s %8d %11.1f %6.1f%%' % (d['kernel'][:64], d['launches'], d['us'], 100 * d['share']))

  # each tensor-core fwd / dgrad call launches one k_conv_fwd*_wgmma kernel, each wgrad call one k_conv_wgrad*_wgmma, in order
  fwd_k = [e for e in kernels if 'k_conv_fwd' in e['name'] and 'wgmma' in e['name']]
  wg_k = [e for e in kernels if 'k_conv_wgrad' in e['name'] and 'wgmma' in e['name']]
  fwd_c = [c for c in calls if c[0] != 'twg_conv_wgrad_planes']
  wg_c = [c for c in calls if c[0] == 'twg_conv_wgrad_planes']
  if len(fwd_k) != len(fwd_c) or len(wg_k) != len(wg_c):
    raise SystemExit('conv launches (%d fwd, %d wgrad) do not match the trace (%d, %d)'
                     % (len(fwd_c), len(wg_c), len(fwd_k), len(wg_k)))
  rows = []
  for c, e in list(zip(fwd_c, fwd_k)) + list(zip(wg_c, wg_k)):
    m = conv_traffic(*c)
    entry, N, H, W, Cin, Cout, k, pad = c
    gemm_k = Cin if entry == 'twg_conv_wgrad_planes' else (Cout if entry == 'twg_conv_dgrad_planes' else Cin)
    rows.append(dict(m, entry=entry, geom=[N, H, W, Cin, Cout, k, pad], kernel=short(e['name']), us=e['dur'],
                     thin=bool(k == 3 and gemm_k <= 64 and H >= 64)))
  groups = collections.OrderedDict()
  for row in rows:
    wgrad = row['entry'] == 'twg_conv_wgrad_planes'
    for gname in ('all tensor-core convs', 'GEMM-K <= 64, 3x3, >= 64^2', 'column-box forward / dgrad',
                  'all weight gradients', 'column-box weight gradients'):
      if gname == 'GEMM-K <= 64, 3x3, >= 64^2' and not row['thin']:
        continue
      if gname == 'column-box forward / dgrad' and not (row['cols'] and not wgrad):
        continue
      if gname == 'all weight gradients' and not wgrad:
        continue
      if gname == 'column-box weight gradients' and not (row['cols'] and wgrad):
        continue
      g = groups.setdefault(gname, {'launches': 0, 'us': 0.0, 'flops': 0.0, 'hbm': 0.0, 'l2_before': 0.0, 'l2_after': 0.0})
      g['launches'] += 1
      for key in ('us', 'flops', 'hbm', 'l2_before', 'l2_after'):
        g[key] += row[key]
  print('\n%-30s %8s %10s %7s %9s %9s %11s %10s' % ('tensor-core convs', 'launches', 'total us', 'share', 'TFLOP', 'HBM GB',
                                                   'L2 GB old', 'L2 GB new'))
  for gname, g in groups.items():
    g['share'] = g['us'] / total
    print('%-30s %8d %10.1f %6.1f%% %9.3f %9.2f %11.2f %10.2f' % (gname, g['launches'], g['us'], 100 * g['share'],
                                                                 g['flops'] / 1e12, g['hbm'] / 1e9, g['l2_before'] / 1e9,
                                                                 g['l2_after'] / 1e9))
  with open(os.path.join(args.out, 'kernels.json'), 'w') as f:
    json.dump({'gpu': gpu, 'library': LIB_PATH, 'kernel_us': total, 'span_us': span, 'kernels': table}, f, indent=1)
  with open(os.path.join(args.out, 'convs.json'), 'w') as f:
    json.dump({'gpu': gpu, 'library': LIB_PATH, 'groups': groups, 'launches': rows}, f, indent=1)

  # each kernel -> the runtime call that launched it (correlation id) -> the library call around it (same thread, time)
  notes = collections.defaultdict(list)
  for e in events:
    if e.get('ph') == 'X' and str(e.get('name', '')).startswith('twg|'):
      notes[e['tid']].append(e)
  launch_at = {}
  for e in events:
    if e.get('ph') == 'X' and e.get('cat') in ('cuda_runtime', 'cuda_driver') and 'correlation' in e.get('args', {}):
      launch_at[e['args']['correlation']] = e
  fill = []
  for k in kernels:
    a = k['args']
    rt = launch_at.get(a.get('correlation'))
    tag = 'torch'
    if rt is not None:
      for n in notes.get(rt['tid'], ()):
        if n['ts'] <= rt['ts'] <= n['ts'] + n['dur']:
          tag = n['name'].split('|')[1]
    grid = int(a['grid'][0]) * int(a['grid'][1]) * int(a['grid'][2])
    block = int(a['block'][0]) * int(a['block'][1]) * int(a['block'][2])
    per_sm = resident_ctas(block, int(a.get('registers per thread', 0)), int(a.get('shared memory', 0)))
    waves, util, tail = launch_fill(grid, per_sm)
    fill.append({'kernel': short(k['name']), 'chain': tag, 'us': k['dur'], 'grid': grid, 'block': block,
                 'ctas_per_sm': per_sm, 'waves': waves, 'util': util, 'tail_us': k['dur'] * tail})
  summary = collections.OrderedDict()
  for tag in CHAINS + ('other',):
    rows_t = [f_ for f_ in fill if (f_['chain'] == tag if tag != 'other' else f_['chain'] not in CHAINS)]
    sub = [f_ for f_ in rows_t if f_['waves'] == 1 and f_['util'] < 1.0]
    summary[tag] = {'launches': len(rows_t), 'us': sum(f_['us'] for f_ in rows_t),
                    'sub_wave_launches': len(sub), 'sub_wave_us': sum(f_['us'] for f_ in sub),
                    'tail_us': sum(f_['tail_us'] for f_ in rows_t),
                    'idle_us': sum(f_['us'] * (1.0 - f_['util']) for f_ in rows_t)}
  pairs = {}
  for a_tag, b_tag in (('Ds', 'Dt'), ('DRs', 'DRt')):
    la = [(f_['us'], f_['util']) for f_ in fill if f_['chain'] == a_tag]
    lb = [(f_['us'], f_['util']) for f_ in fill if f_['chain'] == b_tag]
    ka = [(f_['kernel'], f_['grid']) for f_ in fill if f_['chain'] == a_tag]
    kb = [(f_['kernel'], f_['grid']) for f_ in fill if f_['chain'] == b_tag]
    pairs[a_tag + '|' + b_tag] = {'launches': [len(la), len(lb)], 'same_kernels_and_grids': ka == kb,
                                  'overlap_bound_us': overlap_bound(la, lb)}
  print('\n%-8s %8s %10s %9s %12s %10s %10s' % ('chain', 'launches', 'total us', 'sub-wave', 'sub-wave us', 'tail us',
                                               'idle us'))
  for tag, d in summary.items():
    print('%-8s %8d %10.1f %9d %12.1f %10.1f %10.1f' % (tag, d['launches'], d['us'], d['sub_wave_launches'],
                                                       d['sub_wave_us'], d['tail_us'], d['idle_us']))
  for key, d in pairs.items():
    print('%s side by side: %s launches, same kernels and grids in order: %s, at most %.1f us saved'
          % (key.replace('|', ' / '), d['launches'], d['same_kernels_and_grids'], d['overlap_bound_us']))
  with open(os.path.join(args.out, 'fill.json'), 'w') as f:
    json.dump({'gpu': gpu, 'library': LIB_PATH, 'sms': SMS, 'chains': summary, 'pairs': pairs, 'launches': fill}, f,
              indent=1)


if __name__ == '__main__':
  main()
