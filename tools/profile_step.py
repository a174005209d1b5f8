#!/usr/bin/env python
"""Where the time of the bench.py workload goes: one warmed-up eager model.train_step (256x256, 16 pairs, instance norm)
under torch.profiler with CUDA activities.

  python tools/profile_step.py --out DIR [--hw 256] [--batch 16]

Prints and writes to DIR:
  * kernels.json / the first table: every kernel name with its launches, total microseconds and share of the GPU time of
    the step (the sum of all kernel durations);
  * convs.json / the second table: every tensor-core conv launch of the step (entry point and geometry, recorded where
    twingan_b200.ops calls the library) matched to its kernel in the trace, with its time, FLOPs, algorithmic HBM bytes and
    the modelled L2 -> shared-memory operand bytes of the kernels before and after the column-box forward (conv_traffic);
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
  L2 into shared memory, per CTA work item summed over the grid.  cols: the forward / dgrad takes the column-box kernel."""
  TW, TH, TN, tiles = _tiles(N, H, W)
  taps, px = k * k, N * H * W
  flops = 2.0 * px * Cin * Cout * taps
  if entry == 'twg_conv_wgrad_planes':
    CN = _chunk(Cin)
    BNW = 64 if (Cout >= 64 and CN < 64) else (32 if Cout >= 32 else Cout)
    items = tiles * (Cout // BNW) * (Cin // CN)
    per_item = 2 * 128 * BNW * 2 + taps * 2 * 128 * CN * 2     # gy tile + one x tile per tap, hi and lo planes
    l2 = float(items * per_item)
    return {'flops': flops, 'hbm': 4.0 * px * (Cin + Cout) + 4.0 * taps * Cin * Cout, 'l2_before': l2, 'l2_after': l2,
            'cols': False}
  K, Nc = (Cout, Cin) if entry == 'twg_conv_dgrad_planes' else (Cin, Cout)
  CC = _chunk(K)
  BN = min(Nc, 128)
  items = tiles * (Nc // BN)
  weights = taps * 2 * BN * K * 2                                 # one weight tile per (tap, chunk), hi and lo
  before = items * (taps * 2 * 128 * K * 2 + weights)            # one shifted 128-pixel A tile per (tap, chunk)
  cols = k == 3 and pad == 1 and K == CC and TW == 16 and TH == 8 and TN == 1 and H >= 10
  after = items * (3 * 2 * 160 * K * 2 + weights) if cols else before   # three {K, 16, 10} column boxes per tile
  return {'flops': flops, 'hbm': 4.0 * px * (K + Nc) + 4.0 * taps * K * Nc, 'l2_before': float(before),
          'l2_after': float(after), 'cols': cols}


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
  from torch.profiler import ProfilerActivity, profile
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

  def spy(name, *a):
    if name in _GEOM_AT:
      i = _GEOM_AT[name]
      calls.append((name,) + tuple(int(v) for v in a[i:i + 7]))
    return call(name, *a)
  L.call = spy
  try:
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
      model.train_step(s, t, r)
      torch.cuda.synchronize()
  finally:
    del L.call
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

  # each tensor-core fwd / dgrad call launches one k_conv_fwd*_wgmma kernel, each wgrad call one k_conv_wgrad_wgmma, in order
  fwd_k = [e for e in kernels if 'k_conv_fwd' in e['name'] and 'wgmma' in e['name']]
  wg_k = [e for e in kernels if 'k_conv_wgrad_wgmma' in e['name']]
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
    for gname in ('all tensor-core convs', 'GEMM-K <= 64, 3x3, >= 64^2', 'column-box forward / dgrad'):
      if gname == 'GEMM-K <= 64, 3x3, >= 64^2' and not row['thin']:
        continue
      if gname == 'column-box forward / dgrad' and not row['cols']:
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


if __name__ == '__main__':
  main()
