#!/usr/bin/env python
"""A/B of two builds of libtwg.so on every tensor-core conv geometry the product launches.

  python tools/conv_ab.py --a OLD/libtwg.so --b twingan_b200/libtwg.so [--iters 50] [--batch 16] [--out DIR]

Each build runs in a process of its own (TWG_LIB selects the library twingan_b200._lib loads through ctypes) on the same
seeded inputs, for every tensor-core key of PRODUCT_CONVS (tests/test_gpu_conv_conformance.py) with its epilogue options.
Per geometry it reports whether every output (y, split planes, sign mask, statistics records, gw) is bit-identical
between the builds, and each build's kernel time from CUDA events over `iters` back-to-back launches.  Needs a GPU."""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TC_ENTRIES = ('twg_conv_fwd_planes', 'twg_conv_affine_act_fwd_planes', 'twg_conv_dgrad_planes', 'twg_conv_wgrad_planes')


def product_cases():
  """(entry, H, W, Cin, Cout, k, pad, options) of every tensor-core conv launch of the product."""
  if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
  from tests.test_gpu_conv_conformance import PRODUCT_CONVS
  return [(e,) + key for e in TC_ENTRIES for key in PRODUCT_CONVS[e]]


def _digest(t) -> str:
  import torch
  return hashlib.sha256(t.detach().contiguous().cpu().view(-1).view(torch.uint8).numpy().tobytes()).hexdigest()


def worker(lib_path, batch, iters):
  """Runs every case on the build at lib_path; prints one JSON line {case key: {'ms': ..., 'digest': {output: sha256}}}."""
  os.environ['TWG_LIB'] = os.path.abspath(lib_path)
  sys.path.insert(0, ROOT)
  import torch
  from twingan_b200 import ops
  from twingan_b200._lib import lib
  L = lib()
  dev = torch.device('cuda', 0)
  st = ops._st()
  res = {}
  for case in product_cases():
    entry = case[0]
    if entry == 'twg_conv_wgrad_planes':     # weight-gradient keys carry their batch (it sets the pixel split)
      N, H, W, Cin, Cout, k, pad, opts = case[1:]
    else:
      H, W, Cin, Cout, k, pad, opts = case[1:]
      N = batch
    opts = set(opts.split('+')) - {''}
    seed = int(hashlib.sha256(repr(case).encode()).hexdigest()[:8], 16)
    gen = torch.Generator(device=dev).manual_seed(seed)
    rnd = lambda *shape, s=1.0: torch.randn(shape, device=dev, generator=gen) * s
    geom = (N, H, W, Cin, Cout, k, pad)
    out = {}
    if entry == 'twg_conv_wgrad_planes':
      xp, gp = ops.split_act(rnd(N, H, W, Cin)), ops.split_act(rnd(N, H, W, Cout))
      out['gw'] = rnd(k, k, Cin, Cout)                 # accumulated into: the product adds into its gradient buffer
      acc = int('accumulate' in opts)
      launch = lambda: L.call(entry, xp.data_ptr(), gp.data_ptr(), out['gw'].data_ptr(), *geom, acc, st)
    elif entry == 'twg_conv_dgrad_planes':
      gp = ops.split_act(rnd(N, H, W, Cout))
      wp = torch.empty((2, k * k * Cin * Cout), device=dev, dtype=torch.bfloat16)
      L.call('twg_split_weights', rnd(k, k, Cin, Cout, s=0.05).data_ptr(), wp.data_ptr(), k, Cin, Cout, 1, st)
      out['gx'] = torch.empty((N, H, W, Cin), device=dev)
      launch = lambda: L.call(entry, gp.data_ptr(), wp.data_ptr(), out['gx'].data_ptr(), *geom, st)
    else:
      xp = ops.split_act(rnd(N, H, W, Cin))
      wp = torch.empty((2, k * k * Cin * Cout), device=dev, dtype=torch.bfloat16)
      L.call('twg_split_weights', rnd(k, k, Cin, Cout, s=0.05).data_ptr(), wp.data_ptr(), k, Cin, Cout, 0, st)
      p = lambda name: out[name].data_ptr() if name in out else None
      if entry == 'twg_conv_affine_act_fwd_planes':
        flags = int(next(o for o in opts if o.startswith('flags'))[5:])
        a, b = 1 + rnd(Cout, s=0.3), rnd(Cout, s=0.2)
        if 'z' in opts:
          out['z'] = torch.empty((N, H, W, Cout), device=dev)
        if 'zp' in opts:
          out['zp'] = torch.empty((2, N, H, W, Cout), device=dev, dtype=torch.bfloat16)
        launch = lambda: L.call(entry, xp.data_ptr(), wp.data_ptr(), a.data_ptr(), b.data_ptr(), flags, p('z'), p('zp'),
                                *geom, st)
      else:
        Ho, Wo = H + 2 * pad - k + 1, W + 2 * pad - k + 1
        bias = rnd(Cout, s=0.5) if 'bias' in opts else None
        out['y'] = torch.empty((N, Ho, Wo, Cout), device=dev)
        if 'zp' in opts:
          out['zp'] = torch.empty((2, N, Ho, Wo, Cout), device=dev, dtype=torch.bfloat16)
        if 'mask' in opts:
          out['mask'] = torch.empty(N * Ho * Wo * Cout // 4, device=dev, dtype=torch.uint8)
        if 'stats' in opts:
          slots = int(L.cdll.twg_conv_epilogue_slots(*geom))
          out['stats'] = torch.empty((N, slots, Cout, 4), device=dev)
        launch = lambda: L.call(entry, xp.data_ptr(), wp.data_ptr(), None if bias is None else bias.data_ptr(),
                                int('act' in opts), out['y'].data_ptr(), p('zp'), p('mask'), p('stats'), *geom, st)
    launch()
    torch.cuda.synchronize()
    digest = {name: _digest(t) for name, t in out.items()}
    for _ in range(3):
      launch()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
      launch()
    e1.record()
    torch.cuda.synchronize()
    res['|'.join(str(v) for v in case)] = {'ms': e0.elapsed_time(e1) / iters, 'digest': digest}
    del out
    torch.cuda.empty_cache()
  print(json.dumps(res), flush=True)


def run_build(lib_path, batch, iters):
  r = subprocess.run([sys.executable, os.path.abspath(__file__), '--worker', lib_path, '--batch', str(batch), '--iters',
                      str(iters)], capture_output=True, text=True)
  if r.returncode:
    raise SystemExit('build %s failed:\n%s' % (lib_path, r.stderr[-4000:]))
  return json.loads([l for l in r.stdout.splitlines() if l.startswith('{')][-1])


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--a', help='library of build A (the old one)')
  ap.add_argument('--b', help='library of build B (the new one)')
  ap.add_argument('--batch', type=int, default=16)
  ap.add_argument('--iters', type=int, default=50)
  ap.add_argument('--out', default=None, help='also write the table as OUT/conv_ab.json')
  ap.add_argument('--worker', default=None, help=argparse.SUPPRESS)
  args = ap.parse_args()
  if args.worker:
    worker(args.worker, args.batch, args.iters)
    return
  ra = run_build(args.a, args.batch, args.iters)
  rb = run_build(args.b, args.batch, args.iters)
  sys.path.insert(0, ROOT)
  from bench import gpu_info
  gpu = gpu_info(0)
  print('card: %s, power limit %s W' % (gpu['name'], gpu['power_limit_w']))
  rows, all_equal, ta, tb = [], True, 0.0, 0.0
  print('%-70s %6s %10s %10s %7s' % ('entry|H|W|Cin|Cout|k|pad|options (N=%d)' % args.batch, 'equal', 'A ms', 'B ms', 'A/B'))
  for key in ra:
    a, b = ra[key], rb[key]
    eq = a['digest'] == b['digest']
    all_equal &= eq
    ta += a['ms']
    tb += b['ms']
    rows.append({'case': key, 'bit_equal': eq, 'outputs': sorted(a['digest']), 'ms_a': a['ms'], 'ms_b': b['ms']})
    print('%-70s %6s %10.4f %10.4f %7.3f' % (key, 'yes' if eq else 'NO', a['ms'], b['ms'], a['ms'] / max(b['ms'], 1e-9)))
  print('all outputs bit-identical: %s; sum of per-launch times A %.3f ms, B %.3f ms' % (all_equal, ta, tb))
  if args.out:
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, 'conv_ab.json'), 'w') as f:
      json.dump({'gpu': gpu, 'a': args.a, 'b': args.b, 'batch': args.batch, 'iters': args.iters, 'all_equal': all_equal, 'rows': rows},
                f, indent=1)
  sys.exit(0 if all_equal else 1)


if __name__ == '__main__':
  main()
