#!/usr/bin/env python
"""A/B of two builds of libtwg.so on the one-block-per-sample normaliser launches of the bench.py step and on the DRAGAN
perturbation.

  python tools/norm_ab.py --a OLD/libtwg.so --b twingan_b200/libtwg.so [--iters 50] [--hw 256] [--batch 16] [--out DIR]

Each build runs in a process of its own (TWG_LIB selects the library twingan_b200._lib loads through ctypes).  The process
runs one training step of the bench workload and keeps the key of every twg_norm_act_bwd_reduce and twg_moments launch
(the key layout of tests/product_norms.py, each at its own N; a key outside that list is an error), then runs every key,
and twg_dragan_xhat on the [batch, hw, hw, 3] images, on seeded inputs.  Per case it reports whether every output (gu and
red; sums; s2 and xhat) is bit-identical between the builds, each build's time per launch from CUDA events over `iters`
back-to-back launches after a warm-up, and the GB/s of the bytes the shapes imply: every operand read once and every
result written once (the pooled gradient is a quarter of a tensor; twg_dragan_xhat reads x twice, in its sum and in its
apply pass).  Needs a GPU."""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
  sys.path.insert(0, ROOT)


def case_bytes(case):
  """Algorithmic HBM bytes of one launch of `case`."""
  name = case[0]
  if name == 'twg_moments':
    _, N, HW, C, _ = case
    return 4.0 * N * HW * C
  if name == 'twg_norm_act_bwd_reduce':
    _, N, HW, W, C, _, opts = case
    t = 4.0 * N * HW * C
    return t * (2 + ('gz' in opts.split('+'))) + (t / 4 if 'gpool' in opts.split('+') else 0.0)
  _, N, per = case
  return 4.0 * N * per * 4


def _digest(t) -> str:
  import torch
  return hashlib.sha256(t.detach().contiguous().cpu().view(-1).view(torch.uint8).numpy().tobytes()).hexdigest()


def step_cases(L, hw, batch):
  """The reduce and moments keys of one training step of the bench workload, and its DRAGAN case."""
  import torch
  from tests.product_norms import PRODUCT_NORMS
  from twingan_b200 import twingan
  dev = torch.device('cuda', 0)
  model = twingan.GanModel(twingan.Flags(train_image_size=hw, pggan_max_num_channels=256, generator_norm_type='instance_norm'),
                           device=dev, seed=1234)
  gen = torch.Generator(device=dev).manual_seed(100)
  s = torch.rand((batch, hw, hw, 3), device=dev, generator=gen)
  t = torch.rand((batch, hw, hw, 3), device=dev, generator=gen)
  r = twingan.make_dragan_rand(batch, hw, dev, gen)
  keys = set()
  call = L.call

  def spy(name, *a):
    if name == 'twg_moments':
      keys.add((name, a[2], a[3], a[4], a[5]))
    elif name == 'twg_norm_act_bwd_reduce':
      keys.add((name, a[10], a[11], a[7] if a[6] else 0, a[12], a[13],
                '+'.join(n for n, i in (('gz', 5), ('gpool', 6)) if a[i])))
    return call(name, *a)
  L.call = spy
  try:
    model.train_step(s, t, r)
    torch.cuda.synchronize()
  finally:
    del L.call
  del model
  torch.cuda.empty_cache()
  for k in keys:
    if hw == 256 and batch == 16 and tuple(k[1:]) not in PRODUCT_NORMS[k[0]]:
      raise SystemExit('launch %r is not a key of tests/product_norms.py' % (k,))
  return sorted(keys, key=str) + [('twg_dragan_xhat', batch, hw * hw * 3)]


def worker(lib_path, hw, batch, iters):
  """Runs every case on the build at lib_path; prints one JSON line {case: {'ms': ..., 'digest': {output: sha256}}}."""
  os.environ['TWG_LIB'] = os.path.abspath(lib_path)
  import torch
  from twingan_b200 import ops
  from twingan_b200._lib import lib
  if not torch.cuda.is_available():
    raise SystemExit('norm_ab.py needs a CUDA device')
  L = lib()
  dev = torch.device('cuda', 0)
  st = ops._st()
  res = {}
  for case in step_cases(L, hw, batch):
    name = case[0]
    seed = int(hashlib.sha256(repr(case).encode()).hexdigest()[:8], 16)
    gen = torch.Generator(device=dev).manual_seed(seed)
    rnd = lambda *shape: torch.randn(shape, device=dev, generator=gen)
    out = {}
    if name == 'twg_moments':
      _, N, HW, C, pg = case
      y = rnd(N, HW, C) * 0.7 + 0.3
      out['sums'] = torch.empty((N, C, 2), device=dev)
      launch = lambda: L.call(name, y.data_ptr(), out['sums'].data_ptr(), N, HW, C, pg, st)
    elif name == 'twg_norm_act_bwd_reduce':
      _, N, HW, W, C, flags, opts = case
      y = rnd(N, HW, C) * 0.7 + 0.3
      mean, var = y.mean(1), y.var(1, unbiased=False)
      rstd = (var + 1e-6).rsqrt()
      a = (1 + 0.2 * rnd(C)) * rstd
      b = 0.1 * rnd(C) - mean * a
      gz = rnd(N, HW, C) if 'gz' in opts.split('+') else None
      gp = rnd(N, HW // W // 2, W // 2, C) if 'gpool' in opts.split('+') else None
      out['gu'], out['red'] = torch.empty_like(y), torch.empty((N, C, 2), device=dev)
      launch = lambda: L.call(name, y.data_ptr(), a.data_ptr(), b.data_ptr(), mean.data_ptr(), rstd.data_ptr(),
                              None if gz is None else gz.data_ptr(), None if gp is None else gp.data_ptr(), W,
                              out['gu'].data_ptr(), out['red'].data_ptr(), N, HW, C, flags, st)
    else:
      _, N, per = case
      x = torch.rand((N, per), device=dev, generator=gen)
      alpha = torch.rand(N, device=dev, generator=gen)
      noise = torch.rand((N, per), device=dev, generator=gen) * 2 - 1
      out['xhat'], out['s2'] = torch.empty_like(x), torch.empty(4, device=dev)
      launch = lambda: L.call(name, x.data_ptr(), alpha.data_ptr(), noise.data_ptr(), out['xhat'].data_ptr(),
                              out['s2'].data_ptr(), N, per, st)
    launch()
    torch.cuda.synchronize()
    digest = {k: _digest(t) for k, t in out.items()}
    for _ in range(3):
      launch()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
      launch()
    e1.record()
    torch.cuda.synchronize()
    res['|'.join(str(v) for v in case)] = {'ms': e0.elapsed_time(e1) / iters, 'digest': digest, 'bytes': case_bytes(case)}
    del out
    torch.cuda.empty_cache()
  print(json.dumps(res), flush=True)


def run_build(lib_path, args):
  r = subprocess.run([sys.executable, os.path.abspath(__file__), '--worker', lib_path, '--hw', str(args.hw), '--batch',
                      str(args.batch), '--iters', str(args.iters)], capture_output=True, text=True)
  if r.returncode:
    raise SystemExit('build %s failed:\n%s' % (lib_path, (r.stdout + r.stderr)[-4000:]))
  return json.loads([l for l in r.stdout.splitlines() if l.startswith('{')][-1])


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--a', help='library of build A (the old one)')
  ap.add_argument('--b', help='library of build B (the new one)')
  ap.add_argument('--hw', type=int, default=256)
  ap.add_argument('--batch', type=int, default=16)
  ap.add_argument('--iters', type=int, default=50)
  ap.add_argument('--out', default=None, help='also write the table as OUT/norm_ab.json')
  ap.add_argument('--worker', default=None, help=argparse.SUPPRESS)
  args = ap.parse_args()
  if args.worker:
    worker(args.worker, args.hw, args.batch, args.iters)
    return
  ra = run_build(args.a, args)
  rb = run_build(args.b, args)
  if sorted(ra) != sorted(rb):
    raise SystemExit('the two builds launch different keys: %s' % sorted(set(ra) ^ set(rb)))
  from bench import gpu_info
  gpu = gpu_info(0)
  print('card: %s, power limit %s W' % (gpu['name'], gpu['power_limit_w']))
  rows, all_equal, ta, tb = [], True, 0.0, 0.0
  print('%-58s %5s %9s %9s %6s %8s %8s' % ('case', 'equal', 'A ms', 'B ms', 'A/B', 'A GB/s', 'B GB/s'))
  for key in ra:
    a, b = ra[key], rb[key]
    eq = a['digest'] == b['digest']
    all_equal &= eq
    ta += a['ms']
    tb += b['ms']
    gbs = [a['bytes'] / (r['ms'] * 1e-3) / 1e9 for r in (a, b)]
    rows.append({'case': key, 'bit_equal': eq, 'outputs': sorted(a['digest']), 'bytes': a['bytes'], 'ms_a': a['ms'],
                 'ms_b': b['ms'], 'gbs_a': gbs[0], 'gbs_b': gbs[1]})
    print('%-58s %5s %9.4f %9.4f %6.2f %8.0f %8.0f' % (key.replace('twg_', ''), 'yes' if eq else 'NO', a['ms'], b['ms'],
                                                      a['ms'] / max(b['ms'], 1e-9), gbs[0], gbs[1]))
  print('all outputs bit-identical: %s; sum of per-launch times A %.3f ms, B %.3f ms' % (all_equal, ta, tb))
  if args.out:
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, 'norm_ab.json'), 'w') as f:
      json.dump({'gpu': gpu, 'a': args.a, 'b': args.b, 'hw': args.hw, 'batch': args.batch, 'iters': args.iters,
                 'all_equal': all_equal, 'rows': rows}, f, indent=1)
  sys.exit(0 if all_equal else 1)


if __name__ == '__main__':
  main()
