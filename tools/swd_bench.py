"""Times the sliced Wasserstein evaluation (twingan_b200/swd.py) on the device, per kernel family and end to end, beside
the work its shapes imply, and the fp64 numpy restatement (oracle/swd_oracle.py) on the host cores at a smaller n.

  python tools/swd_bench.py [--n 8192] [--res 256] [--host-n 64] [--out result.json]

The images are seeded synthetic ones made on the device (smooth random images as the real set, noisier ones as the
fake set), fed in batches of --batch.  One full evaluation at the timed shape warms up first.  End-to-end time is taken
with a host clock between device synchronisations; per-family time with CUDA events around every library call of the
timed evaluation.  The card name and power limit are read in the same run.  Needs a GPU."""
from __future__ import annotations

import argparse
import json
import math
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
  sys.path.insert(0, ROOT)

import torch  # noqa: E402

FAMILY = {'twg_swd_pyramid': 'pyramid', 'twg_swd_gather': 'gather', 'twg_swd_stats': 'stats',
          'twg_swd_project': 'project', 'twg_swd_sort': 'sort', 'twg_swd_sorted_l1': 'sorted_l1'}


def work(n, R, nhood=7, nhoods=128, repeats=4, ndirs=128, floor=True):
  """Algorithmic FLOPs / bytes / keys of one evaluation from its shapes.  Bytes count each kernel's compulsory HBM
  traffic: the sort's 4 passes read every key twice (digit counts, scatter) and write it once."""
  D = 3 * nhood * nhood
  levels = [R >> l for l in range(int(math.log2(R)) - 3)]
  rows = n * nhoods
  # distance computations per level, as (rows per set): the fake one, and the floor's two halves
  dists = [rows] + ([rows // 2] if floor else [])
  w = {k: {'flops': 0.0, 'bytes': 0.0} for k in FAMILY.values()}
  keys = 0.0
  for r in levels:
    w['gather']['bytes'] += 2 * rows * D * 4                  # write descriptors (reads hit cache)
    for m in dists:
      w['stats']['bytes'] += 2 * m * D * 4
      w['project']['flops'] += repeats * 2 * (2.0 * m * D * ndirs)
      w['project']['bytes'] += repeats * 2 * (m * D * 4 + m * ndirs * 4)
      k = repeats * 2 * m * ndirs
      keys += k
      w['sort']['bytes'] += k * 4 * 12
      w['sorted_l1']['bytes'] += k * 4
  for s in (n, n):                                               # both sets' pyramids: read the images, write all levels
    w['pyramid']['bytes'] += s * R * R * 3 * 4 * (1 + sum((r / R) ** 2 for r in levels) * 2)
  proj_no_floor = repeats * 2 * 2.0 * rows * D * ndirs * len(levels)
  keys_no_floor = repeats * 2 * rows * ndirs * len(levels)
  return w, keys, proj_no_floor, keys_no_floor


def synthetic(n, R, seed, device):
  g = torch.Generator(device=device).manual_seed(seed)
  lo = torch.rand((n, 3, max(R // 8, 2), max(R // 8, 2)), device=device, generator=g)
  real = torch.nn.functional.interpolate(lo, size=(R, R), mode='bilinear', align_corners=False).permute(0, 2, 3, 1)
  fake = 0.7 * real + 0.3 * torch.rand((n, R, R, 3), device=device, generator=g) ** 2
  return real.contiguous(), fake.contiguous()


def evaluate(n, R, real, fake, batch, seed=0):
  from twingan_b200 import swd
  m = swd.SlicedWasserstein(R, n, real.device, seed)
  for i in range(0, n, batch):
    m.feed('real', real[i:i + batch])
    m.feed('fake', fake[i:i + batch])
  return m.result()


class _Timed(object):
  """Stands in for swd.lib(): every call is bracketed by CUDA events, collected per family."""

  def __init__(self, inner):
    self.inner, self.cdll, self.events = inner, inner.cdll, []

  def call(self, name, *args):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    self.inner.call(name, *args)
    e1.record()
    self.events.append((FAMILY[name], e0, e1))

  def last_error(self):
    return self.inner.last_error()


def main():
  ap = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
  ap.add_argument('--n', type=int, default=8192)
  ap.add_argument('--res', type=int, default=256)
  ap.add_argument('--batch', type=int, default=256)
  ap.add_argument('--host-n', type=int, default=64, help='images per set of the host fp64 timing (0: skip it)')
  ap.add_argument('--out', default=None, help='also write the result as JSON here')
  args = ap.parse_args()
  assert torch.cuda.is_available(), 'tools/swd_bench.py needs a GPU'
  import __graft_entry__ as graft
  graft.build()
  from bench import gpu_info
  from twingan_b200 import _lib, swd
  gpu = gpu_info(0)
  dev = torch.device('cuda')
  n, R = args.n, args.res
  real, fake = synthetic(n, R, 1, dev)

  warm = evaluate(n, R, real, fake, args.batch)                 # module load, allocator, the whole shape once
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  res = evaluate(n, R, real, fake, args.batch)
  torch.cuda.synchronize()
  wall = time.perf_counter() - t0
  assert res == warm, 'two evaluations of the same inputs differ'

  timed = _Timed(_lib.lib())
  swd.lib = lambda: timed                                        # per-family CUDA events, in a run of their own
  evaluate(n, R, real, fake, args.batch)
  torch.cuda.synchronize()
  swd.lib = _lib.lib
  w, keys, proj_nf, keys_nf = work(n, R)
  fam = {k: {'calls': 0, 'ms': 0.0} for k in FAMILY.values()}
  for f, e0, e1 in timed.events:
    fam[f]['calls'] += 1
    fam[f]['ms'] += e0.elapsed_time(e1)
  for k, d in fam.items():
    d['ms'] = round(d['ms'], 3)
    d['flops'] = w[k]['flops']
    d['bytes'] = w[k]['bytes']
    d['tflops'] = round(d['flops'] / (d['ms'] * 1e9), 2) if d['ms'] and d['flops'] else None
    d['gbs'] = round(d['bytes'] / (d['ms'] * 1e6), 1) if d['ms'] else None
  out = {'card': gpu['name'], 'power_limit_w': gpu['power_limit_w'], 'n': n, 'res': R, 'batch': args.batch,
         'evaluation_s': round(wall, 4), 'result': res, 'families': fam,
         'projection_flops': sum(d['flops'] for d in fam.values()), 'projection_flops_without_floor': proj_nf,
         'keys_sorted': keys, 'keys_sorted_without_floor': keys_nf}
  del real, fake
  torch.cuda.empty_cache()

  if args.host_n:
    import numpy as np
    from oracle import swd_oracle as O
    hr, hf = synthetic(args.host_n, R, 1, dev)
    hr, hf = hr.cpu().numpy(), hf.cpu().numpy()
    draws = swd.make_draws(R, args.host_n, 0)
    t0 = time.perf_counter()
    O.swd(hr, hf, draws)
    host = time.perf_counter() - t0
    hw, hkeys, _, _ = work(args.host_n, R)
    out['host_fp64'] = {'n': args.host_n, 'seconds': round(host, 3), 'cores': os.cpu_count(), 'keys_sorted': hkeys,
                        'projection_flops': hw['project']['flops'], 'numpy': np.__version__}

  print('card: %s, power limit %s W' % (gpu['name'], gpu['power_limit_w']))
  print('SWD of %d + %d images at %d^2 (with the real-vs-real floor): %.3f s end to end' % (n, n, R, wall))
  print('  projections %.3g FLOP (%.3g without the floor), %.3g keys sorted (%.3g without the floor)'
        % (out['projection_flops'], proj_nf, keys, keys_nf))
  print('%-10s %6s %10s %12s %12s %9s %9s' % ('family', 'calls', 'ms', 'FLOP', 'bytes', 'TFLOP/s', 'GB/s'))
  for k, d in fam.items():
    print('%-10s %6d %10.2f %12.3g %12.3g %9s %9s' % (k, d['calls'], d['ms'], d['flops'], d['bytes'], d['tflops'], d['gbs']))
  if 'host_fp64' in out:
    h = out['host_fp64']
    print('host fp64 restatement, n=%d on %d cores: %.2f s' % (h['n'], h['cores'], h['seconds']))
  print(json.dumps(out))
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'w') as f:
      json.dump(out, f, indent=1)


if __name__ == '__main__':
  main()
