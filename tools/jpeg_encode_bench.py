"""Times the device JPEG encoder (csrc/twg_jenc.cu) against PIL, and `translate_files` with .jpg outputs end to end.

  python tools/jpeg_encode_bench.py [--n 256] [--batch_size 64] [--parent <parent commit's checkout>] [--out r.json]

Device: CUDA events around windows of `--iters` calls after a warm-up, `--repeats` windows, on 64 seeded photo-like
images of 256 x 256 and 64 of 128 x 128: the three kernel entries on buffers allocated beforehand, and whole
ops.jpeg_encode calls (allocations and launches included).  PIL: the same arrays encoded
(Image.fromarray(a).save(buf, 'JPEG')) on 1 and 8 host threads, host clock, passes repeated until they add up to a
second; min / median / max of each.  End to end: images/s of translate_files with a seeded 256 x 256 model on `--n`
JPEG inputs with .jpg outputs, at 1 and 8 threads, host clock after a warm-up run, each tree's runs in a fresh process;
two corpora: photo-like 368 x 371, 1024 x 768 and 512 x 512 inputs, whose host decoding is heavy, and 256 x 256
inputs, where the device's share of a batch is larger.  With --parent, the same runs of the parent's tree alternate
with this tree's, run for run, `--rounds` times.  Also reported: the device-to-host bytes per output image, the raw
uint8 image before, the scan and its offset after.  The card name and power limit are read in the same run.
Needs a GPU."""
from __future__ import annotations

import argparse
import io
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPES = ((368, 371), (1024, 768), (512, 512))
HEADER_BYTES, EOI_BYTES = 623, 2


def _photo(h, w, rng):
  import numpy as np
  from PIL import Image
  lo = rng.integers(0, 256, (h // 8 + 1, w // 8 + 1, 3), dtype=np.uint8)           # smooth-ish content, like photos
  a = np.asarray(Image.fromarray(lo).resize((w, h), Image.BILINEAR)).astype(np.int32)
  return np.clip(a + rng.integers(-8, 9, a.shape), 0, 255).astype(np.uint8)


def _spread(xs):
  xs = sorted(xs)
  return {'min': round(xs[0], 4), 'median': round(xs[len(xs) // 2], 4), 'max': round(xs[-1], 4)}


def device_encode(arrs, iters, repeats):
  """CUDA-event ms of the three kernel entries on buffers allocated beforehand (`kernels`), and of whole ops.jpeg_encode
  calls, which add five allocations and the ctypes launches (`call`); each a window of `iters` calls, `repeats`
  times."""
  import numpy as np
  import torch
  from twingan_b200 import jpeg, ops
  from twingan_b200._lib import lib
  L = lib()
  x = torch.from_numpy(np.stack(arrs)).cuda()
  n, h, w = x.shape[:3]
  blocks = 6 * ((h + 15) // 16) * ((w + 15) // 16)
  qt = torch.from_numpy(jpeg.encoder_qt()).cuda()
  coefs = torch.empty(n * blocks * 64, dtype=torch.int16, device='cuda')
  bitpos = torch.empty(n * (blocks + 1), dtype=torch.int32, device='cuda')
  work = torch.empty(L.cdll.twgjenc_workspace_bytes(n, h, w), dtype=torch.uint8, device='cuda')
  out = torch.empty(L.cdll.twgjenc_scan_capacity(n, h, w), dtype=torch.uint8, device='cuda')
  offsets = torch.empty(n + 1, dtype=torch.int64, device='cuda')
  st = torch.cuda.current_stream().cuda_stream

  def kernels():
    L.call('twgjenc_dct', x.data_ptr(), n, h, w, qt.data_ptr(), coefs.data_ptr(), st)
    L.call('twgjenc_bits', coefs.data_ptr(), n, h, w, bitpos.data_ptr(), st)
    L.call('twgjenc_pack', coefs.data_ptr(), bitpos.data_ptr(), n, h, w, work.data_ptr(), out.data_ptr(),
           offsets.data_ptr(), st)

  def timed(fn):
    fn()
    torch.cuda.synchronize()
    res = []
    for _ in range(repeats):
      e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      e0.record()
      for _ in range(iters):
        fn()
      e1.record()
      torch.cuda.synchronize()
      res.append(e0.elapsed_time(e1) / iters)
    return _spread(res)
  k = timed(kernels)
  c = timed(lambda: ops.jpeg_encode(x))
  return {'images': int(n), 'hw': int(h), 'kernels_ms': k, 'call_ms': c,
          'images_per_s_kernels': round(int(n) / k['median'] * 1e3, 1),
          'scan_bytes_per_image': round(int(offsets[-1].item()) / int(n), 1)}


def pil_encode(arrs, threads, min_s=1.0, min_passes=5):
  """Host-clock ms of one pass over the arrays, repeated until the passes together take `min_s` (at least
  `min_passes`): min / median / max over the passes."""
  from PIL import Image

  def enc(a):
    b = io.BytesIO()
    Image.fromarray(a).save(b, 'JPEG')
    return b.getvalue()
  passes = []
  with ThreadPoolExecutor(threads) as pool:
    list(pool.map(enc, arrs))                                               # warm-up
    while len(passes) < min_passes or sum(passes) < min_s * 1e3:
      t0 = time.perf_counter()
      list(pool.map(enc, arrs))
      passes.append((time.perf_counter() - t0) * 1e3)
  sp = _spread(passes)
  return {'images': len(arrs), 'hw': arrs[0].shape[0], 'threads': threads, 'passes': len(passes), 'ms': sp,
          'images_per_s_median': round(len(arrs) / sp['median'] * 1e3, 1)}


def end_to_end_worker(root, n, batch_size):
  """One end-to-end measurement with the package of the tree at `root` (run in its own process)."""
  sys.path.insert(0, root)
  import numpy as np
  import torch
  from PIL import Image
  import __graft_entry__ as graft
  graft.build()
  from twingan_b200 import translate, twingan
  d = tempfile.mkdtemp(prefix='twg_jenc_bench_')
  try:
    model = twingan.GanModel(twingan.Flags(train_image_size=256), device='cuda', seed=3)
    out = {}
    for corpus, shapes in (('photos', SHAPES), ('256x256', ((256, 256),))):
      rng = np.random.default_rng(1)
      ins = []
      for i in range(n):
        p = os.path.join(d, corpus, 'in', '%05d.jpg' % i)
        os.makedirs(os.path.dirname(p), exist_ok=True)
        Image.fromarray(_photo(*shapes[i % len(shapes)], rng)).save(p)
        ins.append(p)
      outs = [os.path.join(d, corpus, 'out', os.path.basename(p)) for p in ins]
      translate.translate_files(model, ins[:batch_size], outs[:batch_size], batch_size=batch_size)    # warm-up
      res = {}
      for t in (1, 8):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        translate.translate_files(model, ins, outs, batch_size=batch_size, num_decode_threads=t)
        torch.cuda.synchronize()
        res['threads_%d' % t] = round(n / (time.perf_counter() - t0), 1)
      scan = float(np.mean([os.path.getsize(o) for o in outs])) - HEADER_BYTES - EOI_BYTES
      out[corpus] = {'images_per_s': res, 'scan_bytes_per_image': round(scan, 1)}
    return out
  finally:
    shutil.rmtree(d, ignore_errors=True)


def end_to_end(trees, n, batch_size, rounds):
  """{tree name: [result of each round]}, the trees' runs alternating."""
  out = {name: [] for name in trees}
  for _ in range(rounds):
    for name, root in trees.items():
      r = subprocess.run([sys.executable, os.path.abspath(__file__), '--worker', root, '--n', str(n), '--batch_size',
                          str(batch_size)], capture_output=True, text=True)
      if r.returncode != 0:
        raise RuntimeError('%s: %s' % (name, r.stderr[-3000:]))
      out[name].append(json.loads(r.stdout.strip().splitlines()[-1]))
  return out


def main():
  ap = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
  ap.add_argument('--n', type=int, default=256, help='files of each end-to-end run (0: skip them)')
  ap.add_argument('--batch_size', type=int, default=64)
  ap.add_argument('--iters', type=int, default=50)
  ap.add_argument('--rounds', type=int, default=2)
  ap.add_argument('--repeats', type=int, default=5, help='event windows of --iters calls for each device time')
  ap.add_argument('--parent', default=None, help='a built checkout of the parent commit, timed alternately')
  ap.add_argument('--worker', default=None, help=argparse.SUPPRESS)
  ap.add_argument('--out', default=None, help='also write the result as JSON here')
  args = ap.parse_args()
  if args.worker:
    print(json.dumps(end_to_end_worker(args.worker, args.n, args.batch_size)))
    return
  sys.path.insert(0, ROOT)
  import numpy as np
  import torch
  assert torch.cuda.is_available(), 'tools/jpeg_encode_bench.py needs a GPU'
  import __graft_entry__ as graft
  graft.build()
  from bench import gpu_info
  gpu = gpu_info(0)
  rng = np.random.default_rng(2)
  sets = [[_photo(hw, hw, rng) for _ in range(64)] for hw in (256, 128)]
  out = {'card': gpu['name'], 'power_limit_w': gpu['power_limit_w'], 'host_cores': os.cpu_count(),
         'device': [device_encode(a, args.iters, args.repeats) for a in sets],
         'pil': [pil_encode(a, t) for a in sets for t in (1, 8)],
         'd2h_bytes_per_image_before': 256 * 256 * 3}
  trees = {'this': ROOT}
  if args.parent:
    trees['parent'] = os.path.abspath(args.parent)
  out['end_to_end'] = end_to_end(trees, args.n, args.batch_size, args.rounds) if args.n else 'not measured'
  if args.n:
    out['d2h_bytes_per_image_after'] = round(out['end_to_end']['this'][0]['photos']['scan_bytes_per_image'] + 8, 1)
  print('card: %s, power limit %s W, %s host cores' % (gpu['name'], gpu['power_limit_w'] or 'not measured',
                                                       out['host_cores']))
  for d in out['device']:
    print('device, %d x %d^2: kernels %s ms, whole call %s ms, %.0f scan bytes per image'
          % (d['images'], d['hw'], d['kernels_ms'], d['call_ms'], d['scan_bytes_per_image']))
  for p in out['pil']:
    print('PIL, %d x %d^2, %d thread(s), %d passes: %s ms' % (p['images'], p['hw'], p['threads'], p['passes'], p['ms']))
  if isinstance(out['end_to_end'], dict):
    for name, runs in out['end_to_end'].items():
      for corpus in runs[0]:
        print('end to end (%s), %d %s .jpg -> .jpg: %s' % (name, args.n, corpus,
                                                          [r[corpus]['images_per_s'] for r in runs]))
    print('D2H bytes per image: %d before, %.1f after' % (out['d2h_bytes_per_image_before'],
                                                           out['d2h_bytes_per_image_after']))
  print(json.dumps(out))
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'w') as f:
      json.dump(out, f, indent=1)


if __name__ == '__main__':
  main()
