"""Times image translation (twingan_b200/translate.py): the two kernels of csrc/twg_image.cu on their own, and the whole
file-to-file path on a directory of seeded PNG and JPEG files.

  python tools/translate_bench.py [--n 256] [--num_decode_threads 8] [--batch_size 64] [--out result.json]

Kernels: CUDA events around `--iters` launches after a warm-up, for 64 images of 368 x 371 (the size of the reference's
demo inputs) and 64 images of 1024 x 768, each to 256 x 256.  Bytes are the compulsory traffic: the image rows the
resize samples plus the fp32 output, and for the quantisation the fp32 input plus the uint8 output; the share is of the
H100 SXM's 3.35 TB/s HBM3.  End to end: images/s of translate_files with a seeded 256 x 256 model, at 1 decode thread and
at --num_decode_threads, host clock, one warm-up run first (the CUDA graph capture of each run is included).  The card
name and power limit are read in the same run.  Needs a GPU."""
from __future__ import annotations

import argparse
import json
import os
import shutil
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
  sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def _time(fn, iters):
  fn()
  torch.cuda.synchronize()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(iters):
    fn()
  e1.record()
  torch.cuda.synchronize()
  return e0.elapsed_time(e1) / iters


def _rows_read(H, hw):
  from oracle import translate_oracle as TO   # the coordinate step only
  lo, hi, _ = TO.taps(hw, H)
  return len(np.union1d(lo, hi))


def kernels(shape, B, hw, iters):
  from twingan_b200 import ops
  H, W = shape
  rng = np.random.default_rng(0)
  payload, table = ops.pack_images([rng.integers(0, 256, (H, W, 3), dtype=np.uint8) for _ in range(B)])
  payload, table = payload.cuda(), table.cuda()
  out = torch.empty((B, hw, hw, 3), device='cuda')
  ms = _time(lambda: ops.images_u8_to_batch(payload, table, hw, out), iters)
  front = B * _rows_read(H, hw) * W * 3 + out.numel() * 4
  ms_q = _time(lambda: ops.batch_to_u8(out), iters)
  back = out.numel() * 5
  r = lambda b, t: {'ms': round(t, 4), 'bytes': b, 'gbs': round(b / (t * 1e6), 1),
                    'hbm_share': round(b / (t * 1e-3) / HBM_BYTES_PER_S, 3)}
  return {'images': B, 'input': '%dx%d' % (H, W), 'hw': hw, 'images_u8_to_batch': r(front, ms), 'batch_to_u8': r(back, ms_q)}


def end_to_end(n, threads, batch_size):
  from PIL import Image
  from twingan_b200 import translate, twingan
  d = tempfile.mkdtemp(prefix='twg_translate_bench_')
  try:
    rng = np.random.default_rng(1)
    ins = []
    for i in range(n):
      h, w = ((368, 371), (1024, 768), (512, 512))[i % 3]
      p = os.path.join(d, 'in', '%05d.%s' % (i, 'png' if i % 2 else 'jpg'))
      os.makedirs(os.path.dirname(p), exist_ok=True)
      lo = rng.integers(0, 256, (h // 8 + 1, w // 8 + 1, 3), dtype=np.uint8)          # smooth-ish content, like photos
      img = np.asarray(Image.fromarray(lo).resize((w, h), Image.BILINEAR))
      Image.fromarray(img).save(p)
      ins.append(p)
    outs = [os.path.join(d, 'out', os.path.basename(p)) for p in ins]
    model = twingan.GanModel(twingan.Flags(train_image_size=256), device='cuda', seed=3)
    translate.translate_files(model, ins[:batch_size], outs[:batch_size], batch_size=batch_size)      # warm-up
    res = {}
    for t in sorted({1, threads}):
      torch.cuda.synchronize()
      t0 = time.perf_counter()
      translate.translate_files(model, ins, outs, batch_size=batch_size, num_decode_threads=t)
      torch.cuda.synchronize()
      res['threads_%d' % t] = round(n / (time.perf_counter() - t0), 1)
    return {'images': n, 'sizes': ['368x371', '1024x768', '512x512'], 'formats': 'half PNG, half JPEG',
            'batch_size': batch_size, 'images_per_s': res}
  finally:
    shutil.rmtree(d, ignore_errors=True)


def main():
  ap = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
  ap.add_argument('--n', type=int, default=256, help='files of the end-to-end run (0: skip it)')
  ap.add_argument('--num_decode_threads', type=int, default=8)
  ap.add_argument('--batch_size', type=int, default=64)
  ap.add_argument('--iters', type=int, default=50)
  ap.add_argument('--out', default=None, help='also write the result as JSON here')
  args = ap.parse_args()
  assert torch.cuda.is_available(), 'tools/translate_bench.py needs a GPU'
  import __graft_entry__ as graft
  graft.build()
  from bench import gpu_info
  gpu = gpu_info(0)
  out = {'card': gpu['name'], 'power_limit_w': gpu['power_limit_w'], 'host_cores': os.cpu_count(),
         'kernels': [kernels((368, 371), 64, 256, args.iters), kernels((1024, 768), 64, 256, args.iters)],
         'end_to_end': end_to_end(args.n, args.num_decode_threads, args.batch_size) if args.n else 'not measured'}
  print('card: %s, power limit %s W' % (gpu['name'], gpu['power_limit_w'] if gpu['power_limit_w'] else 'not measured'))
  for k in out['kernels']:
    for name in ('images_u8_to_batch', 'batch_to_u8'):
      r = k[name]
      print('%-19s %3d x %-9s -> %d: %8.4f ms %10.3g B %8.1f GB/s %5.1f %% of HBM'
            % (name, k['images'], k['input'], k['hw'], r['ms'], r['bytes'], r['gbs'], 100 * r['hbm_share']))
  e = out['end_to_end']
  if isinstance(e, dict):
    for t, v in e['images_per_s'].items():
      print('end to end, %d files, %s: %.1f images/s' % (e['images'], t.replace('_', ' '), v))
  else:
    print('end to end: not measured')
  print(json.dumps(out))
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'w') as f:
      json.dump(out, f, indent=1)


if __name__ == '__main__':
  main()
