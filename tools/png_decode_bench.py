"""Times the device PNG decoder (csrc/twg_png.cu) against PIL, and `translate_files` end to end against PIL decoding.

  python tools/png_decode_bench.py [--n 256] [--batch_size 64] [--rounds 2] [--out result.json]

Device: CUDA events around each of the three entries (inflate / unfilter / rgb) of one batch of `--batch_size` PNG files:
seeded photo-like 368 x 371, 1024 x 768 and 512 x 512 images written by PIL at its defaults, and the two photographs of
tests/golden (another encoder, several IDAT chunks), `--iters` runs after a warm-up.  PIL: the same files decoded
(Image.open + convert('RGB')) on 1 and 8 host threads, host clock.  End to end: images/s of translate_files with a seeded
256 x 256 model on a directory of `--n` such PNG files, with .jpg outputs and with .png outputs, on 1 and 8 host threads;
each run of the device path alternates with a run where every file goes to PIL (the decoding before this decoder), for
`--rounds` rounds.  The card name and power limit are read in the same run.  Needs a GPU."""
from __future__ import annotations

import argparse
import io
import json
import os
import shutil
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
  sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

SHAPES = ((368, 371), (1024, 768), (512, 512))
FIXTURES = ('ROJFO5Y2C4CT1SI51NBI8G8QVD42QK39_0.png', 'IVW7BL5WMJRWF8TMXF9RNYE2O1VIPF13_0.png')


def _photo(h, w, rng):
  from PIL import Image
  lo = rng.integers(0, 256, (h // 8 + 1, w // 8 + 1, 3), dtype=np.uint8)           # smooth-ish content, like photos
  a = np.asarray(Image.fromarray(lo).resize((w, h), Image.BILINEAR)).astype(np.int16)
  return np.clip(a + rng.integers(-6, 7, a.shape), 0, 255).astype(np.uint8)        # with sensor-like noise


def _pngs(n, seed=1):
  from PIL import Image
  rng = np.random.default_rng(seed)
  out = [open(os.path.join(ROOT, 'tests', 'golden', f), 'rb').read() for f in FIXTURES]
  while len(out) < n:
    b = io.BytesIO()
    Image.fromarray(_photo(*SHAPES[len(out) % 3], rng)).save(b, 'PNG')
    out.append(b.getvalue())
  return out[:n]


def device_stages(files, iters):
  from twingan_b200 import ops, png
  infos = [png.parse(f) for f in files]
  offs = np.cumsum([0] + [i.H * i.W * 3 for i in infos])
  b = png.pack(files, infos, offs[:-1].tolist())
  payload = torch.empty(int(offs[-1]), dtype=torch.uint8, device='cuda')
  t = [torch.from_numpy(a).cuda() for a in (b.data, b.images, b.palettes)]
  run = lambda hook=None: ops.png_decode(payload, *t, b.raw_bytes, b.pixels, stage_hook=hook)
  assert not run().any().item()
  torch.cuda.synchronize()
  ms = {s: [] for s in ops.PNG_STAGES}
  for _ in range(iters):
    evs = [torch.cuda.Event(enable_timing=True)]
    evs[0].record()

    def hook(name):
      e = torch.cuda.Event(enable_timing=True)
      e.record()
      evs.append(e)
    run(hook)
    torch.cuda.synchronize()
    for s, a, z in zip(ops.PNG_STAGES, evs, evs[1:]):
      ms[s].append(a.elapsed_time(z))
  spread = {k.replace('twgpng_', ''): [round(min(v), 3), round(float(np.median(v)), 3), round(max(v), 3)]
            for k, v in ms.items()}
  total = sum(float(np.median(v)) for v in ms.values())
  return {'images': len(files), 'compressed_bytes': int(len(b.data)), 'inflated_bytes': int(b.images[:, 3].sum()),
          'pixels': b.pixels, 'ms_min_median_max': spread, 'ms_total_median': round(total, 3),
          'images_per_s': round(len(files) / (total * 1e-3), 1)}


def pil_decode(files, threads):
  from PIL import Image
  dec = lambda f: np.asarray(Image.open(io.BytesIO(f)).convert('RGB'))
  with ThreadPoolExecutor(threads) as pool:
    list(pool.map(dec, files))                                              # warm-up
    t0 = time.perf_counter()
    list(pool.map(dec, files))
    s = time.perf_counter() - t0
  return {'threads': threads, 'ms': round(s * 1e3, 2), 'images_per_s': round(len(files) / s, 1)}


def end_to_end(n, batch_size, rounds):
  """{output extension: {path: {threads: [images/s of each round]}}}, the device and PIL paths alternating."""
  from PIL import Image
  from twingan_b200 import translate, twingan
  d = tempfile.mkdtemp(prefix='twg_png_bench_')
  device_png = translate._device_png
  try:
    rng = np.random.default_rng(2)
    ins = []
    for i in range(n):
      p = os.path.join(d, 'in', '%05d.png' % i)
      os.makedirs(os.path.dirname(p), exist_ok=True)
      Image.fromarray(_photo(*SHAPES[i % 3], rng)).save(p)
      ins.append(p)
    model = twingan.GanModel(twingan.Flags(train_image_size=256), device='cuda', seed=3)
    paths = {'device': device_png, 'pil': lambda data: None}
    res = {}
    for ext in ('.jpg', '.png'):
      outs = [os.path.join(d, 'out', os.path.splitext(os.path.basename(p))[0] + ext) for p in ins]
      res[ext] = {name: {1: [], 8: []} for name in paths}
      for name, fn in paths.items():                                        # warm-up
        translate._device_png = fn
        translate.translate_files(model, ins[:batch_size], outs[:batch_size], batch_size=batch_size)
      for _ in range(rounds):
        for t in (1, 8):
          for name, fn in paths.items():
            translate._device_png = fn
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            translate.translate_files(model, ins, outs, batch_size=batch_size, num_decode_threads=t)
            torch.cuda.synchronize()
            res[ext][name][t].append(round(n / (time.perf_counter() - t0), 1))
    return res
  finally:
    translate._device_png = device_png
    shutil.rmtree(d, ignore_errors=True)


def main():
  ap = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
  ap.add_argument('--n', type=int, default=256, help='files of each end-to-end run (0: skip them)')
  ap.add_argument('--batch_size', type=int, default=64)
  ap.add_argument('--iters', type=int, default=10)
  ap.add_argument('--rounds', type=int, default=2)
  ap.add_argument('--out', default=None, help='also write the result as JSON here')
  args = ap.parse_args()
  assert torch.cuda.is_available(), 'tools/png_decode_bench.py needs a GPU'
  import __graft_entry__ as graft
  graft.build()
  from bench import gpu_info
  gpu = gpu_info(0)
  files = _pngs(args.batch_size)
  out = {'card': gpu['name'], 'power_limit_w': gpu['power_limit_w'], 'host_cores': os.cpu_count(),
         'device': device_stages(files, args.iters), 'pil': [pil_decode(files, t) for t in (1, 8)],
         'end_to_end': end_to_end(args.n, args.batch_size, args.rounds) if args.n else 'not measured'}
  print('card: %s, power limit %s W, %d host cores' % (gpu['name'], gpu['power_limit_w'] or 'not measured',
                                                       out['host_cores']))
  dv = out['device']
  print('device, %d files (%d compressed bytes, %d inflated): %s ms (min, median, max), %.1f images/s'
        % (dv['images'], dv['compressed_bytes'], dv['inflated_bytes'], dv['ms_min_median_max'], dv['images_per_s']))
  for p in out['pil']:
    print('PIL, %d thread(s): %.2f ms, %.1f images/s' % (p['threads'], p['ms'], p['images_per_s']))
  if isinstance(out['end_to_end'], dict):
    for ext, r in out['end_to_end'].items():
      for name, per in r.items():
        print('end to end, %d PNG -> %s, %s decoding: %s images/s by threads' % (args.n, ext, name, per))
  print(json.dumps(out))
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'w') as f:
      json.dump(out, f, indent=1)


if __name__ == '__main__':
  main()
