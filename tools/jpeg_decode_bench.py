"""Times the device JPEG decoder (csrc/twg_jpeg.cu) against PIL, and `translate_files` end to end.

  python tools/jpeg_decode_bench.py [--n 192] [--batch_size 64] [--out result.json]

Device: CUDA events around each of the three stages (entropy / IDCT / upsample + colour) of one batch of `--batch_size`
seeded photo-like JPEG files of 368 x 371, 1024 x 768 and 512 x 512 (quality 90, 4:2:0, no restart markers, as PIL
writes them by default), `--iters` runs after a warm-up.  PIL: the same files decoded (Image.open + convert('RGB')) on 1
and 8 host threads, host clock.  End to end: images/s of translate_files with a seeded 256 x 256 model and .jpg outputs on
an all-JPEG directory of `--n` files, and on the mixed corpus of tools/translate_bench.py (half PNG, half JPEG), host clock
after a warm-up run.  The card name and power limit are read in the same run.  Needs a GPU.

  python tools/jpeg_decode_bench.py --progressive [--parent <checkout of the commit before>] [--runs 5]

Progressive files instead (csrc/twg_jpegp.cu): CUDA events around the coefficient reset, each level of scans, the IDCT
and the colour stage of one batch of `--batch_size` files of the same shapes written by PIL with progressive=True
(libjpeg's standard 10-scan script, 3 levels), and PIL on 1 and 8 threads.  End to end: images/s of translate_files (8
decode threads, .jpg outputs) on `--n` such files, each run in a fresh process after a warm-up, alternating run for run
between this tree and `--parent` (which decodes progressive files with PIL), so that both see the same machine state."""
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


def _photo(h, w, rng):
  from PIL import Image
  lo = rng.integers(0, 256, (h // 8 + 1, w // 8 + 1, 3), dtype=np.uint8)           # smooth-ish content, like photos
  return np.asarray(Image.fromarray(lo).resize((w, h), Image.BILINEAR))


def _jpegs(n, seed=1, **kw):
  from PIL import Image
  rng = np.random.default_rng(seed)
  out = []
  for i in range(n):
    b = io.BytesIO()
    Image.fromarray(_photo(*SHAPES[i % 3], rng)).save(b, 'JPEG', quality=90, **kw)
    out.append(b.getvalue())
  return out


def device_stages(files, iters):
  from twingan_b200 import jpeg, ops
  infos = [jpeg.parse(f) for f in files]
  offs = np.cumsum([0] + [i.H * i.W * 3 for i in infos])
  b = jpeg.pack(files, infos, offs[:-1].tolist())
  payload = torch.empty(int(offs[-1]), dtype=torch.uint8, device='cuda')
  t = [torch.from_numpy(a).cuda() for a in (b.data, b.segs, b.comps, b.images, b.qt, b.huff)]
  run = lambda hook=None: ops.jpeg_decode(payload, *t, b.blocks, b.plane_bytes, b.pixels, stage_hook=hook)
  assert not run().any().item()
  torch.cuda.synchronize()
  ms = {s: 0.0 for s in ops.JPEG_STAGES}
  for _ in range(iters):
    evs = [torch.cuda.Event(enable_timing=True)]
    evs[0].record()

    def hook(name):
      e = torch.cuda.Event(enable_timing=True)
      e.record()
      evs.append(e)
    run(hook)
    torch.cuda.synchronize()
    for s, a, z in zip(ops.JPEG_STAGES, evs, evs[1:]):
      ms[s] += a.elapsed_time(z) / iters
  total = sum(ms.values())
  return {'images': len(files), 'compressed_bytes': int(sum(len(f) for f in files)), 'pixels': b.pixels,
          'segments': len(b.segs), 'ms': {k.replace('twgjpeg_', ''): round(v, 3) for k, v in ms.items()},
          'ms_total': round(total, 3), 'images_per_s': round(len(files) / (total * 1e-3), 1)}


def progressive_stages(files, iters):
  from twingan_b200 import jpeg_progressive as jp, ops
  infos = [jp.parse(f) for f in files]
  offs = np.cumsum([0] + [i.H * i.W * 3 for i in infos])
  b = jp.pack(files, infos, offs[:-1].tolist())
  payload = torch.empty(int(offs[-1]), dtype=torch.uint8, device='cuda')
  t = [torch.from_numpy(a).cuda() for a in (b.data, b.segs, b.scans, b.comps, b.images, b.qt, b.huff)]
  run = lambda hook=None: ops.jpeg_progressive_decode(payload, *t, b.blocks, b.plane_bytes, b.pixels, b.levels,
                                                      stage_hook=hook)
  assert not run().any().item()
  torch.cuda.synchronize()
  ms = {}
  for _ in range(iters):
    evs, names = [torch.cuda.Event(enable_timing=True)], []
    evs[0].record()

    def hook(name):
      e = torch.cuda.Event(enable_timing=True)
      e.record()
      evs.append(e)
      names.append(name)
    run(hook)
    torch.cuda.synchronize()
    for s, a, z in zip(names, evs, evs[1:]):
      ms[s] = ms.get(s, 0.0) + a.elapsed_time(z) / iters
  total = sum(ms.values())
  short = lambda k: k.replace('twgjpegp_', '').replace('twgjpeg_', '')
  return {'images': len(files), 'compressed_bytes': int(sum(len(f) for f in files)), 'pixels': b.pixels,
          'scans': len(b.scans), 'segments': len(b.segs), 'levels': len(b.levels) - 1,
          'ms': {short(k): round(v, 3) for k, v in ms.items()}, 'ms_total': round(total, 3),
          'images_per_s': round(len(files) / (total * 1e-3), 1)}


# one end-to-end run in a fresh process: argv = tree, input directory, output directory, batch size
_E2E_RUN = r"""
import os, sys, time
sys.path.insert(0, sys.argv[1])
import torch
import __graft_entry__ as graft
graft.build()
from twingan_b200 import translate, twingan
ins = sorted(os.path.join(sys.argv[2], f) for f in os.listdir(sys.argv[2]))
outs = [os.path.join(sys.argv[3], os.path.basename(p)) for p in ins]
bs = int(sys.argv[4])
model = twingan.GanModel(twingan.Flags(train_image_size=256), device='cuda', seed=3)
translate.translate_files(model, ins[:bs], outs[:bs], batch_size=bs)
torch.cuda.synchronize()
t0 = time.perf_counter()
translate.translate_files(model, ins, outs, batch_size=bs, num_decode_threads=8)
torch.cuda.synchronize()
print('IMAGES_PER_S %.3f' % (len(ins) / (time.perf_counter() - t0)))
"""


def progressive_end_to_end(n, batch_size, parent, runs):
  import subprocess
  from statistics import median
  d = tempfile.mkdtemp(prefix='twg_jpegp_bench_')
  try:
    os.makedirs(os.path.join(d, 'in'))
    for i, f in enumerate(_jpegs(n, seed=2, progressive=True)):
      with open(os.path.join(d, 'in', '%05d.jpg' % i), 'wb') as fh:
        fh.write(f)
    trees = {'this': ROOT}
    if parent:
      trees['parent'] = os.path.abspath(parent)
    res = {k: [] for k in trees}
    for _ in range(runs):
      for k, tree in trees.items():
        out = os.path.join(d, 'out_' + k)
        os.makedirs(out, exist_ok=True)
        p = subprocess.run([sys.executable, '-c', _E2E_RUN, tree, os.path.join(d, 'in'), out, str(batch_size)],
                           capture_output=True, text=True, cwd=d)
        line = [l for l in p.stdout.splitlines() if l.startswith('IMAGES_PER_S')]
        assert p.returncode == 0 and line, p.stdout[-2000:] + p.stderr[-2000:]
        res[k].append(float(line[0].split()[1]))
    return {'images': n, 'inputs': 'all progressive JPEG', 'outputs': '.jpg', 'batch_size': batch_size,
            'decode_threads': 8, 'alternated_runs': runs,
            'images_per_s': {k: {'runs': [round(v, 1) for v in vs], 'median': round(median(vs), 1)}
                             for k, vs in res.items()}}
  finally:
    shutil.rmtree(d, ignore_errors=True)


def pil_decode(files, threads):
  from PIL import Image
  dec = lambda f: np.asarray(Image.open(io.BytesIO(f)).convert('RGB'))
  with ThreadPoolExecutor(threads) as pool:
    list(pool.map(dec, files))                                              # warm-up
    t0 = time.perf_counter()
    list(pool.map(dec, files))
    s = time.perf_counter() - t0
  return {'threads': threads, 'ms': round(s * 1e3, 2), 'images_per_s': round(len(files) / s, 1)}


def end_to_end(n, batch_size, mixed):
  from PIL import Image
  from twingan_b200 import translate, twingan
  d = tempfile.mkdtemp(prefix='twg_jpeg_bench_')
  try:
    rng = np.random.default_rng(1)
    ins = []
    for i in range(n):
      ext = ('png' if i % 2 else 'jpg') if mixed else 'jpg'
      p = os.path.join(d, 'in', '%05d.%s' % (i, ext))
      os.makedirs(os.path.dirname(p), exist_ok=True)
      Image.fromarray(_photo(*SHAPES[i % 3], rng)).save(p)
      ins.append(p)
    outs = [os.path.join(d, 'out', os.path.splitext(os.path.basename(p))[0] + ('.png' if mixed else '.jpg')) for p in ins]
    model = twingan.GanModel(twingan.Flags(train_image_size=256), device='cuda', seed=3)
    translate.translate_files(model, ins[:batch_size], outs[:batch_size], batch_size=batch_size)      # warm-up
    res = {}
    for t in (1, 8):
      torch.cuda.synchronize()
      t0 = time.perf_counter()
      translate.translate_files(model, ins, outs, batch_size=batch_size, num_decode_threads=t)
      torch.cuda.synchronize()
      res['threads_%d' % t] = round(n / (time.perf_counter() - t0), 1)
    return {'images': n, 'inputs': 'half PNG, half JPEG' if mixed else 'all JPEG',
            'outputs': '.png' if mixed else '.jpg', 'batch_size': batch_size, 'images_per_s': res}
  finally:
    shutil.rmtree(d, ignore_errors=True)


def main():
  ap = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
  ap.add_argument('--n', type=int, default=192, help='files of each end-to-end run (0: skip them)')
  ap.add_argument('--batch_size', type=int, default=64)
  ap.add_argument('--iters', type=int, default=20)
  ap.add_argument('--out', default=None, help='also write the result as JSON here')
  ap.add_argument('--progressive', action='store_true', help='time progressive files instead (see above)')
  ap.add_argument('--parent', default=None, help='with --progressive: a checkout of the commit before, to alternate with')
  ap.add_argument('--runs', type=int, default=5, help='with --progressive: end-to-end runs of each tree')
  args = ap.parse_args()
  assert torch.cuda.is_available(), 'tools/jpeg_decode_bench.py needs a GPU'
  import __graft_entry__ as graft
  graft.build()
  from bench import gpu_info
  gpu = gpu_info(0)
  if args.progressive:
    files = _jpegs(args.batch_size, progressive=True)
    out = {'card': gpu['name'], 'power_limit_w': gpu['power_limit_w'], 'host_cores': os.cpu_count(),
           'device': progressive_stages(files, args.iters), 'pil': [pil_decode(files, t) for t in (1, 8)],
           'end_to_end': (progressive_end_to_end(args.n, args.batch_size, args.parent, args.runs)
                          if args.n else 'not measured')}
    print(json.dumps(out))
    if args.out:
      os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
      with open(args.out, 'w') as f:
        json.dump(out, f, indent=1)
    return
  files = _jpegs(args.batch_size)
  out = {'card': gpu['name'], 'power_limit_w': gpu['power_limit_w'], 'host_cores': os.cpu_count(),
         'device': device_stages(files, args.iters), 'pil': [pil_decode(files, t) for t in (1, 8)],
         'end_to_end': ([end_to_end(args.n, args.batch_size, False), end_to_end(args.n, args.batch_size, True)]
                        if args.n else 'not measured')}
  print('card: %s, power limit %s W' % (gpu['name'], gpu['power_limit_w'] if gpu['power_limit_w'] else 'not measured'))
  dv = out['device']
  print('device, %d files (%d bytes, %d segments): %s ms = %.3f ms, %.1f images/s'
        % (dv['images'], dv['compressed_bytes'], dv['segments'], dv['ms'], dv['ms_total'], dv['images_per_s']))
  for p in out['pil']:
    print('PIL, %d thread(s): %.2f ms, %.1f images/s' % (p['threads'], p['ms'], p['images_per_s']))
  if isinstance(out['end_to_end'], list):
    for e in out['end_to_end']:
      print('end to end, %d files, %s -> %s: %s images/s' % (e['images'], e['inputs'], e['outputs'], e['images_per_s']))
  print(json.dumps(out))
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'w') as f:
      json.dump(out, f, indent=1)


if __name__ == '__main__':
  main()
