"""`python -m twingan_b200.translate`: translate image files with a trained model -- the reference's
inference/image_translation_infer.py (docs/infer_and_eval.md), with its flag names.

  python -m twingan_b200.translate --model_path=<train_dir>/256 --image_hw=256 \\
      --input_image_path=<file or directory> --output_image_path=<file or directory>

Decoding and encoding run on the host (PIL, as util_io.imread / imsave); everything between runs on the device.  Per batch:
  * a background thread decodes the files of batch k+1 on a pool of `--num_decode_threads` threads and packs them into
    one uint8 payload + a table of {offset, H, W} (HostPrefetcher, pinned memory) while batch k computes;
  * the payload and table are copied to the device on a side stream (DevicePrefetcher);
  * one kernel converts and resizes the ragged batch to the model input (ops.images_u8_to_batch: convert_image_dtype +
    TF-1 bilinear resize_images), the model translates it (InferencePipeline._infer: a CUDA graph per batch shape), one
    kernel quantises the result (ops.batch_to_u8: util_io.imsave's clip(x * 255).astype(uint8));
  * the uint8 images come back on a side stream (HostReturner) and are encoded and written on a thread pool.
A short last batch is padded with repeats of its last image, so one graph serves the whole run; the padded outputs are
dropped.  The outputs are image_hw x image_hw: like the reference, nothing resizes them back to the input's size.
"""
from __future__ import annotations

import argparse
import collections
import os
import sys
from concurrent.futures import ThreadPoolExecutor
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

IMAGE_EXTENSIONS = ('.jpg', '.jpeg', '.png')
INPUT_TENSORS = {'sources_ph': 't', 'targets_ph': 's'}      # placeholder -> target domain of its translation
# twingan.py:337-365: the outputs of the placeholder graph.  Without style embedding the four style variants of a direction
# are the same function of the input.
OUTPUT_TENSORS = {'custom_generated_%s_style_%s' % (d, v): d for d in ('t', 's') for v in ('source', 'target', 'rand', 'ph')}


def direction_of(input_tensor_name: str, output_tensor_name: str) -> str:
  """The target domain ('t' or 's') that an --input_tensor_name / --output_tensor_name pair of the reference selects:
  sources_ph pairs with custom_generated_t_style_*, targets_ph with custom_generated_s_style_* (an optional ':0' is
  accepted).  Unknown names and mismatched pairs raise ValueError."""
  strip = lambda n: n[:-2] if n.endswith(':0') else n
  i, o = strip(input_tensor_name), strip(output_tensor_name)
  if i not in INPUT_TENSORS:
    raise ValueError('unknown input tensor %r (one of %s)' % (input_tensor_name, ', '.join(sorted(INPUT_TENSORS))))
  if o not in OUTPUT_TENSORS:
    raise ValueError('unknown output tensor %r (one of %s)' % (output_tensor_name, ', '.join(sorted(OUTPUT_TENSORS))))
  if INPUT_TENSORS[i] != OUTPUT_TENSORS[o]:
    raise ValueError('output tensor %r is not computed from input tensor %r (sources_ph pairs with '
                     'custom_generated_t_style_*, targets_ph with custom_generated_s_style_*)'
                     % (output_tensor_name, input_tensor_name))
  return INPUT_TENSORS[i]


def list_images(input_image_path: str, output_image_path: str) -> Tuple[List[str], List[str]]:
  """(input files, output files).  A file maps to `output_image_path` itself.  A directory is walked recursively for
  .jpg / .jpeg / .png files (extension compared in lower case), sorted like util_io.get_files_in_dir(do_sort=True); each
  output is <output_image_path>/<basename>.  Two inputs with one basename, or an empty directory, raise ValueError."""
  if os.path.isfile(input_image_path):
    return [input_image_path], [output_image_path]
  if not os.path.isdir(input_image_path):
    raise FileNotFoundError('no image file or directory at %s' % input_image_path)
  found = []
  for root, dirs, files in os.walk(input_image_path):
    for fn in files:
      if os.path.splitext(fn)[1].lower() in IMAGE_EXTENSIONS:
        found.append(os.path.join(root, fn))
  found.sort()
  if not found:
    raise ValueError('no .jpg, .jpeg or .png files under %s' % input_image_path)
  seen = {}
  for p in found:
    b = os.path.basename(p)
    if b in seen:
      raise ValueError('%s and %s would both be written to %s' % (seen[b], p, os.path.join(output_image_path, b)))
    seen[b] = p
  return found, [os.path.join(output_image_path, os.path.basename(p)) for p in found]


def decode(path: str) -> np.ndarray:
  """uint8 [H, W, 3] RGB at full size (util_io.imread: PIL open + convert('RGB'))."""
  from PIL import Image
  try:
    with Image.open(path) as im:
      return np.asarray(im.convert('RGB'), dtype=np.uint8)
  except Exception as e:       # noqa: BLE001 -- re-raised with the path
    raise ValueError('cannot decode %s: %s' % (path, e)) from e


def save(arr: np.ndarray, path: str) -> None:
  """PIL's defaults for the format the extension implies, as scipy.misc.imsave did."""
  from PIL import Image
  Image.fromarray(arr).save(path)


def _padded_batches(images: Sequence[np.ndarray], batch_size: int):
  """(payload, table) of consecutive batches; the last one padded to batch_size rows with its last row."""
  from . import ops
  for start in range(0, len(images), batch_size):
    chunk = images[start:start + batch_size]
    payload, table = ops.pack_images(chunk)
    if len(chunk) < batch_size:
      table = torch.cat([table, table[-1:].expand(batch_size - len(chunk), 3)], 0)
    yield (payload, table), len(chunk)


class Translator(object):
  """The device path of a run: payload/table batches in, uint8 [n, hw, hw, 3] host arrays out, in order.  The staging
  buffers, result slots and CUDA graphs persist across `run` calls."""

  def __init__(self, model, target_domain: str = 't', use_graph: bool = True, depth: int = 2):
    from . import twingan
    from .prefetch import HostReturner
    self.model = model
    self.hw = int(model.flags.train_image_size)
    self.pipe = twingan.InferencePipeline(model, depth, use_graph=use_graph, target_domain=target_domain)
    self.back = HostReturner(model.device, depth)
    self.depth = depth

  def run(self, host_batches):
    """host_batches: iterable of ((payload, table), count).  Yields the first `count` translated images of each batch."""
    from . import ops
    from .prefetch import DevicePrefetcher
    counts = collections.deque()

    def tensors():
      for pair, n in host_batches:
        counts.append(n)
        yield pair

    feed = DevicePrefetcher(tensors(), self.model.device, self.depth)
    pending = None
    for payload, table in feed:
      x = ops.images_u8_to_batch(payload, table, self.hw)
      y = ops.batch_to_u8(self.pipe._infer(x))
      feed.release()
      done = self.back.put(y) + (counts.popleft(),)
      if pending is not None:
        yield self._finish(pending)
      pending = done
    if pending is not None:
      yield self._finish(pending)

  @staticmethod
  def _finish(pending):
    out, ev, n = pending
    if ev is not None:
      ev.synchronize()
    return out[:n].numpy().copy()             # the pinned slot is reused two batches later


def translate_arrays(model, images: Sequence[np.ndarray], target_domain: str = 't', batch_size: int = 64,
                     use_graph: bool = True) -> List[np.ndarray]:
  """Decoded uint8 [H, W, 3] RGB images of any sizes -> translated uint8 [hw, hw, 3] images (hw = the model's)."""
  if batch_size < 1:
    raise ValueError('batch_size must be positive')
  images = list(images)
  if not images:
    return []
  out = []
  for arr in Translator(model, target_domain, use_graph).run(_padded_batches(images, batch_size)):
    out.extend(arr)
  return out


def translate_files(model, input_paths: Sequence[str], output_paths: Sequence[str], target_domain: str = 't',
                    batch_size: int = 64, num_decode_threads: int = 8, use_graph: bool = True) -> int:
  """Translate input_paths[i] into output_paths[i] (created directories included); returns the number written."""
  from . import ops
  from .prefetch import HostPrefetcher
  if len(input_paths) != len(output_paths):
    raise ValueError('%d inputs but %d outputs' % (len(input_paths), len(output_paths)))
  if batch_size < 1 or num_decode_threads < 1:
    raise ValueError('batch_size and num_decode_threads must be positive')
  n = len(input_paths)
  if n == 0:
    return 0
  nb = (n + batch_size - 1) // batch_size
  decoders = ThreadPoolExecutor(num_decode_threads, thread_name_prefix='twg-decode')
  writers = ThreadPoolExecutor(num_decode_threads, thread_name_prefix='twg-encode')

  def produce(k):
    paths = input_paths[k * batch_size:(k + 1) * batch_size]
    payload, table = ops.pack_images(list(decoders.map(decode, paths)))
    if len(paths) < batch_size:
      table = torch.cat([table, table[-1:].expand(batch_size - len(paths), 3)], 0)
    return payload, table, torch.tensor(len(paths))

  host = HostPrefetcher(produce, capacity=2, num_batches=nb)
  for d in sorted({os.path.dirname(os.path.abspath(p)) for p in output_paths}):
    os.makedirs(d, exist_ok=True)
  written, in_flight = 0, collections.deque()
  try:
    batches = (((p, t), int(c)) for p, t, c in host)
    for k, arr in enumerate(Translator(model, target_domain, use_graph).run(batches)):
      outs = output_paths[k * batch_size:k * batch_size + len(arr)]
      in_flight.append([writers.submit(save, a, p) for a, p in zip(arr, outs)])
      while len(in_flight) > 2:                 # bound the images waiting to be encoded
        for f in in_flight.popleft():
          f.result()
          written += 1
    while in_flight:
      for f in in_flight.popleft():
        f.result()
        written += 1
  finally:
    host.close()
    decoders.shutdown(wait=True, cancel_futures=True)
    writers.shutdown(wait=True, cancel_futures=True)
  return written


def _parser() -> argparse.ArgumentParser:
  p = argparse.ArgumentParser(prog='python -m twingan_b200.translate', description=__doc__.split('\n\n')[0])
  p.add_argument('--model_path', required=True,
                 help='a model.ckpt-<step>.pt of pggan_runner, a directory of them (the newest), a TensorFlow checkpoint '
                      'prefix, or a directory holding a TensorFlow `checkpoint` file')
  p.add_argument('--image_hw', type=int, default=None,
                 help="the model's resolution: must match a .pt checkpoint's (taken from it when omitted); required for a "
                      'TensorFlow checkpoint')
  p.add_argument('--input_tensor_name', default='sources_ph', help='sources_ph (source -> target) or targets_ph')
  p.add_argument('--output_tensor_name', default='custom_generated_t_style_source',
                 help='custom_generated_{t,s}_style_{source,target,rand,ph}[:0], the direction of --input_tensor_name')
  p.add_argument('--input_image_path', required=True, help='an image file, or a directory walked for .jpg/.jpeg/.png')
  p.add_argument('--output_image_path', required=True, help='the output file, or the output directory')
  p.add_argument('--batch_size', type=int, default=64, help='images per model call')
  p.add_argument('--generator_norm_type', default='instance_norm')
  p.add_argument('--pggan_max_num_channels', type=int, default=256)
  p.add_argument('--num_decode_threads', type=int, default=8, help='host threads decoding (and encoding) images')
  p.add_argument('--no_graph', action='store_true', help='launch the kernels of every batch instead of a CUDA graph')
  return p


def main(argv=None) -> int:
  parser = _parser()
  args = parser.parse_args(argv)
  try:
    target_domain = direction_of(args.input_tensor_name, args.output_tensor_name)
  except ValueError as e:
    parser.error(str(e))
  if args.batch_size < 1 or args.num_decode_threads < 1:
    parser.error('--batch_size and --num_decode_threads must be positive')
  if args.image_hw is not None and (args.image_hw < 4 or args.image_hw & (args.image_hw - 1)):
    parser.error('--image_hw must be a power of two, at least 4 (got %d)' % args.image_hw)
  try:
    inputs, outputs = list_images(args.input_image_path, args.output_image_path)
  except (ValueError, FileNotFoundError) as e:
    parser.error(str(e))
  from . import pggan_runner, twingan
  flags = twingan.Flags(train_image_size=args.image_hw, pggan_max_num_channels=args.pggan_max_num_channels,
                        generator_norm_type=args.generator_norm_type)
  try:
    model, _ = pggan_runner.load_for_inference(args.model_path, flags)
  except ValueError as e:
    parser.error('--model_path: %s' % e)
  n = translate_files(model, inputs, outputs, target_domain, args.batch_size, args.num_decode_threads,
                      use_graph=not args.no_graph)
  print('translated %d image%s to %s' % (n, '' if n == 1 else 's', args.output_image_path))
  return n


if __name__ == '__main__':
  main(sys.argv[1:])
