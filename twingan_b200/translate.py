"""`python -m twingan_b200.translate`: translate image files with a trained model -- the reference's
inference/image_translation_infer.py (docs/infer_and_eval.md), with its flag names.

  python -m twingan_b200.translate --model_path=<train_dir>/256 --image_hw=256 \\
      --input_image_path=<file or directory> --output_image_path=<file or directory>

JPEG (baseline and progressive) and PNG files are decoded on the device, pixel for pixel as PIL decodes them, and JPEG outputs are encoded there,
byte for byte as PIL does; PIL decodes every other input (as util_io.imread) and encodes every other output (as
util_io.imsave); everything between runs on the device.  Per batch:
  * a background thread reads the files of batch k+1 on a pool of `--num_decode_threads` threads.  A JPEG that
    twingan_b200/jpeg.py accepts (baseline Huffman, grey or YCbCr, 4:4:4 / 4:2:2 / 4:2:0), a progressive JPEG that
    twingan_b200/jpeg_progressive.py accepts (the same frames, every coefficient refined to its last bit) or a PNG that
    twingan_b200/png.py accepts (not interlaced, not animated, no palette transparency, known chunks, every CRC right)
    travels compressed, with its descriptors; PIL decodes every other file into its region of one uint8 payload + a
    table of {offset, H, W} (HostPrefetcher, pinned memory; the headers give the device files' rows before any
    decoding) while batch k computes;
  * the payload, table and compressed data are copied to the device on a side stream (DevicePrefetcher);
  * three kernels decode the JPEG scans (ops.jpeg_decode), three the PNG streams (ops.png_decode), and the progressive
    JPEG files are entropy-decoded one level of scans at a time before the same inverse DCT and colour kernels
    (ops.jpeg_progressive_decode), into their regions of a copy of the payload, on a stream of the batch's own, up to Translator.DECODE_AHEAD batches ahead of the one
    translated (_DeviceDecoder: the decoders are serial within a file, so batches decode side by side); the batch's
    status is read once, when it is translated, and an image the device could not decode exactly is decoded by PIL and
    written into its region instead (a file PIL refuses fails as before);
  * one kernel converts and resizes the ragged batch to the model input (ops.images_u8_to_batch: convert_image_dtype +
    TF-1 bilinear resize_images), the model translates it (InferencePipeline._infer: a CUDA graph per batch shape), one
    kernel quantises the result (ops.batch_to_u8: util_io.imsave's clip(x * 255).astype(uint8));
  * the outputs PIL would save as JPEG (their extension maps to 'JPEG' in Image.registered_extensions()) are encoded on
    the device (ops.jpeg_encode: the entropy-coded scans packed back to back, jpeg.py writes the header PIL writes);
    their offsets come back on a side stream; a batch later, when the host waits for that batch anyway, exactly their
    bytes follow on a stream that holds nothing of the batch computing meanwhile (ScanReturner).  A batch with any other
    output returns its uint8 images (HostReturner) for PIL to encode.  A thread pool writes the files.
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


class _DeviceFiles(object):
  """The files of a batch one device decoder decodes: their paths, their table rows {offset, H, W}, and the host sizes
  its ops call takes after the descriptor tensors.  (Not a tuple: the prefetcher maps over tuples.)"""

  def __init__(self, paths, rows, sizes):
    self.paths, self.rows, self.sizes = paths, rows, sizes


def _read(path: str) -> Optional[bytes]:
  """The file's bytes, or None when it cannot be read (decode() then raises its usual error)."""
  try:
    with open(path, 'rb') as f:
      return f.read()
  except OSError:
    return None


def _device_jpeg(data: Optional[bytes]):
  """jpeg.JpegInfo when the device decodes this file, else None.  Images above PIL's decompression-bomb limit stay with
  PIL, which warns or refuses as before."""
  from PIL import Image
  from . import jpeg
  info = jpeg.probe(data) if data else None
  if info is not None and Image.MAX_IMAGE_PIXELS and info.H * info.W > Image.MAX_IMAGE_PIXELS:
    return None
  return info


def _device_png(data: Optional[bytes]):
  """png.PngInfo when the device decodes this file, else None; as _device_jpeg, above PIL's decompression-bomb limit
  PIL decides."""
  from PIL import Image
  from . import png
  info = png.probe(data) if data and data[:8] == png.SIGNATURE else None
  if info is not None and Image.MAX_IMAGE_PIXELS and info.H * info.W > Image.MAX_IMAGE_PIXELS:
    return None
  return info


def _device_jpegp(data: Optional[bytes]):
  """jpeg_progressive.ProgressiveInfo when the device decodes this file, else None; as _device_jpeg, above PIL's
  decompression-bomb limit PIL decides."""
  from PIL import Image
  from . import jpeg_progressive
  info = jpeg_progressive.probe(data) if data else None
  if info is not None and Image.MAX_IMAGE_PIXELS and info.H * info.W > Image.MAX_IMAGE_PIXELS:
    return None
  return info


DEVICE_KINDS = ('jpeg', 'png', 'jpegp')      # the device decoders, in the order a batch packs and decodes their files


def _device_file(data: Optional[bytes]):
  """('jpeg', 'png' or 'jpegp', its info) when the device decodes this file, else None."""
  info = _device_jpeg(data)
  if info is not None:
    return 'jpeg', info
  info = _device_png(data)
  if info is not None:
    return 'png', info
  info = _device_jpegp(data)
  return ('jpegp', info) if info is not None else None


def _redecode(payload: torch.Tensor, status: torch.Tensor, files: '_DeviceFiles') -> None:
  """PIL decodes (decode(), so a file PIL refuses raises as before) each image whose status is not 0 into its region of
  the device payload."""
  for i in torch.nonzero(status).flatten().tolist():
    off, h, w = files.rows[i]
    arr = decode(files.paths[i])
    if arr.shape != (h, w, 3):
      raise ValueError('cannot decode %s: PIL reads %s, the header says %dx%d' % (files.paths[i], arr.shape[:2], h, w))
    payload[off:off + arr.size].copy_(torch.from_numpy(arr.reshape(-1).copy()))


class _DeviceDecoder(object):
  """Decodes batches' JPEG, PNG and progressive JPEG files on the device with `ahead` batches in flight behind the one being translated.

  Entropy decoding and inflate are serial within a file (a thread or a warp each), so one batch keeps a few SMs busy
  for as long as its largest file takes.  Each batch therefore decodes on a stream of its own, concurrently with the
  batches around it and with the model, and the host reads its status only when the batch is translated.  `start`
  copies the batch out of the prefetcher's staging slot (on the main stream, so the slot can be refilled at once) and
  enqueues the decoders on that batch's stream; `finish` waits for the status, lets PIL decode the images the device
  flagged, and orders the main stream after the decoding."""

  def __init__(self, device, ahead: int):
    self.device = torch.device(device)
    self.streams = [torch.cuda.Stream(device=self.device) for _ in range(ahead + 1)]
    self._n = 0

  def start(self, payload: torch.Tensor, table: torch.Tensor, descriptors, jpegs: Optional['_DeviceFiles'],
            pngs: Optional['_DeviceFiles'], jpegps: Optional['_DeviceFiles'] = None):
    """(payload, table, handle) of a batch (the six tensors of a jpeg.Batch, then the three of a png.Batch, then the
    seven of a jpeg_progressive.Batch, each present when its files are), the first two copies owned by the caller from
    now on."""
    from . import ops
    payload, table = payload.clone(), table.clone()
    descriptors = [d.clone() for d in descriptors]
    copied = torch.cuda.Event()
    copied.record(torch.cuda.current_stream(self.device))
    stream = self.streams[self._n % len(self.streams)]   # its last batch was finished before this one started
    self._n += 1
    if jpegs is None and pngs is None and jpegps is None:
      return payload, table, None
    stream.wait_event(copied)
    for t in [payload] + descriptors:
      t.record_stream(stream)
    with torch.cuda.stream(stream):
      status = []
      if jpegs is not None:
        status.append(ops.jpeg_decode(payload, *descriptors[:6], *jpegs.sizes))
        descriptors = descriptors[6:]
      if pngs is not None:
        status.append(ops.png_decode(payload, *descriptors[:3], *pngs.sizes))
        descriptors = descriptors[3:]
      if jpegps is not None:
        status.append(ops.jpeg_progressive_decode(payload, *descriptors[:7], *jpegps.sizes))
      status = torch.cat(status) if len(status) > 1 else status[0]
      host = torch.empty(status.numel(), dtype=torch.int32).pin_memory()
      host.copy_(status, non_blocking=True)
      done = torch.cuda.Event()
      done.record(stream)
    return payload, table, (host, done, (jpegs, pngs, jpegps))

  def finish(self, payload: torch.Tensor, handle) -> None:
    if handle is None:
      return
    host, done, groups = handle
    done.synchronize()
    torch.cuda.current_stream(self.device).wait_event(done)
    status = host.clone()
    at = 0
    for files in groups:                       # the groups' statuses follow one another, as start decoded them
      if files is not None:
        _redecode(payload, status[at:at + len(files.paths)], files)
        at += len(files.paths)


def _produce_batch(paths: Sequence[str], batch_size: int, pool: ThreadPoolExecutor):
  """(tensors, (count, jpegs, pngs, jpegps)) of one batch for Translator.run: PIL decodes the files the device does
  not."""
  from . import jpeg, jpeg_progressive, ops, png
  blobs = list(pool.map(_read, paths))
  kinds = list(pool.map(_device_file, blobs))
  host = [i for i, k in enumerate(kinds) if k is None]
  arrays = dict(zip(host, pool.map(decode, [paths[i] for i in host])))
  shapes = [(k[1].H, k[1].W) if k is not None else arrays[i].shape[:2] for i, k in enumerate(kinds)]
  table = np.zeros((batch_size, 3), np.int64)
  off = 0
  for i, (h, w) in enumerate(shapes):
    table[i] = (off, h, w)
    off += h * w * 3
  table[len(paths):] = table[len(paths) - 1]
  payload = np.empty(off, np.uint8)
  for i, a in arrays.items():
    payload[table[i, 0]:table[i, 0] + a.size] = a.reshape(-1)
  payload, table_t = torch.from_numpy(payload), torch.from_numpy(table)
  ops.check_table(table_t, payload.numel())
  tensors, files = (payload, table_t), []
  for kind in DEVICE_KINDS:
    dev = [i for i, k in enumerate(kinds) if k is not None and k[0] == kind]
    if not dev:
      files.append(None)
      continue
    args = [blobs[i] for i in dev], [kinds[i][1] for i in dev], [int(table[i, 0]) for i in dev]
    if kind == 'jpeg':
      b = jpeg.pack(*args)
      tensors += tuple(torch.from_numpy(a) for a in (b.data, b.segs, b.comps, b.images, b.qt, b.huff))
      sizes = (b.blocks, b.plane_bytes, b.pixels)
    elif kind == 'png':
      b = png.pack(*args)
      tensors += tuple(torch.from_numpy(a) for a in (b.data, b.images, b.palettes))
      sizes = (b.raw_bytes, b.pixels)
    else:
      b = jpeg_progressive.pack(*args)
      tensors += tuple(torch.from_numpy(a) for a in (b.data, b.segs, b.scans, b.comps, b.images, b.qt, b.huff))
      sizes = (b.blocks, b.plane_bytes, b.pixels, b.levels)
    files.append(_DeviceFiles([paths[i] for i in dev], [tuple(int(v) for v in table[i]) for i in dev], sizes))
  return tensors, (len(paths),) + tuple(files)


def save(arr: np.ndarray, path: str) -> None:
  """PIL's defaults for the format the extension implies, as scipy.misc.imsave did."""
  from PIL import Image
  Image.fromarray(arr).save(path)


def saves_as_jpeg(path: str) -> bool:
  """Whether `save` writes this path as a JPEG file: PIL picks the format from the lower-cased extension."""
  from PIL import Image
  return Image.registered_extensions().get(os.path.splitext(path)[1].lower()) == 'JPEG'


def _write(data: bytes, path: str) -> None:
  with open(path, 'wb') as f:
    f.write(data)


class ScanReturner(object):
  """The JPEG scans of ops.jpeg_encode device -> host, only the bytes of the rows asked for.  `put` enqueues the copy of
  the offsets on a side stream behind the main stream's work.  `fetch` waits for that copy, which already implies the
  batch's encode is done, then copies the rows' bytes on a second stream that holds nothing else, so the host waits for
  that batch alone and not for the batch queued after it.  Pinned buffers are reused, growing only when a batch needs
  more."""

  def __init__(self, device, depth: int = 2):
    self.device = torch.device(device)
    self.depth = max(2, int(depth))
    self._stream = torch.cuda.Stream(device=self.device)
    self._copy = torch.cuda.Stream(device=self.device)
    self._offsets = [None] * self.depth
    self._bytes = None
    self._n = 0
    self.d2h_bytes = 0

  def put(self, scans: torch.Tensor, offsets: torch.Tensor):
    slot = self._n % self.depth                # fetch runs in order and is synchronous: the slot's last use is over
    self._n += 1
    k = int(offsets.numel())
    if self._offsets[slot] is None or self._offsets[slot].numel() < k:
      self._offsets[slot] = torch.empty(k, dtype=torch.int64).pin_memory()
    ready = torch.cuda.Event()
    ready.record(torch.cuda.current_stream(self.device))
    with torch.cuda.stream(self._stream):
      self._stream.wait_event(ready)
      self._offsets[slot][:k].copy_(offsets, non_blocking=True)
      ev = torch.cuda.Event()
      ev.record(self._stream)
    self.d2h_bytes += k * 8
    return slot, k, scans, offsets, ev

  def fetch(self, handle, rows: Sequence[int]) -> List[bytes]:
    """The scans of `rows` (ascending) of a batch `put` returned `handle` for."""
    slot, k, scans, _, ev = handle
    ev.synchronize()
    off = self._offsets[slot][:k].numpy().copy()
    runs = []                                  # [first row, last row] of each run of consecutive rows
    for r in rows:
      if runs and runs[-1][1] == r - 1:
        runs[-1][1] = r
      else:
        runs.append([r, r])
    total = int(sum(off[b + 1] - off[a] for a, b in runs))
    if self._bytes is None or self._bytes.numel() < total:
      size = max(total, 2 * (self._bytes.numel() if self._bytes is not None else 0))
      self._bytes = torch.empty(size, dtype=torch.uint8).pin_memory()
    at, where = 0, {}
    with torch.cuda.stream(self._copy):        # the batch's encode is done: nothing to wait for on the device
      for a, b in runs:
        m = int(off[b + 1] - off[a])
        self._bytes[at:at + m].copy_(scans[int(off[a]):int(off[b + 1])], non_blocking=True)
        for r in range(a, b + 1):
          where[r] = at + int(off[r] - off[a])
        at += m
      done = torch.cuda.Event()
      done.record(self._copy)
    done.synchronize()
    self.d2h_bytes += total
    data = self._bytes[:total].numpy()
    return [data[where[r]:where[r] + int(off[r + 1] - off[r])].tobytes() for r in rows]


def _padded_batches(images: Sequence[np.ndarray], batch_size: int):
  """(payload, table) of consecutive batches; the last one padded to batch_size rows with its last row."""
  from . import ops
  for start in range(0, len(images), batch_size):
    chunk = images[start:start + batch_size]
    payload, table = ops.pack_images(chunk)
    if len(chunk) < batch_size:
      table = torch.cat([table, table[-1:].expand(batch_size - len(chunk), 3)], 0)
    yield (payload, table), (len(chunk), None, None, None)


class Translator(object):
  """The device path of a run: payload/table batches in, uint8 [n, hw, hw, 3] host arrays out, in order.  The staging
  buffers, result slots and CUDA graphs persist across `run` calls."""

  # batches whose device decoding runs behind the one being translated: enough that the serial decoders of several
  # batches share the GPU (tools/png_decode_bench.py)
  DECODE_AHEAD = 3

  def __init__(self, model, target_domain: str = 't', use_graph: bool = True, depth: int = 2):
    from . import twingan
    from .prefetch import HostReturner
    self.model = model
    self.hw = int(model.flags.train_image_size)
    self.pipe = twingan.InferencePipeline(model, depth, use_graph=use_graph, target_domain=target_domain)
    self.back = HostReturner(model.device, depth)
    self.scans = ScanReturner(model.device, depth) if self.back.cuda else None
    self.depth = depth
    self.decoder = _DeviceDecoder(model.device, self.DECODE_AHEAD) if self.back.cuda else None

  def run(self, host_batches, jpeg_rows=None):
    """host_batches: iterable of (tensors, (count, jpegs, pngs, jpegps)): tensors = (payload, table) host tensors,
    followed by the six descriptor tensors of a jpeg.Batch when `jpegs` (a _DeviceFiles) names JPEG images the device
    decodes, then the three of a png.Batch when `pngs` names PNG images, then the seven of a jpeg_progressive.Batch when
    `jpegps` names progressive JPEG images.  Yields the first
    `count` translated images of each batch.  With `jpeg_rows` (per batch, `count` booleans), yields (images or None,
    {row: JPEG scan bytes}) instead: the marked rows are encoded on the device, and the images come back only when
    some row is not marked.  From the first batch with files the device decodes, the batches go through the decoder
    in order, up to DECODE_AHEAD of them decoding behind the one translated."""
    from . import ops
    from .prefetch import DevicePrefetcher
    counts = collections.deque()

    def tensors():
      for t, info in host_batches:
        counts.append(info)
        yield t

    feed = DevicePrefetcher(tensors(), self.model.device, self.depth)
    decoding = collections.deque()               # (k, n, payload, table, handle) in order

    def ready():
      """(k, n, payload, table, staged): the batches in order, each once its images are in its payload; `staged`: the
      payload is the prefetcher's slot, to be released once the batch has been enqueued."""
      for k, batch in enumerate(feed):
        n, jpegs, pngs, jpegps = counts.popleft()
        if jpegs is None and pngs is None and jpegps is None and not decoding:
          yield k, n, batch[0], batch[1], True
          continue
        decoding.append((k, n) + self.decoder.start(batch[0], batch[1], batch[2:], jpegs, pngs, jpegps))
        feed.release()                           # start copied the batch out of its slot
        while len(decoding) > self.DECODE_AHEAD:
          k0, n0, payload, table, handle = decoding.popleft()
          self.decoder.finish(payload, handle)
          yield k0, n0, payload, table, False
      while decoding:
        k0, n0, payload, table, handle = decoding.popleft()
        self.decoder.finish(payload, handle)
        yield k0, n0, payload, table, False

    pending = None
    for k, n, payload, table, staged in ready():
      x = ops.images_u8_to_batch(payload, table, self.hw)
      y = ops.batch_to_u8(self.pipe._infer(x))
      if staged:
        feed.release()
      rows = None if jpeg_rows is None else [i for i, j in enumerate(jpeg_rows[k]) if j]
      scans = None
      if rows:                                  # every row is encoded; only the marked rows' bytes come back
        scans = self.scans.put(*ops.jpeg_encode(y[:n])), rows
      raw = self.back.put(y) if rows is None or len(rows) < n else None
      if pending is not None:
        yield self._finish(pending)
      pending = (raw, scans, n, jpeg_rows is not None)
    if pending is not None:
      yield self._finish(pending)

  def _finish(self, pending):
    raw, scans, n, files = pending
    arrays = None
    if raw is not None:
      out, ev = raw
      if ev is not None:
        ev.synchronize()
      arrays = out[:n].numpy().copy()           # the pinned slot is reused two batches later
    if not files:
      return arrays
    return arrays, (dict(zip(scans[1], self.scans.fetch(*scans))) if scans is not None else {})


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
  from . import jpeg
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
  writers = ThreadPoolExecutor(num_decode_threads, thread_name_prefix='twg-encode')   # PIL encodes non-JPEG outputs

  def produce(k):
    return _produce_batch(input_paths[k * batch_size:(k + 1) * batch_size], batch_size, decoders)

  host = HostPrefetcher(produce, capacity=2, num_batches=nb)
  for d in sorted({os.path.dirname(os.path.abspath(p)) for p in output_paths}):
    os.makedirs(d, exist_ok=True)
  written, in_flight = 0, collections.deque()
  as_jpeg = [saves_as_jpeg(p) for p in output_paths]
  jpeg_rows = [as_jpeg[k * batch_size:(k + 1) * batch_size] for k in range(nb)]
  try:
    translator = Translator(model, target_domain, use_graph)
    header = jpeg.encoder_header(translator.hw, translator.hw) if any(as_jpeg) else b''
    for k, (arr, scans) in enumerate(translator.run(host, jpeg_rows)):
      outs = output_paths[k * batch_size:(k + 1) * batch_size]
      in_flight.append([writers.submit(_write, header + scans[i] + jpeg.EOI, p) if i in scans else
                        writers.submit(save, arr[i], p) for i, p in enumerate(outs)])
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
