"""A golden vector set stored as several compressed .npz parts (<stem>_0.npz, <stem>_1.npz, ...) so that no file in the
repository exceeds 1 MB; loaded back as one read-only mapping with the interface of np.load's NpzFile."""
import glob
import io
import os

import numpy as np

PART_BYTES = 640 * 1024     # compressed size one part may reach (estimated per array, so parts stay below 1 MB)


class NpzParts:
  def __init__(self, paths):
    self._parts = [np.load(p) for p in paths]
    self._where = {k: part for part in self._parts for k in part.files}
    self.files = list(self._where)

  def __getitem__(self, key):
    return self._where[key][key]

  def __contains__(self, key):
    return key in self._where


def load(stem):
  """stem: path without the _<i>.npz suffix."""
  paths = sorted(glob.glob(stem + '_*.npz'), key=lambda p: int(p[len(stem) + 1:-4]))
  if not paths:
    raise FileNotFoundError(stem + '_*.npz')
  return NpzParts(paths)


def save(stem, arrays):
  """Writes `arrays` (name -> array) as compressed parts of at most PART_BYTES each (an array larger than that on its own
  gets a part of its own), in the order given."""
  for old in glob.glob(stem + '_*.npz'):
    os.remove(old)
  part, size, i = {}, 0, 0

  def flush():
    nonlocal part, size, i
    if part:
      np.savez_compressed('%s_%d.npz' % (stem, i), **part)
      part, size, i = {}, 0, i + 1

  for k, v in arrays.items():
    buf = io.BytesIO()
    np.savez_compressed(buf, a=v)
    n = buf.tell()
    if size + n > PART_BYTES:
      flush()
    part[k] = v
    size += n
  flush()
