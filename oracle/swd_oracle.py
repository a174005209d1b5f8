"""fp64 restatement of PGGAN's sliced Wasserstein distance (Karras et al., ICLR 2018, section 5 and appendix D) for the
tests of twingan_b200/swd.py: plain numpy / scipy, consuming the same explicit draws (twingan_b200.swd.make_draws).

  1. Laplacian pyramid per image and channel: pyr_down = convolve(x, g)[::2, ::2], pyr_up = zeros inserted (values at the
     even indices) then convolve with 4 g, g = [1,4,6,4,1]^T [1,4,6,4,1] / 256, scipy.ndimage.convolve(mode='mirror');
     P[0] = x, then P[i] = pyr_down(P[i-1]) and P[i-1] -= pyr_up(P[i]); the last level stays Gaussian.
  2. Descriptors: nhood_size^2 neighbourhoods at the drawn centres, component order c*s*s + dy*s + dx.
  3. Per set and level, per-channel mean / population std over all neighbourhoods and positions (a zero std normalises
     the channel to 0, the library's rule).
  4. Per level and repeat: project both sets on the same unit directions, sort every column, mean |sortA - sortB|; the
     level's value is the mean over the repeats x 1e3.
  5. One value per level plus their average; the real-vs-real floor is the same between the two halves of the real set.
"""
import numpy as np
import scipy.ndimage

G = np.outer([1., 4., 6., 4., 1.], [1., 4., 6., 4., 1.]) / 256.0
_G4 = G[None, :, :, None]       # NHWC: filter over H, W only


def pyr_down(x):
  return scipy.ndimage.convolve(x, _G4, mode='mirror')[:, ::2, ::2, :]


def pyr_up(x):
  n, h, w, c = x.shape
  u = np.zeros((n, 2 * h, 2 * w, c), dtype=x.dtype)
  u[:, ::2, ::2, :] = x
  return scipy.ndimage.convolve(u, 4.0 * _G4, mode='mirror')


def laplacian_pyramid(images, levels):
  """images [N, R, R, C] -> list of `levels` arrays [N, R >> l, R >> l, C] in fp64."""
  p = [np.asarray(images, dtype=np.float64)]
  for _ in range(1, levels):
    p.append(pyr_down(p[-1]))
    p[-2] = p[-2] - pyr_up(p[-1])
  return p


def collapse(pyramid):
  """Inverse of laplacian_pyramid."""
  x = pyramid[-1]
  for lap in reversed(pyramid[:-1]):
    x = lap + pyr_up(x)
  return x


def descriptors(level, centres, nhood_size):
  """level [N, Rl, Rl, 3], centres int [N, nhoods, 2] = {y, x} -> [N * nhoods, 3 * s * s]."""
  h = nhood_size // 2
  centres = np.asarray(centres, dtype=np.int64)
  n, k = centres.shape[:2]
  off = np.arange(nhood_size) - h
  ys = centres[:, :, 0, None, None] + off[:, None]          # [n, k, s, 1]
  xs = centres[:, :, 1, None, None] + off[None, :]          # [n, k, 1, s]
  patches = level[np.arange(n)[:, None, None, None], ys, xs, :]     # [n, k, s, s, 3]
  return patches.transpose(0, 1, 4, 2, 3).reshape(n * k, -1)


def normalise(desc):
  """Per-channel mean / population std over all rows and positions (PGGAN finalize_descriptors)."""
  d = desc.reshape(desc.shape[0], 3, -1)
  mean = d.mean(axis=(0, 2), keepdims=True)
  std = d.std(axis=(0, 2), keepdims=True)
  scale = np.where(std > 0, 1.0 / np.where(std > 0, std, 1.0), 0.0)
  return ((d - mean) * scale).reshape(desc.shape)


def sliced_wasserstein(a, b, dirs):
  """a, b normalised [rows, D]; dirs [repeats, D, ndirs] -> mean over repeats of mean |sort(a dirs) - sort(b dirs)|."""
  vals = []
  for d in np.asarray(dirs, dtype=np.float64):
    pa = np.sort(a @ d, axis=0)
    pb = np.sort(b @ d, axis=0)
    vals.append(np.abs(pa - pb).mean())
  return float(np.mean(vals))


def swd(real, fake, draws, nhood_size=7, real_floor=True):
  """real, fake [n, R, R, 3] -> {'SWDx1e3_<res>', 'SWDx1e3_avg'} (+ 'real_' keys of the real-vs-real floor)."""
  real = np.asarray(real, dtype=np.float64)
  fake = np.asarray(fake, dtype=np.float64)
  R = real.shape[1]
  levels = int(np.log2(R)) - 3
  pr, pf = laplacian_pyramid(real, levels), laplacian_pyramid(fake, levels)
  out, floor = {}, {}
  for l in range(levels):
    c = np.asarray(draws['centres'][l])
    dirs = np.asarray(draws['dirs'][l], dtype=np.float64)
    da, db = descriptors(pr[l], c, nhood_size), descriptors(pf[l], c, nhood_size)
    out['SWDx1e3_%d' % (R >> l)] = sliced_wasserstein(normalise(da), normalise(db), dirs) * 1e3
    if real_floor:
      half = da.shape[0] // 2
      floor['real_SWDx1e3_%d' % (R >> l)] = sliced_wasserstein(normalise(da[:half]), normalise(da[half:]), dirs) * 1e3
  out['SWDx1e3_avg'] = float(np.mean(list(out.values())))
  if real_floor:
    floor['real_SWDx1e3_avg'] = float(np.mean(list(floor.values())))
    out.update(floor)
  return out
