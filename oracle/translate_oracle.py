"""fp64 restatement of the image translation front and back end (twingan_b200/csrc/twg_image.cu), for tests only.

Front end (inference/image_translation_infer.py:54-58): tf.image.convert_image_dtype (p = u8 * fl32(1/255)) followed by
TF 1.8's resize_bilinear with align_corners=False and no half-pixel centres (resize_bilinear_op.cc).  The coordinate step
is taken in fp32 as TF takes it -- scale = fl32(H / hw), in = fl32(y * scale), y0 = int(in), y1 = min(y0 + 1, H - 1),
l = in - y0 -- so the taps and weights are exactly the kernel's; the interpolation is then evaluated in fp64.

Back end (util_io.imsave): clip(fl32(x * 255), 0, 255) truncated to uint8.
"""
import numpy as np

INV255 = np.float64(np.float32(1.0) / np.float32(255.0))       # fl32(1/255), exactly representable in fp64


def taps(out_size: int, in_size: int):
  """(lower, upper, lerp) per output coordinate, fp32 as compute_interpolation_weights of resize_bilinear_op.cc."""
  scale = np.float32(in_size) / np.float32(out_size)
  pos = np.arange(out_size, dtype=np.float32) * scale
  lo = np.minimum(pos.astype(np.int64), in_size - 1)
  hi = np.minimum(lo + 1, in_size - 1)
  return lo, hi, (pos - lo.astype(np.float32)).astype(np.float64)


def resize(image_u8: np.ndarray, hw: int) -> np.ndarray:
  """uint8 [H, W, 3] -> fp64 [hw, hw, 3]."""
  y0, y1, ly = taps(hw, image_u8.shape[0])
  x0, x1, lx = taps(hw, image_u8.shape[1])
  p = lambda ys, xs: image_u8[ys][:, xs].astype(np.float64) * INV255      # only the sampled pixels
  lx = lx[None, :, None]
  top = p(y0, x0) + (p(y0, x1) - p(y0, x0)) * lx
  bot = p(y1, x0) + (p(y1, x1) - p(y1, x0)) * lx
  return top + (bot - top) * ly[:, None, None]


def images_to_batch(images, hw: int) -> np.ndarray:
  return np.stack([resize(im, hw) for im in images])


def to_u8(x) -> np.ndarray:
  """NaN maps to 0."""
  v = np.asarray(x, dtype=np.float32) * np.float32(255)
  v = np.where(np.isnan(v), np.float32(0), v)
  return np.clip(v, 0, 255).astype(np.uint8)
