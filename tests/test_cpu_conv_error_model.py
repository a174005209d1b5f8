"""Calibration of the per-element conv bound |dev - ref| <= c * S (tests/parity.py conv_error_ratio, tc_elem_c) on the CPU.

The tensor-core convolutions multiply split-bf16 operands: a = hi + lo with hi = bf16(a), lo = bf16(a - hi), and each
product is formed from three MMAs, lo.hi + hi.lo + hi.hi.  Emulated exactly in fp64, that arithmetic stays 4x inside
c = tc_elem_c(K) at every tensor-core edge shape of the kernel suite, in all three directions, while the kernel bugs the bound
is there to catch -- a dropped cross term, hi.hi only, a missing K chunk, a border tap reading a pixel instead of the
zero padding -- exceed it by more than 4x."""
import pytest
import torch
import torch.nn.functional as F

from tests.parity import conv_error_ratio, tc_elem_c
from tests.test_gpu_kernels import TC_EDGE_SHAPES, _rand

MARGIN = 4.0


def _nchw(t):
  return t.permute(0, 3, 1, 2)


def _nhwc(t):
  return t.permute(0, 2, 3, 1)


def _ops(shape):
  """The three directions as bilinear functions of NHWC / HWIO fp64 operands."""
  N, H, W, Cin, Cout, k, pad = shape

  def fwd(x, w):
    return _nhwc(F.conv2d(_nchw(x), w.permute(3, 2, 0, 1), padding=pad))

  def dgrad(gy, w):
    return _nhwc(torch.nn.grad.conv2d_input((N, Cin, H, W), w.permute(3, 2, 0, 1), _nchw(gy), padding=pad))

  def wgrad(x, gy):
    return torch.nn.grad.conv2d_weight(_nchw(x), (Cout, Cin, k, k), _nchw(gy), padding=pad).permute(2, 3, 1, 0)

  return {'fwd': fwd, 'dgrad': dgrad, 'wgrad': wgrad}


def _split(t):
  """fp64 -> the fp32 value the device holds -> its bf16 hi / lo planes (round to nearest even), as fp64."""
  t32 = t.to(torch.float32)
  hi = t32.to(torch.bfloat16)
  lo = (t32 - hi.to(torch.float32)).to(torch.bfloat16)
  return hi.double(), lo.double()


def _operands(shape):
  N, H, W, Cin, Cout, k, pad = shape
  Ho, Wo = H + 2 * pad - k + 1, W + 2 * pad - k + 1
  x = _rand((N, H, W, Cin), 1)         # the operands of test_conv_fwd_dgrad_wgrad
  w = _rand((k, k, Cin, Cout), 2, 0.05)
  gy = _rand((N, Ho, Wo, Cout), 3)
  return {'fwd': (x, w), 'dgrad': (gy, w), 'wgrad': (x, gy)}


def _drop_k_chunk(d, a, b, shape):
  """The operands with one K chunk zeroed: 16 channels of the centre tap (forward / dgrad K = taps x channels), or the first
  128-pixel tile (weight-gradient K = pixels)."""
  k = shape[5]
  if d == 'wgrad':
    flat = a.clone().reshape(-1, a.shape[-1])
    flat[:128] = 0
    return flat.reshape(a.shape), b
  b = b.clone()
  if d == 'fwd':
    b[k // 2, k // 2, :16, :] = 0
  else:
    b[k // 2, k // 2, :, :16] = 0
  return a, b


@pytest.mark.parametrize('shape', TC_EDGE_SHAPES)
def test_split_bf16_model_error_is_within_the_bound_and_kernel_bugs_are_not(shape):
  ops = _ops(shape)
  for d, (a, b) in _operands(shape).items():
    op = ops[d]
    ref, S, c = op(a, b), op(a.abs(), b.abs()), tc_elem_c(op(torch.ones_like(a), torch.ones_like(b)))
    (ah, al), (bh, bl) = _split(a), _split(b)
    hh, hl, lh = op(ah, bh), op(ah, bl), op(al, bh)
    ratio = lambda got: conv_error_ratio(got, ref, S, c)
    model = ratio(hh + hl + lh)
    assert model <= 1.0 / MARGIN, (d, model)
    mutants = {'no lo.hi': hh + hl, 'no hi.lo': hh + lh, 'hi.hi only': hh, 'K chunk missing': op(*_drop_k_chunk(d, a, b, shape))}
    for name, got in mutants.items():
      assert ratio(got) >= MARGIN, (d, name, ratio(got))


@pytest.mark.parametrize('shape', [s for s in TC_EDGE_SHAPES if s[5] == 3])
def test_a_border_tap_shifted_by_one_pixel_exceeds_the_bound(shape):
  """The left zero-padding column replaced by the image's first column: the kw = 0 tap of every border output reads the
  pixel one to its right instead of zero."""
  x, w = _operands(shape)['fwd']
  fwd = _ops(shape)['fwd']
  ref, S, c = fwd(x, w), fwd(x.abs(), w.abs()), tc_elem_c(fwd(torch.ones_like(x), torch.ones_like(w)))
  xp = F.pad(_nchw(x), (1, 1, 1, 1))
  xp[:, :, :, 0] = xp[:, :, :, 1]
  got = _nhwc(F.conv2d(xp, w.permute(3, 2, 0, 1)))
  assert conv_error_ratio(got, ref, S, c) >= MARGIN
