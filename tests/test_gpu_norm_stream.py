"""GPU tests of the kernels that read their input through a shared-memory ring (twg_stream.cuh): the normaliser's backward
reduce, its moments and the DRAGAN batch variance, against fp64 with the bounds of tests/parity.py, at geometries chosen
for the ring rather than for the product.

A stage holds T = 4096 / C pixels of each operand (16 KB); a sample of at least two stages is streamed, a smaller one
takes the direct-load kernel.  Cases: the largest kept size (2 T - 1 pixels) and the smallest streamed one (2 T, whole
stages), one pixel short of and one pixel past a whole number of stages, and more stages than the ring is deep (14 stages
against rings of 6 and 12, the last one a single pixel); gz only, gpool only and both (the pooled cases on 14 image rows,
with whole and short last stages); each channel-vector layout (V = 1 with 4 and 32 lanes per pixel, V = 2, V = 4); N = 1,
3 and 64; leaky-ReLU and pixel norm on and off.  Each case runs twice into fresh buffers, the results must be
bit-identical, and the words after gu, red, sums and the variance's two doubles must be untouched."""
import pytest
import torch

from tests.parity import U32, conv_error_ratio, dragan_var_rel_bound, exact_elem_c, norm_sum_c, serial_run
from tests.test_gpu_norm_conformance import DEV, _ab, _check_moments, _gen, _gu_ref, _p, _pool_bcast, _st, _y

pytestmark = pytest.mark.gpu

STAGE = 16384                     # bytes of one operand in one ring stage (kStreamStage)
CANARY = 12345.0
PAD = 256                         # canary words after each output


def _T(C):
  return STAGE // (4 * C)


def _lib():
  from twingan_b200._lib import lib
  return lib()


def _out(n):
  """n result words followed by PAD canary words."""
  return torch.full((n + PAD,), CANARY, device=DEV)


def _clean(buf, n):
  return bool((buf[n:] == CANARY).all())


def _reduce_cases():
  cases = []
  for C in (16, 128, 256, 512):
    T = _T(C)
    for HW in (2 * T - 1, 2 * T, 3 * T - 1, 3 * T + 1, 13 * T + 1):
      cases.append((3, HW, 0, C, 3, 'gz'))
    for flags in (0, 1, 2):
      cases.append((1, 13 * T + 1, 0, C, flags, 'gz'))
    cases.append((64, 3 * T + 1, 0, C, 3, 'gz'))
    for W in (T, T + 2):                                   # 14 image rows: whole stages / a short last stage
      cases.append((3, 14 * W, W, C, 3, 'gpool'))
      cases.append((3, 14 * W, W, C, 1, 'gz+gpool'))
  return cases


def _moments_cases():
  cases = []
  for C in (16, 128, 256, 512):
    T = _T(C)
    for HW in (2 * T - 1, 2 * T, 3 * T - 1, 3 * T + 1, 13 * T + 1):
      cases.append((3, HW, C, 1))
    cases += [(1, 13 * T + 1, C, 1), (64, 3 * T + 1, C, 16)]
  return cases


def _id(case):
  return '-'.join(str(v) for v in case)


@pytest.mark.parametrize('case', _reduce_cases(), ids=_id)
def test_streamed_reduce(case):
  N, HW, W, C, flags, opts = case
  o = opts.split('+')
  L = _lib()
  y = _y(N, HW, C, 931)
  a, b, mean, rstd = _ab(y, 932)
  H = HW // W if W else 0
  gz = torch.randn((N, HW, C), device=DEV, generator=_gen(933)) if 'gz' in o else None
  gp = torch.randn((N, H // 2, W // 2, C), device=DEV, generator=_gen(934)) if 'gpool' in o else None
  outs = []
  for _ in range(2):
    gu, red = _out(N * HW * C), _out(N * C * 2)
    L.call('twg_norm_act_bwd_reduce', _p(y), _p(a), _p(b), _p(mean), _p(rstd), _p(gz), _p(gp), W, _p(gu), _p(red), N, HW, C,
           flags, _st())
    outs.append((gu, red))
  torch.cuda.synchronize()
  (gu, red), (gu2, red2) = outs
  assert torch.equal(gu, gu2) and torch.equal(red, red2)
  assert _clean(gu, N * HW * C) and _clean(red, N * C * 2)
  gu, red = gu[:N * HW * C].view(N, HW, C), red[:N * C * 2].view(N, C, 2)
  g = torch.zeros((N, HW, C), device=DEV, dtype=torch.float64)
  if gz is not None:
    g += gz.double()
  if gp is not None:
    g += 0.25 * _pool_bcast(gp.double(), H, W)
  gu_ref, S = _gu_ref(y, a, b, flags, g)
  assert conv_error_ratio(gu, gu_ref, S, exact_elem_c(C)) <= 1.0
  gu64 = gu.double()
  yhat = (y.double() - mean.double()[:, None]) * rstd.double()[:, None]
  c = norm_sum_c(serial_run(HW, C)) + 4 * U32
  assert conv_error_ratio(red[..., 0], gu64.sum(1), gu64.abs().sum(1), c) <= 1.0
  assert conv_error_ratio(red[..., 1], (gu64 * yhat).sum(1), (gu64 * yhat).abs().sum(1), c) <= 1.0


@pytest.mark.parametrize('case', _moments_cases(), ids=_id)
def test_streamed_moments(case):
  N, HW, C, pg = case
  L = _lib()
  y = _y(N, HW, C, 941)
  outs = []
  for _ in range(2):
    sums = _out(N * C * 2)
    L.call('twg_moments', _p(y), _p(sums), N, HW, C, pg, _st())
    outs.append(sums)
  torch.cuda.synchronize()
  assert torch.equal(outs[0], outs[1])
  assert _clean(outs[0], N * C * 2)
  assert _check_moments(outs[0][:N * C * 2].view(N, C, 2), y, pg) <= 1.0


# total elements: the largest kept size and the smallest streamed one, one 16-byte unit short of and past whole stages
# beyond the ring's depth, and a total that is not a multiple of four elements (bulk copies move 16-byte units: kept)
@pytest.mark.parametrize('N,per', [(1, 8188), (1, 8192), (4, 3 * 1024 - 1), (1, 13 * 4096 + 4), (2, 13 * 2048 + 1),
                                   (16, 64 * 64 * 3)], ids=lambda v: str(v))
def test_streamed_variance(N, per):
  L = _lib()
  g = _gen(951)
  x = torch.rand((N, per), device=DEV, generator=g)
  x[:, 0::3] = x[:, 0::3] * 0.1 + 0.8
  alpha = torch.rand(N, device=DEV, generator=g)
  noise = torch.rand((N, per), device=DEV, generator=g) * 2 - 1
  outs = []
  for _ in range(2):
    xhat, scratch = _out(N * per), _out(4)
    L.call('twg_dragan_xhat', _p(x), _p(alpha), _p(noise), _p(xhat), _p(scratch), N, per, _st())
    outs.append((xhat, scratch))
  torch.cuda.synchronize()
  assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
  xhat, scratch = outs[0]
  assert _clean(xhat, N * per) and _clean(scratch, 4)
  x64 = x.double()
  R = -(-N * per // 256)
  s2 = scratch[:4].view(torch.float64)
  c = norm_sum_c(R)
  assert abs(float(s2[0]) - float(x64.sum())) <= c * float(x64.abs().sum())
  assert abs(float(s2[1]) - float((x64 * x64).sum())) <= (c + U32) * float((x64 * x64).sum())
  m = x64.mean()
  var = ((x64 - m) ** 2).mean()
  pert = alpha.double()[:, None] * (0.5 * var * noise.double())
  ref = x64 + pert
  bound = (dragan_var_rel_bound(R, 1 + m * m / var) + 4 * U32) * pert.abs() + 2 * U32 * ref.abs()
  assert float(((xhat[:N * per].view(N, per).double() - ref).abs() / (bound + 1e-30)).max()) <= 1.0
