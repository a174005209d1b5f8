"""Calibration of the projection bound of test_gpu_swd_conformance.py on the CPU.

k_swd_project normalises each descriptor component in fp32, (a - mean) * rstd (two roundings), and adds the K = 3 s^2
products for one output in one fp32 accumulator by FMA, k ascending.  This file emulates that in numpy (the product of
two fp32 values is exact in fp64, so an FMA is one rounding of the fp64 sum to fp32) on descriptors like the suite's,
one channel with |mean| >> std, and shows that the error against fp64 on the same fp32 inputs stays 4x inside the
suite's bound PROJECT_C * K * u * sum |a b| at every neighbourhood size the evaluation accepts, while a projection that
drops one term, or normalises one channel with another channel's statistics, exceeds it by more than 4x.  The emulated
error is 3-5 u sum |a b| at every K (it grows like sqrt(K), not K), so the smallest neighbourhood (K = 3) sets c."""
import numpy as np
import pytest

from tests.parity import U32
from tests.test_gpu_swd_conformance import PROJECT_C

MARGIN = 4.0
F32 = np.float32


def _inputs(rows, s, nd, seed):
  rng = np.random.default_rng(seed)
  ss = s * s
  A = (rng.standard_normal((rows, 3 * ss)) * 0.2).astype(F32)
  A[:, ss:2 * ss] += F32(3.0)
  d = rng.standard_normal((3 * ss, nd))
  B = (d / np.sqrt((d * d).sum(0, keepdims=True))).astype(F32)
  c = np.arange(3 * ss) // ss
  v = [A[:, c == i].astype(np.float64) for i in range(3)]
  mean = np.array([x.mean() for x in v]).astype(F32)
  rstd = np.array([1.0 / x.std() for x in v]).astype(F32)
  return A, B, c, mean, rstd


def _emulate(A, B, c, mean, rstd, mutant=None):
  cm = c.copy()
  if mutant == 'wrong_channel':
    cm[c == 1] = 0
  V = ((A - mean[cm]).astype(F32) * rstd[cm]).astype(F32)
  acc = np.zeros((A.shape[0], B.shape[1]), F32)
  for k in range(A.shape[1]):
    if mutant == 'drop_last' and k == A.shape[1] - 1:
      continue
    acc = (V[:, k:k + 1].astype(np.float64) * B[k].astype(np.float64) + acc.astype(np.float64)).astype(F32)
  return acc


def _ratio(A, B, c, mean, rstd, got):
  a = (A.astype(np.float64) - mean[c].astype(np.float64)) * rstd[c].astype(np.float64)
  b = B.astype(np.float64)
  ref, S = a @ b, np.abs(a) @ np.abs(b)
  return float(np.max(np.abs(got - ref) / (PROJECT_C * A.shape[1] * U32 * S)))


@pytest.mark.parametrize('s', [1, 3, 7, 15])
def test_projection_bound_holds_the_emulation_4x_inside(s):
  A, B, c, mean, rstd = _inputs(1024, s, 128, seed=s)
  r = _ratio(A, B, c, mean, rstd, _emulate(A, B, c, mean, rstd))
  assert r * MARGIN <= 1.0, (s, r)


@pytest.mark.parametrize('mutant', ['drop_last', 'wrong_channel'])
def test_projection_bound_catches_a_wrong_projection(mutant):
  A, B, c, mean, rstd = _inputs(1024, 7, 128, seed=11)
  r = _ratio(A, B, c, mean, rstd, _emulate(A, B, c, mean, rstd, mutant))
  assert r >= MARGIN, (mutant, r)
