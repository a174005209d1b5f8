"""GPU tests of the split route of twg_norm_act_bwd_reduce: a sample spread over a cluster of K CTAs (K = 2, 4, 8) when it
has at least 512 KB and the batch's clusters run in one wave.  The split kernel adds every sum in the order of the
one-block kernels, and a sample's sums do not depend on the rest of its batch, so each case runs its samples twice: at
its own N (the split route) and as the first samples of a batch too large for any cluster size (the one-block streamed
kernel).  gu and red of those samples must be bit-identical between the two.

The host's choice of K is restated here (split_k); the device's cluster occupancy comes from the library.  Cases: every
twg_norm_act_bwd_reduce key of tests/product_norms.py that takes the split route on this device; each channel-vector
layout (V = 1, 2, 4) at each K; HW not a multiple of the pixel groups per block (gpb) nor of a batch; one chain a pixel
longer than the others; gz, gpool and both; flags 0-3.  Every launch runs twice into fresh buffers with canary words
after the outputs."""
import pytest
import torch

from tests.product_norms import PRODUCT_NORMS
from tests.test_gpu_norm_conformance import DEV, _ab, _gen, _p, _st, _y

pytestmark = pytest.mark.gpu

SPLIT_MIN = 512 << 10             # bytes of the smallest sample the route splits (kSplitMinBytes)
CANARY = 12345.0
PAD = 256


def _lib():
  from twingan_b200._lib import lib
  return lib()


def vec_geom(C):
  """(G lanes per pixel, V float4 per lane) of a vectorisable channel count, else None (vec_geom in twg_common.cuh)."""
  if C % 4:
    return None
  q = C // 4
  if q <= 32:
    return (q, 1) if q & (q - 1) == 0 else None
  return (32, q // 32) if q % 32 == 0 and q // 32 in (1, 2, 4) else None


def clusters(C, K):
  return int(_lib().cdll.twg_norm_bwd_reduce_split_clusters(C, K))


def split_k(N, HW, C):
  """K of the reduce's launch: the largest of 8, 4, 2 that divides gpb and for which N clusters of K CTAs run at once,
  for a vectorisable sample of at least SPLIT_MIN bytes; 1 (the one-block kernels) otherwise."""
  geom = vec_geom(C)
  if geom is None or HW * C * 4 < SPLIT_MIN:
    return 1
  gpb = 256 // geom[0]
  for K in (8, 4, 2):
    if gpb % K == 0 and N <= clusters(C, K):
      return K
  return 1


def _unsplit_batch(C):
  return max(clusters(C, K) for K in (2, 4, 8)) + 1


def _run(L, N, HW, W, C, flags, t):
  """Two launches into fresh canaried buffers; returns gu [N, HW, C] and red [N, C, 2] of the first."""
  outs = []
  for _ in range(2):
    gu = torch.full((N * HW * C + PAD,), CANARY, device=DEV)
    red = torch.full((N * C * 2 + PAD,), CANARY, device=DEV)
    L.call('twg_norm_act_bwd_reduce', _p(t['y']), _p(t['a']), _p(t['b']), _p(t['mean']), _p(t['rstd']), _p(t['gz']),
           _p(t['gp']), W, _p(gu), _p(red), N, HW, C, flags, _st())
    outs.append((gu, red))
  torch.cuda.synchronize()
  (gu, red), (gu2, red2) = outs
  assert torch.equal(gu, gu2) and torch.equal(red, red2), 'two launches differ'
  assert bool((gu[N * HW * C:] == CANARY).all()) and bool((red[N * C * 2:] == CANARY).all()), 'canary overwritten'
  return gu[:N * HW * C].view(N, HW, C), red[:N * C * 2].view(N, C, 2)


def _inputs(N, HW, W, C, opts, seed):
  y = _y(N, HW, C, seed)
  a, b, mean, rstd = _ab(y, seed + 1)
  o = opts.split('+')
  gz = torch.randn((N, HW, C), device=DEV, generator=_gen(seed + 2)) if 'gz' in o else None
  gp = torch.randn((N, HW // W // 2, W // 2, C), device=DEV, generator=_gen(seed + 3)) if 'gpool' in o else None
  return {'y': y, 'a': a, 'b': b, 'mean': mean, 'rstd': rstd, 'gz': gz, 'gp': gp}


def check_split_equals_one_block(N, HW, W, C, flags, opts, seed=961):
  """Runs the case on the split route and embedded in a one-block batch; returns the K it was split over."""
  K = split_k(N, HW, C)
  assert K > 1, 'not a split-route case: N=%d HW=%d C=%d' % (N, HW, C)
  Nb = _unsplit_batch(C)
  assert split_k(Nb, HW, C) == 1
  L = _lib()
  t = _inputs(N, HW, W, C, opts, seed)
  rest = _inputs(Nb - N, HW, W, C, opts, seed + 10)
  tb = {k: None if v is None else torch.cat([v, rest[k]]) for k, v in t.items()}
  gu, red = _run(L, N, HW, W, C, flags, t)
  gub, redb = _run(L, Nb, HW, W, C, flags, tb)
  assert torch.equal(gu, gub[:N]), 'gu differs from the one-block kernel (K=%d)' % K
  assert torch.equal(red, redb[:N]), 'red differs from the one-block kernel (K=%d)' % K
  return K


def _product_cases():
  return [k for k in PRODUCT_NORMS['twg_norm_act_bwd_reduce'] if vec_geom(k[3]) and k[1] * k[3] * 4 >= SPLIT_MIN]


def _id(case):
  return '-'.join(str(v) for v in case)


@pytest.mark.parametrize('case', _product_cases(), ids=_id)
def test_product_key(case):
  N, HW, W, C, flags, opts = case
  if split_k(N, HW, C) == 1:
    pytest.skip('one-block route on this device: N=%d exceeds the clusters that run at once' % N)
  check_split_equals_one_block(N, HW, W, C, flags, opts)


def test_product_keys_reach_the_split_route():
  """The bench step's streamed keys at N = 32 take the split route."""
  assert all(split_k(*k[:2], k[3]) > 1 for k in _product_cases() if k[0] == 32)


# each layout at each K: C = 16 (G = 4), 256 (V = 2), 512 (V = 4) and 128 (G = 32, V = 1, gpb = 8)
@pytest.mark.parametrize('C', [16, 128, 256, 512])
@pytest.mark.parametrize('K', [8, 4, 2])
def test_every_cluster_size(C, K):
  G, V = vec_geom(C)
  gpb = 256 // G
  lo = 1 if K == 8 else clusters(C, 2 * K) + 1       # the smallest N that no longer fits clusters of 2 K
  assert lo <= clusters(C, K), 'K=%d is never chosen for C=%d' % (K, C)
  HW = max(SPLIT_MIN // (4 * C), gpb * 4 * K) + gpb // 2 + 1
  assert check_split_equals_one_block(lo, HW, 0, C, 3, 'gz') == K


# (N, HW, W, C, flags, opts): HW not a multiple of gpb nor of a batch (4 / V pixels x K per chain), one chain a pixel
# longer than its neighbours (HW = m gpb + 1), pooled gradients with whole and short batches, flags 0-3
def _edge_cases():
  cases = []
  for C in (16, 32, 64, 128, 256, 512):
    G, V = vec_geom(C)
    gpb = 256 // G
    base = -(-SPLIT_MIN // (4 * C))
    for HW in (gpb * (base // gpb + 3) + 1, gpb * (base // gpb + 5) + gpb // 2 + 3):
      for flags in (0, 1, 2, 3):
        cases.append((3, HW, 0, C, flags, 'gz'))
    for W in (2 * gpb, 2 * gpb + 2):
      H = 2 * (-(-base // (2 * W)) + 1)
      cases.append((2, H * W, W, C, 3, 'gpool'))
      cases.append((2, H * W, W, C, 1, 'gz+gpool'))
  return cases


@pytest.mark.parametrize('case', _edge_cases(), ids=_id)
def test_edge_geometry(case):
  check_split_equals_one_block(*case)
