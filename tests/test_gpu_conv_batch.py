"""The convolutions of the product at the batch sizes it launches them with.

The kernel suite (test_gpu_kernels.CONV_SHAPES) runs each layer at N = 1 .. 12, but N decides how the weight gradients
split their pixels (launch_wgrad's tiles per CTA and whether the last CTA is short, the SIMT splits and the pointwise
blocks: test_gpu_conv_conformance's restated host rules) and whether the last batch tile of a tensor-core conv is ragged.
Here every product weight-gradient key runs at its own N, and every tensor-core forward / dgrad key of images below
16 x 16 (several images a tile) at a batch of whole tiles or, where ragged, one whose last tile holds a single image:
each against the fp64 reference with the kernel suite's per-element bounds, twice (bit-identical), the weight gradients
also with accumulate = 1."""
import pytest
import torch

from oracle import twingan_oracle as O
from tests.parity import _log_result, conv_error_ratio, exact_elem_c, tc_elem_c
from tests.product_launches import Recorder
from tests.test_gpu_conv_conformance import (PRODUCT_CONV_KEYS, WGRAD_ENTRIES, _bits, _split_ref, conv_keys, pick_tile,
                                             pw_wgrad_blocks, simt_wgrad_splits, tc_wgrad_grid)

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'


def _batch_cases():
  """(key, N): each product weight-gradient key at its N; each tensor-core forward / dgrad key whose tiles hold several
  images (TN > 1) at N = TN + 1 when it is ragged (one full tile and one of a single image) and N = TN when not (the
  per-sample arithmetic of these kernels is batch-invariant, so one such batch stands for every other).  Pure Python:
  collected without the library."""
  cases = []
  for key in sorted(PRODUCT_CONV_KEYS, key=str):
    if key[0] in WGRAD_ENTRIES:
      cases.append((key, key[1]))
    elif key[0] in ('twg_conv_fwd_planes', 'twg_conv_dgrad_planes'):
      TN = pick_tile(1, key[1], key[2])[2]
      if TN > 1:
        cases.append((key, TN + 1 if 'ragged' in key[-1].split('+') else TN))
  return cases


BATCH_CONV_CASES = _batch_cases()


def _case_id(case):
  return '-'.join(str(v) for v in case[0]).replace('twg_conv_', '') + '-N%d' % case[1]


def _randn(shape, seed, scale=1.0):
  return torch.randn(shape, device=DEV, generator=torch.Generator(device=DEV).manual_seed(seed)) * scale


def _wgrad64(x, gy, k, pad):
  """fp64 weight gradient of conv2d(x, w) for the output gradient gy."""
  w = torch.zeros((k, k, x.shape[3], gy.shape[3]), device=DEV, dtype=torch.float64, requires_grad=True)
  y = O.conv2d_nhwc(x.double(), w, 'SAME' if pad else 'VALID')
  return torch.autograd.grad(y, w, gy.double())[0]


def _wgrad_geometry(N, H, W, Cin, Cout, k, pad, tc):
  if tc:
    return tc_wgrad_grid(N, H, W, Cin, Cout, k, pad)
  if k == 1 and pad == 0 and min(Cin, Cout) <= 4:
    blocks, chunk = pw_wgrad_blocks(N, H, W, Cin, Cout)
    return {'pw_blocks': blocks, 'pixels_per_block': chunk}
  splits, mps = simt_wgrad_splits(N, H, W, Cin, Cout, k, pad)
  return {'simt_splits': splits, 'pixels_per_split': mps}


def _run_wgrad(key, N, rec):
  from twingan_b200 import ops
  name, _, H, W, Cin, Cout, k, pad, opts = key
  Ho, Wo = H + 2 * pad - k + 1, W + 2 * pad - k + 1
  x, gy = _randn((N, H, W, Cin), 901), _randn((N, Ho, Wo, Cout), 902)
  before = _randn((k, k, Cin, Cout), 903)
  with rec.spying():
    first, second = ops.conv_wgrad_raw(x, gy, k, pad), ops.conv_wgrad_raw(x, gy, k, pad)
    buf = before.clone()
    ops._conv_wgrad(x, gy, k, pad, out=buf)
  torch.cuda.synchronize()
  assert torch.equal(first, second)
  assert torch.equal(buf, before + first)               # accumulate = 1 adds the same sum to what the buffer holds
  tc = name == 'twg_conv_wgrad_planes'
  ref = _wgrad64(x, gy, k, pad)
  S = _wgrad64(x.abs(), gy.abs(), k, pad)
  del x, gy
  K = _wgrad64(torch.ones((N, H, W, 1), device=DEV), torch.ones((N, Ho, Wo, 1), device=DEV), k, pad).expand_as(ref)
  c = tc_elem_c(K) if tc else exact_elem_c(K)
  res = {'wgrad': conv_error_ratio(first, ref, S, c),
         'geometry': _wgrad_geometry(N, H, W, Cin, Cout, k, pad, tc)}
  return res


def _run_fwd_dgrad(key, N, rec):
  from twingan_b200 import ops
  name, H, W, Cin, Cout, k, pad, opts = key
  opts = tuple(o for o in opts.split('+') if o and o != 'ragged')
  x, w, gy = _randn((N, H, W, Cin), 911), _randn((k, k, Cin, Cout), 912, 0.05), _randn((N, H, W, Cout), 913)
  with rec.spying():
    if name == 'twg_conv_dgrad_planes':
      assert not opts, key
      run = lambda xs, gys: ops.conv_dgrad_raw(gys, w, tuple(xs.shape), k, pad)
    else:
      assert name == 'twg_conv_fwd_planes', key
      run = lambda xs, gys: ops.conv_fwd_raw(xs, w, k, pad)
    out, again = run(x, gy), run(x, gy)
    per_sample = torch.cat([run(x[i:i + 1], gy[i:i + 1]) for i in range(N)])
    if opts:
      # the key's epilogue options on the same output: one fp32 rounding per operation, like torch's.  (Ragged tiles
      # are those of images below 16 x 16, which have no fused epilogue: no sign mask, no statistics.)
      assert set(opts) <= {'bias', 'act', 'zp'}, key
      bias = _randn((Cout,), 914, 0.5)
      zp = torch.empty((2,) + tuple(out.shape), device=DEV, dtype=torch.bfloat16) if 'zp' in opts else None
      y, _ = ops._conv_fwd(x, w, k, pad, bias=bias if 'bias' in opts else None, act='act' in opts, zp=zp)
  torch.cuda.synchronize()
  assert torch.equal(out, again)
  assert torch.equal(out, per_sample)
  if opts:
    t = out + bias
    want = torch.maximum(0.2 * t, t) if 'act' in opts else t
    assert torch.equal(y, want if 'bias' in opts else out)
    if 'zp' in opts:
      assert torch.equal(_bits(zp), _bits(_split_ref(y)))
  a, b = x.double().requires_grad_(True), w.double().requires_grad_(True)
  ones = (torch.ones_like(a), torch.ones_like(b))
  if name == 'twg_conv_dgrad_planes':
    f = lambda u, v, g: torch.autograd.grad(O.conv2d_nhwc(u, v, 'SAME' if pad else 'VALID'), u, g)[0]
    ref = f(a, b, gy.double())
    S = f(a.detach().abs().requires_grad_(True), b.detach().abs(), gy.double().abs())
    K = f(ones[0].requires_grad_(True), ones[1], torch.ones_like(gy, dtype=torch.float64))
  else:
    f = lambda u, v: O.conv2d_nhwc(u, v, 'SAME' if pad else 'VALID').detach()
    ref, S, K = f(a, b), f(a.abs(), b.abs()), f(*ones)
  return {name.replace('twg_conv_', '').replace('_planes', ''): conv_error_ratio(out, ref, S, tc_elem_c(K)),
          'geometry': dict(zip(('TW', 'TH', 'TN', 'tiles_w', 'tiles_h', 'tiles_n'), pick_tile(N, H, W)))}


@pytest.mark.parametrize('case', BATCH_CONV_CASES, ids=_case_id)
def test_conv_at_the_product_batch_against_fp64(built_lib, case):
  from twingan_b200 import ops
  key, N = case
  ops.set_precision(1)
  rec = Recorder(built_lib, conv_keys)
  try:
    res = _run_wgrad(key, N, rec) if key[0] in WGRAD_ENTRIES else _run_fwd_dgrad(key, N, rec)
  finally:
    torch.cuda.empty_cache()
  assert key in rec.keys(), (key, sorted(rec.keys(), key=str))
  _log_result({'test': 'conv_batch', 'key': list(key), 'N': N, 'ratios': res})
  bad = {k: v for k, v in res.items() if k != 'geometry' and not v <= 1.0}
  assert not bad, (key, N, res)


def test_batch_cases_reach_short_ctas_and_ragged_tiles(built_lib):
  """The product batches put the per-tap tensor-core weight gradient (not the column-box kernel) into launches whose last
  CTA is cut short, and ragged batch tiles into the forward and dgrad; the cases above run them."""
  short = [(key, N) for key, N in BATCH_CONV_CASES if key[0] == 'twg_conv_wgrad_planes'
           and not tc_wgrad_grid(*key[1:8])['cols'] and tc_wgrad_grid(*key[1:8])['last_cta_tiles'] <
           tc_wgrad_grid(*key[1:8])['tiles_per_cta']]
  ragged = [(key, N) for key, N in BATCH_CONV_CASES if key[0] != 'twg_conv_wgrad_planes' and 'ragged' in key[-1]]
  _log_result({'test': 'conv_batch_reach', 'short_last_cta': len(short), 'ragged': len(ragged)})
  assert short and ragged
  assert ('twg_conv_wgrad_planes', 9, 8, 8, 256, 256, 3, 1, 'accumulate') in PRODUCT_CONV_KEYS
