"""The column-box forward / dgrad keys that keep their weights in shared memory (GEMM K <= 32, BN <= 64), at the
work splits their scheduling creates: fewer work items than CTAs (a warpgroup with no tile), an odd number of items per
CTA (one warpgroup takes one tile fewer than the other), and border tiles.  Each result is held to fp64 and computed twice,
bit for bit the same both times."""
import pytest
import torch

from tests.parity import conv_error_ratio, tc_elem_c
from tests.test_gpu_conv_cols import _stats_reference
from tests.test_gpu_conv_conformance import _all_option_sets, _bits, _fwd_planes, _split_ref, expected_rc
from tests.test_gpu_kernels import _dev, _rand, conv_refs

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'

# (GEMM K, BN) of every resident-weight key: the forward runs Cin = K, Cout = BN, the data gradient Cout = K, Cin = BN
KEYS = [(16, 16), (16, 32), (16, 64), (32, 16), (32, 32), (32, 64)]
# N, H, W
GEOMS = {
    'few_items': (1, 16, 32),     # 4 work items for up to 132 CTAs
    'odd_items': (12, 88, 48),    # 11 x 3 tiles x 12 images = 396 = 3 x 132: three items per CTA
    'border': (2, 20, 40),        # 3 x 3 tiles per image, all at a border, ragged on both sides
}


def _twice(fn):
  a = fn()
  torch.cuda.synchronize()
  b = fn()
  torch.cuda.synchronize()
  assert torch.equal(_bits(a), _bits(b))
  return a


@pytest.mark.parametrize('geom', sorted(GEOMS))
@pytest.mark.parametrize('key', KEYS)
def test_resident_fwd_and_dgrad_against_fp64(built_lib, key, geom):
  from twingan_b200 import ops
  K, BN = key
  N, H, W = GEOMS[geom]
  for Cin, Cout, seed in ((K, BN, 401), (BN, K, 411)):      # forward key (K, BN), then dgrad key (K, BN)
    x, w, gy = _rand((N, H, W, Cin), seed), _rand((3, 3, Cin, Cout), seed + 1, 0.05), _rand((N, H, W, Cout), seed + 2)
    (yr, gxr, _), (sy, sgx, _), (ky, kgx, _) = conv_refs(x, w, gy, 3, 1, DEV)
    if Cin == K:
      y = _twice(lambda: ops.conv_fwd_raw(_dev(x), _dev(w), 3, 1))
      assert conv_error_ratio(y, yr, sy, tc_elem_c(ky)) <= 1.0, (Cin, Cout)
    if Cout == K:
      gx = _twice(lambda: ops.conv_dgrad_raw(_dev(gy), _dev(w), (N, H, W, Cin), 3, 1))
      assert conv_error_ratio(gx, gxr, sgx, tc_elem_c(kgx)) <= 1.0, (Cin, Cout)


@pytest.mark.parametrize('geom', ['odd_items', 'border'])
@pytest.mark.parametrize('key', KEYS)
def test_resident_fwd_epilogues(built_lib, key, geom):
  """Every option set of twg_conv_fwd_planes and the affine entry, each run twice: y bit for bit the plain output's bias /
  leaky-ReLU, planes and sign mask from y, statistics records at their (tile, consumer warp) slots against fp64, and the
  affine result against fp64."""
  from twingan_b200 import ops
  L = built_lib
  Cin, Cout = key
  N, H, W = GEOMS[geom]
  shape = (N, H, W, Cin, Cout, 3, 1)
  slots = ops._epilogue_slots(*shape)
  tiles_h, tiles_w = -(-H // 8), -(-W // 16)
  assert slots == tiles_h * tiles_w * 8
  x, w = _rand((N, H, W, Cin), 421), _rand((3, 3, Cin, Cout), 422, 0.08)
  xp, wp = ops.split_act(_dev(x)), ops.weight_planes(_dev(w), False)
  bias = _dev(_rand((Cout,), 423, 0.5))
  y_plain = _twice(lambda: ops._conv_fwd(None, _dev(w), 3, 1, xp=xp)[0])
  (yr, _, _), (sy, _, _), (ky, _, _) = conv_refs(x, w, _rand((N, H, W, Cout), 424), 3, 1, DEV)
  assert conv_error_ratio(y_plain, yr, sy, tc_elem_c(ky)) <= 1.0
  t = y_plain + bias
  ref = {False: y_plain, True: {False: t, True: torch.maximum(0.2 * t, t)}}
  cnt, first, first_in, mean, m2 = _stats_reference(y_plain, tiles_h, tiles_w)
  for opts in _all_option_sets():
    if expected_rc(opts, True)[0]:
      continue
    runs = []
    for _ in range(2):
      y = torch.full_like(y_plain, float('nan'))
      zp = torch.empty((2,) + tuple(y.shape), device=DEV, dtype=torch.bfloat16)
      mask = torch.empty(y.numel() // 4, device=DEV, dtype=torch.uint8)
      stats = torch.full((N, slots, Cout, 4), float('nan'), device=DEV)
      assert _fwd_planes(L, xp, wp, shape, opts, bias, y, zp, mask, stats) == 0, (opts, L.last_error())
      torch.cuda.synchronize()
      runs.append((y, zp, mask, stats))
    (y, zp, mask, stats), again = runs
    assert torch.equal(_bits(y), _bits(again[0])), opts
    assert torch.equal(y, ref[True]['act' in opts] if 'bias' in opts else ref[False]), opts
    if 'zp' in opts:
      assert torch.equal(_bits(zp), _bits(again[1])), opts
      assert torch.equal(_bits(zp), _bits(_split_ref(y))), opts
    if 'mask' in opts:
      assert torch.equal(mask, again[2]), opts
      pos = (y.reshape(-1, 4) > 0).to(torch.int32)
      assert torch.equal(mask, (pos * torch.tensor([1, 2, 4, 8], device=DEV, dtype=torch.int32)).sum(1).to(torch.uint8))
    if 'stats' in opts:
      assert torch.equal(_bits(stats), _bits(again[3])), opts
      s = stats.double()
      assert torch.equal(s[..., 0], cnt[:, :, None].expand_as(s[..., 0])), opts
      assert torch.equal(s[..., 1][first_in], first[first_in]), opts          # the pivot is the row's first pixel
      n = s[..., 0].clamp(min=1)
      scale = float(y_plain.double().abs().max())
      live = s[..., 0] > 0
      assert float((s[..., 1] + s[..., 2] / n - mean)[live].abs().max()) <= 1e-5 * scale, opts
      assert float((s[..., 3] - s[..., 2] ** 2 / n - m2)[live].abs().max()) <= 1e-4 * scale * scale, opts
  a, b = _dev(1 + _rand((Cout,), 425, 0.3)), _dev(_rand((Cout,), 426, 0.2))
  for flags in (0, ops.FLAG_LRELU, ops.FLAG_PIXNORM, ops.FLAG_LRELU | ops.FLAG_PIXNORM):
    u = a.double() * y_plain.double() + b.double()
    if flags & ops.FLAG_LRELU:
      u = torch.maximum(0.2 * u, u)
    if flags & ops.FLAG_PIXNORM:
      u = u * torch.rsqrt((u * u).mean(-1, keepdim=True) + 1e-6)

    def affine():
      z = torch.empty_like(y_plain)
      zp = torch.empty((2,) + tuple(z.shape), device=DEV, dtype=torch.bfloat16)
      L.call('twg_conv_affine_act_fwd_planes', xp.data_ptr(), wp.data_ptr(), a.data_ptr(), b.data_ptr(), flags,
             z.data_ptr(), zp.data_ptr(), *shape, ops._st())
      torch.cuda.synchronize()
      assert torch.equal(_bits(zp), _bits(_split_ref(z))), flags
      return z
    z = _twice(affine)
    assert float(((z.double() - u).abs() / (u.abs() + 1e-3)).max()) < 2e-6, flags
