"""The column-box forward / dgrad kernel (3x3 SAME, GEMM K = one channel chunk of 16, 32 or 64, 16 x 8 pixel tiles) where it
differs from the per-tap kernel: tiles at every image border with non-zero data in the halo, persistent CTAs that run
several tiles each with a short last round, and every epilogue option, each result held to fp64."""
import pytest
import torch

from tests.parity import conv_error_ratio, tc_elem_c
from tests.test_gpu_conv_conformance import _all_option_sets, _bits, _fwd_planes, _split_ref, expected_rc
from tests.test_gpu_kernels import _dev, _rand, conv_refs

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'

# N, H, W, Cin, Cout.  H % 8 and W % 16 != 0 where possible, so the bottom and right tiles hang over the image; the grid is at
# most 132 (one CTA per SM) or 264 CTAs, so the shapes with 189 .. 432 work items run several tiles per CTA and end in a
# short round; 256 channels on the other side of the GEMM give two 128-channel output blocks.
COLS_SHAPES = [
    (2, 20, 40, 16, 16),     # 3 x 3 tiles per image: every tile touches a border
    (2, 18, 24, 64, 32),
    (3, 36, 72, 32, 64),
    (6, 72, 120, 16, 32),    # 432 work items
    (3, 66, 100, 64, 16),    # 189 work items of the 64-channel forward (one A buffer)
    (12, 64, 64, 32, 128),   # 384 work items, BN = 128
    (2, 40, 48, 64, 256),    # forward: two output-channel blocks
    (3, 48, 64, 256, 64),    # dgrad: two output-channel blocks
]
# the shapes above that have the fused epilogue (Cout <= 64, Cin * Cout <= 2048)
FUSED_SHAPES = [s for s in COLS_SHAPES if s[4] <= 64 and s[3] * s[4] <= 2048]


@pytest.mark.parametrize('shape', COLS_SHAPES)
def test_cols_fwd_and_dgrad_against_fp64(built_lib, shape):
  """Forward (GEMM K = Cin) and data gradient (GEMM K = Cout) per element against fp64; randn data, so every halo pixel
  a border tile reads from inside the image is non-zero and every one outside must read as zero."""
  from twingan_b200 import ops
  N, H, W, Cin, Cout = shape
  x, w, gy = _rand((N, H, W, Cin), 301), _rand((3, 3, Cin, Cout), 302, 0.05), _rand((N, H, W, Cout), 303)
  (yr, gxr, _), (sy, sgx, _), (ky, kgx, _) = conv_refs(x, w, gy, 3, 1, DEV)
  y = ops.conv_fwd_raw(_dev(x), _dev(w), 3, 1)
  gx = ops.conv_dgrad_raw(_dev(gy), _dev(w), (N, H, W, Cin), 3, 1)
  torch.cuda.synchronize()
  assert conv_error_ratio(y, yr, sy, tc_elem_c(ky)) <= 1.0
  assert conv_error_ratio(gx, gxr, sgx, tc_elem_c(kgx)) <= 1.0


def _stats_reference(y, tiles_h, tiles_w):
  """Per statistics slot ((tile row, tile column) * 8 + consumer warp; warp w drains pixel row w of its 16 x 8 tile): the
  in-image pixel count, the first pixel of the row, and the mean and sum of squared deviations in fp64."""
  N, H, W, C = y.shape
  pad = torch.zeros((N, tiles_h * 8, tiles_w * 16, C), device=y.device, dtype=torch.float64)
  inside = torch.zeros((N, tiles_h * 8, tiles_w * 16, 1), device=y.device, dtype=torch.float64)
  pad[:, :H, :W] = y.double()
  inside[:, :H, :W] = 1.0
  slot = lambda t: t.reshape(N, tiles_h, 8, tiles_w, 16, -1).permute(0, 1, 3, 2, 4, 5).reshape(N, -1, 16, t.shape[-1])
  v, m = slot(pad), slot(inside)
  cnt = m.sum(2)                                                    # [N, slots, 1]
  mean = (v * m).sum(2) / cnt.clamp(min=1)
  m2 = (((v - mean[:, :, None]) * m) ** 2).sum(2)
  return cnt[..., 0], v[:, :, 0], m[:, :, 0, 0] > 0, mean, m2


@pytest.mark.parametrize('shape', FUSED_SHAPES)
def test_cols_fwd_every_epilogue_option(built_lib, shape):
  """Every option set twg_conv_fwd_planes accepts, and the evaluation-mode affine with each flag set: y bit for bit the
  plain output's bias / leaky-ReLU, planes and sign mask bit for bit from y, each statistics record at its slot with the
  count, pivot, mean and squared deviations of its pixels, and the affine result against the same operations in fp64 on the plain output."""
  from twingan_b200 import ops
  L = built_lib
  N, H, W, Cin, Cout = shape
  geom = (N, H, W, Cin, Cout, 3, 1)
  slots = ops._epilogue_slots(*geom)
  tiles_h, tiles_w = -(-H // 8), -(-W // 16)
  assert slots == tiles_h * tiles_w * 8
  x, w = _rand((N, H, W, Cin), 311), _rand((3, 3, Cin, Cout), 312, 0.08)
  xp, wp = ops.split_act(_dev(x)), ops.weight_planes(_dev(w), False)
  bias = _dev(_rand((Cout,), 313, 0.5))
  y_plain, _ = ops._conv_fwd(None, _dev(w), 3, 1, xp=xp)
  (yr, _, _), (sy, _, _), (ky, _, _) = conv_refs(x, w, _rand((N, H, W, Cout), 314), 3, 1, DEV)
  torch.cuda.synchronize()
  assert conv_error_ratio(y_plain, yr, sy, tc_elem_c(ky)) <= 1.0
  t = y_plain + bias
  ref = {False: {False: y_plain, True: y_plain}, True: {False: t, True: torch.maximum(0.2 * t, t)}}
  cnt, first, first_in, mean, m2 = _stats_reference(y_plain, tiles_h, tiles_w)
  for opts in _all_option_sets():
    if expected_rc(opts, True)[0]:
      continue
    y = torch.full_like(y_plain, float('nan'))
    zp = torch.empty((2,) + tuple(y.shape), device=DEV, dtype=torch.bfloat16)
    mask = torch.empty(y.numel() // 4, device=DEV, dtype=torch.uint8)
    stats = torch.full((N, slots, Cout, 4), float('nan'), device=DEV)
    assert _fwd_planes(L, xp, wp, geom, opts, bias, y, zp, mask, stats) == 0, (opts, L.last_error())
    torch.cuda.synchronize()
    assert torch.equal(y, ref['bias' in opts]['act' in opts]), opts
    if 'zp' in opts:
      assert torch.equal(_bits(zp), _bits(_split_ref(y))), opts
    if 'mask' in opts:
      pos = (y.reshape(-1, 4) > 0).to(torch.int32)
      assert torch.equal(mask, (pos * torch.tensor([1, 2, 4, 8], device=DEV, dtype=torch.int32)).sum(1).to(torch.uint8))
    if 'stats' in opts:
      s = stats.double()
      assert torch.equal(s[..., 0], cnt[:, :, None].expand_as(s[..., 0])), opts
      got_first = s[..., 1][first_in]
      assert torch.equal(got_first, first[first_in]), opts            # the pivot is the row's first pixel
      n = s[..., 0].clamp(min=1)
      scale = float(y_plain.double().abs().max())
      live = s[..., 0] > 0
      got_mean = s[..., 1] + s[..., 2] / n
      got_m2 = s[..., 3] - s[..., 2] ** 2 / n
      assert float((got_mean - mean)[live].abs().max()) <= 1e-5 * scale, opts
      assert float((got_m2 - m2)[live].abs().max()) <= 1e-4 * scale * scale, opts
  a, b = _dev(1 + _rand((Cout,), 315, 0.3)), _dev(_rand((Cout,), 316, 0.2))
  for flags in (0, ops.FLAG_LRELU, ops.FLAG_PIXNORM, ops.FLAG_LRELU | ops.FLAG_PIXNORM):
    u = a.double() * y_plain.double() + b.double()
    if flags & ops.FLAG_LRELU:
      u = torch.maximum(0.2 * u, u)
    if flags & ops.FLAG_PIXNORM:
      u = u * torch.rsqrt((u * u).mean(-1, keepdim=True) + 1e-6)
    z = torch.empty_like(y_plain)
    zp = torch.empty((2,) + tuple(z.shape), device=DEV, dtype=torch.bfloat16)
    L.call('twg_conv_affine_act_fwd_planes', xp.data_ptr(), wp.data_ptr(), a.data_ptr(), b.data_ptr(), flags,
           z.data_ptr(), zp.data_ptr(), *geom, ops._st())
    torch.cuda.synchronize()
    assert float(((z.double() - u).abs() / (u.abs() + 1e-3)).max()) < 2e-6, flags
    assert torch.equal(_bits(zp), _bits(_split_ref(z))), flags
