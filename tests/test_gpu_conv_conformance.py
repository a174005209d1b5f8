"""Conformance of the convolution layer as the training step and inference use it.

  * coverage: every conv launch of the product (entry point, geometry, fused-epilogue options) is a case of the kernel
    suite, so a new layer shape or a new dispatch choice fails here until a case is added for it;
  * the forward epilogue of twg_conv_fwd_planes: bias + leaky-ReLU, split planes and sign mask bit for bit against the
    plain output, every refused option combination refused before anything is launched;
  * the split kernels bit for bit against torch's round-to-nearest-even bf16;
  * run-to-run reproducibility of all three kernel families, and batch invariance of the tensor-core forward and dgrad."""
import pytest
import torch

from tests import product_launches
from tests.parity import _log_result, conv_error_ratio, tc_elem_c
from tests.product_launches import harvest_product_launches, key_configs
from tests.test_gpu_kernels import CONV_SHAPES, conv_refs, _dev, _rand

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'


# ---------------------------------------------------------------------------------------------------------------------
# forward-epilogue matrix
# ---------------------------------------------------------------------------------------------------------------------
# N, H, W, Cin, Cout, k, pad: one fused shape per fused forward instantiation <Cin chunk, Cout>, one of them ragged
# (24 x 40); shapes without a fused epilogue, incl. two Cout blocks of 128 (the bias index is offset by the block); and
# every geometry at which the product asks for an epilogue option
EPI_SHAPES = [
    (2, 16, 16, 16, 16, 3, 1), (2, 24, 40, 16, 32, 3, 1), (2, 16, 32, 16, 64, 3, 1), (2, 32, 16, 32, 16, 3, 1),
    (2, 16, 16, 32, 32, 3, 1), (2, 16, 16, 32, 64, 3, 1), (2, 16, 16, 64, 16, 3, 1), (2, 32, 32, 64, 32, 3, 1),
    (2, 16, 16, 64, 128, 3, 1), (2, 16, 16, 128, 256, 3, 1), (3, 8, 8, 256, 256, 3, 1),
    (2, 16, 16, 512, 256, 1, 0), (2, 32, 32, 128, 128, 3, 1), (2, 32, 32, 128, 256, 1, 0), (2, 32, 32, 128, 256, 3, 1),
    (2, 32, 32, 512, 128, 1, 0), (2, 64, 64, 64, 64, 3, 1), (2, 64, 64, 64, 128, 1, 0), (2, 64, 64, 64, 128, 3, 1),
    (2, 64, 64, 256, 64, 1, 0), (1, 128, 128, 32, 32, 3, 1), (1, 128, 128, 32, 64, 1, 0), (1, 128, 128, 32, 64, 3, 1),
    (1, 128, 128, 128, 32, 1, 0), (1, 256, 256, 16, 16, 3, 1), (1, 256, 256, 16, 32, 1, 0), (1, 256, 256, 16, 32, 3, 1),
    (1, 256, 256, 64, 16, 1, 0), (1, 256, 256, 64, 16, 3, 1),
]
# the fused instantiations, and the evaluation-mode generator / encoder layers of inference (3x3 SAME)
AFFINE_SHAPES = [s[:5] for s in EPI_SHAPES[:8]] + [(1, 128, 128, 32, 32), (1, 128, 128, 32, 64), (1, 256, 256, 16, 16),
                                                   (1, 256, 256, 16, 32), (1, 256, 256, 64, 16)]
OPTS = ('bias', 'act', 'zp', 'mask', 'stats')


def expected_rc(opts, fused):
  """What twg_conv_fwd_planes returns for a set of options: 0, -1 (invalid) or -2 (unsupported), and the message."""
  if 'act' in opts and 'bias' not in opts:
    return -1, 'activation needs a bias'
  if 'mask' in opts and not ('bias' in opts and 'act' in opts and fused):
    return -2, 'no activation mask'
  if 'stats' in opts and ('bias' in opts or 'zp' in opts or not fused):
    return -2, 'no epilogue statistics'
  return 0, None


def _all_option_sets():
  for m in range(1 << len(OPTS)):
    yield tuple(o for i, o in enumerate(OPTS) if m >> i & 1)


def _split_ref(t):
  hi = t.to(torch.bfloat16)
  return torch.stack([hi, (t - hi.float()).to(torch.bfloat16)])


def _bits(t):
  return t.contiguous().view(torch.int16)


def _fwd_planes(L, xp, wp, shape, opts, bias, y, zp, mask, stats):
  from twingan_b200 import ops
  p = lambda name, t: t.data_ptr() if name in opts else None
  return L.try_call('twg_conv_fwd_planes', xp.data_ptr(), wp.data_ptr(), p('bias', bias), int('act' in opts), y.data_ptr(),
                    p('zp', zp), p('mask', mask), p('stats', stats), *shape, ops._st())


@pytest.mark.parametrize('shape', EPI_SHAPES)
def test_conv_fwd_planes_epilogue_matrix(built_lib, shape):
  from twingan_b200 import ops
  L = built_lib
  N, H, W, Cin, Cout, k, pad = shape
  assert ops.tc_eligible(*shape)
  slots = ops._epilogue_slots(*shape)
  fused = slots > 0
  assert fused == (k == 3 and Cout <= 64 and Cin * Cout <= 2048 and H >= 16 and W >= 16)
  x, w = _rand((N, H, W, Cin), 201), _rand((k, k, Cin, Cout), 202, 0.08)
  xp, wp = ops.split_act(_dev(x)), ops.weight_planes(_dev(w), False)
  bias = _dev(_rand((Cout,), 203, 0.5))
  y_plain, _ = ops._conv_fwd(None, _dev(w), k, pad, xp=xp)
  torch.cuda.synchronize()
  # the plain output itself against fp64, per element
  (yr, _, _), (sy, _, _), (ky, _, _) = conv_refs(x, w, _rand((N, H, W, Cout), 204), k, pad, DEV)
  assert conv_error_ratio(y_plain, yr, sy, tc_elem_c(ky)) <= 1.0
  t = y_plain + bias
  ref = {False: {False: y_plain, True: y_plain}, True: {False: t, True: torch.maximum(0.2 * t, t)}}
  accepted = 0
  for opts in _all_option_sets():
    y = torch.full_like(y_plain, float('nan'))
    zp = torch.empty((2,) + tuple(y.shape), device=DEV, dtype=torch.bfloat16)
    mask = torch.empty(y.numel() // 4, device=DEV, dtype=torch.uint8)
    stats = torch.empty((N, max(slots, 1), Cout, 4), device=DEV)
    want, msg = expected_rc(opts, fused)
    n0 = L.launch_count()
    rc = _fwd_planes(L, xp, wp, shape, opts, bias, y, zp, mask, stats)
    torch.cuda.synchronize()
    if want:
      assert rc == want and msg in L.last_error(), (opts, rc, L.last_error())
      assert L.launch_count() == n0, opts          # refused before anything was launched
      continue
    accepted += 1
    assert rc == 0, (opts, L.last_error())
    z = ref['bias' in opts]['act' in opts]
    assert torch.equal(y, z), opts                  # one fp32 rounding per operation, like torch's
    if 'zp' in opts:
      assert torch.equal(_bits(zp), _bits(_split_ref(y))), opts
    if 'mask' in opts:
      pos = (y.reshape(-1, 4) > 0).to(torch.int32)
      want_mask = (pos * torch.tensor([1, 2, 4, 8], device=DEV, dtype=torch.int32)).sum(1).to(torch.uint8)
      assert torch.equal(mask, want_mask), opts
    if 'stats' in opts:
      assert bool(torch.isfinite(stats).all()), opts
  # fused shapes accept 9 of the 32 option sets (plain, zp, stats, bias, bias+zp, bias+act(+zp)(+mask)), the others 6
  assert accepted == (9 if fused else 6)


@pytest.mark.parametrize('shape', AFFINE_SHAPES)
def test_conv_affine_epilogue_all_flags(built_lib, shape):
  """twg_conv_affine_act_fwd_planes with each of the four flag sets (none, leaky-ReLU, pixel norm, both) against the same
  operations in fp64 on the plain conv output; fp32 output alone, with planes, and planes alone: the same values, the
  planes bit for bit the split of the fp32 output."""
  from twingan_b200 import ops
  L = built_lib
  N, H, W, Cin, Cout = shape
  x, w = _rand((N, H, W, Cin), 211), _rand((3, 3, Cin, Cout), 212, 0.08)
  a, b = _dev(1 + _rand((Cout,), 213, 0.3)), _dev(_rand((Cout,), 214, 0.2))
  xp, wp = ops.split_act(_dev(x)), ops.weight_planes(_dev(w), False)
  y_plain, _ = ops._conv_fwd(None, _dev(w), 3, 1, xp=xp)
  for flags in (0, ops.FLAG_LRELU, ops.FLAG_PIXNORM, ops.FLAG_LRELU | ops.FLAG_PIXNORM):
    u = a.double() * y_plain.double() + b.double()
    if flags & ops.FLAG_LRELU:
      u = torch.maximum(0.2 * u, u)
    if flags & ops.FLAG_PIXNORM:
      u = u * torch.rsqrt((u * u).mean(-1, keepdim=True) + 1e-6)
    z, z_only = torch.empty_like(y_plain), torch.empty_like(y_plain)
    zp = torch.empty((2,) + tuple(z.shape), device=DEV, dtype=torch.bfloat16)
    zp_only = torch.empty_like(zp)
    for out, planes in ((z_only, None), (z, zp), (None, zp_only)):
      L.call('twg_conv_affine_act_fwd_planes', xp.data_ptr(), wp.data_ptr(), a.data_ptr(), b.data_ptr(), flags,
             None if out is None else out.data_ptr(), None if planes is None else planes.data_ptr(), N, H, W, Cin, Cout,
             3, 1, ops._st())
    torch.cuda.synchronize()
    assert float(((z.double() - u).abs() / (u.abs() + 1e-3)).max()) < 2e-6, flags
    assert torch.equal(z_only, z), flags
    assert torch.equal(_bits(zp), _bits(_split_ref(z))), flags
    assert torch.equal(_bits(zp_only), _bits(zp)), flags


# ---------------------------------------------------------------------------------------------------------------------
# split kernels
# ---------------------------------------------------------------------------------------------------------------------
def test_split_act_is_round_to_nearest_even(built_lib):
  from twingan_b200 import ops
  one = 1.0
  special = [0.0, -0.0, 1e-45, -1e-45, 1e-40, -3e-39, 1.2e-38, 3e38, -1e38, 65504.0, -7.5e30,
             one + 2 ** -8, one + 3 * 2 ** -8, -(one + 2 ** -8), 2 ** -20 * (1 + 2 ** -8), 3 + 2 ** -7,   # bf16 ties
             one + 2 ** -8 + 2 ** -16, one + 2 ** -8 + 2 ** -17 + 2 ** -23]                              # lo ties
  g = torch.Generator().manual_seed(5)
  x = torch.cat([torch.tensor(special, dtype=torch.float32), torch.randn(4096 - len(special), generator=g) * 10])
  xd = x.to(DEV).reshape(1, 1, -1, 4)
  planes = ops.split_act(xd)
  torch.cuda.synchronize()
  assert torch.equal(_bits(planes), _bits(_split_ref(xd)))


@pytest.mark.parametrize('k,Cin,Cout', [(3, 16, 32), (3, 64, 128), (1, 128, 16), (1, 4096, 256)])
def test_split_weights_layouts(built_lib, k, Cin, Cout):
  """Forward layout [tap][Cout][Cin] and dgrad layout [flipped tap][Cin][Cout], each as hi plane then lo plane."""
  from twingan_b200 import ops
  w = _dev(_rand((k, k, Cin, Cout), 221, 0.3))
  taps = w.reshape(k * k, Cin, Cout)
  for dgrad, want in ((False, taps.permute(0, 2, 1)), (True, taps.flip(0))):
    planes = torch.empty((2, k * k * Cin * Cout), device=DEV, dtype=torch.bfloat16)
    built_lib.call('twg_split_weights', w.data_ptr(), planes.data_ptr(), k, Cin, Cout, int(dgrad), ops._st())
    torch.cuda.synchronize()
    assert torch.equal(_bits(planes), _bits(_split_ref(want.contiguous().reshape(-1)))), dgrad


def test_weight_plane_table_equals_per_weight_split(built_lib):
  """The model's one-launch twg_split_weights_table gives the planes twg_split_weights gives weight by weight."""
  from twingan_b200 import ops, twingan
  model = twingan.GanModel(twingan.Flags(train_image_size=32, pggan_max_num_channels=256), device=DEV)
  table = model.variables.weight_table
  assert table.rows > 0
  table.dirty = True
  n = 0
  for name, t in model.variables.vars.items():
    for dgrad in (False, True):
      if (t.data_ptr(), dgrad) not in table.index:
        continue
      k, _, Cin, Cout = t.shape
      want = torch.empty((2, k * k * Cin * Cout), device=DEV, dtype=torch.bfloat16)
      built_lib.call('twg_split_weights', t.data_ptr(), want.data_ptr(), k, Cin, Cout, int(dgrad), ops._st())
      got = table.get(t.data_ptr(), dgrad)
      torch.cuda.synchronize()
      assert torch.equal(_bits(got), _bits(want)), (name, dgrad)
      n += 1
  assert n == table.rows


# ---------------------------------------------------------------------------------------------------------------------
# reproducibility and batch invariance
# ---------------------------------------------------------------------------------------------------------------------
REPRO_SHAPES = [(2, 16, 16, 3, 16, 1, 0), (2, 16, 16, 16, 3, 1, 0),          # pointwise
                (3, 8, 8, 257, 256, 3, 1), (4, 4, 4, 256, 256, 4, 0),        # SIMT
                (2, 24, 40, 16, 32, 3, 1), (9, 3, 5, 64, 64, 3, 1), (130, 1, 1, 4096, 256, 1, 0),
                (4, 40, 36, 128, 256, 3, 1)]


@pytest.mark.parametrize('prec', [0, 1])
@pytest.mark.parametrize('shape', REPRO_SHAPES)
def test_conv_results_are_bit_identical_from_run_to_run(built_lib, shape, prec):
  from twingan_b200 import ops
  ops.set_precision(prec)
  try:
    N, H, W, Cin, Cout, k, pad = shape
    Ho, Wo = H + 2 * pad - k + 1, W + 2 * pad - k + 1
    x, w, gy = _dev(_rand((N, H, W, Cin), 231)), _dev(_rand((k, k, Cin, Cout), 232, 0.05)), _dev(_rand((N, Ho, Wo, Cout), 233))
    run = lambda: (ops.conv_fwd_raw(x, w, k, pad), ops.conv_dgrad_raw(gy, w, (N, H, W, Cin), k, pad),
                   ops.conv_wgrad_raw(x, gy, k, pad))
    first, second = run(), run()
    torch.cuda.synchronize()
    for d, a, b in zip(('fwd', 'dgrad', 'wgrad'), first, second):
      assert torch.equal(a, b), d
  finally:
    ops.set_precision(1)


@pytest.mark.parametrize('shape', [(9, 3, 5, 64, 64, 3, 1), (130, 1, 1, 4096, 256, 1, 0), (6, 4, 4, 384, 256, 3, 1),
                                   (3, 2, 2, 128, 128, 3, 1), (3, 24, 40, 16, 32, 3, 1), (2, 16, 16, 128, 256, 1, 0)])
def test_tensor_core_fwd_and_dgrad_are_per_sample(built_lib, shape):
  """A sample's forward output and input gradient do not depend on the batch it is computed in, also where one tile spans
  several images.  (The weight gradient is not batch-invariant: its pixel split depends on N.)"""
  from twingan_b200 import ops
  N, H, W, Cin, Cout, k, pad = shape
  assert ops.tc_eligible(*shape)
  x, w, gy = _dev(_rand((N, H, W, Cin), 241)), _dev(_rand((k, k, Cin, Cout), 242, 0.05)), _dev(_rand((N, H, W, Cout), 243))
  y = ops.conv_fwd_raw(x, w, k, pad)
  gx = ops.conv_dgrad_raw(gy, w, (N, H, W, Cin), k, pad)
  ys = torch.cat([ops.conv_fwd_raw(x[i:i + 1], w, k, pad) for i in range(N)])
  gxs = torch.cat([ops.conv_dgrad_raw(gy[i:i + 1], w, (1, H, W, Cin), k, pad) for i in range(N)])
  torch.cuda.synchronize()
  assert torch.equal(y, ys)
  assert torch.equal(gx, gxs)


# ---------------------------------------------------------------------------------------------------------------------
# the batch-dependent host rules of the conv launchers (twg_conv_tc.cu, twg_conv_simt.cu, twg_conv_pw.cu), restated
# ---------------------------------------------------------------------------------------------------------------------
NUM_SMS = 132            # kNumSMs of twg_common.cuh


def _cdiv(a, b):
  return -(-a // b)


def _pow2_le(v):
  p = 1
  while p * 2 <= v:
    p *= 2
  return p


def pick_tile(N, H, W):
  """(TW, TH, TN, tiles_w, tiles_h, tiles_n) of pick_tile: a 128-pixel tile of TN images of TH x TW pixels."""
  TW = _pow2_le(min(W, 16))
  TH = _pow2_le(min(H, 128 // TW))
  TN = 128 // (TW * TH)
  return TW, TH, TN, _cdiv(W, TW), _cdiv(H, TH), _cdiv(N, TN)


def tc_ragged(N, H, W):
  """The last batch tile of a tensor-core conv holds fewer than TN images."""
  TN = pick_tile(N, H, W)[2]
  return TN > 1 and N % TN != 0


def _chunk_for(c):
  return 64 if c % 64 == 0 else (32 if c % 32 == 0 else (16 if c % 16 == 0 else 0))


def tc_wgrad_grid(N, H, W, Cin, Cout, k, pad):
  """launch_wgrad's pixel split: {tiles_per_cta, ctas (xb), last_cta_tiles, total_tiles, cols}.  The CTAs of one
  channel block take consecutive runs of tiles_per_cta tiles; the last run is cut short by total_tiles when
  last_cta_tiles < tiles_per_cta."""
  TW, TH, TN, tw, th, tn = pick_tile(N, H, W)
  CN = _chunk_for(Cin)
  BNW = 64 if (Cout >= 64 and CN < 64) else (32 if Cout >= 32 else Cout)
  total = tw * th * tn
  want = max(1, min(NUM_SMS // ((Cout // BNW) * (Cin // CN)), total))
  per = _cdiv(total, want)
  xb = _cdiv(total, per)
  return {'tiles_per_cta': per, 'ctas': xb, 'last_cta_tiles': total - (xb - 1) * per, 'total_tiles': total,
          'cols': k == 3 and pad == 1 and TW == 16 and TH == 8 and TN == 1 and H >= 10}


def simt_wgrad_splits(N, H, W, Cin, Cout, k, pad):
  """(splits, pixels per split) of conv_wgrad_simt."""
  M = N * (H + 2 * pad - k + 1) * (W + 2 * pad - k + 1)
  tiles = k * k * _cdiv(Cin, 16 if Cin <= 16 else 64) * _cdiv(Cout, 16 if Cout <= 16 else 64)
  splits = max(1, min(_cdiv(4 * NUM_SMS, tiles), _cdiv(M, 64)))
  mps = _cdiv(_cdiv(M, splits), 16) * 16
  return _cdiv(M, mps), mps


def pw_wgrad_blocks(N, H, W, Cin, Cout):
  """(blocks, pixels per block) of pw_wgrad: the wide side L = max(Cin, Cout) gives G = min(L / 4, 32) threads a pixel."""
  P = N * H * W
  G = min(max(Cin, Cout) // 4, 32)
  blocks = min(_cdiv(P, (256 // G) * 16), 4 * NUM_SMS)
  chunk = _cdiv(P, blocks)
  return _cdiv(P, chunk), chunk


# ---------------------------------------------------------------------------------------------------------------------
# coverage audit
# ---------------------------------------------------------------------------------------------------------------------
# argument positions of the geometry (N, H, W, Cin, Cout, k, pad) in each conv entry point
_GEOM_AT = {'twg_conv_fwd': 3, 'twg_conv_dgrad': 3, 'twg_conv_wgrad': 3, 'twg_conv_fwd_planes': 8,
            'twg_conv_affine_act_fwd_planes': 7, 'twg_conv_dgrad_planes': 3, 'twg_conv_wgrad_planes': 3}
WGRAD_ENTRIES = ('twg_conv_wgrad', 'twg_conv_wgrad_planes')
_TC_ENTRIES = ('twg_conv_fwd_planes', 'twg_conv_affine_act_fwd_planes', 'twg_conv_dgrad_planes')


def conv_key(name, args):
  """(entry, [N,] H, W, Cin, Cout, k, pad, options) of one conv launch.  The weight gradients carry N: it sets their
  pixel split (the summation order, and whether the last CTA is short) and whether the last batch tile is ragged.  The
  tensor-core forward, dgrad and affine forward carry 'ragged' when their last batch tile is; their per-sample arithmetic
  does not depend on N otherwise (test_tensor_core_fwd_and_dgrad_are_per_sample).  The exact-fp32 forward and dgrad the
  product launches are the pointwise kernels, one output pixel at a time."""
  i = _GEOM_AT[name]
  geom = tuple(int(v) for v in args[i + 1:i + 7])
  N = int(args[i])
  opts = []
  if name in WGRAD_ENTRIES and args[i + 7]:
    opts.append('accumulate')
  if name == 'twg_conv_fwd_planes':
    opts += [o for o, v in (('bias', args[2]), ('act', args[3]), ('zp', args[5]), ('mask', args[6]), ('stats', args[7])) if v]
  if name == 'twg_conv_affine_act_fwd_planes':
    opts += ['flags%d' % int(args[4])] + [o for o, v in (('z', args[5]), ('zp', args[6])) if v]
  if name in _TC_ENTRIES and tc_ragged(N, geom[0], geom[1]):
    opts.append('ragged')
  return (name,) + ((N,) if name in WGRAD_ENTRIES else ()) + geom + ('+'.join(opts),)


def _with_ragged(opts, N, H, W):
  return '+'.join(filter(None, (opts, 'ragged' if tc_ragged(N, H, W) else '')))


def kernel_suite_keys():
  """The keys the kernel suite runs: test_conv_fwd_dgrad_wgrad at both precisions (with the accumulate check), the
  epilogue matrix and the affine-epilogue test."""
  from twingan_b200 import ops
  keys = set()
  for N, H, W, Cin, Cout, k, pad in CONV_SHAPES:
    g = (H, W, Cin, Cout, k, pad)
    keys |= {('twg_conv_fwd',) + g + ('',), ('twg_conv_dgrad',) + g + ('',), ('twg_conv_wgrad', N) + g + ('',),
             ('twg_conv_wgrad', N) + g + ('accumulate',)}
    if ops.conv_path(N, H, W, Cin, Cout, k, pad) == ops.CONV_TC:
      keys |= {('twg_conv_fwd_planes',) + g + (_with_ragged('', N, H, W),),
               ('twg_conv_dgrad_planes',) + g + (_with_ragged('', N, H, W),),
               ('twg_conv_wgrad_planes', N) + g + ('',), ('twg_conv_wgrad_planes', N) + g + ('accumulate',)}
  for N, H, W, Cin, Cout, k, pad in EPI_SHAPES:
    fused = ops._epilogue_slots(N, H, W, Cin, Cout, k, pad) > 0
    for opts in _all_option_sets():
      if expected_rc(opts, fused)[0] == 0:
        keys.add(('twg_conv_fwd_planes', H, W, Cin, Cout, k, pad, _with_ragged('+'.join(opts), N, H, W)))
  for N, H, W, Cin, Cout in AFFINE_SHAPES:
    for flags in range(4):
      for outs in ('z', 'z+zp', 'zp'):
        keys.add(('twg_conv_affine_act_fwd_planes', H, W, Cin, Cout, 3, 1,
                  _with_ragged('flags%d+%s' % (flags, outs), N, H, W)))
  return keys


def suite_keys():
  """The keys of the kernel suite and of the product-batch cases of test_gpu_conv_batch.py."""
  from tests.test_gpu_conv_batch import BATCH_CONV_CASES
  return kernel_suite_keys() | {key for key, _ in BATCH_CONV_CASES}


def harvest_product_convs():
  """The keys of every conv launch in the shared harvest of the product (tests/product_launches.py)."""
  return conv_keys(harvest_product_launches())


def conv_keys(launches):
  return {conv_key(name, args) for name, args in launches if name in _GEOM_AT}


# The conv launches of the product, harvested by harvest_product_convs.  A change that adds, removes or re-dispatches a conv
# must update this set and, for each new key, add a case to the kernel suite.
PRODUCT_CONVS = {
    'twg_conv_affine_act_fwd_planes': [
        (128, 128, 32, 32, 3, 1, 'flags3+z'), (128, 128, 32, 32, 3, 1, 'flags3+zp'), (128, 128, 32, 64, 3, 1, 'flags3+z'),
        (256, 256, 16, 16, 3, 1, 'flags3+z'), (256, 256, 16, 16, 3, 1, 'flags3+zp'), (256, 256, 16, 32, 3, 1, 'flags3+z'),
        (256, 256, 64, 16, 3, 1, 'flags3+zp')],
    'twg_conv_dgrad': [
        (1, 1, 256, 1, 1, 0, ''), (128, 128, 3, 32, 1, 0, ''), (128, 128, 32, 3, 1, 0, ''), (16, 16, 256, 3, 1, 0, ''), (16,
        16, 3, 256, 1, 0, ''), (256, 256, 16, 3, 1, 0, ''), (256, 256, 3, 16, 1, 0, ''), (32, 32, 128, 3, 1, 0, ''), (32,
        32, 3, 128, 1, 0, ''), (4, 4, 256, 3, 1, 0, ''), (4, 4, 3, 256, 1, 0, ''), (64, 64, 3, 64, 1, 0, ''), (64, 64, 64,
        3, 1, 0, ''), (8, 8, 256, 3, 1, 0, ''), (8, 8, 3, 256, 1, 0, '')],
    'twg_conv_dgrad_planes': [
        (1, 1, 4096, 256, 1, 0, 'ragged'), (128, 128, 128, 32, 1, 0, ''), (128, 128, 128, 32, 3, 1, ''), (128, 128, 32, 32,
        3, 1, ''), (128, 128, 32, 64, 1, 0, ''), (128, 128, 32, 64, 3, 1, ''), (16, 16, 256, 256, 3, 1, ''), (16, 16, 512,
        256, 1, 0, ''), (16, 16, 512, 256, 3, 1, ''), (256, 256, 16, 16, 3, 1, ''), (256, 256, 16, 32, 1, 0, ''), (256, 256,
        16, 32, 3, 1, ''), (256, 256, 64, 16, 1, 0, ''), (256, 256, 64, 16, 3, 1, ''), (32, 32, 128, 128, 3, 1, ''), (32,
        32, 128, 256, 1, 0, ''), (32, 32, 128, 256, 3, 1, ''), (32, 32, 512, 128, 1, 0, ''), (32, 32, 512, 128, 3, 1, ''),
        (4, 4, 256, 256, 3, 1, ''), (4, 4, 256, 256, 3, 1, 'ragged'), (4, 4, 384, 256, 3, 1, ''), (4, 4, 384, 256, 3, 1,
        'ragged'), (64, 64, 256, 64, 1, 0, ''), (64, 64, 256, 64, 3, 1, ''), (64, 64, 64, 128, 1, 0, ''), (64, 64, 64, 128,
        3, 1, ''), (64, 64, 64, 64, 3, 1, ''), (8, 8, 256, 256, 3, 1, ''), (8, 8, 256, 256, 3, 1, 'ragged'), (8, 8, 512,
        256, 1, 0, ''), (8, 8, 512, 256, 3, 1, '')],
    'twg_conv_fwd': [
        (1, 1, 256, 1, 1, 0, ''), (128, 128, 3, 32, 1, 0, ''), (128, 128, 32, 3, 1, 0, ''), (16, 16, 256, 3, 1, 0, ''), (16,
        16, 3, 256, 1, 0, ''), (256, 256, 16, 3, 1, 0, ''), (256, 256, 3, 16, 1, 0, ''), (32, 32, 128, 3, 1, 0, ''), (32,
        32, 3, 128, 1, 0, ''), (4, 4, 256, 3, 1, 0, ''), (4, 4, 3, 256, 1, 0, ''), (64, 64, 3, 64, 1, 0, ''), (64, 64, 64,
        3, 1, 0, ''), (8, 8, 256, 3, 1, 0, ''), (8, 8, 3, 256, 1, 0, '')],
    'twg_conv_fwd_planes': [
        (1, 1, 4096, 256, 1, 0, 'ragged'), (128, 128, 128, 32, 1, 0, ''), (128, 128, 128, 32, 1, 0, 'bias'), (128, 128, 128,
        32, 3, 1, ''), (128, 128, 32, 32, 3, 1, ''), (128, 128, 32, 32, 3, 1, 'bias+act+zp+mask'), (128, 128, 32, 32, 3, 1,
        'stats'), (128, 128, 32, 64, 1, 0, ''), (128, 128, 32, 64, 1, 0, 'bias'), (128, 128, 32, 64, 3, 1, ''), (128, 128,
        32, 64, 3, 1, 'bias+act+mask'), (128, 128, 32, 64, 3, 1, 'stats'), (16, 16, 256, 256, 3, 1, ''), (16, 16, 512, 256,
        1, 0, ''), (16, 16, 512, 256, 1, 0, 'bias'), (16, 16, 512, 256, 3, 1, ''), (256, 256, 16, 16, 3, 1, ''), (256, 256,
        16, 16, 3, 1, 'bias+act+zp+mask'), (256, 256, 16, 16, 3, 1, 'stats'), (256, 256, 16, 32, 1, 0, ''), (256, 256, 16,
        32, 1, 0, 'bias'), (256, 256, 16, 32, 3, 1, ''), (256, 256, 16, 32, 3, 1, 'bias+act+mask'), (256, 256, 16, 32, 3, 1,
        'stats'), (256, 256, 64, 16, 1, 0, ''), (256, 256, 64, 16, 1, 0, 'bias'), (256, 256, 64, 16, 3, 1, ''), (256, 256,
        64, 16, 3, 1, 'stats'), (32, 32, 128, 128, 3, 1, ''), (32, 32, 128, 128, 3, 1, 'bias+act+zp'), (32, 32, 128, 256, 1,
        0, ''), (32, 32, 128, 256, 1, 0, 'bias'), (32, 32, 128, 256, 3, 1, ''), (32, 32, 128, 256, 3, 1, 'bias+act'), (32,
        32, 512, 128, 1, 0, ''), (32, 32, 512, 128, 1, 0, 'bias'), (32, 32, 512, 128, 3, 1, ''), (4, 4, 256, 256, 3, 1, ''),
        (4, 4, 256, 256, 3, 1, 'ragged'), (4, 4, 384, 256, 3, 1, ''), (4, 4, 384, 256, 3, 1, 'ragged'), (64, 64, 256, 64, 1,
        0, ''), (64, 64, 256, 64, 1, 0, 'bias'), (64, 64, 256, 64, 3, 1, ''), (64, 64, 64, 128, 1, 0, ''), (64, 64, 64, 128,
        1, 0, 'bias'), (64, 64, 64, 128, 3, 1, ''), (64, 64, 64, 128, 3, 1, 'bias+act'), (64, 64, 64, 64, 3, 1, ''), (64,
        64, 64, 64, 3, 1, 'bias+act+zp'), (8, 8, 256, 256, 3, 1, ''), (8, 8, 256, 256, 3, 1, 'ragged'), (8, 8, 512, 256, 1,
        0, ''), (8, 8, 512, 256, 1, 0, 'ragged'), (8, 8, 512, 256, 3, 1, ''), (8, 8, 512, 256, 3, 1, 'ragged')],
    'twg_conv_wgrad': [
        (12, 1, 1, 256, 1, 1, 0, 'accumulate'), (12, 128, 128, 3, 32, 1, 0, 'accumulate'), (12, 128, 128, 32, 3, 1, 0,
        'accumulate'), (12, 256, 256, 16, 3, 1, 0, 'accumulate'), (12, 256, 256, 3, 16, 1, 0, 'accumulate'), (12, 32, 32, 3,
        128, 1, 0, 'accumulate'), (12, 64, 64, 3, 64, 1, 0, 'accumulate'), (16, 1, 1, 256, 1, 1, 0, 'accumulate'), (16, 128,
        128, 3, 32, 1, 0, 'accumulate'), (16, 128, 128, 32, 3, 1, 0, 'accumulate'), (16, 16, 16, 3, 256, 1, 0,
        'accumulate'), (16, 256, 256, 16, 3, 1, 0, 'accumulate'), (16, 256, 256, 3, 16, 1, 0, 'accumulate'), (16, 32, 32,
        128, 3, 1, 0, 'accumulate'), (16, 32, 32, 3, 128, 1, 0, 'accumulate'), (16, 4, 4, 3, 256, 1, 0, 'accumulate'), (16,
        64, 64, 3, 64, 1, 0, 'accumulate'), (16, 64, 64, 64, 3, 1, 0, 'accumulate'), (16, 8, 8, 3, 256, 1, 0, 'accumulate'),
        (24, 1, 1, 256, 1, 1, 0, 'accumulate'), (24, 128, 128, 3, 32, 1, 0, 'accumulate'), (24, 16, 16, 3, 256, 1, 0,
        'accumulate'), (24, 256, 256, 3, 16, 1, 0, 'accumulate'), (24, 32, 32, 3, 128, 1, 0, 'accumulate'), (24, 4, 4, 3,
        256, 1, 0, 'accumulate'), (24, 64, 64, 3, 64, 1, 0, 'accumulate'), (24, 8, 8, 3, 256, 1, 0, 'accumulate'), (3, 1, 1,
        256, 1, 1, 0, 'accumulate'), (3, 128, 128, 3, 32, 1, 0, 'accumulate'), (3, 256, 256, 3, 16, 1, 0, 'accumulate'),
        (32, 128, 128, 3, 32, 1, 0, 'accumulate'), (32, 16, 16, 256, 3, 1, 0, 'accumulate'), (32, 16, 16, 3, 256, 1, 0,
        'accumulate'), (32, 256, 256, 3, 16, 1, 0, 'accumulate'), (32, 32, 32, 128, 3, 1, 0, 'accumulate'), (32, 32, 32, 3,
        128, 1, 0, 'accumulate'), (32, 4, 4, 256, 3, 1, 0, 'accumulate'), (32, 4, 4, 3, 256, 1, 0, 'accumulate'), (32, 64,
        64, 3, 64, 1, 0, 'accumulate'), (32, 64, 64, 64, 3, 1, 0, 'accumulate'), (32, 8, 8, 256, 3, 1, 0, 'accumulate'),
        (32, 8, 8, 3, 256, 1, 0, 'accumulate'), (36, 1, 1, 256, 1, 1, 0, 'accumulate'), (36, 128, 128, 3, 32, 1, 0,
        'accumulate'), (36, 256, 256, 3, 16, 1, 0, 'accumulate'), (36, 32, 32, 3, 128, 1, 0, 'accumulate'), (36, 64, 64, 3,
        64, 1, 0, 'accumulate'), (4, 1, 1, 256, 1, 1, 0, 'accumulate'), (4, 128, 128, 3, 32, 1, 0, 'accumulate'), (4, 64,
        64, 3, 64, 1, 0, 'accumulate'), (48, 1, 1, 256, 1, 1, 0, 'accumulate'), (48, 128, 128, 3, 32, 1, 0, 'accumulate'),
        (48, 128, 128, 32, 3, 1, 0, 'accumulate'), (48, 16, 16, 3, 256, 1, 0, 'accumulate'), (48, 256, 256, 16, 3, 1, 0,
        'accumulate'), (48, 256, 256, 3, 16, 1, 0, 'accumulate'), (48, 32, 32, 128, 3, 1, 0, 'accumulate'), (48, 32, 32, 3,
        128, 1, 0, 'accumulate'), (48, 4, 4, 3, 256, 1, 0, 'accumulate'), (48, 64, 64, 3, 64, 1, 0, 'accumulate'), (48, 64,
        64, 64, 3, 1, 0, 'accumulate'), (48, 8, 8, 3, 256, 1, 0, 'accumulate'), (6, 128, 128, 3, 32, 1, 0, 'accumulate'),
        (6, 256, 256, 3, 16, 1, 0, 'accumulate'), (64, 128, 128, 32, 3, 1, 0, 'accumulate'), (64, 16, 16, 256, 3, 1, 0,
        'accumulate'), (64, 256, 256, 16, 3, 1, 0, 'accumulate'), (64, 32, 32, 128, 3, 1, 0, 'accumulate'), (64, 4, 4, 256,
        3, 1, 0, 'accumulate'), (64, 64, 64, 64, 3, 1, 0, 'accumulate'), (64, 8, 8, 256, 3, 1, 0, 'accumulate'), (8, 1, 1,
        256, 1, 1, 0, 'accumulate'), (8, 128, 128, 3, 32, 1, 0, 'accumulate'), (8, 16, 16, 3, 256, 1, 0, 'accumulate'), (8,
        32, 32, 3, 128, 1, 0, 'accumulate'), (8, 4, 4, 3, 256, 1, 0, 'accumulate'), (8, 64, 64, 3, 64, 1, 0, 'accumulate'),
        (8, 8, 8, 3, 256, 1, 0, 'accumulate'), (9, 1, 1, 256, 1, 1, 0, 'accumulate'), (9, 128, 128, 3, 32, 1, 0,
        'accumulate'), (9, 256, 256, 3, 16, 1, 0, 'accumulate')],
    'twg_conv_wgrad_planes': [
        (12, 1, 1, 4096, 256, 1, 0, 'accumulate'), (12, 128, 128, 128, 32, 1, 0, 'accumulate'), (12, 128, 128, 128, 32, 3,
        1, 'accumulate'), (12, 128, 128, 32, 32, 3, 1, 'accumulate'), (12, 128, 128, 32, 64, 1, 0, 'accumulate'), (12, 128,
        128, 32, 64, 3, 1, 'accumulate'), (12, 16, 16, 256, 256, 3, 1, 'accumulate'), (12, 16, 16, 512, 256, 1, 0,
        'accumulate'), (12, 16, 16, 512, 256, 3, 1, 'accumulate'), (12, 256, 256, 16, 16, 3, 1, 'accumulate'), (12, 256,
        256, 16, 32, 1, 0, 'accumulate'), (12, 256, 256, 16, 32, 3, 1, 'accumulate'), (12, 256, 256, 64, 16, 1, 0,
        'accumulate'), (12, 256, 256, 64, 16, 3, 1, 'accumulate'), (12, 32, 32, 128, 128, 3, 1, 'accumulate'), (12, 32, 32,
        128, 256, 1, 0, 'accumulate'), (12, 32, 32, 128, 256, 3, 1, 'accumulate'), (12, 32, 32, 512, 128, 1, 0,
        'accumulate'), (12, 32, 32, 512, 128, 3, 1, 'accumulate'), (12, 4, 4, 256, 256, 3, 1, 'accumulate'), (12, 4, 4, 384,
        256, 3, 1, 'accumulate'), (12, 64, 64, 256, 64, 1, 0, 'accumulate'), (12, 64, 64, 256, 64, 3, 1, 'accumulate'), (12,
        64, 64, 64, 128, 1, 0, 'accumulate'), (12, 64, 64, 64, 128, 3, 1, 'accumulate'), (12, 64, 64, 64, 64, 3, 1,
        'accumulate'), (12, 8, 8, 256, 256, 3, 1, 'accumulate'), (12, 8, 8, 512, 256, 1, 0, 'accumulate'), (12, 8, 8, 512,
        256, 3, 1, 'accumulate'), (16, 1, 1, 4096, 256, 1, 0, 'accumulate'), (16, 128, 128, 128, 32, 1, 0, 'accumulate'),
        (16, 128, 128, 128, 32, 3, 1, 'accumulate'), (16, 128, 128, 32, 32, 3, 1, 'accumulate'), (16, 128, 128, 32, 64, 1,
        0, 'accumulate'), (16, 128, 128, 32, 64, 3, 1, 'accumulate'), (16, 16, 16, 256, 256, 3, 1, 'accumulate'), (16, 16,
        16, 512, 256, 1, 0, 'accumulate'), (16, 16, 16, 512, 256, 3, 1, 'accumulate'), (16, 256, 256, 16, 16, 3, 1,
        'accumulate'), (16, 256, 256, 16, 32, 1, 0, 'accumulate'), (16, 256, 256, 16, 32, 3, 1, 'accumulate'), (16, 256,
        256, 64, 16, 3, 1, 'accumulate'), (16, 32, 32, 128, 128, 3, 1, 'accumulate'), (16, 32, 32, 128, 256, 1, 0,
        'accumulate'), (16, 32, 32, 128, 256, 3, 1, 'accumulate'), (16, 32, 32, 512, 128, 1, 0, 'accumulate'), (16, 32, 32,
        512, 128, 3, 1, 'accumulate'), (16, 4, 4, 256, 256, 3, 1, 'accumulate'), (16, 4, 4, 384, 256, 3, 1, 'accumulate'),
        (16, 64, 64, 256, 64, 1, 0, 'accumulate'), (16, 64, 64, 256, 64, 3, 1, 'accumulate'), (16, 64, 64, 64, 128, 1, 0,
        'accumulate'), (16, 64, 64, 64, 128, 3, 1, 'accumulate'), (16, 64, 64, 64, 64, 3, 1, 'accumulate'), (16, 8, 8, 256,
        256, 3, 1, 'accumulate'), (16, 8, 8, 512, 256, 1, 0, 'accumulate'), (16, 8, 8, 512, 256, 3, 1, 'accumulate'), (24,
        1, 1, 4096, 256, 1, 0, 'accumulate'), (24, 128, 128, 32, 32, 3, 1, 'accumulate'), (24, 128, 128, 32, 64, 1, 0,
        'accumulate'), (24, 128, 128, 32, 64, 3, 1, 'accumulate'), (24, 16, 16, 256, 256, 3, 1, 'accumulate'), (24, 256,
        256, 16, 16, 3, 1, 'accumulate'), (24, 256, 256, 16, 32, 1, 0, 'accumulate'), (24, 256, 256, 16, 32, 3, 1,
        'accumulate'), (24, 32, 32, 128, 128, 3, 1, 'accumulate'), (24, 32, 32, 128, 256, 1, 0, 'accumulate'), (24, 32, 32,
        128, 256, 3, 1, 'accumulate'), (24, 4, 4, 384, 256, 3, 1, 'accumulate'), (24, 64, 64, 64, 128, 1, 0, 'accumulate'),
        (24, 64, 64, 64, 128, 3, 1, 'accumulate'), (24, 64, 64, 64, 64, 3, 1, 'accumulate'), (24, 8, 8, 256, 256, 3, 1,
        'accumulate'), (3, 1, 1, 4096, 256, 1, 0, 'accumulate'), (3, 128, 128, 32, 32, 3, 1, 'accumulate'), (3, 128, 128,
        32, 64, 1, 0, 'accumulate'), (3, 128, 128, 32, 64, 3, 1, 'accumulate'), (3, 16, 16, 256, 256, 3, 1, 'accumulate'),
        (3, 256, 256, 16, 16, 3, 1, 'accumulate'), (3, 256, 256, 16, 32, 1, 0, 'accumulate'), (3, 256, 256, 16, 32, 3, 1,
        'accumulate'), (3, 32, 32, 128, 128, 3, 1, 'accumulate'), (3, 32, 32, 128, 256, 1, 0, 'accumulate'), (3, 32, 32,
        128, 256, 3, 1, 'accumulate'), (3, 4, 4, 384, 256, 3, 1, 'accumulate'), (3, 64, 64, 64, 128, 1, 0, 'accumulate'),
        (3, 64, 64, 64, 128, 3, 1, 'accumulate'), (3, 64, 64, 64, 64, 3, 1, 'accumulate'), (3, 8, 8, 256, 256, 3, 1,
        'accumulate'), (32, 128, 128, 32, 32, 3, 1, 'accumulate'), (32, 128, 128, 32, 64, 1, 0, 'accumulate'), (32, 128,
        128, 32, 64, 3, 1, 'accumulate'), (32, 16, 16, 256, 256, 3, 1, 'accumulate'), (32, 16, 16, 512, 256, 1, 0,
        'accumulate'), (32, 16, 16, 512, 256, 3, 1, 'accumulate'), (32, 256, 256, 16, 16, 3, 1, 'accumulate'), (32, 256,
        256, 16, 32, 1, 0, 'accumulate'), (32, 256, 256, 16, 32, 3, 1, 'accumulate'), (32, 32, 32, 128, 128, 3, 1,
        'accumulate'), (32, 32, 32, 128, 256, 1, 0, 'accumulate'), (32, 32, 32, 128, 256, 3, 1, 'accumulate'), (32, 32, 32,
        512, 128, 1, 0, 'accumulate'), (32, 32, 32, 512, 128, 3, 1, 'accumulate'), (32, 4, 4, 256, 256, 3, 1, 'accumulate'),
        (32, 64, 64, 256, 64, 1, 0, 'accumulate'), (32, 64, 64, 256, 64, 3, 1, 'accumulate'), (32, 64, 64, 64, 128, 1, 0,
        'accumulate'), (32, 64, 64, 64, 128, 3, 1, 'accumulate'), (32, 64, 64, 64, 64, 3, 1, 'accumulate'), (32, 8, 8, 256,
        256, 3, 1, 'accumulate'), (32, 8, 8, 512, 256, 1, 0, 'accumulate'), (32, 8, 8, 512, 256, 3, 1, 'accumulate'), (36,
        1, 1, 4096, 256, 1, 0, 'accumulate'), (36, 128, 128, 32, 32, 3, 1, 'accumulate'), (36, 128, 128, 32, 64, 1, 0,
        'accumulate'), (36, 128, 128, 32, 64, 3, 1, 'accumulate'), (36, 16, 16, 256, 256, 3, 1, 'accumulate'), (36, 256,
        256, 16, 16, 3, 1, 'accumulate'), (36, 256, 256, 16, 32, 1, 0, 'accumulate'), (36, 256, 256, 16, 32, 3, 1,
        'accumulate'), (36, 32, 32, 128, 128, 3, 1, 'accumulate'), (36, 32, 32, 128, 256, 1, 0, 'accumulate'), (36, 32, 32,
        128, 256, 3, 1, 'accumulate'), (36, 4, 4, 384, 256, 3, 1, 'accumulate'), (36, 64, 64, 64, 128, 1, 0, 'accumulate'),
        (36, 64, 64, 64, 128, 3, 1, 'accumulate'), (36, 64, 64, 64, 64, 3, 1, 'accumulate'), (36, 8, 8, 256, 256, 3, 1,
        'accumulate'), (4, 1, 1, 4096, 256, 1, 0, 'accumulate'), (4, 128, 128, 32, 32, 3, 1, 'accumulate'), (4, 128, 128,
        32, 64, 1, 0, 'accumulate'), (4, 128, 128, 32, 64, 3, 1, 'accumulate'), (4, 16, 16, 256, 256, 3, 1, 'accumulate'),
        (4, 32, 32, 128, 128, 3, 1, 'accumulate'), (4, 32, 32, 128, 256, 1, 0, 'accumulate'), (4, 32, 32, 128, 256, 3, 1,
        'accumulate'), (4, 4, 4, 384, 256, 3, 1, 'accumulate'), (4, 64, 64, 64, 128, 1, 0, 'accumulate'), (4, 64, 64, 64,
        128, 3, 1, 'accumulate'), (4, 64, 64, 64, 64, 3, 1, 'accumulate'), (4, 8, 8, 256, 256, 3, 1, 'accumulate'), (48, 1,
        1, 4096, 256, 1, 0, 'accumulate'), (48, 128, 128, 128, 32, 1, 0, 'accumulate'), (48, 128, 128, 128, 32, 3, 1,
        'accumulate'), (48, 128, 128, 32, 32, 3, 1, 'accumulate'), (48, 128, 128, 32, 64, 1, 0, 'accumulate'), (48, 128,
        128, 32, 64, 3, 1, 'accumulate'), (48, 16, 16, 256, 256, 3, 1, 'accumulate'), (48, 16, 16, 512, 256, 1, 0,
        'accumulate'), (48, 16, 16, 512, 256, 3, 1, 'accumulate'), (48, 256, 256, 16, 16, 3, 1, 'accumulate'), (48, 256,
        256, 16, 32, 1, 0, 'accumulate'), (48, 256, 256, 16, 32, 3, 1, 'accumulate'), (48, 256, 256, 64, 16, 1, 0,
        'accumulate'), (48, 256, 256, 64, 16, 3, 1, 'accumulate'), (48, 32, 32, 128, 128, 3, 1, 'accumulate'), (48, 32, 32,
        128, 256, 1, 0, 'accumulate'), (48, 32, 32, 128, 256, 3, 1, 'accumulate'), (48, 32, 32, 512, 128, 1, 0,
        'accumulate'), (48, 32, 32, 512, 128, 3, 1, 'accumulate'), (48, 4, 4, 256, 256, 3, 1, 'accumulate'), (48, 4, 4, 384,
        256, 3, 1, 'accumulate'), (48, 64, 64, 256, 64, 1, 0, 'accumulate'), (48, 64, 64, 256, 64, 3, 1, 'accumulate'), (48,
        64, 64, 64, 128, 1, 0, 'accumulate'), (48, 64, 64, 64, 128, 3, 1, 'accumulate'), (48, 64, 64, 64, 64, 3, 1,
        'accumulate'), (48, 8, 8, 256, 256, 3, 1, 'accumulate'), (48, 8, 8, 512, 256, 1, 0, 'accumulate'), (48, 8, 8, 512,
        256, 3, 1, 'accumulate'), (6, 128, 128, 32, 32, 3, 1, 'accumulate'), (6, 128, 128, 32, 64, 1, 0, 'accumulate'), (6,
        128, 128, 32, 64, 3, 1, 'accumulate'), (6, 16, 16, 256, 256, 3, 1, 'accumulate'), (6, 256, 256, 16, 16, 3, 1,
        'accumulate'), (6, 256, 256, 16, 32, 1, 0, 'accumulate'), (6, 256, 256, 16, 32, 3, 1, 'accumulate'), (6, 32, 32,
        128, 128, 3, 1, 'accumulate'), (6, 32, 32, 128, 256, 1, 0, 'accumulate'), (6, 32, 32, 128, 256, 3, 1, 'accumulate'),
        (6, 64, 64, 64, 128, 1, 0, 'accumulate'), (6, 64, 64, 64, 128, 3, 1, 'accumulate'), (6, 64, 64, 64, 64, 3, 1,
        'accumulate'), (6, 8, 8, 256, 256, 3, 1, 'accumulate'), (64, 128, 128, 128, 32, 1, 0, 'accumulate'), (64, 128, 128,
        128, 32, 3, 1, 'accumulate'), (64, 128, 128, 32, 32, 3, 1, 'accumulate'), (64, 16, 16, 256, 256, 3, 1,
        'accumulate'), (64, 16, 16, 512, 256, 1, 0, 'accumulate'), (64, 16, 16, 512, 256, 3, 1, 'accumulate'), (64, 256,
        256, 16, 16, 3, 1, 'accumulate'), (64, 256, 256, 64, 16, 1, 0, 'accumulate'), (64, 256, 256, 64, 16, 3, 1,
        'accumulate'), (64, 32, 32, 128, 128, 3, 1, 'accumulate'), (64, 32, 32, 512, 128, 1, 0, 'accumulate'), (64, 32, 32,
        512, 128, 3, 1, 'accumulate'), (64, 4, 4, 256, 256, 3, 1, 'accumulate'), (64, 64, 64, 256, 64, 1, 0, 'accumulate'),
        (64, 64, 64, 256, 64, 3, 1, 'accumulate'), (64, 64, 64, 64, 64, 3, 1, 'accumulate'), (64, 8, 8, 256, 256, 3, 1,
        'accumulate'), (64, 8, 8, 512, 256, 1, 0, 'accumulate'), (64, 8, 8, 512, 256, 3, 1, 'accumulate'), (8, 1, 1, 4096,
        256, 1, 0, 'accumulate'), (8, 128, 128, 32, 32, 3, 1, 'accumulate'), (8, 128, 128, 32, 64, 1, 0, 'accumulate'), (8,
        128, 128, 32, 64, 3, 1, 'accumulate'), (8, 16, 16, 256, 256, 3, 1, 'accumulate'), (8, 32, 32, 128, 128, 3, 1,
        'accumulate'), (8, 32, 32, 128, 256, 1, 0, 'accumulate'), (8, 32, 32, 128, 256, 3, 1, 'accumulate'), (8, 4, 4, 384,
        256, 3, 1, 'accumulate'), (8, 64, 64, 64, 128, 1, 0, 'accumulate'), (8, 64, 64, 64, 128, 3, 1, 'accumulate'), (8,
        64, 64, 64, 64, 3, 1, 'accumulate'), (8, 8, 8, 256, 256, 3, 1, 'accumulate'), (9, 1, 1, 4096, 256, 1, 0,
        'accumulate'), (9, 128, 128, 32, 32, 3, 1, 'accumulate'), (9, 128, 128, 32, 64, 1, 0, 'accumulate'), (9, 128, 128,
        32, 64, 3, 1, 'accumulate'), (9, 16, 16, 256, 256, 3, 1, 'accumulate'), (9, 256, 256, 16, 16, 3, 1, 'accumulate'),
        (9, 256, 256, 16, 32, 1, 0, 'accumulate'), (9, 256, 256, 16, 32, 3, 1, 'accumulate'), (9, 32, 32, 128, 128, 3, 1,
        'accumulate'), (9, 32, 32, 128, 256, 1, 0, 'accumulate'), (9, 32, 32, 128, 256, 3, 1, 'accumulate'), (9, 4, 4, 384,
        256, 3, 1, 'accumulate'), (9, 64, 64, 64, 128, 1, 0, 'accumulate'), (9, 64, 64, 64, 128, 3, 1, 'accumulate'), (9,
        64, 64, 64, 64, 3, 1, 'accumulate'), (9, 8, 8, 256, 256, 3, 1, 'accumulate')],
}
PRODUCT_CONV_KEYS = {(entry,) + key for entry, keys in PRODUCT_CONVS.items() for key in keys}


def test_every_product_conv_is_a_kernel_suite_case(built_lib):
  seen = harvest_product_convs()
  where = key_configs(conv_keys)
  _log_result({'test': 'conv_coverage', 'harvested': len(seen), 'harvest_s': product_launches.HARVEST_SECONDS,
               'keys': sorted(seen, key=str)})
  assert seen == PRODUCT_CONV_KEYS, ('new', sorted(((k, where[k]) for k in seen - PRODUCT_CONV_KEYS), key=str),
                                     'gone', sorted(PRODUCT_CONV_KEYS - seen, key=str))
  missing = sorted(((k, where[k]) for k in seen - suite_keys()), key=str)
  assert not missing, missing
