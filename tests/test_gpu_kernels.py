"""Per-kernel parity on the GPU: every C-ABI kernel family against the CPU oracle's primitive
(oracle/twingan_oracle.py) on identical seeded inputs.  Tolerance 1e-3 relative (north_star), written
next to each check; most fp32 kernels are compared far tighter."""
import math

import pytest
import torch

from tests.parity import rel_err, REL_TOL, conv_error_ratio, exact_elem_c, tc_elem_c, _log_result

pytestmark = pytest.mark.gpu

from oracle import twingan_oracle as O  # noqa: E402


def _dev(t):
  return t.to('cuda:0', torch.float32).contiguous()


def _rand(shape, seed, scale=1.0):
  g = torch.Generator().manual_seed(seed)
  return torch.randn(shape, generator=g, dtype=torch.float64) * scale


CONV_SHAPES = [
    # N, H, W, Cin, Cout, k, pad
    (2, 8, 8, 3, 16, 1, 0),       # fromRGB
    (2, 8, 8, 16, 3, 1, 0),       # toRGB
    (2, 16, 16, 16, 16, 3, 1),
    (3, 8, 8, 32, 64, 3, 1),
    (2, 12, 20, 64, 32, 3, 1),    # non-square, ragged tiles
    (4, 4, 4, 257, 256, 3, 1),    # minibatch-stddev conv
    (4, 4, 4, 256, 256, 4, 0),    # 4x4 VALID head
    (4, 1, 1, 256, 1, 1, 0),      # FC as 1x1
    (1, 32, 32, 128, 128, 3, 1),
    (2, 16, 16, 512, 256, 3, 1),  # UNet-concat width
    (12, 32, 32, 64, 128, 3, 1),  # wide layer, BN = 128
    (4, 40, 36, 128, 256, 3, 1),  # same, ragged tiles, two Cout blocks, two Cin chunks
    (3, 64, 64, 64, 64, 3, 1),    # same, BN = 64
    (2, 32, 32, 32, 64, 3, 1),    # row-box weight gradient (16/32-channel layers, W >= 16)
    (2, 24, 40, 16, 32, 3, 1),    # same, ragged tiles in both directions
    (1, 64, 64, 32, 32, 3, 1),
    (2, 16, 16, 16, 64, 3, 1),
    (3, 16, 48, 32, 16, 3, 1),
    (2, 24, 40, 64, 16, 3, 1),    # row-shift weight gradient, two M groups (64-channel chunk)
    (2, 20, 36, 64, 32, 3, 1),
]
# tensor-core geometries the network runs and the shapes above do not reach (tests/test_cpu_conv_error_model.py
# calibrates the per-element bound on these)
TC_EDGE_SHAPES = [
    # the discriminator's 4x4 VALID head as ops.conv2d runs it: a 1x1 tensor-core conv over the flattened 4x4x256 input
    # (one 128-image tile of 1x1 pixels, 64 K chunks); 130 images = two batch tiles, the last one ragged
    (5, 1, 1, 4096, 256, 1, 0),
    (130, 1, 1, 4096, 256, 1, 0),
    (6, 4, 4, 384, 256, 3, 1),    # the minibatch-stddev conv as run: 257 input channels zero-padded to 384 (tc_channel_pad)
    (2, 16, 16, 16, 128, 3, 1),   # forward kernels <16, 128> and <32, 128>, and the dgrads that select them
    (2, 16, 16, 128, 16, 3, 1),
    (2, 12, 20, 32, 128, 3, 1),
    (2, 12, 20, 128, 32, 3, 1),
    (2, 8, 8, 128, 256, 1, 0),    # 1x1 tensor-core conv over an image
    (9, 3, 5, 64, 64, 3, 1),      # several images per tile (TN > 1), ragged batch, odd image
    (3, 2, 2, 128, 128, 3, 1),    # 2x2 images: only some taps of each pixel are inside
    (5, 1, 1, 64, 64, 3, 1),      # 1x1 images: only the centre tap is inside
]
CONV_SHAPES += TC_EDGE_SHAPES
# every other conv geometry of the training step and of inference at 4x4 .. 256x256 (fromRGB / toRGB, 3x3 layers, 1x1
# residual shortcuts; test_gpu_conv_conformance.py checks that this list and the rest of the suite cover them all)
STEP_SHAPES = [
    (2, 4, 4, 3, 256, 1, 0), (2, 4, 4, 256, 3, 1, 0), (2, 4, 4, 256, 256, 3, 1), (2, 8, 8, 3, 256, 1, 0),
    (2, 8, 8, 256, 3, 1, 0), (2, 8, 8, 256, 256, 3, 1), (2, 8, 8, 512, 256, 1, 0), (2, 8, 8, 512, 256, 3, 1),
    (2, 16, 16, 3, 256, 1, 0), (2, 16, 16, 256, 3, 1, 0), (2, 16, 16, 256, 256, 3, 1), (2, 16, 16, 512, 256, 1, 0),
    (2, 32, 32, 3, 128, 1, 0), (2, 32, 32, 128, 3, 1, 0), (2, 32, 32, 128, 256, 1, 0), (2, 32, 32, 128, 256, 3, 1),
    (2, 32, 32, 512, 128, 1, 0), (2, 32, 32, 512, 128, 3, 1), (2, 64, 64, 3, 64, 1, 0), (2, 64, 64, 64, 3, 1, 0),
    (2, 64, 64, 64, 128, 1, 0), (2, 64, 64, 64, 128, 3, 1), (2, 64, 64, 256, 64, 1, 0), (2, 64, 64, 256, 64, 3, 1),
    (1, 128, 128, 3, 32, 1, 0), (1, 128, 128, 32, 3, 1, 0), (1, 128, 128, 32, 32, 3, 1), (1, 128, 128, 32, 64, 1, 0),
    (1, 128, 128, 32, 64, 3, 1), (1, 128, 128, 128, 32, 1, 0), (1, 128, 128, 128, 32, 3, 1), (1, 256, 256, 3, 16, 1, 0),
    (1, 256, 256, 16, 3, 1, 0), (1, 256, 256, 16, 16, 3, 1), (1, 256, 256, 16, 32, 1, 0), (1, 256, 256, 16, 32, 3, 1),
    (1, 256, 256, 64, 16, 1, 0), (1, 256, 256, 64, 16, 3, 1),
]
CONV_SHAPES += STEP_SHAPES

_CPU_REF_MACS = 2e8     # fp64 references above this many multiply-adds run on the GPU (F.conv2d), below it on the CPU


def conv_refs(x, w, gy, k, pad, device):
  """fp64 references of the three directions on `device`, the same operations on absolute values (the S of
  parity.conv_error_ratio) and on all-ones operands (the number of products each output element adds):
  (y, gx, gw), (S_y, S_gx, S_gw), (K_y, K_gx, K_gw)."""
  pad_s = 'SAME' if pad else 'VALID'
  out = []
  for a, b, g in ((x, w, gy), (x.abs(), w.abs(), gy.abs()), (torch.ones_like(x), torch.ones_like(w), torch.ones_like(gy))):
    a = a.detach().to(device).requires_grad_(True)
    b = b.detach().to(device).requires_grad_(True)
    y = O.conv2d_nhwc(a, b, pad_s)
    ga, gb = torch.autograd.grad(y, (a, b), g.to(device))
    out.append((y.detach(), ga, gb))
  return out


@pytest.mark.parametrize('prec', [0, 1])
@pytest.mark.parametrize('shape', CONV_SHAPES)
def test_conv_fwd_dgrad_wgrad(built_lib, shape, prec):
  """Each direction against fp64, on the whole tensor (rel_err) and per element: |dev - ref| <= c * S with S the same
  operation on absolute values (parity.conv_error_ratio).  Also the weight gradient's accumulate mode."""
  from twingan_b200 import ops
  ops.set_precision(prec)
  try:
    N, H, W, Cin, Cout, k, pad = shape
    Ho, Wo = H + 2 * pad - k + 1, W + 2 * pad - k + 1
    x = _rand((N, H, W, Cin), 1)
    w = _rand((k, k, Cin, Cout), 2, 0.05)
    gy = _rand((N, Ho, Wo, Cout), 3)
    macs = N * Ho * Wo * Cin * Cout * k * k
    refs, sums, counts = conv_refs(x, w, gy, k, pad, 'cpu' if macs < _CPU_REF_MACS else 'cuda:0')
    yd = ops.conv_fwd_raw(_dev(x), _dev(w), k, pad)
    gxd = ops.conv_dgrad_raw(_dev(gy), _dev(w), (N, H, W, Cin), k, pad)
    gwd = ops.conv_wgrad_raw(_dev(x), _dev(gy), k, pad)
    torch.cuda.synchronize()
    tol = 2e-5 if prec == 0 else 1e-4   # << 1e-3 north_star tolerance
    for got, ref in zip((yd, gxd, gwd), refs):
      assert rel_err(got, ref) < tol
    tc = ops.tc_eligible(*shape)
    rec = {'test': 'conv_elem', 'shape': list(shape), 'prec': prec, 'family': 'tc' if tc else 'exact'}
    for d, got, ref, S, K in zip(('fwd', 'dgrad', 'wgrad'), (yd, gxd, gwd), refs, sums, counts):
      c = tc_elem_c(K) if tc else exact_elem_c(K)
      r = conv_error_ratio(got, ref, S, c)
      # the worst |err| / S over the elements with the family's plain constant (K >= 128), for the record
      rec[d] = {'ratio_to_bound': r, 'max_err_over_S': conv_error_ratio(got, ref, S, 1.0)}
    _log_result(rec)
    for d in ('fwd', 'dgrad', 'wgrad'):
      assert rec[d]['ratio_to_bound'] <= 1.0, rec
    # accumulate = 1: the weight gradient is added to what the buffer holds
    buf = _dev(_rand((k, k, Cin, Cout), 4))
    before = buf.clone()
    out = ops._conv_wgrad(_dev(x), _dev(gy), k, pad, out=buf)
    torch.cuda.synchronize()
    assert out is buf
    assert torch.equal(buf, before + gwd)
  finally:
    ops.set_precision(1)


def test_conv_reference_on_the_gpu_matches_the_cpu_oracle(built_lib):
  """The large cases above take their fp64 reference from F.conv2d on the GPU: it agrees with the CPU oracle."""
  shape = (3, 8, 8, 64, 32, 3, 1)
  N, H, W, Cin, Cout, k, pad = shape
  x, w, gy = _rand((N, H, W, Cin), 1), _rand((k, k, Cin, Cout), 2, 0.05), _rand((N, H, W, Cout), 3)
  cpu, gpu = conv_refs(x, w, gy, k, pad, 'cpu'), conv_refs(x, w, gy, k, pad, 'cuda:0')
  for a, b, s in zip(gpu[0], cpu[0], cpu[1]):
    assert conv_error_ratio(a, b.to('cuda:0'), s, 1e-13) <= 1.0


def test_bias_lrelu_pool_upsample_lerp_double_backward(built_lib):
  """Discriminator-side operators are twice differentiable: check d/dtheta of ||d out/dx||^2."""
  from twingan_b200 import ops
  N, H, W, C, Co = 3, 8, 8, 16, 32
  x = _rand((N, H, W, C), 11).requires_grad_(True)
  w = _rand((3, 3, C, Co), 12, 0.1).requires_grad_(True)
  b = _rand((Co,), 13, 0.1).requires_grad_(True)

  def net(x, w, b, conv, act, pool, up, lerp):
    h = act(conv(x, w), b)
    h2 = pool(h)
    h3 = up(h2)
    return lerp(h, h3, 0.3)

  ref_out = net(x, w, b, lambda a, ww: O.conv2d_nhwc(a, ww, 'SAME'), lambda a, bb: O.leaky_relu(a + bb), O.avg_pool2,
                O.resize_twice_as_big, lambda a, c, al: al * a + (1 - al) * c)
  seed = _rand(tuple(ref_out.shape), 14)
  (gx,) = torch.autograd.grad(ref_out, x, seed, create_graph=True)

  xd, wd, bd = (_dev(t.detach()).requires_grad_(True) for t in (x, w, b))
  out = net(xd, wd, bd, lambda a, ww: ops.conv2d(a, ww, 1, 'D'), lambda a, bb: ops.bias_act(a, bb, True, 'D'),
            ops.avg_pool2, ops.resize_twice_as_big, ops.lerp)
  (gxd,) = torch.autograd.grad(out, xd, _dev(seed), create_graph=True)
  pend = ops.gradient_penalty(gxd, 1.0)   # lambda*mean_n (||g||-1)^2
  ref_pen = ((torch.sqrt((gx ** 2).sum(dim=(1, 2, 3))) - 1) ** 2).mean()
  gw_ref2, = torch.autograd.grad(ref_pen, (w,))
  (gwd,) = torch.autograd.grad(pend, (wd,))
  torch.cuda.synchronize()
  assert rel_err(out, ref_out) < 1e-4
  assert rel_err(gxd, gx) < 1e-4
  assert abs(pend.item() - ref_pen.item()) / ref_pen.item() < 1e-4
  assert rel_err(gwd, gw_ref2) < REL_TOL * 0.5


@pytest.mark.parametrize('N,C', [(4, 32), (16, 256), (3, 8)])
def test_mbstd_fwd_bwd_bwd2(built_lib, N, C):
  from twingan_b200 import ops
  x = _rand((N, 4, 4, C), 21).requires_grad_(True)
  out = O.minibatch_state_concat(x)
  go = _rand(tuple(out.shape), 22)
  (gx,) = torch.autograd.grad(out, x, go, create_graph=True)
  v = _rand(tuple(gx.shape), 23)
  (ddx,) = torch.autograd.grad((gx * v).sum(), x)
  xd = _dev(x.detach()).requires_grad_(True)
  outd = ops.minibatch_state_concat(xd)
  (gxd,) = torch.autograd.grad(outd, xd, _dev(go), create_graph=True)
  (ddxd,) = torch.autograd.grad((gxd * _dev(v)).sum(), xd)
  torch.cuda.synchronize()
  assert rel_err(outd, out) < 1e-5
  assert rel_err(gxd, gx) < 1e-4
  assert rel_err(ddxd, ddx) < REL_TOL * 0.5


def test_losses_and_dragan(built_lib):
  from twingan_b200 import ops
  logits = _rand((16, 1), 31, 2.0).requires_grad_(True)
  for label in (0.0, 1.0):
    ref = O.sigmoid_cross_entropy(label, logits, 0.7)
    (g,) = torch.autograd.grad(ref, logits)
    ld = _dev(logits.detach()).requires_grad_(True)
    got = ops.sigmoid_cross_entropy(label, ld, 0.7)
    (gd,) = torch.autograd.grad(got, ld)
    assert abs(got.item() - ref.item()) < 1e-5 * abs(ref.item())
    assert rel_err(gd, g) < 1e-5
  a = _rand((4, 16, 16, 3), 32).requires_grad_(True)
  b = _rand((4, 16, 16, 3), 33).requires_grad_(True)
  ref = O.absolute_difference(a, b, 0.1)
  ga, gb = torch.autograd.grad(ref, (a, b))
  ad, bd = _dev(a.detach()).requires_grad_(True), _dev(b.detach()).requires_grad_(True)
  got = ops.absolute_difference(ad, bd, 0.1)
  gad, gbd = torch.autograd.grad(got, (ad, bd))
  assert abs(got.item() - ref.item()) < 1e-5 * abs(ref.item())
  assert rel_err(gad, ga) < 1e-6 and rel_err(gbd, gb) < 1e-6
  # DRAGAN perturbation: variance (not std) scaling, image_generation.py:445
  real = torch.rand((4, 8, 8, 3), dtype=torch.float64)
  alpha = torch.rand((4, 1, 1, 1), dtype=torch.float64)
  noise = torch.rand((4, 8, 8, 3), dtype=torch.float64) * 2 - 1
  ref = O.dragan_interpolates(real, alpha, noise)
  got = ops.dragan_xhat(_dev(real), _dev(alpha), _dev(noise))
  assert rel_err(got, ref) < 1e-6


def test_adam_tf_epsilon_placement(built_lib):
  """tf.train.AdamOptimizer: eps outside the bias correction (SURVEY 8a.4-5)."""
  from twingan_b200 import ops
  cfg = O.Config()
  p, g = _rand((1000,), 41, 0.05), _rand((1000,), 42, 1e-3)
  m, v = _rand((1000,), 43, 1e-3), _rand((1000,), 44, 1e-3).abs() * 1e-3
  t = 7
  rp, rm, rv = O.adam_apply(cfg, p, g, m, v, t)
  pd, gd, md, vd = _dev(p), _dev(g), _dev(m), _dev(v)
  lr_t = cfg.learning_rate * math.sqrt(1 - cfg.adam_beta2 ** t) / (1 - cfg.adam_beta1 ** t)
  ops.adam_(pd, gd, md, vd, lr_t, cfg.adam_beta1, cfg.adam_beta2, cfg.adam_eps)
  assert rel_err(pd, rp) < 1e-6 and rel_err(md, rm) < 1e-6 and rel_err(vd, rv) < 1e-6


def test_conv_and_pool_entries_reject_bad_arguments_on_gpu(built_lib):
  """Error behaviour of the C-ABI: invalid geometry returns a negative status and a message, never aborts."""
  L = built_lib
  x = torch.zeros(16, device='cuda:0')
  rc = L.try_call('twg_conv_fwd', x.data_ptr(), x.data_ptr(), x.data_ptr(), 1, 2, 2, 1, 1, 5, 0, None)
  assert rc == -1 and 'empty output' in L.last_error()
  rc = L.try_call('twg_conv_fwd', None, x.data_ptr(), x.data_ptr(), 1, 2, 2, 1, 1, 1, 0, None)
  assert rc == -1 and 'null' in L.last_error()
  rc = L.try_call('twg_pool2', x.data_ptr(), x.data_ptr(), None, 1, 3, 3, 1, 0.25, None)
  assert rc == -1


@pytest.mark.parametrize('prec', [0, 1])
@pytest.mark.parametrize('cout', [64, 128])
def test_baseline_config2_fused_layer_family(built_lib, cout, prec):
  """BASELINE.json configs[1] / SURVEY 8d config 2 at its stated size: x ~ N(0,1) [32,64,64,64], W ~ N(0,0.02)
  [3,3,64,64] and [3,3,64,128], gamma ~ U(0.5,1.5), beta ~ N(0,0.1), instance_norm (eps 1e-6) and batch_renorm (eps 1e-3,
  step 0) with leaky-ReLU and pixel-norm, forward + backward with upstream gradient ~ N(0,1), seeds 0/1/2, against the
  fp64 oracle cast to fp32: 1e-3 relative (inf-norm over inf-norm) on every tensor, and per element on the forward
  output with rtol 1e-3 / atol 1e-5 -- met by every element on the exact-fp32 path (prec 0).  The split-bf16 tensor-core
  path (prec 1) carries ~5e-6 relative error per product, i.e. absolute errors up to ~5e-5 on O(1) outputs: a small
  fraction of the elements exceeds atol 1e-5 (worst ~5e-5, ~6e-6 of max|z|); the test bounds that tail
  (fraction <= 1e-3, worst <= 2e-4) instead of pretending it is not there.  The leaky-ReLU active set is
  transferred like in the whole-step tests (DESIGN.md 4, kinks)."""
  from twingan_b200 import ops
  from twingan_b200 import pggan_utils as pu
  ops.set_precision(prec)
  try:
    for seed in ((0, 1, 2) if prec == 1 else (0,)):   # the exact-fp32 path is checked on one seed (CPU oracle time)
      g = torch.Generator().manual_seed(seed)
      x = torch.randn((32, 64, 64, 64), generator=g, dtype=torch.float64).requires_grad_(True)
      w = (torch.randn((3, 3, 64, cout), generator=g, dtype=torch.float64) * 0.02).requires_grad_(True)
      gamma = (0.5 + torch.rand((cout,), generator=g, dtype=torch.float64)).requires_grad_(True)
      beta = (torch.randn((cout,), generator=g, dtype=torch.float64) * 0.1).requires_grad_(True)
      gz = torch.randn((32, 64, 64, cout), generator=g, dtype=torch.float64)
      y_ref = O.conv2d_nhwc(x, w, 'SAME')
      for kind in ('instance_norm', 'batch_renorm'):
        kid = pu._KIND[kind]
        xd, wd = _dev(x.detach()).requires_grad_(True), _dev(w.detach()).requires_grad_(True)
        gd, bd = _dev(gamma.detach()).requires_grad_(True), _dev(beta.detach()).requires_grad_(True)
        snap = torch.zeros(4 * cout + 2, device='cuda:0')      # step 0: renorm statistics and their weights are zero
        snap[cout:2 * cout] = 1.0
        bs = torch.empty((2, cout), device='cuda:0') if kid == ops.NORM_RENORM else None
        ops.ACTIVE_SET_TRACE = {'lrelu': [], 'l1': []}
        try:
          clip = torch.tensor(pu.get_renorm_clipping_params(0), device='cuda:0') if kid == ops.NORM_RENORM else None
          zd = ops.GenLayerFn.apply(xd, wd, gd, bd, None, None, 3, 1, kid, ops.FLAG_LRELU | ops.FLAG_PIXNORM, pu._EPS[kid],
                                    clip, snap, None, bs, 0, 0, 'G', 'fp32')
          got = torch.autograd.grad(zd, (xd, wd, gd, bd), _dev(gz))
          torch.cuda.synchronize()
          trace = ops.ACTIVE_SET_TRACE
        finally:
          ops.ACTIVE_SET_TRACE = None
        assert len(trace['lrelu']) == 1
        O.ACTIVE_SET = {'lrelu': iter([t for _, t in trace['lrelu']]), 'l1': iter(()), 'flips': [0, 0]}
        try:
          if kind == 'instance_norm':
            u = O.instance_norm(y_ref, gamma, beta)
          else:
            zero = torch.zeros(cout, dtype=torch.float64)
            stats = {'renorm_mean': zero, 'renorm_stddev': zero, 'renorm_mean_weight': torch.tensor(0.0, dtype=torch.float64),
                     'renorm_stddev_weight': torch.tensor(0.0, dtype=torch.float64)}
            u = O.batch_norm_train(y_ref, gamma, beta, stats, True, O.renorm_clipping(0))
          z_ref = O.pixel_norm(O.leaky_relu(u))
        finally:
          O.ACTIVE_SET = None
        ref = torch.autograd.grad(z_ref, (x, w, gamma, beta), gz, retain_graph=True)
        tag = (kind, cout, seed, prec)
        assert rel_err(zd, z_ref) < REL_TOL, tag
        for name, a, b in zip(('gx', 'gw', 'ggamma', 'gbeta'), got, ref):
          assert rel_err(a, b) < REL_TOL, tag + (name, rel_err(a, b))
        zr = z_ref.detach().to(torch.float32)
        diff = (zd.detach().cpu() - zr).abs()
        bad = diff > (1e-5 + 1e-3 * zr.abs())
        if prec == 0:
          assert not bool(bad.any()), tag + (int(bad.sum()),)
        else:
          assert float(bad.float().mean()) <= 1e-3 and float(diff.max()) <= 2e-4, tag + (int(bad.sum()), float(diff.max()))
  finally:
    ops.set_precision(1)


@pytest.mark.parametrize('kind', ['instance_norm', 'batch_norm', 'batch_renorm'])
def test_norm_variance_is_stable_far_from_zero_mean(built_lib, kind):
  """tf.nn.moments is two-pass.  With mean = 10 and std = 0.05 (mean^2/var = 4e4) a single-pass fp32 E[y^2] - E[y]^2
  loses the variance (relative error ~ 6e-8 * 4e4 = 2.4e-3 at best, far worse after accumulation); the shifted sums of
  twg_moments keep the forward and the backward within 1e-3 of the fp64 oracle."""
  from twingan_b200 import ops
  from twingan_b200 import pggan_utils as pu
  N, H, W, C = 4, 32, 32, 32
  y = (10.0 + 0.05 * _rand((N, H, W, C), 51)).requires_grad_(True)
  gamma = (1 + _rand((C,), 52, 0.2)).requires_grad_(True)
  beta = _rand((C,), 53, 0.1).requires_grad_(True)
  gz = _rand((N, H, W, C), 54)
  clip = {'rmin': 0.9, 'rmax': 1.1, 'dmax': 0.1}
  stats = {'renorm_mean': torch.full((C,), 6.0, dtype=torch.float64), 'renorm_stddev': torch.full((C,), 0.036, dtype=torch.float64),
           'renorm_mean_weight': torch.tensor(0.6, dtype=torch.float64),
           'renorm_stddev_weight': torch.tensor(0.6, dtype=torch.float64)}
  if kind == 'instance_norm':
    u = O.instance_norm(y, gamma, beta)
  elif kind == 'batch_norm':
    u = O.batch_norm_train(y, gamma, beta, None, False, None)
  else:
    u = O.batch_norm_train(y, gamma, beta, stats, True, clip)
  z = O.pixel_norm(u)      # no leaky-ReLU: its kink would turn the (reference-shared) 1e-5 noise of a*y + b into sign flips
  ref = torch.autograd.grad(z, (y, gamma, beta), gz)
  yd = _dev(y.detach()).requires_grad_(True)
  gd = _dev(gamma.detach()).requires_grad_(True)
  bd = _dev(beta.detach()).requires_grad_(True)
  kid = pu._KIND[kind]
  snap = torch.zeros(4 * C + 2, device='cuda:0')
  snap[2 * C:3 * C] = 6.0
  snap[3 * C:4 * C] = 0.036
  snap[4 * C] = 0.6
  snap[4 * C + 1] = 0.6
  bs = torch.empty((2, C), device='cuda:0')
  zd = ops.NormActFn.apply(yd, gd, bd, kid, ops.FLAG_PIXNORM, pu._EPS[kid], (0.9, 1.1, 0.1), snap,
                           bs if kid != ops.NORM_INSTANCE else None, 'G')
  got = torch.autograd.grad(zd, (yd, gd, bd), _dev(gz))
  torch.cuda.synchronize()
  assert rel_err(zd, z) < REL_TOL
  for a, b in zip(got, ref):
    assert rel_err(a, b) < REL_TOL, (kind, rel_err(a, b))
  if kid != ops.NORM_INSTANCE:
    m_ref = y.detach().mean(dim=(0, 1, 2))
    v_ref = y.detach().var(dim=(0, 1, 2), unbiased=False)
    assert rel_err(bs[0], m_ref) < 1e-6
    second = (v_ref + 1e-3).sqrt() if kid == ops.NORM_RENORM else v_ref
    assert rel_err(bs[1], second) < REL_TOL


@pytest.mark.parametrize('kind', ['instance_norm', 'batch_renorm'])
def test_gen_layer_batched_passes_equal_separate_passes(built_lib, kind):
  """One GenLayerFn call over [pass0 | pass1 | pass2 | pass3] with domains (s, t, t, s) == four calls with one domain
  each: outputs, input gradients, per-domain gamma/beta gradients (summed over the passes of a domain), weight
  gradient, batch statistics per pass."""
  from twingan_b200 import ops
  from twingan_b200 import pggan_utils as pu
  ops.set_precision(0)
  try:
    Bp, H, Ci, Co = 3, 8, 16, 32
    kid = pu._KIND[kind]
    x = _dev(_rand((4 * Bp, H, H, Ci), 61))
    w = _dev(_rand((3, 3, Ci, Co), 62, 0.1))
    gam = [_dev(1 + _rand((Co,), 63 + i, 0.2)) for i in range(2)]
    bet = [_dev(_rand((Co,), 65 + i, 0.1)) for i in range(2)]
    gz = _dev(_rand((4 * Bp, H, H, Co), 67))
    snaps = []
    for i in range(2):
      sn = torch.zeros(4 * Co + 2, device='cuda:0')
      sn[2 * Co:3 * Co] = 0.01 * (i + 1)
      sn[3 * Co:4 * Co] = 0.3 + 0.1 * i
      sn[4 * Co] = 0.5
      sn[4 * Co + 1] = 0.5
      snaps.append(sn)
    clip = torch.tensor([0.9, 1.1, 0.1], device='cuda:0')
    flags = ops.FLAG_LRELU | ops.FLAG_PIXNORM
    doms = (0, 1, 1, 0)
    leaf = lambda t: t.clone().requires_grad_(True)
    xb, wb, g0, b0, g1, b1 = leaf(x), leaf(w), leaf(gam[0]), leaf(bet[0]), leaf(gam[1]), leaf(bet[1])
    bs = torch.empty((4, 2, Co), device='cuda:0') if kid == ops.NORM_RENORM else None
    zb = ops.GenLayerFn.apply(xb, wb, g0, b0, g1, b1, 3, 1, kid, flags, pu._EPS[kid], clip, snaps[0], snaps[1], bs, Bp,
                              sum(d << i for i, d in enumerate(doms)), 'G', 'fp32')
    gb = torch.autograd.grad(zb, (xb, wb, g0, b0, g1, b1), gz)
    zs, gxs = [], []
    acc = {'w': 0, 0: [0, 0], 1: [0, 0]}
    for i, d in enumerate(doms):
      xi, wi, gi, bi = leaf(x[i * Bp:(i + 1) * Bp]), leaf(w), leaf(gam[d]), leaf(bet[d])
      bsi = torch.empty((1, 2, Co), device='cuda:0') if kid == ops.NORM_RENORM else None
      zi = ops.GenLayerFn.apply(xi, wi, gi, bi, None, None, 3, 1, kid, flags, pu._EPS[kid], clip, snaps[d], None, bsi, 0, 0,
                                'G', 'fp32')
      gi_ = torch.autograd.grad(zi, (xi, wi, gi, bi), gz[i * Bp:(i + 1) * Bp])
      zs.append(zi)
      gxs.append(gi_[0])
      acc['w'] = acc['w'] + gi_[1]
      acc[d][0] = acc[d][0] + gi_[2]
      acc[d][1] = acc[d][1] + gi_[3]
      if bs is not None:
        assert rel_err(bs[i], bsi[0]) < 1e-6
    torch.cuda.synchronize()
    assert rel_err(zb, torch.cat(zs)) < 1e-6
    assert rel_err(gb[0], torch.cat(gxs)) < 1e-5
    assert rel_err(gb[1], acc['w']) < 1e-5
    for d in (0, 1):
      assert rel_err(gb[2 + 2 * d], acc[d][0]) < 1e-5
      assert rel_err(gb[3 + 2 * d], acc[d][1]) < 1e-5
  finally:
    ops.set_precision(1)


def test_mbstd_groups_equal_separate_minibatches(built_lib):
  from twingan_b200 import ops
  N, C, G = 4, 32, 3
  x = _dev(_rand((G * N, 4, 4, C), 71))
  go = _dev(_rand((G * N, 4, 4, C + 1), 72))
  v = _dev(_rand((G * N, 4, 4, C), 73))
  xa = x.clone().requires_grad_(True)
  outa = ops.minibatch_state_concat(xa, G)
  (gxa,) = torch.autograd.grad(outa, xa, go, create_graph=True)
  (dda,) = torch.autograd.grad((gxa * v).sum(), xa)
  for g in range(G):
    sl = slice(g * N, (g + 1) * N)
    xg = x[sl].clone().requires_grad_(True)
    outg = ops.minibatch_state_concat(xg)
    (gxg,) = torch.autograd.grad(outg, xg, go[sl].contiguous(), create_graph=True)
    (ddg,) = torch.autograd.grad((gxg * v[sl]).sum(), xg)
    assert rel_err(outa[sl], outg) < 1e-6 and rel_err(gxa[sl], gxg) < 1e-5 and rel_err(dda[sl], ddg) < 1e-5


def test_mbstd_padded_channels_and_padded_weights(built_lib):
  """minibatch_state_concat with zero pad channels + the following 3x3 conv with zero-padded weight rows (tensor-core
  path) == the unpadded pair (C+1 channels, CUDA-core path): values, first and second derivatives, and the weight
  gradient through the temporary padded sink."""
  from twingan_b200 import ops
  N, C, Co, G = 6, 32, 32, 3
  ct = ops.tc_channel_pad(C + 1)
  assert ct == 64 and ops.tc_channel_pad(257) == 384 and ops.tc_channel_pad(16) == 16
  assert ops.tc_eligible(N, 4, 4, ct, Co, 3, 1) and not ops.tc_eligible(N, 4, 4, C + 1, Co, 3, 1)
  x = _dev(_rand((N, 4, 4, C), 91))
  w = _dev(_rand((3, 3, C + 1, Co), 92, 0.2)).requires_grad_(True)
  go = _dev(_rand((N, 4, 4, Co), 93))
  v = _dev(_rand((N, 4, 4, C), 94))

  def run(padded, sink=None):
    xa = x.clone().requires_grad_(True)
    if sink is not None:
      ops.register_grad_sinks({w.data_ptr(): sink})
    try:
      m = ops.minibatch_state_concat(xa, G, ct if padded else None)
      ww = ops.pad_cin(w, ct) if padded else w
      y = ops.conv2d(m, ww, 1, 'D')
      if sink is None:
        gx, gw = torch.autograd.grad(y, [xa, w], go, create_graph=True)
        (dd,) = torch.autograd.grad((gx * v).sum(), xa)
        return y.detach(), gx.detach(), gw.detach(), dd
      (gx,) = torch.autograd.grad(y, xa, go)
      ops.flush_padded_sinks()
      return y.detach(), gx, sink.clone(), None
    finally:
      ops.register_grad_sinks({})
      ops.drop_padded_sinks()

  y0, gx0, gw0, dd0 = run(False)
  y1, gx1, gw1, dd1 = run(True)
  assert rel_err(y1, y0) < 1e-5 and rel_err(gx1, gx0) < 1e-5 and rel_err(gw1, gw0) < 1e-5 and rel_err(dd1, dd0) < 1e-4
  sink = torch.zeros_like(w.detach())
  y2, gx2, gw2, _ = run(True, sink)
  assert rel_err(y2, y0) < 1e-5 and rel_err(gx2, gx0) < 1e-5 and rel_err(gw2, gw0) < 1e-5


def test_batched_wiring_ops(built_lib):
  """FanoutFn, L1GroupsFn, GanLossesFn, sum_scalars, UpsampleConcatFn with a shared skip, RepeatBatchFn against plain
  torch on the CPU in fp64."""
  from twingan_b200 import ops
  B, H = 2, 8
  gout = _rand((4 * B, H, H, 3), 81)
  x = _rand((2 * B, H, H, 3), 82)
  gd = _dev(gout).requires_grad_(True)
  ds, dt, e2, ls, lt = ops.FanoutFn.apply(gd, _dev(x), 0.7)
  sc, tc, tp, sp = gout[0:B], gout[B:2 * B], gout[2 * B:3 * B], gout[3 * B:]
  f32 = lambda t: t.to(torch.float32)
  assert rel_err(ds, f32(torch.cat([x[:B], sc, sp]))) == 0 and rel_err(dt, f32(torch.cat([x[B:], tc, tp]))) == 0
  assert rel_err(e2, f32(torch.cat([tp, sp]))) == 0
  assert abs(ls.item() - 0.7 * (sc - x[:B]).abs().mean().item()) < 1e-6
  assert abs(lt.item() - 0.7 * (tc - x[B:]).abs().mean().item()) < 1e-6
  gds, gdt, ge2 = _rand(tuple(ds.shape), 83), _rand(tuple(dt.shape), 84), _rand(tuple(e2.shape), 85)
  total = (ds * _dev(gds)).sum() + (dt * _dev(gdt)).sum() + (e2 * _dev(ge2)).sum() + 2.0 * ls + 3.0 * lt
  (gg,) = torch.autograd.grad(total, gd)
  n = sc.numel()
  ref = torch.cat([gds[B:2 * B] + 2.0 * 0.7 / n * torch.sign(sc - x[:B]), gdt[B:2 * B] + 3.0 * 0.7 / n * torch.sign(tc - x[B:]),
                   gdt[2 * B:] + ge2[:B], gds[2 * B:] + ge2[B:]])
  assert rel_err(gg, ref) < 1e-6
  # grouped L1
  a, b = _rand((2 * B, 4, 4, 8), 86), _rand((2 * B, 4, 4, 8), 87)
  ad, bd = _dev(a).requires_grad_(True), _dev(b).requires_grad_(True)
  l0, l1 = ops.L1GroupsFn.apply(ad, bd, 0.1)
  assert abs(l0.item() - 0.1 * (a[:B] - b[:B]).abs().mean().item()) < 1e-7
  assert abs(l1.item() - 0.1 * (a[B:] - b[B:]).abs().mean().item()) < 1e-7
  ga, gb_ = torch.autograd.grad(ops.sum_scalars([l0, l1], 0.5), (ad, bd))
  sg = torch.sign(a - b) * 0.1 / a[:B].numel() * 0.5
  assert rel_err(ga, sg) < 1e-6 and rel_err(gb_, -sg) < 1e-6
  # GAN losses
  logits = _rand((3 * B, 1), 88, 2.0)
  ld = _dev(logits).requires_grad_(True)
  out = ops.GanLossesFn.apply(ld, 0.9)
  lg = logits.clone().requires_grad_(True)
  real, cyc, pri = lg[:B], lg[B:2 * B], lg[2 * B:]
  ref6 = [O.sigmoid_cross_entropy(1.0, cyc, 0.9), O.sigmoid_cross_entropy(1.0, pri, 0.9), O.sigmoid_cross_entropy(0.0, cyc, 0.9),
          O.sigmoid_cross_entropy(1.0, real, 0.9), O.sigmoid_cross_entropy(0.0, pri, 0.9), O.sigmoid_cross_entropy(1.0, real, 0.9)]
  for got, want in zip(out, ref6):
    assert abs(got.item() - want.item()) < 1e-5 * abs(want.item())
  for subset in ((0, 1), (2, 3, 4, 5)):
    (g_dev,) = torch.autograd.grad(ops.sum_scalars([out[i] for i in subset], 1.0), ld, retain_graph=True)
    (g_ref,) = torch.autograd.grad(sum(ref6[i] for i in subset), lg, retain_graph=True)
    assert rel_err(g_dev, g_ref) < 1e-5
  # UNet join with a skip shared by two halves of the batch, and its gradient
  a2, b2 = _rand((4, 4, 4, 8), 89), _rand((2, 8, 8, 4), 90)
  a2d, b2d = _dev(a2).requires_grad_(True), _dev(b2).requires_grad_(True)
  j = ops.UpsampleConcatFn.apply(a2d, b2d, False)
  a2c, b2c = a2.clone().requires_grad_(True), b2.clone().requires_grad_(True)
  jr = torch.cat([O.resize_twice_as_big(a2c), torch.cat([b2c, b2c])], dim=3)
  gj = _rand(tuple(jr.shape), 91)
  assert rel_err(j, jr.to(torch.float32)) == 0
  g1 = torch.autograd.grad(j, (a2d, b2d), _dev(gj))
  g2 = torch.autograd.grad(jr, (a2c, b2c), gj)
  assert rel_err(g1[0], g2[0]) < 1e-6 and rel_err(g1[1], g2[1]) < 1e-6
  # repeat
  e = _dev(_rand((3, 4, 4, 8), 92)).requires_grad_(True)
  r = ops.repeat_batch(e)
  gr = _dev(_rand((6, 4, 4, 8), 93))
  (ge,) = torch.autograd.grad(r, e, gr)
  assert rel_err(r, torch.cat([e, e]).detach()) == 0 and rel_err(ge, gr[:3] + gr[3:]) < 1e-6


def test_wide_conv_and_fused_discriminator_epilogue(built_lib):
  """A wide layer (128 -> 128 channels) on the tensor-core path: forward, dgrad, and the fused bias + leaky-ReLU +
  split-plane epilogue of the discriminator layers, against the fp64 convolution."""
  from twingan_b200 import ops
  ops.set_precision(1)
  N, H, W, Ci, Co = 16, 32, 32, 128, 128          # >= 16384 pixels: the fused discriminator epilogue is used
  x = _dev(_rand((N, H, W, Ci), 101))
  w = _dev(_rand((3, 3, Ci, Co), 102, 0.05))
  b = _dev(_rand((Co,), 103, 0.1))
  gy = _dev(_rand((N, H, W, Co), 104))
  y = ops.conv_fwd_raw(x, w, 3, 1)
  gx = ops.conv_dgrad_raw(gy, w, (N, H, W, Ci), 3, 1)
  z = ops.conv_bias_act(x, w, b, 1, True, 'D', emit_planes=True)
  zp = ops._take_planes(z)
  torch.cuda.synchronize()
  x64, w64 = x.double().cpu().requires_grad_(True), w.double().cpu()
  y64 = O.conv2d_nhwc(x64, w64, 'SAME')
  (gx64,) = torch.autograd.grad(y64, x64, gy.double().cpu())
  assert rel_err(y, y64) < 1e-4
  assert rel_err(gx, gx64) < 1e-4
  ref = O.leaky_relu(y64.detach() + b.double().cpu())
  assert rel_err(z.detach(), ref) < 1e-4
  assert rel_err(zp.float().sum(0), z.detach()) < 1e-5          # planes: hi + lo == z


@pytest.mark.parametrize('shape', [(16, 128, 128, 16, 16), (8, 72, 80, 16, 32), (16, 64, 64, 32, 64), (16, 64, 64, 64, 16),
                                   (6, 64, 64, 32, 32), (5, 40, 48, 16, 64), (5, 40, 48, 32, 16), (9, 64, 64, 64, 32)])
def test_row_shift_wgrad_matches_the_halo_wgrad(built_lib, shape):
  """Two weight-gradient kernels on the same operands, on shapes with several pixel tiles per CTA (the stage rings wrap):
  the tensor-core kernel (split-bf16 wgmma, taps stacked along M) against the exact-fp32 CUDA-core kernel, and both
  against the fp64 convolution.  (The id is kept from the kernels this A/B was first written for.)"""
  from twingan_b200 import ops
  N, H, W, Ci, Co = shape
  x = _rand((N, H, W, Ci), 111).requires_grad_(False)
  gy = _rand((N, H, W, Co), 112)
  w = torch.zeros((3, 3, Ci, Co), dtype=torch.float64, requires_grad=True)
  (ref,) = torch.autograd.grad(O.conv2d_nhwc(x, w, 'SAME'), w, gy)
  xd, gd = _dev(x), _dev(gy)
  res = {}
  for prec in (1, 0):
    ops.set_precision(prec)
    res[prec] = ops.conv_wgrad_raw(xd, gd, 3, 1)
  ops.set_precision(1)
  torch.cuda.synchronize()
  assert rel_err(res[1], res[0]) < 2e-5
  assert rel_err(res[1], ref) < 1e-4 and rel_err(res[0], ref) < 1e-4


# N, H, W, Cin, Cout: shapes with epilogue statistics, incl. ragged tiles in both directions
STATS_SHAPES = [(3, 64, 64, 16, 16), (2, 24, 40, 16, 32), (2, 128, 128, 32, 32), (2, 20, 36, 64, 16), (4, 16, 16, 32, 64),
                (2, 72, 80, 16, 16)]


@pytest.mark.parametrize('offset', [0.0, 40.0])
@pytest.mark.parametrize('shape', STATS_SHAPES)
def test_conv_fwd_planes_epilogue_statistics(built_lib, shape, offset):
  """Instance-norm statistics taken in the conv epilogue (twg_conv_fwd_planes + twg_norm_finalize_partials) against
  tf.nn.moments' two-pass definition on the conv output, incl. |mean| >> std (a constant input offset makes every output
  channel's mean large): mean to 1e-6 of its scale, rstd to 1e-4 relative."""
  from twingan_b200 import ops
  from twingan_b200._lib import lib
  N, H, W, Cin, Cout = shape
  L = lib()
  x = _rand((N, H, W, Cin), 21) * 0.5 + offset
  w = _rand((3, 3, Cin, Cout), 22, 0.05) + (0.02 if offset else 0.0)
  gamma0 = 1 + _rand((Cout,), 23, 0.2)
  beta0 = _rand((Cout,), 24, 0.1)
  gamma1 = 1 + _rand((Cout,), 25, 0.2)
  beta1 = _rand((Cout,), 26, 0.1)
  xd, wd = _dev(x), _dev(w)
  xp = ops.split_act(xd)
  slots = ops._epilogue_slots(N, H, W, Cin, Cout, 3, 1)
  assert slots > 0, 'this shape must offer epilogue statistics'
  stats = torch.empty((N, slots, Cout, 4), device='cuda:0')
  y, _ = ops._conv_fwd(None, wd, 3, 1, xp=xp, stats=stats)
  y_plain, _ = ops._conv_fwd(None, wd, 3, 1, xp=xp)
  assert torch.equal(y, y_plain)                       # the statistics epilogue does not change y
  buf = torch.empty((4, N, Cout), device='cuda:0')
  dom_mask, gs = 0b10 if N % 2 == 0 else 0, (N // 2 if N % 2 == 0 else N)
  g0, b0, g1, b1 = _dev(gamma0), _dev(beta0), _dev(gamma1), _dev(beta1)
  L.call('twg_norm_finalize_partials', stats.data_ptr(), slots, g0.data_ptr(), b0.data_ptr(), g1.data_ptr(), b1.data_ptr(),
         dom_mask, gs, 1e-6, buf[0].data_ptr(), buf[1].data_ptr(), buf[2].data_ptr(), buf[3].data_ptr(), N, Cout, ops._st())
  torch.cuda.synchronize()
  y64 = y.double().cpu()
  mean = y64.mean(dim=(1, 2))
  var = ((y64 - mean[:, None, None, :]) ** 2).mean(dim=(1, 2))
  rstd = (var + 1e-6).rsqrt()
  dom = torch.tensor([(dom_mask >> (n // gs)) & 1 for n in range(N)])
  gam = torch.where(dom[:, None] == 1, gamma1[None], gamma0[None])
  bet = torch.where(dom[:, None] == 1, beta1[None], beta0[None])
  a_ref = gam * rstd
  b_ref = bet - mean * a_ref
  scale = y64.abs().max().item()
  assert (buf[2].double().cpu() - mean).abs().max().item() < 1e-6 * scale
  assert ((buf[3].double().cpu() - rstd) / rstd).abs().max().item() < 1e-4
  assert rel_err(buf[0], a_ref) < 1e-4
  assert rel_err(buf[1], b_ref) < 1e-4


def test_generator_layer_epilogue_statistics_match_moments_pass(built_lib):
  """The generator layer (conv -> instance norm -> leaky-ReLU -> pixel norm) gives the same forward tensor and gradients
  whether its statistics come from the conv epilogue or from the twg_moments pass over y."""
  from twingan_b200 import ops
  N, H, W, Cin, Cout = 4, 64, 64, 16, 32
  x = _dev(_rand((N, H, W, Cin), 31))
  w = _dev(_rand((3, 3, Cin, Cout), 32, 0.05))
  gam = [_dev(1 + _rand((Cout,), 33 + i, 0.2)) for i in range(2)]
  bet = [_dev(_rand((Cout,), 35 + i, 0.1)) for i in range(2)]
  gz = _dev(_rand((N, H, W, Cout), 37))
  out = {}
  for on in (True, False):
    ops.EPILOGUE_STATS = on
    ops.begin_step()
    xs = x.clone().requires_grad_(True)
    ws = w.clone().requires_grad_(True)
    ps = [t.clone().requires_grad_(True) for t in (gam[0], bet[0], gam[1], bet[1])]
    z = ops.GenLayerFn.apply(xs, ws, ps[0], ps[1], ps[2], ps[3], 3, 1, ops.NORM_INSTANCE, ops.FLAG_LRELU | ops.FLAG_PIXNORM,
                             1e-6, None, None, None, None, N // 2, 0b10, 'G', 'fp32', None)
    grads = torch.autograd.grad(z, [xs, ws] + ps, gz)
    torch.cuda.synchronize()
    out[on] = [z.detach()] + [g.detach() for g in grads]
  ops.EPILOGUE_STATS = True
  for a, b in zip(out[True], out[False]):
    assert rel_err(a, b) < 2e-5


@pytest.mark.parametrize('pool', [None, 'planes'])
@pytest.mark.parametrize('shape', [(3, 64, 64, 16, 16), (2, 24, 40, 16, 32), (2, 32, 32, 64, 32), (2, 128, 128, 16, 16),
                                   (1, 64, 64, 32, 32)])   # the last two are wide enough for the image-row backward kernel
def test_discriminator_layer_sign_mask_backward_is_bit_identical(built_lib, shape, pool):
  """The discriminator layer's first-order backward reads the activation's sign from the byte mask the conv epilogue wrote
  (twg_conv_fwd_planes -> twg_lrelu_bwd_colsum) instead of z: same forward tensors and,
  bit for bit, the same input / weight / bias gradients as the path that reads z (util_misc.py:86: the gradient of
  tf.maximum(0.2 x, x) depends on x only through its sign)."""
  from twingan_b200 import ops
  N, H, W, Cin, Cout = shape
  x = _dev(_rand((N, H, W, Cin), 41))
  w = _dev(_rand((3, 3, Cin, Cout), 42, 0.08))
  b = _dev(_rand((Cout,), 43, 0.1))
  ho, wo = (H // 2, W // 2) if pool else (H, W)
  g = _dev(_rand((N, ho, wo, Cout), 44))
  out = {}
  for on in (True, False):
    ops.ACT_SIGN_MASK = on
    ops.begin_step()
    xs, ws, bs = (t.clone().requires_grad_(True) for t in (x, w, b))
    res = ops.conv_bias_act(xs, ws, bs, 1, True, 'D', emit_planes=False, pool=pool)
    z, head = (res if pool else (res, res))
    target = res[1] if pool else res
    grads = torch.autograd.grad(target, [xs, ws, bs], g)
    torch.cuda.synchronize()
    out[on] = [z.detach().clone(), target.detach().clone()] + [t.detach().clone() for t in grads]
  ops.ACT_SIGN_MASK = True
  for a, c in zip(out[True][:3], out[False][:3]):
    assert torch.equal(a, c)                       # z, pooled z, input gradient: deterministic kernels
  for a, c in zip(out[True][3:], out[False][3:]):
    assert rel_err(a, c) < 1e-6                    # weight / bias gradients: fp32 atomics order only
  # and against the fp64 oracle primitives (conv + bias -> leaky-ReLU -> 2x2 average pool)
  x64, w64, b64 = (t.double().cpu().requires_grad_(True) for t in (x, w, b))
  z64 = O.leaky_relu(O.conv2d_nhwc(x64, w64, 'SAME') + b64)
  t64 = O.avg_pool2(z64) if pool else z64
  ref = torch.autograd.grad(t64, [x64, w64, b64], g.double().cpu())
  assert rel_err(out[True][1], t64) < 1e-4
  # gradients in the L2 norm: an element of z within fp32 rounding of the kink takes the other slope in fp64, which moves a
  # few entries of the gradient by O(1) of their size (the step tests fix the active set instead; here a norm that a handful
  # of such entries cannot dominate is enough)
  for got, want in zip(out[True][2:], ref):
    got = got.double().cpu()
    assert float((got - want).norm() / want.norm()) < 5e-3


@pytest.mark.parametrize('flags_pix', [True, False])
@pytest.mark.parametrize('shape', [(3, 64, 64, 16, 16), (2, 24, 40, 16, 32), (2, 32, 32, 64, 32), (2, 128, 128, 32, 32),
                                   # the other fused instantiations <Cin chunk, Cout>: <16, 64>, <32, 16>, <32, 64>, <64, 16>
                                   (2, 16, 32, 16, 64), (2, 32, 16, 32, 16), (2, 16, 16, 32, 64), (2, 16, 16, 64, 16)])
def test_inference_layer_in_one_kernel(built_lib, shape, flags_pix):
  """twg_conv_affine_act_fwd_planes: conv -> evaluation-mode normaliser (moving statistics = per-channel affine,
  libs/batch_norm.py:266-278) -> leaky-ReLU -> pixel norm in the conv epilogue, against the fp64 oracle primitives and
  against the unfused path (conv, then the normaliser/activation pass); fp32 output, and the split planes of the same values."""
  from twingan_b200 import ops
  N, H, W, Cin, Cout = shape
  x = _rand((N, H, W, Cin), 51)
  w = _rand((3, 3, Cin, Cout), 52, 0.08)
  gamma = 1 + _rand((Cout,), 53, 0.2)
  beta = _rand((Cout,), 54, 0.1)
  mm = _rand((Cout,), 55, 0.1)
  mv = 0.5 + _rand((Cout,), 56).abs()
  y = O.conv2d_nhwc(x, w, 'SAME')
  z = O.leaky_relu(O.batch_norm_eval(y, gamma, beta, mm, mv, 1e-3))
  if flags_pix:
    z = O.pixel_norm(z)
  flags = ops.FLAG_LRELU | (ops.FLAG_PIXNORM if flags_pix else 0)
  assert ops.affine_epilogue_ok(N, H, W, Cin, Cout, 3, 1)
  xd, wd = _dev(x), _dev(w)
  args = (_dev(gamma), _dev(beta), _dev(mm), _dev(mv), flags, 1e-3)
  with torch.no_grad():
    fused = ops.conv_affine_act_eval(xd, wd, *args, emit='both')
    planes = ops._take_planes(fused)
    only = ops.conv_affine_act_eval(xd, wd, *args, emit='planes')
    planes_only = ops._take_planes(only)
    unfused = ops.norm_act_eval(ops.conv2d(xd, wd, 1, 'G'), args[0], args[1], ops.NORM_RENORM, flags, 1e-3, args[2], args[3])
  torch.cuda.synchronize()
  assert rel_err(fused, z) < 1e-4
  assert rel_err(fused, unfused) < 2e-5
  rebuilt = planes[0].float() + planes[1].float()
  assert rel_err(rebuilt, fused) < 2e-5               # hi + lo = z to ~2^-17
  assert torch.equal(planes, planes_only)


@pytest.mark.parametrize('shape', [(4, 16, 16, 32, 16, 2), (2, 64, 64, 16, 16, 2), (4, 4, 4, 64, 32, 4), (3, 32, 24, 8, 8, 3)])
def test_upsample_concat_and_pool_row_kernels(built_lib, shape):
  """resize_twice_as_big + maybe_concat_unet_layer (nets/pggan_utils.py:349, 281-298; the skip batch is shared by
  n % Nb) and tf.nn.avg_pool 2x2 (nets/pggan.py:436) at widths that take the row-decomposed kernels, fp32 and planes output,
  against plain torch indexing; the backward of the join against autograd of the same indexing."""
  from twingan_b200 import ops
  N, H, W, Ca, Cb, Nb = shape
  a = _rand((N, H, W, Ca), 61)
  b = _rand((Nb, 2 * H, 2 * W, Cb), 62)
  up = a.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)
  skip = b[[n % Nb for n in range(N)]]
  want = torch.cat((up, skip), dim=-1)
  ad, bd = _dev(a).requires_grad_(True), _dev(b).requires_grad_(True)
  got = ops.UpsampleConcatFn.apply(ad, bd, False)
  assert rel_err(got, want) < 1e-7          # a pure copy: only the fp64 -> fp32 rounding of the inputs
  g = _rand(tuple(want.shape), 63)
  ga, gb = torch.autograd.grad(got, (ad, bd), _dev(g))
  a64, b64 = a.clone().requires_grad_(True), b.clone().requires_grad_(True)
  ref = torch.cat((a64.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2), b64[[n % Nb for n in range(N)]]), dim=-1)
  ra, rb = torch.autograd.grad(ref, (a64, b64), g)
  assert rel_err(ga, ra) < 1e-6 and rel_err(gb, rb) < 1e-6
  if (Ca + Cb) % 16 == 0:
    planes_only = ops.UpsampleConcatFn.apply(_dev(a), _dev(b), True)
    pl = ops._take_planes(planes_only)
    assert rel_err(pl[0].float() + pl[1].float(), want) < 2e-5
  # 2x2 average pool of the joined tensor (fp32 + planes)
  pooled = ops.avg_pool2(got.detach(), emit_planes=True)
  wantp = want.reshape(N, H, 2, W, 2, Ca + Cb).mean(dim=(2, 4))
  assert rel_err(pooled, wantp) < 1e-6
  pp = ops._take_planes(pooled)
  if pp is not None:
    assert rel_err(pp[0].float() + pp[1].float(), wantp) < 2e-5
