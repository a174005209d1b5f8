"""Size-independent properties at BASELINE.json's FULL sizes (256x256, 16 pairs per GPU; inference 64 images), where the
CPU oracle is too slow to be the checker:

  * the three conv kernels are mutually adjoint:  <conv(x,w), gy> == <x, dgrad(gy,w)> == <w, wgrad(x,gy)>
  * conv is linear in x
  * the whole step's gradients agree with central finite differences of its own losses (generator set on the
    generator loss, discriminator set on the discriminator loss incl. the DRAGAN double backward)
  * inference is per-sample: running a 64-image batch gives, bit for bit, what running its two halves gives

Everything goes through the C-ABI (twingan_b200.ops / twingan_b200.twingan); the oracle is not involved."""
import math

import pytest
import torch

from tests.parity import _log_result

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
# the full-resolution layers of the 256^2 stage at 16 images (SURVEY 8a.1): narrow, wide and mixed channel counts
FULL_SHAPES = [
    (16, 256, 256, 16, 16),    # E/D block256 conv1
    (16, 256, 256, 16, 32),    # E/D block256 conv2
    (16, 256, 256, 64, 16),    # G block256 conv1 (UNet concat width)
    (16, 128, 128, 32, 64),
    (16, 64, 64, 64, 128),
    (16, 32, 32, 512, 128),    # G block32 conv1
    (16, 16, 16, 256, 256),
]


def _dot(a, b):
  return float((a.double() * b.double()).sum())


@pytest.mark.parametrize('shape', FULL_SHAPES)
def test_conv_kernels_are_mutually_adjoint_and_linear_at_full_size(built_lib, shape):
  from twingan_b200 import ops
  N, H, W, Ci, Co = shape
  ops.set_precision(1)
  g = torch.Generator(device=DEV).manual_seed(11)
  x = torch.randn((N, H, W, Ci), device=DEV, generator=g)
  x2 = torch.randn((N, H, W, Ci), device=DEV, generator=g)
  w = torch.randn((3, 3, Ci, Co), device=DEV, generator=g) * 0.05
  gy = torch.randn((N, H, W, Co), device=DEV, generator=g)
  y = ops.conv_fwd_raw(x, w, 3, 1)
  gx = ops.conv_dgrad_raw(gy, w, (N, H, W, Ci), 3, 1)
  gw = ops.conv_wgrad_raw(x, gy, 3, 1)
  a, b, c = _dot(y, gy), _dot(x, gx), _dot(w, gw)
  # typical magnitude of such an inner product: |y| |gy| / sqrt(n); split-bf16 products carry ~5e-6 relative error each
  scale = float(y.double().norm() * gy.double().norm()) / math.sqrt(y.numel())
  _log_result({'test': 'fullsize_adjoint', 'shape': list(shape), 'fwd_vs_dgrad': abs(a - b) / scale, 'fwd_vs_wgrad': abs(a - c) / scale})
  assert abs(a - b) <= 1e-3 * scale, (shape, a, b, scale)
  assert abs(a - c) <= 1e-3 * scale, (shape, a, c, scale)
  # linearity in x
  y2 = ops.conv_fwd_raw(x2, w, 3, 1)
  ylin = ops.conv_fwd_raw(0.75 * x - 1.5 * x2, w, 3, 1)
  err = float((ylin - (0.75 * y - 1.5 * y2)).abs().max() / ylin.abs().max())
  assert err < 1e-4, (shape, err)    # bf16x3: ~5e-6 per product
  # zero padding really is zero: an input supported on the interior only produces nothing two pixels away from it
  xi = torch.zeros_like(x)
  xi[:, 8:H - 8, 8:W - 8, :] = x[:, 8:H - 8, 8:W - 8, :]
  yi = ops.conv_fwd_raw(xi, w, 3, 1)
  assert float(yi[:, :7].abs().max()) == 0.0 and float(yi[:, :, :7].abs().max()) == 0.0
  assert float(yi[:, H - 7:].abs().max()) == 0.0 and float(yi[:, :, W - 7:].abs().max()) == 0.0


def _losses(model, s, t, r):
  from twingan_b200 import ops
  ops.begin_step()
  ops.invalidate_weight_cache()
  g_loss, d_loss, _, _, _ = model.clone_fn(s, t, r)
  return float(g_loss.detach()), float(d_loss.detach())


def test_full_step_gradients_match_finite_differences_of_the_losses(built_lib):
  """configs[3] shape: 256x256, 16 pairs, instance norm, DRAGAN.  d(loss)/d(theta) . d  vs  (L(theta+d) - L(theta-d))/2
  along the gradient direction and along a gradient + random mixture, separately for the generator set (generator
  loss) and the discriminator set (discriminator loss, which contains the gradient penalty => double backward)."""
  from twingan_b200 import ops, twingan
  ops.set_precision(1)
  model = twingan.GanModel(twingan.Flags(train_image_size=256), device=DEV)
  v = model.variables
  gen = torch.Generator(device=DEV).manual_seed(3)
  s = torch.rand((16, 256, 256, 3), device=DEV, generator=gen)
  t = torch.rand((16, 256, 256, 3), device=DEV, generator=gen)
  r = twingan.make_dragan_rand(16, 256, DEV, gen)
  # move the normaliser gammas/betas and biases off their symmetric initial values so every gradient path is exercised
  with torch.no_grad():
    for n, (o, shp) in v.offsets.items():
      if not n.endswith('/weights'):
        k = int(math.prod(shp))
        v.flat[o:o + k].add_(0.1 * torch.randn(k, device=DEV, generator=gen))
  ops.invalidate_weight_cache()
  model.compute_gradients(s, t, r)
  grad = model.flat_grad.clone()
  theta0 = v.flat.clone()
  assert torch.isfinite(grad).all()
  for group, which in (('G', 0), ('D', 1)):
    lo, hi = v.group_range[group]
    gvec = torch.zeros_like(grad)
    gvec[lo:hi] = grad[lo:hi]
    gn2 = _dot(gvec, gvec)
    assert gn2 > 0
    rnd = torch.zeros_like(grad)
    rnd[lo:hi] = torch.randn(hi - lo, device=DEV, generator=gen)
    # only perturb real variables, not the alignment padding between them (its gradient is identically zero anyway)
    rnd = rnd * (gvec != 0)
    rnd = rnd * (math.sqrt(gn2) / float(rnd.double().norm()))
    for direction in (gvec, gvec + rnd):
      slope = _dot(gvec, direction)                    # analytic directional derivative per unit step
      step = 2e-3 / abs(slope)                         # predicted loss change of +-2e-3 each way (losses are O(1))
      with torch.no_grad():
        v.flat.copy_(theta0 + step * direction)
      lp = _losses(model, s, t, r)[which]
      with torch.no_grad():
        v.flat.copy_(theta0 - step * direction)
      lm = _losses(model, s, t, r)[which]
      fd = (lp - lm) / (2 * step)
      _log_result({'test': 'fullsize_fd', 'group': group, 'fd': fd, 'slope': slope, 'ratio': fd / slope, 'lp': lp, 'lm': lm})
      assert abs(fd - slope) <= 0.05 * abs(slope), (group, fd, slope, lp, lm, step)
  with torch.no_grad():
    v.flat.copy_(theta0)
  ops.invalidate_weight_cache()


def test_inference_is_per_sample_at_config5_size(built_lib):
  """configs[4]: 64 images at 256x256 through E(.;'_s', eval) -> G(.;'_t', eval): the batch equals its two halves."""
  from twingan_b200 import ops, twingan
  ops.set_precision(1)
  model = twingan.GanModel(twingan.Flags(train_image_size=256, generator_norm_type='batch_renorm'), device=DEV)
  v = model.variables
  gen = torch.Generator(device=DEV).manual_seed(9)
  with torch.no_grad():   # moving_mean ~ N(0, 0.1), moving_variance ~ U(0.5, 1.5) (SURVEY 8d config 5)
    for key, (o, C) in v.state_offsets.items():
      v.state[o:o + C] = 0.1 * torch.randn(C, device=DEV, generator=gen)
      v.state[o + C:o + 2 * C] = 0.5 + torch.rand(C, device=DEV, generator=gen)
  x = torch.rand((64, 256, 256, 3), device=DEV, generator=gen)
  full = model.infer(x)
  assert tuple(full.shape) == (64, 256, 256, 3) and torch.isfinite(full).all()
  halves = torch.cat([model.infer(x[:32].contiguous()), model.infer(x[32:].contiguous())], 0)
  err = float((full - halves).abs().max() / full.abs().max())
  _log_result({'test': 'fullsize_infer_split', 'err': err, 'bit_equal': bool(torch.equal(full, halves))})
  # bit for bit: the evaluation path has no cross-sample reduction, no conv splits K, and the tensor-core tile shape
  # depends on the layer, not the batch
  assert torch.equal(full, halves), err
  # and the translation really depends on its input
  assert float((full[0] - full[1]).abs().max()) > 0


@pytest.mark.parametrize('norm', ['instance_norm', 'batch_renorm'])
def test_batched_passes_equal_the_reference_pass_structure_at_full_size(built_lib, norm):
  """configs[3] size (256x256, 16 pairs): the step with the weight-sharing passes batched (E 2x16 -> 32, G 4x16 -> 64,
  D 3x16 -> 48 per domain) against the same step run as the reference's 16 separate passes -- every named loss, forward
  tensors, the flat gradient and the normaliser statistics pushed afterwards.  Both are CUDA paths; what this checks is
  the wiring of the batched step (domains, per-pass statistics, gradient fan-in) at the size where the CPU checker cannot.

  The two structures do not add in the same order: the batched step's weight gradients split their pixel sums by the
  batched N, and its per-variable gradients are one sum where the pass-by-pass step adds one per pass.  Instance norm
  with eps 1e-6 amplifies such last-bit differences, and a few of the 1.6e9 leaky-ReLU pre-activations land on the other
  side of their kink (the oracle tests transfer the active set, two 16 GB device runs cannot).  So the pass-by-pass step
  is run twice, and its distance to itself (zero when the kernels are reproducible, as they are) plus the stated floors
  is what the batched step is held to."""
  from twingan_b200 import ops, twingan
  ops.set_precision(1)
  gen = torch.Generator(device=DEV).manual_seed(21)
  s = torch.rand((16, 256, 256, 3), device=DEV, generator=gen)
  t = torch.rand((16, 256, 256, 3), device=DEV, generator=gen)
  r = twingan.make_dragan_rand(16, 256, DEV, gen)

  def run(batched):
    model = twingan.GanModel(twingan.Flags(train_image_size=256, generator_norm_type=norm, batch_passes=batched,
                                           global_step=15000), device=DEV, seed=11)
    v = model.variables
    g2 = torch.Generator(device=DEV).manual_seed(5)
    with torch.no_grad():
      for n, (o, shp) in v.offsets.items():
        if not n.endswith('/weights'):
          k = int(math.prod(shp))
          v.flat[o:o + k].add_(0.1 * torch.randn(k, device=DEV, generator=g2))
    ops.invalidate_weight_cache()
    _, _, ends, stats = model.compute_gradients(s, t, r)
    model.apply_stat_updates(stats)
    torch.cuda.synchronize()
    fw = torch.cat([ends[k].detach().reshape(-1).float() for k in ('s_prime', 't_cycle', 'enc_t_prime', 'pred_s_prime',
                                                                     'pred_real_t')])
    return (model.flat_grad.clone(), {k: float(x) for k, x in model.last_losses.items()}, v.state.clone(), fw, v.group_range)

  rel = lambda a, b: float((a.double() - b.double()).norm() / b.double().norm())
  ref1, ref2, bat = run(False), run(False), run(True)
  assert set(bat[1]) == set(ref1[1])
  for k in ref1[1]:
    noise = abs(ref1[1][k] - ref2[1][k])
    assert abs(bat[1][k] - ref1[1][k]) <= 3 * noise + 1e-4 * abs(ref1[1][k]) + 1e-7, (k, bat[1][k], ref1[1][k], ref2[1][k])
  rec = {'test': 'fullsize_batched_vs_pass_by_pass', 'norm': norm, 'fwd_noise': rel(ref2[3], ref1[3]), 'fwd_gap': rel(bat[3], ref1[3])}
  assert rec['fwd_gap'] <= 3 * rec['fwd_noise'] + 1e-5, rec
  for group in ('G', 'D'):
    lo, hi = ref1[4][group]
    rec['grad_noise_' + group] = rel(ref2[0][lo:hi], ref1[0][lo:hi])
    rec['grad_gap_' + group] = rel(bat[0][lo:hi], ref1[0][lo:hi])
  _log_result(rec)
  print(rec)
  for group in ('G', 'D'):
    assert rec['grad_gap_' + group] <= 3 * rec['grad_noise_' + group] + 1e-4, rec
    assert rec['grad_gap_' + group] < 5e-2, rec
  if ref1[2].numel() > 4:
    noise = float((ref2[2] - ref1[2]).abs().max())
    assert float((bat[2] - ref1[2]).abs().max()) <= 3 * noise + 1e-4 * max(float(ref1[2].abs().max()), 1.0)
