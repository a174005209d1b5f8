"""The step that runs is usually a replayed CUDA graph: bench.py times train_step_graphed, pggan_runner.run_stage captures
every stable stage and replays it, and InferencePipeline(use_graph=True) replays one graph per batch shape.  No reduction
of the step depends on launch timing (no fp32 atomics), so a replay must compute what the eager launches compute, bit
for bit: losses, gradient buffer, parameters, Adam slots, normaliser state and the device step counters, after every
step, at every stable configuration of the launch harvest (tests/product_launches.py) -- including the 256x256 stages,
where the cluster-launched reductions, the bulk-copy rings, the column-box convs and the conv partials scratch run inside
the capture."""
import gc

import pytest
import torch

from tests.product_launches import harvest_configs, inference_configs

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
STEPS = 3
STABLE = [c for c in harvest_configs() if not c[2]]          # the stages the runner captures
INFER_BATCHES = (64, 1, 37)


def _free():
  gc.collect()
  torch.cuda.empty_cache()


def _batches(hw, pairs, seed):
  from twingan_b200 import twingan
  g = torch.Generator(device=DEV).manual_seed(seed)
  return [(torch.rand((pairs, hw, hw, 3), device=DEV, generator=g), torch.rand((pairs, hw, hw, 3), device=DEV, generator=g),
           twingan.make_dragan_rand(pairs, hw, DEV, g)) for _ in range(STEPS)]


def _record(model, gl, dl):
  v = model.variables
  return {'generator_loss': gl.clone(), 'discriminator_loss': dl.clone(), 'flat_grad': model.flat_grad.clone(),
          'variables': v.flat.clone(), 'adam_m': v.adam_m.clone(), 'adam_v': v.adam_v.clone(), 'state': v.state.clone(),
          'counters': model._counters.clone(), 'lr': model._lr_dev.clone(), 'clip': model._clip_dev.clone()}


def _train(hw, kw, batches, graphed, between=None):
  """STEPS steps of a fresh model (seed 5); the record after each step and whatever `between(model, step)` returned."""
  from twingan_b200 import twingan
  model = twingan.GanModel(twingan.Flags(train_image_size=hw, **kw), device=DEV, seed=5)
  if graphed:
    model.capture(*batches[0])
  recs, extra = [], []
  for i, (s, t, r) in enumerate(batches):
    gl, dl = (model.train_step_graphed if graphed else model.train_step)(s, t, r)
    recs.append(_record(model, gl, dl))
    if between is not None:
      extra.append(between(model, i + 1))
  torch.cuda.synchronize()
  del model
  _free()
  return recs, extra


def _assert_equal_records(eager, replay):
  assert len(eager) == len(replay) == STEPS
  for step, (a, b) in enumerate(zip(eager, replay)):
    for key in a:
      if not torch.equal(a[key], b[key]):
        d = (a[key] - b[key]).abs()
        raise AssertionError('step %d: %s of the replayed step differs from the eager step at %d elements (max |diff| %g)'
                             % (step, key, int((d != 0).sum()), float(d.max())))


@pytest.mark.parametrize('label,hw,pairs,kw', [(c[0], c[1], c[3], c[4]) for c in STABLE], ids=[c[0] for c in STABLE])
def test_replayed_step_equals_eager_step(built_lib, label, hw, pairs, kw):
  batches = _batches(hw, pairs, 17)
  eager, _ = _train(hw, kw, batches, graphed=False)
  replay, _ = _train(hw, kw, batches, graphed=True)
  _assert_equal_records(eager, replay)
  assert not torch.equal(eager[0]['variables'], eager[-1]['variables'])


def _bump_autograd_sequence(n):
  """Create n autograd nodes on this thread: moves its node sequence counter, and no other state, ahead of the counter of
  autograd's CUDA worker thread."""
  x = torch.zeros(1, requires_grad=True)
  for _ in range(n):
    x * 1.0


_HISTORY = [('4 B=16 instance_norm res', 4, False, 16, {'use_res_block': True}),
            ('8 growing B=16 instance_norm res', 8, True, 16, {'use_res_block': True}),
            ('64 B=8 batch_renorm res', 64, False, 8, {'generator_norm_type': 'batch_renorm', 'use_res_block': True}),
            ('16 B=8 wgan_gp res', 16, False, 8, {'loss_architecture': 'wgan_gp', 'use_res_block': True}),
            ('8 growing B=16 instance_norm', 8, True, 16, {}),
            ('64 B=16 instance_norm', 64, False, 16, {})]


@pytest.mark.parametrize('label,hw,growing,pairs,kw', _HISTORY, ids=[c[0] for c in _HISTORY])
def test_eager_step_does_not_depend_on_autograd_history(built_lib, label, hw, growing, pairs, kw):
  """Autograd picks the next ready node by per-thread sequence numbers, and the penalty's double-backward nodes are made on
  its CUDA worker thread.  The gradient of a fresh model's step must not depend on how far the two counters have drifted:
  the same after steps that advance the worker's counter and after 200 000 nodes that advance the main thread's (before
  the residual-block weight gradients were summed in a fixed order, the 4x4 residual case differed in its last bits)."""
  from twingan_b200 import twingan
  s, t, r = _batches(hw, pairs, 31)[0]

  def grad(steps=0):
    model = twingan.GanModel(twingan.Flags(train_image_size=hw, is_growing=growing, alpha_grow=0.5 if growing else 0.0,
                                           **kw), device=DEV, seed=5)
    for _ in range(steps):
      model.compute_gradients(s, t, r)
    model.compute_gradients(s, t, r)
    out = model.flat_grad.clone()
    del model
    return out
  first = grad()
  for when, g in (('after 4 more steps', grad(4)), ('after 200000 main-thread nodes', (_bump_autograd_sequence(200000), grad())[1])):
    assert torch.equal(first, g), '%s: %d gradient elements differ (max |diff| %g)' % (
        when, int((first != g).sum()), float((first - g).abs().max()))
  _free()


class _Images(object):
  """uint8 HWC images made from a seed (len() and image(i) like image_only.ImageOnlyDataset)."""

  def __init__(self, n, seed, hw=20):
    self.imgs = (torch.rand((n, hw, hw, 3), generator=torch.Generator().manual_seed(seed)) * 255).to(torch.uint8).numpy()

  def __len__(self):
    return len(self.imgs)

  def image(self, i):
    return self.imgs[i]


@pytest.mark.parametrize('hw', [64, 256])
def test_replay_after_the_swd_hook_and_inference_equals_eager(built_lib, tmp_path, hw):
  """run_stage calls eval_fn(model, step) between replays: the SWD hook runs model.infer in evaluation mode, and so does a
  caller that samples from the model.  Neither may disturb the captured step, and both give what the eager twin gets."""
  from twingan_b200 import swd
  x = torch.rand((5, hw, hw, 3), device=DEV, generator=torch.Generator(device=DEV).manual_seed(3))
  batches = _batches(hw, 16, 23)

  def between(tag):
    eval_fn = swd.make_eval_fn(_Images(8, 1), _Images(8, 2), 8, str(tmp_path / tag))

    def run(model, step):
      return eval_fn(model, step), model.infer(x).clone(), model.infer(x, 's').clone()
    return run
  eager, e_extra = _train(hw, {}, batches, False, between('eager'))
  replay, r_extra = _train(hw, {}, batches, True, between('replay'))
  _assert_equal_records(eager, replay)
  for step, ((swd_a, t_a, s_a), (swd_b, t_b, s_b)) in enumerate(zip(e_extra, r_extra)):
    assert swd_a is not None and swd_a == swd_b, (step, swd_a, swd_b)
    assert torch.equal(t_a, t_b) and torch.equal(s_a, s_b), step


@pytest.mark.parametrize('hw', [64, 256])
def test_replay_sees_weights_loaded_between_steps(built_lib, hw):
  """variables.load_dict between replays marks the weight-plane table dirty: the next replay must read the new planes."""
  batches = _batches(hw, 16, 29)

  def perturb(model, step):
    v = model.variables
    v.load_dict({n: t * (1.0 - 2.0 ** -5) + 1e-3 * step for n, t in v.to_dict().items()})
    return None
  eager, _ = _train(hw, {}, batches, False, perturb)
  replay, _ = _train(hw, {}, batches, True, perturb)
  _assert_equal_records(eager, replay)


def _inference_stages():
  """The distinct models of inference_configs(): (label, hw, growing, alpha, Flags keyword arguments)."""
  out, seen = [], set()
  for label, hw, growing, alpha, _, kw in inference_configs():
    key = (hw, growing, alpha, tuple(sorted(kw.items())))
    if key not in seen:
      seen.add(key)
      out.append((label.rsplit(' ', 1)[0], hw, growing, alpha, kw))
  return out


INFER_STAGES = _inference_stages()


@pytest.mark.parametrize('label,hw,growing,alpha,kw', INFER_STAGES, ids=[c[0] for c in INFER_STAGES])
def test_graphed_inference_pipeline_equals_infer(built_lib, label, hw, growing, alpha, kw):
  """InferencePipeline(use_graph=True) captures one graph per batch shape; every replay equals GanModel.infer bit for bit,
  on 64, 1 and 37 images, in both directions, and a second run through the same graphs again."""
  from twingan_b200 import twingan
  model = twingan.GanModel(twingan.Flags(train_image_size=hw, is_growing=growing, alpha_grow=alpha, **kw), device=DEV)
  g = torch.Generator().manual_seed(hw + 7)
  host = [torch.rand((n, hw, hw, 3), generator=g).pin_memory() for n in INFER_BATCHES]
  for d in ('t', 's'):
    want = [model.infer(h.to(DEV), d).cpu() for h in host]
    pipe = twingan.InferencePipeline(model, use_graph=True, target_domain=d)
    for rnd in range(2):
      got = []
      for out, ev in pipe.run(iter(host)):
        ev.synchronize()
        got.append(out.clone())
      assert len(got) == len(host)
      for n, a, b in zip(INFER_BATCHES, got, want):
        assert torch.equal(a, b), (d, rnd, n, float((a - b).abs().max()))
    assert len(pipe._graphs) == len(INFER_BATCHES)
  del model, pipe
  _free()
