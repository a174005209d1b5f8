"""The training step runs the domain-t discriminator chain on a second stream beside the domain-s chain
(Flags.concurrent_domains).  The domains share no variable, gradient sink or partial-sum region, and every kernel keeps
its inputs, grid and order within its domain, so the two-stream step must compute what the serial schedule computes,
bit for bit -- losses, gradient buffer, parameters, Adam slots, normaliser state and device counters after every step --
eager and graph-replayed, at the bench configuration, a small and a large stage of the stage runner's batch tables, the
residual blocks, the WGAN-GP and hinge losses, the equalized learning rate and the alternating (mode A) step."""
import gc
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
STEPS = 2
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CONFIGS = [
    ('bench 256 B=16', 256, 16, {}),
    ('TWINGAN_HW_TO_BATCH_SIZE 16 B=8', 16, 8, {}),
    ('DEFAULT_HW_TO_BATCH_SIZE 256 B=12', 256, 12, {}),
    ('use_res_block 64 B=16', 64, 16, {'use_res_block': True}),
    ('wgan_gp 64 B=16', 64, 16, {'loss_architecture': 'wgan_gp'}),
    ('hinge 64 B=16', 64, 16, {'loss_architecture': 'hinge'}),
    ('equalized_learning_rate 64 B=16', 64, 16, {'equalized_learning_rate': True}),
]


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
          'counters': model._counters.clone()}


def _train(hw, kw, batches, concurrent, mode='eager'):
  """STEPS steps of a fresh model (seed 5) and the record after each: mode 'eager' (train_step), 'graphed'
  (train_step_graphed) or 'alternating' (train_step_alternating)."""
  from twingan_b200 import twingan
  model = twingan.GanModel(twingan.Flags(train_image_size=hw, concurrent_domains=concurrent, **kw), device=DEV, seed=5)
  if mode == 'graphed':
    model.capture(*batches[0])
  step = {'eager': model.train_step, 'graphed': model.train_step_graphed,
          'alternating': model.train_step_alternating}[mode]
  recs = []
  for s, t, r in batches:
    gl, dl = step(s, t, r)[:2]
    recs.append(_record(model, gl, dl))
  recs[0]['names'] = {n: (o, int(torch.Size(shape).numel())) for n, (o, shape) in model.variables.offsets.items()}
  torch.cuda.synchronize()
  del model
  _free()
  return recs


def _serial(hw, kw, batches, mode='eager'):
  """The serial schedule's records, from the second of two serial runs.  The first model a process trains does not
  reproduce the later ones bit for bit, with either schedule (DESIGN §1, known issue).  The first-model case is compared
  across two fresh processes by test_first_model_of_a_process_equals_serial_step."""
  _train(hw, kw, batches, concurrent=False, mode=mode)
  return _train(hw, kw, batches, concurrent=False, mode=mode)


def _assert_equal(serial, concurrent, what):
  assert len(serial) == len(concurrent) == STEPS
  names = serial[0]['names']
  for step, (a, b) in enumerate(zip(serial, concurrent)):
    for key in a:
      if key == 'names' or torch.equal(a[key], b[key]):
        continue
      d = (a[key] - b[key]).abs()
      where = ''
      if key in ('flat_grad', 'variables', 'adam_m', 'adam_v'):
        hit = set(int(i) for i in torch.nonzero(d).flatten().tolist())
        where = ' in ' + ', '.join(sorted(n for n, (o, c) in names.items() if any(o <= i < o + c for i in hit)))
      raise AssertionError('%s, step %d: %s differs from the serial schedule at %d elements (max |diff| %g)%s'
                           % (what, step, key, int((d != 0).sum()), float(d.max()), where))


@pytest.mark.parametrize('label,hw,pairs,kw', CONFIGS, ids=[c[0] for c in CONFIGS])
def test_two_stream_step_equals_serial_step(built_lib, label, hw, pairs, kw):
  batches = _batches(hw, pairs, 23)
  serial = _serial(hw, kw, batches)
  _assert_equal(serial, _train(hw, kw, batches, concurrent=True), 'eager')
  _assert_equal(serial, _train(hw, kw, batches, concurrent=True, mode='graphed'), 'graph-replayed')
  assert not torch.equal(serial[0]['variables'], serial[-1]['variables'])


def test_two_stream_alternating_step_equals_serial(built_lib):
  batches = _batches(64, 16, 29)
  serial = _serial(64, {}, batches, mode='alternating')
  _assert_equal(serial, _train(64, {}, batches, concurrent=True, mode='alternating'), 'mode A')


def test_two_stream_step_repeats_with_other_work_between(built_lib):
  """The same two-stream run twice in one process, with unrelated device work and allocations between the two."""
  batches = _batches(256, 16, 31)
  _train(256, {}, batches, concurrent=True, mode='graphed')
  first = _train(256, {}, batches, concurrent=True, mode='graphed')
  junk = [torch.randn((1024, 1024), device=DEV) for _ in range(8)]
  for a in junk:
    torch.mm(a, a, out=a)
  del junk
  _assert_equal(first, _train(256, {}, batches, concurrent=True, mode='graphed'), 'second run')


_FRESH = r'''
import sys
sys.path.insert(0, sys.argv[1])
import torch
from tests.test_gpu_concurrent_d import _batches, _train
recs = _train(64, {'loss_architecture': 'wgan_gp'}, _batches(64, 16, 37), concurrent=sys.argv[2] == '1')
torch.save(recs, sys.argv[3])
'''


def test_first_model_of_a_process_equals_serial_step(built_lib, tmp_path):
  """The two-stream step as the first model of a fresh process, where every lazily made constant is made during the
  step, against the serial step as the first model of another: WGAN-GP, whose interpolate reads ops._one."""
  recs = {}
  for concurrent in (0, 1):
    out = str(tmp_path / ('%d.pt' % concurrent))
    run = subprocess.run([sys.executable, '-c', _FRESH, ROOT, str(concurrent), out], cwd=ROOT, capture_output=True,
                         text=True, timeout=600)
    assert run.returncode == 0, run.stderr[-3000:]
    recs[concurrent] = torch.load(out)
  _assert_equal(recs[0], recs[1], 'first model of its process')


def test_domain_chains_use_disjoint_partial_regions(built_lib):
  """The domain-t stream owns a partial-sum region of its own, the library refuses it to any other stream, and the
  two-stream step's reductions on that stream are served from it: the serial step never touches it."""
  from twingan_b200 import ops
  from twingan_b200._lib import lib
  L = lib()
  side = ops.domain_stream(DEV)
  main = torch.cuda.current_stream(DEV)
  assert L.cdll.twg_partials_region(side.cuda_stream) == 1
  assert L.cdll.twg_partials_region(main.cuda_stream) == 0
  other = torch.cuda.Stream(device=DEV)
  assert L.try_call('twg_partials_bind', other.cuda_stream, 1) != 0
  assert 'another stream' in L.last_error()
  assert L.cdll.twg_partials_region(other.cuda_stream) == 0
  assert ops.domain_stream(DEV) is side
  batches = _batches(64, 16, 41)
  uses = []
  for concurrent in (False, True):
    before = [L.cdll.twg_partials_region_uses(r) for r in (0, 1)]
    _train(64, {}, batches, concurrent=concurrent)
    uses.append([L.cdll.twg_partials_region_uses(r) - b for r, b in zip((0, 1), before)])
  (serial0, serial1), (two0, two1) = uses
  assert serial1 == 0 and serial0 > 0, uses
  assert two1 > 0 and two0 + two1 == serial0, uses       # the same reductions, the domain-t chain's on region 1
