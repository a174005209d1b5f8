"""Data-parallel training all-reduces the generator-set gradient on a side stream while the discriminator backward still
runs (GanModel.train_step, train_step_graphed).  That is only right if the generator-set slice of the gradient buffer is
final when compute_gradients calls after_generator_backward -- with every optional flag, e.g. --equalized_learning_rate,
whose scaled weights collect their gradients in scratch buffers first.  These tests hold that precondition on one GPU,
run the real stream choreography with a stand-in all-reduce, and run ddp.selfcheck on two gloo ranks sharing the GPU."""
import gc
import json
import os
import traceback

import pytest
import torch

from tests.product_launches import harvest_configs

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
# the scaled weights of the pass-by-pass step get one scratch buffer per pass
EXTRA_CONFIGS = [('equalized_learning_rate+pass_by_pass %d%s B=16' % (hw, ' growing' if growing else ''), hw, growing, 16,
                  {'equalized_learning_rate': True, 'batch_passes': False}) for hw, growing in ((256, False), (64, True))]
CONFIGS = harvest_configs() + EXTRA_CONFIGS


def _free():
  gc.collect()
  torch.cuda.empty_cache()


def _flags(hw, growing, kw, **more):
  from twingan_b200 import twingan
  return twingan.Flags(train_image_size=hw, is_growing=growing, alpha_grow=0.5 if growing else 0.0, **kw, **more)


def _batch(hw, pairs, g):
  from twingan_b200 import twingan
  return (torch.rand((pairs, hw, hw, 3), device=DEV, generator=g), torch.rand((pairs, hw, hw, 3), device=DEV, generator=g),
          twingan.make_dragan_rand(pairs, hw, DEV, g))


@pytest.mark.parametrize('label,hw,growing,pairs,kw', CONFIGS, ids=[c[0] for c in CONFIGS])
def test_generator_set_is_final_when_its_allreduce_starts(built_lib, label, hw, growing, pairs, kw):
  """Eager: a clone of the generator-set slice taken in after_generator_backward equals the slice compute_gradients
  returns.  Graphed: the slice after replaying graph 1a (forward + generator-set backward) equals the slice after graph
  1b (discriminator-set backward)."""
  from twingan_b200 import twingan
  g = torch.Generator(device=DEV).manual_seed(41)
  model = twingan.GanModel(_flags(hw, growing, kw), device=DEV)
  v = model.variables
  at_callback = []
  model.compute_gradients(*_batch(hw, pairs, g),
                          after_generator_backward=lambda: at_callback.append(v.group_slice(model.flat_grad, 'G').clone()))
  final = v.group_slice(model.flat_grad, 'G')
  assert float(final.abs().max()) > 0
  assert len(at_callback) == 1 and torch.equal(at_callback[0], final), \
      'eager: %d elements of the generator set change after the callback' % int((at_callback[0] != final).sum())

  s, t, r = _batch(hw, pairs, g)
  model.capture(s, t, r)
  st = model._static
  st['s'].copy_(s)
  st['t'].copy_(t)
  for k, x in r.items():
    st['r'][k].copy_(x)
  model._g1a.replay()
  mid = v.group_slice(model.flat_grad, 'G').clone()
  model._g1b.replay()
  final = v.group_slice(model.flat_grad, 'G')
  assert float(final.abs().max()) > 0
  assert torch.equal(mid, final), 'graphed: %d elements of the generator set change in graph 1b' % int((mid != final).sum())
  del model, st
  _free()


_CHOREOGRAPHY = [('instance_norm 64 B=8', 64, 8, {}),
                 ('batch_renorm 64 B=8', 64, 8, {'generator_norm_type': 'batch_renorm'}),
                 ('equalized_learning_rate 64 B=8', 64, 8, {'equalized_learning_rate': True}),
                 ('equalized_learning_rate+pass_by_pass 64 B=8', 64, 8, {'equalized_learning_rate': True, 'batch_passes': False}),
                 ('bench 256 B=16', 256, 16, {}),
                 ('equalized_learning_rate 256 B=16', 256, 16, {'equalized_learning_rate': True})]


@pytest.mark.parametrize('graphed', [False, True], ids=['eager', 'graphed'])
@pytest.mark.parametrize('label,hw,pairs,kw', _CHOREOGRAPHY, ids=[c[0] for c in _CHOREOGRAPHY])
def test_overlapped_allreduce_stream_choreography(built_lib, monkeypatch, label, hw, pairs, kw, graphed):
  """With a process group, train_step / train_step_graphed all-reduce the generator set on the comm stream between the two
  backward passes and the discriminator set after them.  ddp.allreduce_flat_ is replaced by t.mul_(2), which runs
  exactly where NCCL would and stands for two ranks fed the same batch (x + x is exact in fp32); the result must equal, bit
  for bit, a model without a process group that doubles its gradient buffer between compute_gradients and the applies."""
  from twingan_b200 import ddp, twingan
  calls = []

  def doubled(t, group=None):
    calls.append(t.numel())
    return t.mul_(2)
  monkeypatch.setattr(ddp, 'allreduce_flat_', doubled)
  g = torch.Generator(device=DEV).manual_seed(43)
  batches = [_batch(hw, pairs, g) for _ in range(2)]
  model = twingan.GanModel(_flags(hw, False, kw), device=DEV, seed=9, process_group=object())
  twin = twingan.GanModel(_flags(hw, False, kw), device=DEV, seed=9)
  if graphed:
    model.capture(*batches[0])
  v, w = model.variables, twin.variables
  for step, (s, t, r) in enumerate(batches):
    gl, dl = (model.train_step_graphed if graphed else model.train_step)(s, t, r)
    tgl, tdl, _, stats = twin.compute_gradients(s, t, r)
    twin.flat_grad.mul_(2)
    twin.apply_gradients()
    twin.apply_stat_updates(stats)
    torch.cuda.synchronize()
    for name, a, b in (('generator_loss', gl, tgl), ('discriminator_loss', dl, tdl), ('flat_grad', model.flat_grad, twin.flat_grad),
                       ('variables', v.flat, w.flat), ('adam_m', v.adam_m, w.adam_m), ('adam_v', v.adam_v, w.adam_v),
                       ('state', v.state, w.state), ('counters', model._counters, twin._counters),
                       ('lr', model._lr_dev, twin._lr_dev), ('clip', model._clip_dev, twin._clip_dev)):
      assert torch.equal(a, b), 'step %d: %s differs at %d elements (max |diff| %g)' % (
          step, name, int((a != b).sum()), float((a.double() - b.double()).abs().max()))
  assert calls == [v.group_slice(v.flat, 'G').numel(), v.group_slice(v.flat, 'D').numel()] * len(batches)
  del model, twin
  _free()


def _selfcheck_worker(rank, ports, out_dir, cases):
  import datetime
  import torch.distributed as dist
  result = {}
  try:
    torch.cuda.set_device(0)
    timeout = datetime.timedelta(seconds=120)
    # rank 0's store binds a free port itself and hands it to rank 1: no window in which another process could take it
    if rank == 0:
      store = dist.TCPStore('127.0.0.1', 0, 2, is_master=True, timeout=timeout, wait_for_workers=False)
      ports.put(store.port)
    else:
      store = dist.TCPStore('127.0.0.1', ports.get(timeout=120), 2, is_master=False, timeout=timeout)
    dist.init_process_group('gloo', store=store, rank=rank, world_size=2, timeout=timeout)
    try:
      from twingan_b200 import ddp
      for name, extra, graphed in cases:
        result[name] = ddp.selfcheck(torch.device(DEV), extra_flags=extra, graphed=graphed)
    finally:
      dist.destroy_process_group()
  except BaseException:
    result['error'] = traceback.format_exc()
  with open(os.path.join(out_dir, 'rank%d.json' % rank), 'w') as f:
    json.dump(result, f)


_SELFCHECK_CASES = [('default', None, False), ('default graphed', None, True),
                    ('equalized_learning_rate', {'equalized_learning_rate': True}, False),
                    ('equalized_learning_rate graphed', {'equalized_learning_rate': True}, True)]


def test_two_gloo_ranks_on_one_gpu_pass_the_ddp_selfcheck(built_lib, tmp_path):
  """ddp.selfcheck on two ranks of a gloo process group that share cuda:0 (gloo all-reduces CUDA tensors): the real
  overlapped step, eager and graphed, with the default flags and with --equalized_learning_rate, leaves both ranks with
  the parameters, Adam slots and normaliser state of a step on the summed gradient of the two micro-batches."""
  import torch.multiprocessing as mp
  ctx = mp.get_context('spawn')
  ports = ctx.Queue()
  procs = [ctx.Process(target=_selfcheck_worker, args=(rank, ports, str(tmp_path), _SELFCHECK_CASES)) for rank in range(2)]
  for p in procs:
    p.start()
  try:
    for p in procs:
      p.join(timeout=300)
  finally:
    for p in procs:
      if p.is_alive():
        p.kill()
        p.join()
  assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
  for rank in range(2):
    with open(os.path.join(str(tmp_path), 'rank%d.json' % rank)) as f:
      res = json.load(f)
    assert 'error' not in res, 'rank %d:\n%s' % (rank, res.get('error'))
    for name, _, _ in _SELFCHECK_CASES:
      assert res[name]['world'] == 2 and res[name]['params_identical_across_ranks'], (rank, name, res[name])
      assert res[name]['equal_to_sequential_sum_step'], (rank, name, res[name])
