"""Data-parallel gradient aggregation: the reference sums per-clone gradients with tf.add_n
(deployment/model_deploy.py:473-503) after scaling each clone's loss by 1/num_clones (:265-267).
Here: one process per GPU, ONE all-reduce(sum) over the flat gradient buffer (NCCL over NVLink on the GPU
box; gloo in the CPU tests).  Batch-coupled statistics (batch-norm moments, minibatch-stddev, DRAGAN variance)
stay per replica exactly like the reference's clones (SURVEY 8e)."""
from __future__ import annotations

import torch
import torch.distributed as dist


def allreduce_flat_(flat_grad: torch.Tensor, group=None) -> torch.Tensor:
  if group is not None or (dist.is_available() and dist.is_initialized()):
    if dist.get_world_size(group) > 1:
      dist.all_reduce(flat_grad, op=dist.ReduceOp.SUM, group=group)
  return flat_grad


def shard_batch(global_batch: int, rank: int, world: int):
  """Weak scaling: every rank owns `global_batch // world` independent (source,target) pairs."""
  if global_batch % world:
    raise ValueError('global batch %d not divisible by world size %d' % (global_batch, world))
  per = global_batch // world
  return rank * per, (rank + 1) * per


def selfcheck(device, group=None, hw: int = 16, batch: int = 2, max_channels: int = 32, norm: str = 'instance_norm',
              extra_flags=None, graphed: bool = False):
  """Data-parallel correctness of the PRODUCT on real ranks (deployment/model_deploy.py:265-267, 473-503): with
  num_clones = world, (1) the all-reduced flat gradient of the ranks' micro-batches equals the sum over the same
  micro-batches run one after the other on one GPU, (2) after a whole train_step (overlapped all-reduces + both Adam
  applies) every rank holds bit-identical parameters, (3) with two ranks, whose sum g0 + g1 does not depend on the order
  of the reduction, that step leaves parameters, Adam slots and normaliser state bit-identical to a model without a
  process group that sums the two micro-batches' gradients itself.  `extra_flags`: further twingan.Flags fields;
  `graphed`: the step is captured and replayed (train_step_graphed) instead of launched eagerly.  Returns a dict of
  measured errors; raises on failure."""
  from . import twingan
  world = dist.get_world_size(group)
  rank = dist.get_rank(group)
  flags = twingan.Flags(train_image_size=hw, pggan_max_num_channels=max_channels, generator_norm_type=norm, num_clones=world,
                        **(extra_flags or {}))
  model = twingan.GanModel(flags, device=device, seed=7, process_group=group if group is not None else dist.group.WORLD)
  micro = []
  for r in range(world):
    g = torch.Generator(device=device).manual_seed(100 + r)
    micro.append((torch.rand((batch, hw, hw, 3), device=device, generator=g), torch.rand((batch, hw, hw, 3), device=device, generator=g),
                  twingan.make_dragan_rand(batch, hw, device, g)))
  model.compute_gradients(*micro[rank])
  model.allreduce_gradients()
  reduced = model.flat_grad.clone()
  ref = twingan.GanModel(twingan.Flags(**{**flags.__dict__}), device=device, seed=7, process_group=None)
  total = torch.zeros_like(reduced)
  for m in micro:
    ref.compute_gradients(*m)
    total += ref.flat_grad
  scale = float(total.abs().max())
  grad_err = float((reduced - total).abs().max()) / max(scale, 1e-30)
  if not grad_err < 1e-4:
    raise AssertionError('rank %d: all-reduced gradient differs from the sequential sum: %g' % (rank, grad_err))
  # a whole step through the public entry point, then compare parameters across ranks bit for bit
  step_model = twingan.GanModel(twingan.Flags(**{**flags.__dict__}), device=device, seed=7,
                                process_group=group if group is not None else dist.group.WORLD)
  if graphed:
    step_model.capture(*micro[rank])
    step_model.train_step_graphed(*micro[rank])
  else:
    step_model.train_step(*micro[rank])
  torch.cuda.synchronize(device)
  mine = step_model.variables.flat
  gathered = [torch.empty_like(mine) for _ in range(world)]
  dist.all_gather(gathered, mine, group=group)
  identical = all(torch.equal(gathered[0], t) for t in gathered)
  if not identical:
    raise AssertionError('rank %d: parameters differ across ranks after the step' % rank)
  moved = float((mine - ref.variables.flat).abs().max())
  if not moved > 0:
    raise AssertionError('parameters did not move')
  out = {'world': world, 'grad_rel_err_vs_sequential_sum': grad_err, 'params_identical_across_ranks': identical,
         'max_param_update': moved}
  if world == 2:
    twin = twingan.GanModel(twingan.Flags(**{**flags.__dict__}), device=device, seed=7, process_group=None)
    twin.compute_gradients(*micro[1 - rank])
    other = twin.flat_grad.clone()
    _, _, _, stats = twin.compute_gradients(*micro[rank])     # this rank's batch statistics feed its EMA pushes
    twin.flat_grad.add_(other)
    twin.apply_gradients()
    twin.apply_stat_updates(stats)
    torch.cuda.synchronize(device)
    sv, tv = step_model.variables, twin.variables
    for name, a, b in (('parameters', sv.flat, tv.flat), ('adam_m', sv.adam_m, tv.adam_m), ('adam_v', sv.adam_v, tv.adam_v),
                       ('normaliser state', sv.state, tv.state)):
      if not torch.equal(a, b):
        raise AssertionError('rank %d: %s after the overlapped step differ from the sequential-sum step (max |diff| %g)'
                             % (rank, name, float((a - b).abs().max())))
    out['equal_to_sequential_sum_step'] = True
  return out


def _main():
  import os
  import sys
  if '--selfcheck' not in sys.argv:
    raise SystemExit('usage: torchrun ... -m twingan_b200.ddp --selfcheck')
  local = int(os.environ.get('LOCAL_RANK', '0'))
  torch.cuda.set_device(local)
  dev = torch.device('cuda', local)
  dist.init_process_group('nccl', device_id=dev)
  try:
    out = selfcheck(dev)
    for norm in ('batch_renorm',):
      out[norm] = selfcheck(dev, norm=norm)
    for graphed in (False, True):
      out['equalized_learning_rate' + (' graphed' if graphed else '')] = selfcheck(
          dev, extra_flags={'equalized_learning_rate': True}, graphed=graphed)
    if dist.get_rank() == 0:
      print('ddp selfcheck ok', out, flush=True)
  finally:
    dist.destroy_process_group()


if __name__ == '__main__':
  _main()
