"""Stage scheduler on the device: 4 -> 4to8 -> 8 for a few steps each, with checkpoint hand-off (SURVEY 8f-1)."""
import math
import os

import pytest
import torch

pytestmark = pytest.mark.gpu


def test_progressive_stages_train_and_hand_off(tmp_path):
  from twingan_b200 import pggan_runner as R
  from twingan_b200 import twingan
  base = twingan.Flags(pggan_max_num_channels=32, generator_norm_type='batch_renorm', learning_rate=1e-3)
  plan = R.stage_plan(4, 8, 16, {4: 4, 8: 4})          # 4 steps per stage
  assert [s.name for s in plan] == ['4', '4to8', '8']
  gen = torch.Generator(device='cuda').manual_seed(5)
  alphas, log = [], []

  def batch_fn(stage, step):
    shape = (stage.batch_size, stage.hw, stage.hw, 3)
    return torch.rand(shape, device='cuda', generator=gen), torch.rand(shape, device='cuda', generator=gen)

  def log_fn(step, losses):
    log.append((step, losses))

  model = R.run(base, str(tmp_path), batch_fn, stages=plan, max_steps_per_stage=4, log_fn=log_fn)
  assert len(log) == 12 and all(math.isfinite(l['generator_loss']) and math.isfinite(l['discriminator_loss']) for _, l in log)
  for name in ('4', '4to8', '8'):
    assert R.latest_checkpoint(os.path.join(str(tmp_path), name))[1] == 4
  assert model.flags.train_image_size == 8 and not model.flags.is_growing
  # Adam time: two applies per step; every stage starts its own optimiser like the reference (init_fn restores model
  # variables only, model/model_inheritor.py:610-644), so the last stage has seen 4 steps
  assert model.variables.adam_t == 2 * 4

  # hand-off: the 4to8 stage started from the 4x4 weights and moved them; the 8 stage started from 4to8's
  c4 = R.load_checkpoint(R.latest_checkpoint(os.path.join(str(tmp_path), '4'))[0])
  c48 = R.load_checkpoint(R.latest_checkpoint(os.path.join(str(tmp_path), '4to8'))[0])
  c8 = R.load_checkpoint(R.latest_checkpoint(os.path.join(str(tmp_path), '8'))[0])
  shared = [n for n in c4['variables'] if n in c48['variables'] and n.endswith('/weights')]
  assert shared
  for n in shared:
    d = (c48['variables'][n] - c4['variables'][n]).abs().max().item()
    assert 0 < d < 0.05, (n, d)                      # 4 Adam steps of lr 1e-3 from the carried-over value
  assert set(c8['variables']) < set(c48['variables'])

  # re-running the plan skips finished stages (pggan_runner.py:117-121) and returns without training
  log.clear()
  assert R.run(base, str(tmp_path), batch_fn, stages=plan, max_steps_per_stage=4, log_fn=log_fn) is None
  assert log == []

  # resume: extend the last stage by two steps from its own checkpoint
  m2 = R.run(base, str(tmp_path), batch_fn, stages=plan[-1:], max_steps_per_stage=6, log_fn=log_fn, use_graph=False)
  assert [s for s, _ in log] == [5, 6] and m2.flags.global_step == 6 and m2.variables.adam_t == 2 * 6


def test_device_prefetcher_overlaps_and_delivers_exact_batches():
  """prefetch.DevicePrefetcher: batch k+1 is copied on a side stream while the main stream is busy with batch k; every
  delivered batch equals its pinned host source bit for bit, staging slots are never overwritten early."""
  from twingan_b200.prefetch import DevicePrefetcher, HostPrefetcher
  g = torch.Generator().manual_seed(3)
  host = [(torch.rand((4, 64, 64, 3), generator=g).pin_memory(), {'alpha': torch.rand((4, 1, 1, 1), generator=g).pin_memory()})
          for _ in range(7)]
  pf = DevicePrefetcher(HostPrefetcher(iter(host), capacity=2), 'cuda', depth=2)
  busy = torch.rand((2048, 2048), device='cuda')
  outs = []
  for s, d in pf:
    for _ in range(20):                     # keep the main stream busy so that the next copy really overlaps
      busy = busy @ busy * 1e-3
    outs.append((s.clone(), d['alpha'].clone()))   # reads the slot on the main stream
    pf.release()
  torch.cuda.synchronize()
  assert len(outs) == 7 and pf.h2d_bytes == sum(a.numel() * 4 + b['alpha'].numel() * 4 for a, b in host)
  for (s, a), (hs, hd) in zip(outs, host):
    assert torch.equal(s.cpu(), hs) and torch.equal(a.cpu(), hd['alpha'])


def test_stage_runs_from_host_batches_through_the_prefetcher(tmp_path):
  from twingan_b200 import pggan_runner as R
  from twingan_b200 import twingan
  base = twingan.Flags(pggan_max_num_channels=16, train_image_size=8, learning_rate=1e-3)
  stage = R.Stage(8, False, 4, 5, '8')
  gen = torch.Generator().manual_seed(9)
  calls = []

  def batch_fn(st, step):                   # host tensors: the prefetcher pins and copies them
    calls.append(step)
    shape = (st.batch_size, st.hw, st.hw, 3)
    return torch.rand(shape, generator=gen), torch.rand(shape, generator=gen)

  model = twingan.GanModel(base, device='cuda')
  log = []
  reached = R.run_stage(model, stage, batch_fn, None, prefetch=2, log_fn=lambda s, l: log.append((s, l)))
  assert reached == 5 and calls == [0, 1, 2, 3, 4] and len(log) == 5
  assert all(math.isfinite(l['generator_loss']) for _, l in log)


def test_pipelined_inference_equals_plain_inference():
  """twingan.infer_batches (host batch in, pinned host result out, copies overlapped with compute on side streams) returns
  what GanModel.infer returns for every batch, in order, bit for bit (no reduction of inference depends on launch
  timing)."""
  from twingan_b200 import twingan
  model = twingan.GanModel(twingan.Flags(train_image_size=32, pggan_max_num_channels=32), device='cuda')
  g = torch.Generator().manual_seed(11)
  host = [torch.rand((3, 32, 32, 3), generator=g).pin_memory() for _ in range(5)]
  want = [model.infer(h.cuda()).cpu() for h in host]
  again = [model.infer(h.cuda()).cpu() for h in host]
  assert all(torch.equal(a, b) for a, b in zip(want, again))
  got = []
  for out, ev in twingan.infer_batches(model, iter(host)):
    ev.synchronize()
    got.append(out.clone())
  assert len(got) == 5
  for i, (a, b) in enumerate(zip(got, want)):
    assert torch.equal(a, b), (i, float((a - b).abs().max()))
  # and the batches did not get mixed up: neighbouring results differ by O(1)
  assert float((got[0] - got[1]).abs().max()) > 1e-2
  # a persistent pipeline reuses its staging / result slots across runs; with use_graph the batch is a CUDA-graph replay
  for use_graph in (False, True):
    pipe = twingan.InferencePipeline(model, use_graph=use_graph)
    for rnd in range(2):
      outs = []
      for out, ev in pipe.run(iter(host[rnd:rnd + 3])):
        ev.synchronize()
        outs.append(out.clone())
      assert len(outs) == 3
      for a, b in zip(outs, want[rnd:rnd + 3]):
        assert torch.equal(a, b), (use_graph, rnd, float((a - b).abs().max()))
