"""Host logic of the progressive stage scheduler (twingan_b200/pggan_runner.py; reference pggan_runner.py:82-160,
twingan.py:834-835).  No kernels run here: variables live on the CPU and only the plan / checkpoint / warm-start code
is exercised."""
import os

import pytest
import torch

from twingan_b200 import pggan_runner as R
from twingan_b200 import twingan


def test_stage_plan_matches_reference_loop():
  # pggan_runner.py:91-115 with the default flag values
  plan = R.stage_plan(4, 256, 300000, R.DEFAULT_HW_TO_BATCH_SIZE)
  assert [s.name for s in plan] == ['4', '4to8', '8', '8to16', '16', '16to32', '32', '32to64', '64', '64to128', '128',
                                    '128to256', '256']
  assert plan[0] == R.Stage(4, False, 16, 300000 // 16, '4')
  by = {s.name: s for s in plan}
  assert by['64to128'].batch_size == 12 and by['64to128'].max_number_of_steps == 25000 and by['64to128'].is_growing
  assert by['64to128'].ignore_missing_vars and not by['128'].ignore_missing_vars          # :143
  assert by['256'].max_number_of_steps == R.LAST_STAGE_STEPS and by['128to256'].max_number_of_steps == 25000   # :103-104
  # the flag is a dict literal in the reference (ast.literal_eval, :92)
  plan2 = R.stage_plan(8, 32, 1000, '{8: 8, 16: 4, 32: 3}')
  assert [(s.name, s.batch_size, s.max_number_of_steps) for s in plan2] == \
      [('8', 8, 125), ('8to16', 4, 250), ('16', 4, 250), ('16to32', 3, 333), ('32', 3, R.LAST_STAGE_STEPS)]
  with pytest.raises(KeyError):
    R.stage_plan(4, 16, 100, {4: 1, 8: 1})
  with pytest.raises(ValueError):
    R.stage_plan(6, 16)


def test_alpha_grow_schedule():
  # twingan.py:834-835
  assert R.alpha_grow(0, 1000) == 0.0
  assert R.alpha_grow(250, 1000) == 0.25
  assert R.alpha_grow(1000, 1000) == 1.0
  assert R.alpha_grow(600, 1000, grow_start_number_of_steps=200) == 0.5


def _model(hw, growing, seed):
  f = twingan.Flags(train_image_size=hw, is_growing=growing, pggan_max_num_channels=16,
                    generator_norm_type='batch_renorm')
  return twingan.GanModel(f, device='cpu', seed=seed)


def test_checkpoint_round_trip_and_growing_hand_off(tmp_path):
  m8 = _model(8, False, seed=1)
  v8 = m8.variables
  v8.adam_m.normal_(); v8.adam_v.uniform_(); v8.adam_t = 14
  v8.state.uniform_()
  m8.flags.global_step = 7
  d = str(tmp_path / '8')
  assert R.latest_checkpoint(d) is None
  R.save_checkpoint(m8, d, 3)
  path = R.save_checkpoint(m8, d, 7)
  assert R.latest_checkpoint(d) == (path, 7) and os.path.basename(path) == 'model.ckpt-7.pt'
  ck = R.load_checkpoint(path)

  # resume of the same stage: everything restored bit-exactly
  m8b = _model(8, False, seed=2)
  assert R.warm_start(m8b, ck, ignore_missing_vars=False, restore_step=True) == []
  for n, (o, shp) in v8.offsets.items():       # (alignment padding between variables is not part of a checkpoint)
    k = int(torch.tensor(shp).prod())
    for a, b in ((m8b.variables.flat, v8.flat), (m8b.variables.adam_m, v8.adam_m), (m8b.variables.adam_v, v8.adam_v)):
      assert torch.equal(a[o:o + k], b[o:o + k]), n
  for key, (o, C) in v8.state_offsets.items():
    assert torch.equal(m8b.variables.state[o:o + 4 * C + 2], v8.state[o:o + 4 * C + 2]), key
  assert m8b.variables.adam_t == 14 and m8b.flags.global_step == 7

  # 8 -> 8to16: the growing model has variables the 8x8 checkpoint lacks (new blocks, from_rgb/to_rgb at 16)
  m16g = _model(16, True, seed=3)
  fresh = m16g.variables.to_dict()
  with pytest.raises(KeyError):
    R.warm_start(m16g, ck, ignore_missing_vars=False)
  missing = R.warm_start(m16g, ck, ignore_missing_vars=True)
  assert missing and all('16x16' in n for n in missing)
  now = m16g.variables.to_dict()
  for n in now:
    if n in ck['variables']:
      assert torch.equal(now[n], ck['variables'][n]), n       # carried over by name
    else:
      assert torch.equal(now[n], fresh[n]), n                 # kept its initialisation
  assert m16g.flags.global_step == 0                            # a new stage counts its own steps

  # 8to16 -> 16: the stable model's variables are a subset of the growing stage's
  R.save_checkpoint(m16g, str(tmp_path / '8to16'), 5)
  ck2 = R.load_checkpoint(R.latest_checkpoint(str(tmp_path / '8to16'))[0])
  m16 = _model(16, False, seed=4)
  assert R.warm_start(m16, ck2, ignore_missing_vars=False) == []
  assert set(m16.variables.offsets) < set(m16g.variables.offsets)

  # same name, different shape is an error, never a silent skip
  bad = dict(ck2)
  bad['variables'] = dict(ck2['variables'])
  n0 = next(iter(m16.variables.offsets))
  bad['variables'][n0] = torch.zeros(3)
  with pytest.raises(ValueError):
    R.warm_start(m16, bad, ignore_missing_vars=True)


class _AlternatingStub(object):
  """The part of GanModel that run_stage(alternating=True) drives: flags, device and a train_step_alternating that records
  what each run was given and keeps the model's counters (turn by n_critic_counter; global_step + 1 on generator turns)."""

  def __init__(self, n_critic_counter=0, global_step=0):
    self.flags = twingan.Flags(train_image_size=8, is_growing=True, global_step=global_step)
    self.device = torch.device('cpu')
    self.n_critic_counter = n_critic_counter
    self.runs = []                       # (batch index, global_step, alpha, turn) of each run

  def train_step_alternating(self, sources, targets, rand):
    turn = 'G' if self.n_critic_counter % self.flags.n_critic == 0 else 'D'
    self.runs.append((int(sources[0, 0, 0, 0]), self.flags.global_step, self.flags.alpha_grow, turn))
    self.n_critic_counter += 1
    if turn == 'G':
      self.flags.global_step += 1
    return torch.zeros(()), torch.zeros(()), turn


def test_alternating_stage_counts_generator_turns_as_global_steps(monkeypatch):
  """image_generation.py:622-651: n_critic_counter counts runs and picks the turn; global_step advances on generator turns
  only, and it is what alpha (twingan.py:834-835), slim's number_of_steps stop (model/model_inheritor.py:1116-1123),
  save_every and the checkpoint names count.  With n_critic = 2 a 4-step growing stage is 7 runs: G D G D G D G."""
  saved = []
  monkeypatch.setattr(R, 'save_checkpoint', lambda m, d, step: saved.append((step, m.flags.global_step, m.n_critic_counter)))
  batch_fn = lambda st, i: (torch.full((st.batch_size, st.hw, st.hw, 3), float(i)),) * 2
  stage = R.Stage(8, True, 2, 4, '4to8')
  m = _AlternatingStub()
  log = []
  assert R.run_stage(m, stage, batch_fn, 'unused', save_every=2, alternating=True, log_fn=lambda s, l: log.append(s)) == 4
  assert [r[0] for r in m.runs] == list(range(7))                    # batch_fn gets the run index
  assert [r[3] for r in m.runs] == ['G', 'D'] * 3 + ['G']
  assert [r[1] for r in m.runs] == [0, 1, 1, 2, 2, 3, 3]              # the global_step each run computes with
  assert [r[2] for r in m.runs] == [g / 4.0 for g in (0, 1, 1, 2, 2, 3, 3)]
  assert log == [1, 1, 2, 2, 3, 3, 4]
  assert m.flags.global_step == 4 and m.n_critic_counter == 7
  assert saved == [(2, 2, 3), (4, 4, 7), (4, 4, 7)]                  # save_every, then the stage's last checkpoint

  # resumed after an odd number of runs (checkpoint of global step 2 at run 3): the next run is a discriminator turn on
  # batch 3, and the stage stops at the same run as the uninterrupted one
  saved.clear()
  r = _AlternatingStub(n_critic_counter=3, global_step=2)
  assert R.run_stage(r, stage, batch_fn, 'unused', start_step=2, save_every=2, alternating=True) == 4
  assert r.runs == m.runs[3:] and saved == [(4, 4, 7), (4, 4, 7)]
  assert R.runs_to_reach(3, 2, 2) == 4 and R.runs_to_reach(0, 2, 4) == 7 and R.runs_to_reach(5, 3, 0) == 0


def test_checkpoint_carries_the_alternating_counter(tmp_path):
  """n_critic_counter is a variable of the reference's checkpoint (image_generation.py:622): a resume restores it, a new
  stage starts it at 0 like global_step."""
  m = _model(8, False, seed=1)
  m.n_critic_counter, m.flags.global_step = 5, 2
  ck = R.load_checkpoint(R.save_checkpoint(m, str(tmp_path), 2))
  assert ck['n_critic_counter'] == 5
  resumed = _model(8, False, seed=2)
  R.warm_start(resumed, ck, restore_step=True)
  assert resumed.n_critic_counter == 5 and resumed.flags.global_step == 2
  fresh = _model(8, False, seed=3)
  R.warm_start(fresh, ck, restore_optimizer=False)
  assert fresh.n_critic_counter == 0 and fresh.flags.global_step == 0
