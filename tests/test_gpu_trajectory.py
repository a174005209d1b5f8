"""Every step of a training run held to the fp64 oracle, not just a first step from a freshly loaded state.

A run spends all but its first step on state the previous step left behind: the split-bf16 weight planes rebuilt after
each Adam apply, the normaliser snapshot that batch renorm's r / d read, the device step counters behind Adam's lr_t and
the renorm clipping, Adam's m and v, and across stages the variables, slots and counters a hand-off or a resume carries.
Each step here runs the real entry point (train_step, train_step_alternating, or pggan_runner's loop around them) and is
compared with the oracle evaluated from exactly the state the device started that step from (tests/parity.check_step),
so errors do not compound and anything carried wrongly shows on the step that reads it.  The reference's counters (Adam
t, global_step, n_critic_counter) are kept here by the reference's rules; global_step and alpha come from them, never
from the model.  Learning rate 1e-3: a step moves every weight by ~5 % of its N(0, 0.02) size, far outside the 1e-3
forward tolerance, so a step that ran on stale planes or state cannot pass."""
import os
from dataclasses import replace

import pytest
import torch

from oracle import twingan_oracle as O
from tests.parity import REL_TOL, RefCounters, check_step, entry_state, oracle_config, rel_err, seeded_model

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
LR = 1e-3


def _assert_ok(res, what):
  top = sorted(((k, e) for k, e in res['details'].items() if k not in res['bad']), key=lambda kv: -kv[1])[:3]
  print('[trajectory] %s: kink flips %d/%d, worst %.3e, largest %s' % (what, res['kink_flips'][0], res['kink_flips'][1],
                                                                     res['worst'], top))
  assert res['ok'], '%s: worst=%g bad=%s' % (what, res['worst'], dict(list(res['bad'].items())[:6]))


def _device_batch(cfg, batch, seed):
  src, tgt, rand = O.make_inputs(cfg, batch, seed=seed)
  f32 = lambda t: t.to(DEV, torch.float32).contiguous()
  return f32(src), f32(tgt), {k: f32(v) for k, v in rand.items()}


def _alpha(cfg, global_step, stage_steps):
  """twingan.py:834-835 for a growing stage of `stage_steps` steps; 0 for a stable one."""
  from twingan_b200 import pggan_runner as R
  return R.alpha_grow(global_step, stage_steps) if cfg.is_growing else 0.0


def _set_precision(prec):
  from twingan_b200 import ops
  ops.set_precision(prec)


@pytest.fixture
def precision():
  """Tests that change the conv precision leave the default (tensor cores) behind."""
  yield _set_precision
  _set_precision(1)


# Split-bf16 tensor-core convs (prec 1) on the discriminator's 32-channel layers: after a few steps at lr 1e-3 the weight
# gradients of the layers before the fc layer -- sums over few pixels whose terms cancel -- and the fc bias of a fresh
# model (mean D(real) against mean D(fake) at D ~ 0) carry up to 3.9e-3 of their largest element (measured on an H100:
# the 16 batch_renorm and 32 no-normaliser cases below, steps 2 to 4; the same steps with exact-fp32 convs stay below
# 1.1e-4, so this is the split-bf16 product error amplified, as at the 256x256 stage of test_gpu_step).  Forward values,
# losses, the generator set's gradients, Adam, normaliser state and counters keep the 1e-3 bar.
TC_LOOSE = {'grad/discriminator': 5e-3}


def _planes_in_use(model, prec):
  if prec == 1:
    assert model.variables.weight_table.rows > 0, 'no conv of this model reads the weight-plane table'


# -- mode B: GanModel.train_step, 4 steps ------------------------------------------------------------------------------
MODE_B = [
    # label, hw, batch, max channels, norm, growing, prec, first global step, stage steps (alpha), extra flags,
    # weight scale, grad floor                     (configurations of test_gpu_step.CASES / F4_CASES)
    ('8 growing instance_norm', 8, 4, 32, 'instance_norm', True, 1, 1, 6, {}, 1.0, 0.0),
    ('16 growing batch_renorm across 10000', 16, 3, 32, 'batch_renorm', True, 1, 9999, 20000, {}, 1.0, 0.0),
    ('16 batch_norm exact fp32', 16, 4, 16, 'batch_norm', False, 0, 0, 0, {}, 1.0, 0.0),
    ('32 growing no normaliser', 32, 2, 32, 'none', True, 1, 1, 6, {}, 1.0, 0.0),
    ('8 growing 3 pairs 256 channels', 8, 3, 256, 'instance_norm', True, 1, 1, 6, {}, 1.0, 0.0),
    ('8 equalized lr res batch_renorm exact fp32', 8, 3, 32, 'batch_renorm', False, 0, 15000, 0,
     dict(use_res_block=True, equalized_learning_rate=True), 50.0, 1e-3),
]
STEPS = 4


@pytest.mark.parametrize('label,hw,batch,mc,norm,growing,prec,gs0,stage_steps,extra,wscale,floor', MODE_B,
                         ids=[c[0] for c in MODE_B])
def test_train_steps_follow_the_oracle(built_lib, precision, label, hw, batch, mc, norm, growing, prec, gs0, stage_steps,
                                       extra, wscale, floor):
  """Four mode-B steps from seeded parameters and normaliser state; alpha follows global_step every step as run_stage sets
  it.  The batch_renorm case starts at global step 9999, so the clipping changes between steps 2 and 3
  (nets/pggan_utils.py:44-47: gs > 10000).  Then inference on the trained weights and moving statistics."""
  precision(prec)
  ref = RefCounters(global_step=gs0)
  base = oracle_config(hw, growing, _alpha(O.Config(is_growing=growing), gs0, stage_steps), mc, norm, global_step=gs0,
                       learning_rate=LR, **extra)
  model, _ = seeded_model(base, batch, seed=0, weight_scale=wscale)
  _planes_in_use(model, prec)
  for i in range(STEPS):
    cfg = replace(base, global_step=ref.global_step, alpha_grow=_alpha(base, ref.global_step, stage_steps))
    model.flags.alpha_grow = cfg.alpha_grow
    s, t, r = _device_batch(cfg, batch, seed=10 + i)
    res = check_step(model, lambda: model.train_step(s, t, r), cfg, s, t, r, ref, grad_floor=floor,
                     loose=TC_LOOSE if prec == 1 else None)
    _assert_ok(res, '%s, step %d' % (label, i + 1))
  assert ref.adam_t == 2 * STEPS and ref.global_step == gs0 + STEPS
  st = entry_state(model, norm == 'batch_renorm')
  src, _, _ = O.make_inputs(cfg, batch, seed=99)
  want = O.inference(cfg, st['params'], st['state'], src)
  got = model.infer(src.to(DEV, torch.float32))
  assert rel_err(got, want) < REL_TOL, rel_err(got, want)


# -- mode A: train_step_alternating, directly and through run_stage ------------------------------------------------------
MODE_A = [
    # label, hw, batch, max channels, norm, growing, first global step, stage steps
    ('8 growing instance_norm', 8, 4, 32, 'instance_norm', True, 0, 3),
    ('16 batch_renorm below 10000', 16, 3, 32, 'batch_renorm', False, 9999, 10002),
]


@pytest.mark.parametrize('label,hw,batch,mc,norm,growing,gs0,stage_steps', MODE_A, ids=[c[0] for c in MODE_A])
def test_alternating_runs_follow_the_oracle(built_lib, label, hw, batch, mc, norm, growing, gs0, stage_steps):
  """Six mode-A runs, G D G D G D (image_generation.py:622-651): one apply per run at the shared Adam time, the EMA pushes on
  every run, global_step (and with it alpha and the renorm clipping) advancing on generator turns only."""
  ref = RefCounters(global_step=gs0)
  base = oracle_config(hw, growing, _alpha(O.Config(is_growing=growing), gs0, stage_steps), mc, norm, global_step=gs0,
                       learning_rate=LR)
  model, _ = seeded_model(base, batch, seed=1)
  _planes_in_use(model, 1)
  turns = []
  for i in range(6):
    cfg = replace(base, global_step=ref.global_step, alpha_grow=_alpha(base, ref.global_step, stage_steps))
    model.flags.alpha_grow = cfg.alpha_grow
    s, t, r = _device_batch(cfg, batch, seed=20 + i)
    res = check_step(model, lambda: model.train_step_alternating(s, t, r), cfg, s, t, r, ref, alternating=True,
                     loose=TC_LOOSE)
    _assert_ok(res, '%s, run %d' % (label, i + 1))
    turns.append(res['turn'])
  assert turns == ['G', 'D'] * 3 and ref.global_step == gs0 + 3 and ref.adam_t == 6


def _patch(monkeypatch, name, on_step):
  """Replace GanModel.<name> at class level: on_step(model, run, sources, targets, rand) gets a callable that runs the real
  entry point and returns what the caller receives."""
  from twingan_b200 import twingan
  orig = getattr(twingan.GanModel, name)

  def wrapper(self, sources, targets, rand):
    return on_step(self, lambda: orig(self, sources, targets, rand), sources, targets, rand)
  monkeypatch.setattr(twingan.GanModel, name, wrapper)


def _index_batches(cfg, batch):
  """batch_fn of the stage runner: batch k of a stage is a function of (stage, k) alone."""
  def batch_fn(stage, k):
    s, t, _ = _device_batch(replace(cfg, hw=stage.hw), stage.batch_size, seed=1000 * stage.hw + k)
    return s, t
  return batch_fn


@pytest.mark.parametrize('label,hw,batch,mc,norm,growing,gs0,stage_steps', MODE_A, ids=[c[0] for c in MODE_A])
def test_alternating_stage_follows_the_oracle(built_lib, monkeypatch, label, hw, batch, mc, norm, growing, gs0, stage_steps):
  """run_stage(alternating=True) from global step gs0 to the stage's step count: five runs G D G D G, each held to the
  oracle at the reference's global_step -- alpha, the renorm clipping and the stop count generator turns, not runs."""
  from twingan_b200 import pggan_runner as R
  ref = RefCounters(global_step=gs0)
  base = oracle_config(hw, growing, 0.0, mc, norm, global_step=gs0, learning_rate=LR)
  model, _ = seeded_model(base, batch, seed=2)
  turns = []

  def on_step(m, run, s, t, r):
    cfg = replace(base, global_step=ref.global_step, alpha_grow=_alpha(base, ref.global_step, stage_steps))
    res = check_step(m, run, cfg, s, t, r, ref, alternating=True, loose=TC_LOOSE)
    _assert_ok(res, '%s, run %d' % (label, len(turns) + 1))
    turns.append(res['turn'])
    return res['result']
  _patch(monkeypatch, 'train_step_alternating', on_step)
  stage = R.Stage(hw, growing, batch, stage_steps, label)
  reached = R.run_stage(model, stage, _index_batches(base, batch), None, start_step=gs0, alternating=True,
                        dragan_generator=torch.Generator(device=DEV).manual_seed(4))
  assert reached == stage_steps and ref.global_step == stage_steps
  assert turns == ['G', 'D', 'G', 'D', 'G'], turns


# -- stage hand-off: pggan_runner.run over 4 -> 4to8 -> 8 ---------------------------------------------------------------
def test_stage_hand_off_follows_the_oracle(built_lib, monkeypatch, tmp_path):
  """Three mode-B steps per stage through pggan_runner.run, every step held to the oracle.  At the first step of each stage:
  variables the previous stage had are its last checkpoint's, bit for bit; new ones are a fresh model's initialisation;
  Adam's slots are zero and its time, global_step and the device counters 0 (a new train_dir; init_fn restores model
  variables only, model/model_inheritor.py:610-644); the normaliser state is carried over."""
  from twingan_b200 import pggan_runner as R
  from twingan_b200 import twingan
  base_flags = twingan.Flags(pggan_max_num_channels=32, generator_norm_type='batch_renorm', learning_rate=LR)
  plan = R.stage_plan(4, 8, 12, {4: 4, 8: 4})
  assert [(s.name, s.max_number_of_steps) for s in plan][:2] == [('4', 3), ('4to8', 3)]
  seen, models, refs = [], [], []

  def on_step(m, run, s, t, r):
    if not models or m is not models[-1]:     # the first step of a stage
      stage = plan[len(seen)]
      _check_hand_off(m, stage, plan[len(seen) - 1] if seen else None, tmp_path, base_flags)
      seen.append(stage)
      models.append(m)
      refs.append(RefCounters())
    stage, ref = seen[-1], refs[-1]
    cfg = oracle_config(stage.hw, stage.is_growing, 0.0, 32, 'batch_renorm', learning_rate=LR)
    cfg = replace(cfg, global_step=ref.global_step, alpha_grow=_alpha(cfg, ref.global_step, stage.max_number_of_steps))
    res = check_step(m, run, cfg, s, t, r, ref, loose=TC_LOOSE)
    _assert_ok(res, 'stage %s, step %d' % (stage.name, ref.global_step))
    return res['result']
  _patch(monkeypatch, 'train_step', on_step)
  model = R.run(base_flags, str(tmp_path), _index_batches(O.Config(), 4), stages=plan, max_steps_per_stage=3,
                use_graph=False, dragan_generator=torch.Generator(device=DEV).manual_seed(6))
  assert [s.name for s in seen] == ['4', '4to8', '8'] and all(ref.global_step == 3 for ref in refs)
  assert model.flags.train_image_size == 8


def _check_hand_off(model, stage, prev, base_dir, base_flags):
  from twingan_b200 import pggan_runner as R
  from twingan_b200 import twingan
  v = model.variables
  now = {n: t.cpu() for n, t in v.to_dict().items()}
  flags = replace(base_flags, train_image_size=stage.hw, is_growing=stage.is_growing)
  fresh = twingan.GanModel(flags, device='cpu').variables.to_dict()    # run()'s seed; the same values on any device
  ck = R.load_checkpoint(R.latest_checkpoint(os.path.join(str(base_dir), prev.name))[0]) if prev else {'variables': {}}
  for n, t in now.items():
    want = ck['variables'][n] if n in ck['variables'] else fresh[n]
    assert torch.equal(t, want), '%s: %s at the first step of stage %s' % (
        n, 'not the previous checkpoint' if n in ck['variables'] else 'not the initialisation', stage.name)
  if prev is not None:
    assert set(ck['variables']) & set(now), stage.name
    state = {k: t.cpu() for k, t in v.state_to_dict().items()}
    for k, t in ck['norm_state'].items():
      if k in state:
        assert torch.equal(state[k], t), (stage.name, k)
  assert float(v.adam_m.abs().max()) == 0.0 and float(v.adam_v.abs().max()) == 0.0, stage.name
  assert v.adam_t == 0 and model.flags.global_step == 0 and model._counters.tolist() == [0, 0], stage.name


# -- resume: an interrupted and resumed run equals the uninterrupted one bit for bit ------------------------------------
def _record(model, out):
  v = model.variables
  return {'generator_loss': out[0].clone(), 'discriminator_loss': out[1].clone(), 'variables': v.flat.clone(),
          'adam_m': v.adam_m.clone(), 'adam_v': v.adam_v.clone(), 'state': v.state.clone(),
          'counters': model._counters.clone(), 'n_critic_counter': torch.tensor(model.n_critic_counter),
          'host_counters': torch.tensor([v.adam_t, model.flags.global_step])}


RESUME = [
    # label, entry points recorded, run() keywords, steps before the interruption, steps in all, DRAGAN draws before it
    ('mode B eager', ('train_step',), dict(use_graph=False), 2, 5, 2),
    ('mode B graph replay', ('train_step', 'train_step_graphed'), dict(use_graph=True), 2, 5, 2),
    ('mode A after 3 runs', ('train_step_alternating',), dict(alternating=True), 2, 4, 3),
]


@pytest.mark.parametrize('label,entries,kw,cut,steps,draws', RESUME, ids=[c[0] for c in RESUME])
def test_resumed_run_equals_the_uninterrupted_run(built_lib, monkeypatch, tmp_path, label, entries, kw, cut, steps, draws):
  """pggan_runner.run for `steps` steps, against run for `cut` steps, a checkpoint, a fresh model that resumes from it
  through run, and the rest: parameters, Adam slots, normaliser state, counters and losses after every step (every run in
  mode A, which is cut after an odd number of runs, so the resumed model starts on a discriminator turn).  The batches are
  a function of their index and the resumed run's DRAGAN generator is advanced by the draws of the runs it skips."""
  from twingan_b200 import pggan_runner as R
  from twingan_b200 import twingan
  records = []

  def on_step(m, run, s, t, r):
    out = run()
    records.append(_record(m, out))
    return out
  for e in entries:
    _patch(monkeypatch, e, on_step)
  stage = R.Stage(8, False, 4, 6, '8') if not kw.get('alternating') else R.Stage(8, True, 4, 4, '4to8')
  base = twingan.Flags(pggan_max_num_channels=32, generator_norm_type='batch_renorm', learning_rate=LR)
  batch_fn = _index_batches(O.Config(), 4)
  gen = lambda: torch.Generator(device=DEV).manual_seed(8)

  R.run(base, str(tmp_path / 'a'), batch_fn, stages=[stage], max_steps_per_stage=steps, dragan_generator=gen(), **kw)
  whole, records[:] = list(records), []
  R.run(base, str(tmp_path / 'b'), batch_fn, stages=[stage], max_steps_per_stage=cut, dragan_generator=gen(), **kw)
  assert R.latest_checkpoint(str(tmp_path / 'b' / stage.name))[1] == cut
  first = len(records)
  resumed_gen = gen()
  for _ in range(draws):
    twingan.make_dragan_rand(stage.batch_size, stage.hw, DEV, resumed_gen)
  R.run(base, str(tmp_path / 'b'), batch_fn, stages=[stage], max_steps_per_stage=steps, dragan_generator=resumed_gen, **kw)
  assert first == draws and len(records) == len(whole), (first, len(records), len(whole))
  for i, (a, b) in enumerate(zip(whole, records)):
    for k in a:
      if not torch.equal(a[k], b[k]):
        d = (a[k].double() - b[k].double()).abs()
        raise AssertionError('%s, %s %d: %s of the resumed run differs from the uninterrupted run at %d elements '
                             '(max |diff| %g)' % (label, 'run' if kw.get('alternating') else 'step', i + 1, k,
                                                  int((d != 0).sum()), float(d.max())))
  assert int(whole[-1]['host_counters'][1]) == steps
