"""Progressive stage scheduler + checkpoint hand-off -- host-side mirror of pggan_runner.py (SURVEY 8f-1).

The reference trains 4 -> 4to8 -> 8 -> 8to16 -> ... -> max_hw, one `model.main()` per stage, each stage warm-started
from the previous stage's checkpoint with `ignore_missing_vars = is_growing` (pggan_runner.py:91-160).  The same
loop here drives `twingan.GanModel`:

  * `stage_plan(...)`            the list of stages with the reference's names, batch sizes and step counts
                                 (pggan_runner.py:91-115,137-143)
  * `alpha_grow(...)`            fade-in coefficient from the global step (twingan.py:834-835)
  * `save_checkpoint / load_checkpoint / latest_checkpoint`
                                 `<train_dir>/model.ckpt-<step>.pt` holding the variables under their TF names
                                 (SURVEY 8a.4-11), the normaliser state, both Adam slots, the Adam time and the
                                 step counters (global_step, mode A's n_critic_counter)
  * `warm_start(model, ckpt, ignore_missing_vars)`
                                 restore-by-name; a growing stage adds from_rgb/to_rgb/block variables that the
                                 previous stage does not have (pggan_runner.py:143; model_inheritor init_fn)
  * `run_stage / run`            the training loop; fixed stages replay the captured CUDA graphs, growing stages run
                                 eagerly because alpha changes every step

Nothing here touches the data path: batches come from a `batch_fn(stage, index) -> (sources, targets)` callable, the
index being the step (mode B) or the run (mode A, run_stage).
"""
from __future__ import annotations

import ast
import math
import os
import re
from dataclasses import dataclass, replace
from typing import Callable, Dict, Iterable, List, Optional, Tuple

import torch

# pggan_runner.py:52-57 (generic default) and the value its help text recommends for TwinGAN
DEFAULT_HW_TO_BATCH_SIZE = {4: 16, 8: 16, 16: 16, 32: 16, 64: 12, 128: 12, 256: 12, 512: 6}
TWINGAN_HW_TO_BATCH_SIZE = {4: 8, 8: 8, 16: 8, 32: 8, 64: 8, 128: 4, 256: 3, 512: 2}
LAST_STAGE_STEPS = 10000000            # "train indefinitely for the last stage", pggan_runner.py:103-104
_CKPT_RE = re.compile(r'model\.ckpt-(\d+)\.pt$')


@dataclass(frozen=True)
class Stage:
  hw: int
  is_growing: bool
  batch_size: int
  max_number_of_steps: int
  name: str                     # sub-directory of train_dir: '8to16' or '16' (pggan_runner.py:106-109)

  @property
  def ignore_missing_vars(self) -> bool:   # pggan_runner.py:143
    return self.is_growing


def parse_hw_to_batch_size(expr) -> Dict[int, int]:
  """The flag is a Python dict literal (pggan_runner.py:92)."""
  if isinstance(expr, dict):
    return {int(k): int(v) for k, v in expr.items()}
  table = ast.literal_eval(expr)
  if not isinstance(table, dict):
    raise ValueError('hw_to_batch_size must be a dict literal, got %r' % (expr,))
  return {int(k): int(v) for k, v in table.items()}


def stage_plan(start_hw: int = 4, max_hw: int = 256, num_images_per_resolution: int = 300000,
               hw_to_batch_size=None) -> List[Stage]:
  """pggan_runner.py:91-115: resolutions are the powers of two from start_hw to max_hw; every resolution but the first
  has a growing stage followed by a stable stage; each runs num_images_per_resolution / batch_size steps except the
  final stable stage, which runs 'indefinitely'."""
  if start_hw < 4 or start_hw & (start_hw - 1) or max_hw & (max_hw - 1) or max_hw < start_hw:
    raise ValueError('start_hw and max_hw must be powers of two with 4 <= start_hw <= max_hw')
  table = parse_hw_to_batch_size(hw_to_batch_size if hw_to_batch_size is not None else DEFAULT_HW_TO_BATCH_SIZE)
  resolutions = [2 ** i for i in range(int(math.log2(start_hw)), int(math.log2(max_hw)) + 1)]
  stages = []
  for res in resolutions:
    if res not in table:
      raise KeyError('hw_to_batch_size has no entry for resolution %d' % res)
    batch = table[res]
    for is_growing in (True, False):
      if is_growing and res == resolutions[0]:
        continue
      steps = int(num_images_per_resolution / batch)
      if res == resolutions[-1] and not is_growing:
        steps = LAST_STAGE_STEPS
      stages.append(Stage(res, is_growing, batch, steps, '%dto%d' % (res // 2, res) if is_growing else '%d' % res))
  return stages


def alpha_grow(global_step: int, max_number_of_steps: int, grow_start_number_of_steps: int = 0) -> float:
  """twingan.py:834-835: (global_step - grow_start) / (max_number_of_steps - grow_start).  The reference does not
  clip; a stage stops at max_number_of_steps so the value stays in [.,1]."""
  return float(global_step - grow_start_number_of_steps) / float(max_number_of_steps - grow_start_number_of_steps)


# -- checkpoints -----------------------------------------------------------------------------------------
def checkpoint_path(train_dir: str, step: int) -> str:
  return os.path.join(train_dir, 'model.ckpt-%d.pt' % step)


def latest_checkpoint(train_dir: Optional[str]) -> Optional[Tuple[str, int]]:
  """(path, step) of the newest checkpoint in train_dir, or None (tf.train.latest_checkpoint + the '.ckpt-' split of
  pggan_runner.py:112-121)."""
  if not train_dir or not os.path.isdir(train_dir):
    return None
  best = None
  for fn in os.listdir(train_dir):
    m = _CKPT_RE.search(fn)
    if m and (best is None or int(m.group(1)) > best[1]):
      best = (os.path.join(train_dir, fn), int(m.group(1)))
  return best


def model_state(model) -> Dict[str, object]:
  """Everything a stage hand-off or resume needs, keyed by the reference's variable names."""
  v = model.variables
  adam_m, adam_v = {}, {}
  for n, (o, s) in v.offsets.items():
    k = int(math.prod(s))
    adam_m[n] = v.adam_m[o:o + k].view(s).detach().cpu().clone()
    adam_v[n] = v.adam_v[o:o + k].view(s).detach().cpu().clone()
  return {
      'variables': {n: t.cpu() for n, t in v.to_dict().items()},
      'norm_state': {n: t.cpu() for n, t in v.state_to_dict().items()},
      'adam_m': adam_m, 'adam_v': adam_v, 'adam_t': int(v.adam_t),
      'global_step': int(model.flags.global_step),
      'n_critic_counter': int(model.n_critic_counter),     # a tf.get_variable of the reference (image_generation.py:622)
      'train_image_size': int(model.flags.train_image_size), 'is_growing': bool(model.flags.is_growing),
  }


def save_checkpoint(model, train_dir: str, step: int) -> str:
  os.makedirs(train_dir, exist_ok=True)
  path = checkpoint_path(train_dir, step)
  tmp = path + '.tmp'
  torch.save(model_state(model), tmp)
  os.replace(tmp, path)
  return path


def load_checkpoint(path: str) -> Dict[str, object]:
  return torch.load(path, map_location='cpu', weights_only=False)


def warm_start(model, ckpt: Dict[str, object], ignore_missing_vars: bool = False, restore_optimizer: bool = True,
               restore_step: bool = False) -> List[str]:
  """Restore by name.  Variables of `model` that the checkpoint lacks keep their fresh initialisation when
  `ignore_missing_vars` (growing stage: new from_rgb / to_rgb / block variables), otherwise raise, like the
  reference's restore (model_inheritor.py init_fn with FLAGS.ignore_missing_vars).  A variable present under the
  same name with a different shape is always an error.  Returns the list of missing variable names."""
  v = model.variables
  src = ckpt['variables']
  missing = [n for n in v.offsets if n not in src]
  if missing and not ignore_missing_vars:
    raise KeyError('checkpoint lacks %d variables (first: %s); set ignore_missing_vars for a growing stage'
                   % (len(missing), missing[0]))
  with torch.no_grad():
    for n, (o, s) in v.offsets.items():
      if n not in src:
        continue
      t = src[n]
      if tuple(t.shape) != tuple(s):
        raise ValueError('variable %s: checkpoint shape %s != model shape %s' % (n, tuple(t.shape), tuple(s)))
      k = int(math.prod(s))
      v.flat[o:o + k].copy_(t.reshape(-1).to(v.device, torch.float32))
      if restore_optimizer and n in ckpt.get('adam_m', {}):
        v.adam_m[o:o + k].copy_(ckpt['adam_m'][n].reshape(-1).to(v.device, torch.float32))
        v.adam_v[o:o + k].copy_(ckpt['adam_v'][n].reshape(-1).to(v.device, torch.float32))
    ns = ckpt.get('norm_state') or {}
    for key, (o, C) in v.state_offsets.items():
      base, dom = key[:-2], key[-2:]
      if base + 'moving_mean' + dom not in ns:
        if not ignore_missing_vars:
          raise KeyError('checkpoint lacks normaliser state %s' % key)
        continue
      rec = v.state[o:o + 4 * C + 2]
      for i, nm in enumerate(('moving_mean', 'moving_variance', 'renorm_mean', 'renorm_stddev')):
        rec[i * C:(i + 1) * C].copy_(ns[base + nm + dom].to(v.device, torch.float32))
      rec[4 * C] = float(ns[base + 'renorm_mean_weight' + dom])
      rec[4 * C + 1] = float(ns[base + 'renorm_stddev_weight' + dom])
    v.state_snapshot.copy_(v.state)
  if restore_optimizer:
    v.adam_t = int(ckpt.get('adam_t', 0))     # one beta-power pair per optimizer (SURVEY 8a.4-5)
  if restore_step:
    model.flags.global_step = int(ckpt.get('global_step', 0))
    model.n_critic_counter = int(ckpt.get('n_critic_counter', 0))
  from . import ops
  ops.invalidate_weight_cache()
  return missing


# -- loading a trained model for inference / evaluation ------------------------------------------------------
_TF_STATE_RE = re.compile(r'^model_checkpoint_path:\s*"([^"]*)"\s*$', re.M)


def step_of(path: str, default: int = 0) -> int:
  """The step a checkpoint's name carries (model.ckpt-<step>[.pt], like the reference's '.ckpt-' split), else `default`."""
  m = re.search(r'-(\d+)(\.pt)?$', path)
  return int(m.group(1)) if m else default


def resolve_model_path(path: str) -> Tuple[str, str]:
  """('pt', file) or ('tf', checkpoint prefix) for a model path given as
    * a model.ckpt-<step>.pt of this runner;
    * a directory holding such files (the newest one);
    * the prefix of a TensorFlow V2 checkpoint of the reference (<prefix>.index exists);
    * a directory holding a TensorFlow `checkpoint` state file (model_checkpoint_path: "...", relative to the directory
      unless absolute: tf.train.get_checkpoint_state, as util_io.get_model_filenames reads it).
  A frozen graph (.pb / .pbtxt) or a metagraph (.meta) is refused: only checkpoints of the variables can be loaded."""
  if path.endswith(('.pb', '.pbtxt', '.meta')):
    raise ValueError('%s: loading a frozen graph or a metagraph is not supported; pass a checkpoint (a model.ckpt-<step>.pt, '
                     'a TensorFlow checkpoint prefix, or a directory holding either)' % path)
  if os.path.isdir(path):
    own = latest_checkpoint(path)
    if own is not None:
      return 'pt', own[0]
    state = os.path.join(path, 'checkpoint')
    if os.path.isfile(state):
      m = _TF_STATE_RE.search(open(state, encoding='utf-8').read())
      if not m:
        raise ValueError('%s has no model_checkpoint_path entry' % state)
      prefix = m.group(1) if os.path.isabs(m.group(1)) else os.path.join(path, m.group(1))
      if not os.path.isfile(prefix + '.index'):
        raise FileNotFoundError('%s names %s, which has no .index file' % (state, prefix))
      return 'tf', prefix
    raise FileNotFoundError('no checkpoint in directory %s (no model.ckpt-<step>.pt, no TensorFlow checkpoint file)' % path)
  if os.path.isfile(path):
    return 'pt', path
  if os.path.isfile(path + '.index'):
    return 'tf', path
  raise FileNotFoundError('no checkpoint at %s (neither a file nor a TensorFlow prefix with a .index file)' % path)


def load_for_inference(path: str, flags, device='cuda'):
  """(twingan.GanModel, step) of the checkpoint `path` names (any form of resolve_model_path), weights and normaliser
  moving statistics restored, optimiser state not.  flags.train_image_size must equal a .pt checkpoint's; None takes it
  from the checkpoint, which a TensorFlow checkpoint does not record, so there it is required."""
  from . import tf_checkpoint, twingan
  kind, where = resolve_model_path(path)
  if kind == 'pt':
    ckpt = load_checkpoint(where)
    trained = int(ckpt['train_image_size']) if 'train_image_size' in ckpt else None
    if flags.train_image_size is None:
      if trained is None:
        raise ValueError('%s does not record its image size; give it explicitly' % where)
      flags = replace(flags, train_image_size=trained)
    elif trained is not None and trained != flags.train_image_size:
      raise ValueError('%s was trained at %d x %d, not %d x %d'
                       % (where, trained, trained, flags.train_image_size, flags.train_image_size))
    model = twingan.GanModel(flags, device=device)
    warm_start(model, ckpt, ignore_missing_vars=False, restore_optimizer=False)
    return model, step_of(where, int(ckpt.get('global_step', 0)))
  if flags.train_image_size is None:
    raise ValueError('%s is a TensorFlow checkpoint, which does not record its image size; give it explicitly' % where)
  model = twingan.GanModel(flags, device=device)
  tf_checkpoint.import_into(model, where, ignore_missing_vars=False, load_adam=False)
  return model, step_of(where)


# -- the loop ----------------------------------------------------------------------------------------------
def runs_to_reach(n_critic_counter: int, n_critic: int, generator_turns: int) -> int:
  """Mode-A runs, from run `n_critic_counter` on, up to and including the `generator_turns`-th generator turn (runs whose
  counter is a multiple of n_critic, image_generation.py:640-646)."""
  if generator_turns <= 0:
    return 0
  first_g = -(-n_critic_counter // n_critic) * n_critic
  return first_g + (generator_turns - 1) * n_critic + 1 - n_critic_counter


BatchFn = Callable[[Stage, int], Tuple[torch.Tensor, torch.Tensor]]
EvalFn = Callable[[object, int], object]


def run_stage(model, stage: Stage, batch_fn: BatchFn, train_dir: Optional[str] = None, start_step: int = 0,
              max_steps: Optional[int] = None, save_every: int = 0, use_graph: bool = True,
              grow_start_number_of_steps: int = 0, dragan_generator: Optional[torch.Generator] = None,
              log_fn: Optional[Callable[[int, Dict[str, float]], None]] = None, alternating: bool = False,
              prefetch: int = 0, eval_every_n_iter_in_training: int = 0, eval_fn: Optional[EvalFn] = None) -> int:
  """Train `model` for one stage, from global step `start_step` to min(stage.max_number_of_steps, start_step + max_steps).
  Returns the step reached.  Growing stages recompute alpha every step (twingan.py:834-835) and therefore run the
  eager step; stable stages capture the step once and replay it.  `alternating`: the reference's own schedule
  (GanModel.train_step_alternating: one Adam apply per run, generator and discriminator turns alternate) instead of
  the simultaneous mode-B step.  Steps, and with them alpha, the renorm clipping, the stop, `save_every`, evaluations and
  checkpoint names, then count generator turns -- global_step advances on those only (image_generation.py:648-651) and
  slim's number_of_steps stops on it (model/model_inheritor.py:1116-1123) -- while the runs are counted by
  model.n_critic_counter (:622, 641-645), which `batch_fn` receives as its index so that a resume replays the same
  batches; `log_fn` is called after every run.
  `prefetch` > 0: `batch_fn` returns HOST tensors; a background thread keeps that many batches ready in pinned memory and
  the host->device copy of batch k+1 runs on a side stream while step k computes (prefetch.py; the reference's
  slim.prefetch_queue, model/model_inheritor.py:425-470).
  `eval_every_n_iter_in_training` > 0 with `eval_fn`: eval_fn(model, step) after every step that reaches a multiple of it
  (twingan.py:679-680), e.g. swd.make_eval_fn; the evaluation must leave the model's training state as it found it."""
  from . import twingan
  end = stage.max_number_of_steps if max_steps is None else min(stage.max_number_of_steps, start_step + max_steps)
  graphed = False
  step = start_step
  feed = host_feed = None
  first = model.n_critic_counter if alternating else start_step     # index of the first batch
  if prefetch > 0 and end > start_step:
    from .prefetch import DevicePrefetcher, HostPrefetcher
    num = runs_to_reach(first, model.flags.n_critic, end - start_step) if alternating else end - start_step
    host_feed = HostPrefetcher(lambda i: tuple(batch_fn(stage, first + i)), capacity=prefetch, num_batches=num)
    feed = DevicePrefetcher(host_feed, model.device)
  while step < end:
    sources, targets = next(feed) if feed is not None else batch_fn(stage, model.n_critic_counter if alternating else step)
    rand = twingan.make_dragan_rand(sources.shape[0], stage.hw, model.device, dragan_generator)
    model.flags.global_step = step
    if stage.is_growing:
      model.flags.alpha_grow = alpha_grow(step, stage.max_number_of_steps, grow_start_number_of_steps)
    if alternating:
      g, d, turn = model.train_step_alternating(sources, targets, rand)
    elif stage.is_growing:
      g, d = model.train_step(sources, targets, rand)
    elif use_graph and model.device.type == 'cuda':
      if not graphed:
        model.capture(sources, targets, rand)
        graphed = True
      g, d = model.train_step_graphed(sources, targets, rand)
    else:
      g, d = model.train_step(sources, targets, rand)
    if feed is not None:
      feed.release()
    if alternating and turn != 'G':      # a discriminator turn leaves global_step where it was
      if log_fn is not None:
        log_fn(step, {'generator_loss': float(g), 'discriminator_loss': float(d)})
      continue
    step += 1
    if log_fn is not None:
      log_fn(step, {'generator_loss': float(g), 'discriminator_loss': float(d)})
    if eval_fn is not None and eval_every_n_iter_in_training > 0 and step % eval_every_n_iter_in_training == 0:
      eval_fn(model, step)
    if train_dir and save_every and step % save_every == 0:
      save_checkpoint(model, train_dir, step)
  model.flags.global_step = step
  if host_feed is not None:
    host_feed.close()
  if train_dir:
    save_checkpoint(model, train_dir, step)
  return step


def run(base_flags, base_dir: str, batch_fn: BatchFn, stages: Optional[Iterable[Stage]] = None,
        max_steps_per_stage: Optional[int] = None, device='cuda', seed: int = 1234, process_group=None,
        save_every: int = 0, use_graph: bool = True, log_fn=None, tf_checkpoint_prefix: Optional[str] = None,
        prefetch: int = 0, eval_every_n_iter_in_training: int = 0, eval_fn: Optional[EvalFn] = None,
        alternating: bool = False, dragan_generator: Optional[torch.Generator] = None):
  """pggan_runner.py main(): walk the stage plan; skip stages whose checkpoint already reached the stage's step count
  (:117-121); resume a partially trained stage from its own directory; otherwise warm-start from the previous
  stage's directory with ignore_missing_vars = is_growing (:137-146).  `tf_checkpoint_prefix`: a TensorFlow V2
  checkpoint of the reference (e.g. its pretrained models) that seeds the first stage that has nothing to start
  from (twingan_b200/tf_checkpoint.py).  `prefetch` > 0: `batch_fn` returns host tensors that are produced on a background
  thread and copied ahead of the step (run_stage).  `eval_every_n_iter_in_training` / `eval_fn`: periodic evaluation as in
  run_stage, for the stages of 16 x 16 and up (the reference skips SWD below 16, image_generation.py:869-871).
  `alternating` / `dragan_generator`: as in run_stage; a resumed stage restores global_step and n_critic_counter from its
  checkpoint, a new stage starts both at 0.  Returns the last model."""
  from . import twingan
  last_train_dir = None
  model = None
  for st in (list(stages) if stages is not None else stage_plan()):
    train_dir = os.path.join(base_dir, st.name)
    target = st.max_number_of_steps if max_steps_per_stage is None else min(st.max_number_of_steps, max_steps_per_stage)
    own = latest_checkpoint(train_dir)
    if own is not None and own[1] >= target:
      last_train_dir = train_dir
      continue
    flags = replace(base_flags, train_image_size=st.hw, is_growing=st.is_growing, alpha_grow=0.0, global_step=0)
    model = twingan.GanModel(flags, device=device, seed=seed, process_group=process_group)
    start = 0
    if own is not None:
      warm_start(model, load_checkpoint(own[0]), ignore_missing_vars=False, restore_step=True)
      start = own[1]
    elif last_train_dir is not None:
      prev = latest_checkpoint(last_train_dir)
      if prev is not None:
        # a new stage starts its own global_step at 0 (a fresh train_dir in the reference).  The reference's init_fn
        # restores slim.get_model_variables() only (model/model_inheritor.py:610-644): weights and normaliser moving
        # statistics -- Adam's slots and beta powers start fresh in every stage.
        warm_start(model, load_checkpoint(prev[0]), ignore_missing_vars=st.ignore_missing_vars, restore_optimizer=False)
    elif tf_checkpoint_prefix is not None:
      from . import tf_checkpoint
      tf_checkpoint.import_into(model, tf_checkpoint_prefix, ignore_missing_vars=True)
    run_stage(model, st, batch_fn, train_dir, start_step=start,
              max_steps=None if max_steps_per_stage is None else target - start, save_every=save_every,
              use_graph=use_graph, log_fn=log_fn, prefetch=prefetch, alternating=alternating,
              dragan_generator=dragan_generator,
              eval_every_n_iter_in_training=eval_every_n_iter_in_training if st.hw >= 16 else 0, eval_fn=eval_fn)
    last_train_dir = train_dir
  return model
