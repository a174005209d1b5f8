"""`python -m twingan_b200.swd_eval`: the reference's evaluation run with --calc_swd=True (docs/infer_and_eval.md;
image_generation.py:868-927), on the device.

  python -m twingan_b200.swd_eval --checkpoint_path=<train_dir>/model.ckpt-<step>.pt | <TF checkpoint prefix> \\
      --dataset_dir=<source domain> --unpaired_target_dataset_dir=<target domain> --dataset_split_name=train \\
      --train_image_size=256 --swd_num_images=8192 --eval_dir=<dir>

writes <eval_dir>/swd_eval_step_<step>_<n>_images.txt in the reference's layout: the SWD x 1e3 of target-domain images
(real) against the translated source-domain images (fake) per pyramid level and on average, and the real-vs-real floor.
"""
from __future__ import annotations

import argparse
import os
import re
import sys

from . import swd


def _parser() -> argparse.ArgumentParser:
  p = argparse.ArgumentParser(prog='python -m twingan_b200.swd_eval', description=__doc__.split('\n\n')[0])
  p.add_argument('--checkpoint_path', required=True,
                 help='a model.ckpt-<step>.pt of pggan_runner, or the prefix of a TensorFlow checkpoint of the reference')
  p.add_argument('--dataset_dir', required=True, help='image_only TFRecords of the source domain')
  p.add_argument('--unpaired_target_dataset_dir', required=True, help='image_only TFRecords of the target domain')
  p.add_argument('--dataset_split_name', default='train')
  p.add_argument('--train_image_size', type=int, default=256)
  p.add_argument('--swd_num_images', type=int, default=1024, help='images per set (the reference recommends 8192)')
  p.add_argument('--eval_dir', required=True)
  p.add_argument('--pggan_max_num_channels', type=int, default=256)
  p.add_argument('--generator_norm_type', default='instance_norm')
  p.add_argument('--batch_size', type=int, default=64, help='images translated per model call')
  p.add_argument('--seed', type=int, default=0, help='seeds the image draws, the neighbourhoods and the directions')
  return p


def _step_of(path: str, default: int = 0) -> int:
  """The step a checkpoint's name carries (model.ckpt-<step>[.pt], like the reference's '.ckpt-' split), else `default`."""
  m = re.search(r'-(\d+)(\.pt)?$', path)
  return int(m.group(1)) if m else default


def _load_model(args):
  from . import pggan_runner, tf_checkpoint, twingan
  flags = twingan.Flags(train_image_size=args.train_image_size, pggan_max_num_channels=args.pggan_max_num_channels,
                        generator_norm_type=args.generator_norm_type)
  path = args.checkpoint_path
  if os.path.isfile(path):
    ckpt = pggan_runner.load_checkpoint(path)
    if int(ckpt.get('train_image_size', args.train_image_size)) != args.train_image_size:
      raise ValueError('%s was trained at %d x %d, not --train_image_size=%d'
                       % (path, ckpt['train_image_size'], ckpt['train_image_size'], args.train_image_size))
    model = twingan.GanModel(flags, device='cuda')
    pggan_runner.warm_start(model, ckpt, ignore_missing_vars=False, restore_optimizer=False)
    return model, _step_of(path, int(ckpt.get('global_step', 0)))
  if os.path.isfile(path + '.index'):
    model = twingan.GanModel(flags, device='cuda')
    tf_checkpoint.import_into(model, path, ignore_missing_vars=False, load_adam=False)
    return model, _step_of(path)
  raise FileNotFoundError('no checkpoint at %s (neither a file nor a TensorFlow prefix with a .index file)' % path)


def main(argv=None):
  parser = _parser()
  args = parser.parse_args(argv)
  try:
    swd.check_resolution(args.train_image_size)
  except ValueError as e:
    parser.error('--train_image_size: %s' % e)
  if args.swd_num_images < 2 or args.swd_num_images % 2:
    parser.error('--swd_num_images must be even and at least 2: the real column of the result is the SWD between the two '
                 'halves of the real set (got %d)' % args.swd_num_images)
  if args.batch_size < 1:
    parser.error('--batch_size must be positive')
  from .image_only import ImageOnlyDataset
  source = ImageOnlyDataset(args.dataset_dir, args.dataset_split_name)
  target = ImageOnlyDataset(args.unpaired_target_dataset_dir, args.dataset_split_name)
  for name, ds in (('--dataset_dir', source), ('--unpaired_target_dataset_dir', target)):
    if len(ds) < args.swd_num_images:
      parser.error('%s has %d %s images, fewer than --swd_num_images=%d'
                   % (name, len(ds), args.dataset_split_name, args.swd_num_images))
  model, step = _load_model(args)
  result = swd.evaluate_translation(model, source, target, args.swd_num_images, args.seed, args.batch_size)
  path = swd.write_result(args.eval_dir, step, args.swd_num_images, result, is_training=False)
  print(open(path).read(), end='')
  return result


if __name__ == '__main__':
  main(sys.argv[1:])
