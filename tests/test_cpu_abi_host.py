"""CPU tests: the C-ABI library loads and exports every symbol include/twg.h declares (no kernel is launched
without a GPU), host-side argument validation, and the host logic (variable layout, layer tables, FLOP table)."""
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_loads_and_exports_every_header_symbol(built_lib):
  from twingan_b200 import _lib
  protos = _lib.parse_header()
  assert len(protos) >= 34
  for name in protos:
    assert hasattr(built_lib.cdll, name), name
  assert built_lib.cdll.twg_version() >= 100
  # every `int twg_*(` in the header was parsed
  hdr = open(_lib.HEADER).read()
  declared = set(re.findall(r'\b(twg_\w+)\s*\(', hdr)) - {'twg_last_error_string'}
  assert declared == set(protos), declared ^ set(protos)


def test_conv_and_pool_entries_reject_bad_arguments_without_gpu(built_lib):
  L = built_lib
  assert L.try_call('twg_conv_fwd', None, None, None, 1, 4, 4, 16, 16, 3, 1, None) == -1
  assert 'null' in L.last_error()
  assert L.try_call('twg_conv_fwd', 8, 8, 8, 1, 2, 2, 4, 4, 5, 0, None) == -1           # empty output
  assert L.try_call('twg_conv_wgrad', 8, 8, 8, 0, 4, 4, 4, 4, 3, 1, 0, None) == -1      # N=0 (empty batch)
  assert L.try_call('twg_pool2', 8, 8, None, 1, 3, 4, 1, 0.25, None) == -1              # odd H


def test_every_library_call_matches_the_header_arity():
  """Every call in the package that names a library function -- `lib().call('twg_...', ...)`, `.try_call(...)`, the conv
  launcher `_conv_launch(family, shape, 'twg_...', ...)`, `.cdll.twg_...(...)` -- passes as many arguments as include/twg.h
  declares.  (ctypes checks the count only when a call is made, and without a GPU no kernel call is.)"""
  import ast
  from twingan_b200 import _lib
  protos = _lib.parse_header()
  pkg = os.path.join(ROOT, 'twingan_b200')
  seen = 0
  for fn in sorted(os.listdir(pkg)):
    if not fn.endswith('.py'):
      continue
    for node in ast.walk(ast.parse(open(os.path.join(pkg, fn)).read())):
      if not isinstance(node, ast.Call):
        continue
      named = [i for i, a in enumerate(node.args) if isinstance(a, ast.Constant) and str(a.value).startswith('twg_')]
      f = node.func
      if named:
        name, args = node.args[named[0]].value, node.args[named[0] + 1:]
      elif isinstance(f, ast.Attribute) and f.attr.startswith('twg_') and isinstance(f.value, ast.Attribute) \
          and f.value.attr == 'cdll':
        name, args = f.attr, node.args
      else:
        continue
      where = '%s:%d %s' % (fn, node.lineno, name)
      assert name in protos, where
      want = len(protos[name][1])
      if any(isinstance(a, ast.Starred) for a in args):    # (..., *ptrs, ...): at least not too many
        assert len([a for a in args if not isinstance(a, ast.Starred)]) < want, where
      else:
        assert len(args) == want, (where, len(args), want)
      seen += 1
  assert seen >= 60, seen


def test_product_never_imports_the_oracle_and_fails_loudly_without_cuda():
  pkg = os.path.join(ROOT, 'twingan_b200')
  for fn in os.listdir(pkg):
    if fn.endswith('.py'):
      src = open(os.path.join(pkg, fn)).read()
      assert 'oracle' not in re.sub(r'#.*', '', src).replace('no CPU fallback', ''), fn
  from twingan_b200 import ops
  from twingan_b200._lib import TwgError
  with pytest.raises(TwgError):
    ops.conv_fwd_raw(torch.zeros(1, 4, 4, 16), torch.zeros(3, 3, 16, 16), 3, 1)


def test_variable_store_layout_and_reference_names():
  from twingan_b200 import pggan
  from twingan_b200.variables import VariableStore
  v = VariableStore('cpu')
  pggan.declare_variables(v, 256, False, 256, True, 'batch_renorm')
  v.materialize()
  g0, g1 = v.group_range['G']
  d0, d1 = v.group_range['D']
  assert g0 == 0 and g1 == d0 and d1 == v.flat.numel()
  for name, (o, shape) in v.offsets.items():
    assert o % 4 == 0, name                       # 16-byte aligned slices (float4 kernels)
  wcount = lambda pre: sum(int(torch.tensor(s).prod()) for n, (o, s) in v.offsets.items() if n.startswith(pre) and n.endswith('/weights'))
  assert abs(wcount('encoder_content') - 2.95e6) < 2e4 and abs(wcount('generator') - 5.7e6) < 2e4   # SURVEY 8a.1
  assert 'encoder_content/encoder_block_256x256x32/Conv_1/BatchNorm/gamma_t' in v
  assert 'generator/generator_to_rgb_256x256/Conv/BatchNorm/beta_s' in v
  assert 'discriminator_t/prediction/fully_connected/weights' in v
  assert 'discriminator_s/before_fc_1x1x256/Conv/weights' in v and tuple(v['discriminator_s/before_fc_1x1x256/Conv/weights'].shape) == (3, 3, 257, 256)
  rec = v.state_record('generator/block_4x4x256/Conv/BatchNorm/_s')
  assert rec.numel() == 4 * 256 + 2 and float(rec[256:512].min()) == 1.0   # moving_variance starts at one
  # names agree with the oracle's (reference) naming
  from oracle import twingan_oracle as O
  ref = O.init_params(O.Config(hw=256, generator_norm_type='batch_renorm'))
  assert set(ref) == set(v.offsets)
  for k in ref:
    assert tuple(ref[k].shape) == tuple(v.offsets[k][1]), k


def test_flop_table_matches_survey():
  from twingan_b200 import flops
  s = flops.step_flops_per_pair(256)
  assert abs(s['F_E'] / 1e9 - 4.385) < 2e-3 and abs(s['F_G'] / 1e9 - 7.216) < 2e-3 and abs(s['F_D'] / 1e9 - 4.406) < 2e-3
  assert abs(s['total'] / 1e9 - 289.0) < 0.1 and abs(s['forward'] / 1e9 - 81.7) < 0.1
  assert abs(flops.step_flops_per_pair(128, True)['total'] / 1e9 - 229.1) < 0.2
  m = flops.mixed_roofline_seconds(256, 16, 1443e12, 6569e9)
  assert abs(m['step'] * 1e3 - 7.6) < 0.1          # SURVEY 8d: 7.6 ms mixed bound with fp32 activations


def test_renorm_clip_schedule_and_unet_lookup():
  from twingan_b200 import pggan_utils as pu
  assert pu.get_renorm_clipping_params(0) == (0.9, 1.1, 0.1)
  assert pu.get_renorm_clipping_params(20001) == (0.5, 2.0, 0.5)
  ep = {'encoder_block_8x8x256': 'plain', 'encoder_block_interpolated_8x8x256': 'interp'}
  assert pu.unet_layer_for(8, ep, 256) == 'interp'          # nets/pggan_utils.py:293
  with pytest.raises(ValueError):
    pu.unet_layer_for(16, ep, 256)
