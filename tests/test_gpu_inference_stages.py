"""GanModel.infer against the fp64 oracle (oracle/twingan_oracle.inference) where the product runs the evaluation-mode
network and test_gpu_step.test_inference_parity does not reach: growing stages mid fade-in and at their last step (the
SWD evaluation during training), stable stages from a stage checkpoint (translate, swd_eval), plain batch norm, residual
blocks, 256 channels on the tensor cores, and the target -> source direction.  Affine parameters and the moving
statistics are randomised, so the evaluation-mode affine is not the identity."""
import pytest
import torch

from tests.parity import REL_TOL, _log_result, rel_err

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'

# (hw, growing, alpha, max channels, normaliser, residual blocks, target domain, batch)
CASES = [(16, True, a, 256, norm, False, 't', 3) for a in (0.3, 1.0) for norm in ('instance_norm', 'batch_renorm')]
CASES += [(64, True, a, 256, norm, False, 't', 2) for a in (0.3, 1.0) for norm in ('instance_norm', 'batch_renorm')]
CASES += [
    (128, True, 0.5, 256, 'batch_renorm', False, 't', 2),
    (64, False, 0.0, 256, 'batch_norm', False, 't', 3),
    (128, False, 0.0, 256, 'batch_norm', False, 't', 2),
    (32, False, 0.0, 256, 'instance_norm', True, 't', 3),
    (32, True, 0.3, 256, 'batch_norm', True, 't', 2),
    (64, True, 0.3, 256, 'batch_renorm', False, 's', 2),
]


def _id(c):
  hw, growing, alpha, mc, norm, res, d, B = c
  return '%s%s-%s%s-%s-B%d' % ('%dto%d' % (hw // 2, hw) if growing else hw, '-a%g' % alpha if growing else '', norm,
                               '-res' if res else '', d, B)


@pytest.mark.parametrize('case', CASES, ids=_id)
def test_infer_matches_the_fp64_oracle(built_lib, case):
  from oracle import twingan_oracle as O
  from twingan_b200 import twingan
  hw, growing, alpha, mc, norm, res, d, B = case
  cfg = O.Config(hw=hw, is_growing=growing, alpha_grow=alpha, max_num_channels=mc, generator_norm_type=norm,
                 use_res_block=res)
  params = O.init_params(cfg, seed=hw + B, randomize_affine=True)
  state = O.init_norm_state(cfg, seed=7)
  src, tgt, _ = O.make_inputs(cfg, B, seed=hw)
  x = src if d == 't' else tgt
  ref = O.inference(cfg, params, state, x, target_domain=d)
  model = twingan.GanModel(twingan.Flags(train_image_size=hw, is_growing=growing, alpha_grow=alpha,
                                         pggan_max_num_channels=mc, generator_norm_type=norm, use_res_block=res),
                           device=DEV)
  model.variables.load_dict(params, state if state else None)
  got = model.infer(x.to(DEV, torch.float32), target_domain=d)
  err = rel_err(got, ref)
  _log_result({'test': 'inference_stage', 'case': _id(case), 'rel_err': err})
  assert err < REL_TOL, (case, err)
