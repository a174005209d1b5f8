"""The column-box weight-gradient kernel (3x3 SAME, 16 x 8 pixel tiles inside one image, every input-channel chunk of 16, 32
or 64) where it differs from the per-tap kernel: tiles at every image border with non-zero data in the halo, CTAs whose pixel
split leaves a short last CTA, several input-channel and output-channel blocks, and accumulate on and off.  Each gw element is
held to fp64, and two runs of the same call must agree bit for bit."""
import pytest
import torch

from tests.parity import conv_error_ratio, tc_elem_c
from tests.test_gpu_kernels import _dev, _rand, conv_refs

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'

# N, H, W, Cin, Cout.  H % 8 and W % 16 != 0 where possible, so the bottom and right tiles hang over the image.  The grid
# splits the tiles over at most 132 / (output-channel blocks x input-channel blocks) CTAs; the tile counts below do not divide
# evenly, so the last CTA runs fewer tiles.  Every (input-channel chunk, output-channel block) pair the dispatch picks occurs:
# CN x BNW = 16 x 16, 32, 64; 32 x 16, 32, 64; 64 x 16, 32.
SHAPES = [
    (2, 20, 40, 16, 16),     # 3 x 3 tiles per image: every tile touches a border
    (3, 18, 24, 16, 32),
    (2, 36, 72, 16, 128),    # two 64-channel output blocks
    (3, 36, 72, 32, 16),
    (2, 66, 100, 32, 32),
    (2, 40, 48, 32, 256),    # four output blocks
    (3, 66, 100, 64, 16),
    (2, 18, 24, 64, 32),
    (2, 40, 48, 128, 64),    # two 64-channel input blocks
    (2, 24, 40, 256, 32),    # four input blocks
    (13, 16, 16, 256, 256),  # 26 tiles over 4 CTAs of 7: the last one runs 5
    (5, 32, 32, 128, 128),   # 40 tiles over 14 CTAs of 3: the last one runs one
]


def _wgrad(L, xp, gp, gw, shape, accumulate):
  from twingan_b200 import ops
  N, H, W, Cin, Cout = shape
  L.call('twg_conv_wgrad_planes', xp.data_ptr(), gp.data_ptr(), gw.data_ptr(), N, H, W, Cin, Cout, 3, 1, int(accumulate),
         ops._st())


@pytest.mark.parametrize('accumulate', [False, True])
@pytest.mark.parametrize('shape', SHAPES)
def test_cols_wgrad_against_fp64(built_lib, shape, accumulate):
  """gw per element against fp64 (randn data, so every halo pixel a border tile reads from inside the image is non-zero and
  every one outside must read as zero); with accumulate, into a non-zero gw.  Two runs agree bit for bit."""
  from twingan_b200 import ops
  L = built_lib
  N, H, W, Cin, Cout = shape
  x, w, gy = _rand((N, H, W, Cin), 401), _rand((3, 3, Cin, Cout), 402, 0.05), _rand((N, H, W, Cout), 403)
  (_, _, gwr), (_, _, sgw), (_, _, kgw) = conv_refs(x, w, gy, 3, 1, DEV)
  xp, gp = ops.split_act(_dev(x)), ops.split_act(_dev(gy))
  g0 = _dev(_rand((3, 3, Cin, Cout), 404)) if accumulate else torch.zeros((3, 3, Cin, Cout), device=DEV)
  runs = []
  for _ in range(2):
    gw = g0.clone() if accumulate else torch.full_like(g0, float('nan'))
    _wgrad(L, xp, gp, gw, shape, accumulate)
    runs.append(gw)
  torch.cuda.synchronize()
  assert torch.equal(runs[0].view(torch.int32), runs[1].view(torch.int32))
  ref = gwr.double() + g0.double().to(gwr.device)
  S = sgw.double() + g0.double().abs().to(gwr.device)
  assert conv_error_ratio(runs[0], ref, S, tc_elem_c(kgw)) <= 1.0
