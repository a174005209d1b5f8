"""CPU test: every instantiation of the split backward reduce (k_norm_act_bwd_reduce_split<V>, one cluster of CTAs per
sample) compiles without a spill.

Compiles twg_norm.cu with the flags of __graft_entry__.build() plus `-Xptxas -v` (no GPU needed).  A thread holds a batch
of pixels in flight, the per-channel affine and its share of the chains' sums in registers, up to about 240 of the 255 it
may have at V = 4; a spill would put local-memory traffic between the loads and the ordered adds."""
import os
import re
import subprocess

import pytest

import __graft_entry__ as graft
from tests.test_cpu_ptxas import _functions, _nvcc

EXPECTED_V = {1, 2, 4}


@pytest.fixture(scope='module')
def report(tmp_path_factory):
  nvcc = _nvcc()
  if not nvcc:
    pytest.skip('nvcc not found')
  out = tmp_path_factory.mktemp('ptxas_split')
  cmd = [nvcc] + graft.NVCC_FLAGS + ['-Xptxas', '-v', '-c', '-o', str(out / 'twg_norm.o'),
                                     os.path.join(graft.CSRC, 'twg_norm.cu')]
  r = subprocess.run(cmd, cwd=str(out), capture_output=True, text=True)
  assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
  return r.stdout + r.stderr


def test_no_split_reduce_spills(report):
  fns = {f: s for f, s in _functions(report).items() if re.match(r'_ZN3twg\d+k_norm_act_bwd_reduce_splitI', f)}
  vs = {int(re.search(r'ILi(\d+)E', f).group(1)) for f in fns}
  assert vs == EXPECTED_V, sorted(fns)
  spilling = {f: s for f, s in fns.items() if s != (0, 0)}
  assert not spilling, spilling
