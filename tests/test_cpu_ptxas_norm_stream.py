"""CPU test: the kernels that read their input through a shared-memory ring (twg_stream.cuh) compile without a spill.

Compiles twg_norm.cu and twg_elementwise.cu with the flags of __graft_entry__.build() plus `-Xptxas -v` (no GPU needed).
The streamed backward reduce holds a stage's pixels, the next stage's pooled gradient and its 8 V sums in registers, about 200 of the
255 a thread may have at V = 4; a spill would put local-memory traffic into the one block a sample has."""
import os
import re
import subprocess

import pytest

import __graft_entry__ as graft
from tests.test_cpu_ptxas import _functions, _nvcc

# kernel -> template instantiations the dispatch can launch
EXPECTED = {'k_norm_act_bwd_reduce_stream': 3, 'k_moments_stream': 3, 'k_sum_sq_stream': 1}


@pytest.fixture(scope='module')
def report(tmp_path_factory):
  nvcc = _nvcc()
  if not nvcc:
    pytest.skip('nvcc not found')
  out = tmp_path_factory.mktemp('ptxas_stream')
  text = ''
  for src in ('twg_norm.cu', 'twg_elementwise.cu'):
    cmd = [nvcc] + graft.NVCC_FLAGS + ['-Xptxas', '-v', '-c', '-o', str(out / (src + '.o')), os.path.join(graft.CSRC, src)]
    r = subprocess.run(cmd, cwd=str(out), capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    text += r.stdout + r.stderr
  return text


def _kernel(mangled):
  m = re.match(r'_ZN3twg\d+(k_\w+?_stream)(?:I|E)', mangled)
  return m.group(1) if m else None


def test_no_streamed_kernel_spills(report):
  fns = {f: s for f, s in _functions(report).items() if _kernel(f)}
  counts = {k: sum(_kernel(f) == k for f in fns) for k in EXPECTED}
  assert counts == EXPECTED, counts
  spilling = {f: s for f, s in fns.items() if s != (0, 0)}
  assert not spilling, spilling
