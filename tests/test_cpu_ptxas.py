"""CPU test: ptxas keeps the tensor-core convolutions asynchronous and in registers.

Compiles twg_conv_tc.cu with the flags of __graft_entry__.build() plus `-Xptxas -v` (no GPU needed) and reads ptxas's
report.  It fails on
  - any C7518 "wgmma.mma_async instructions are serialized" line: ptxas then makes every wgmma wait for the one before it,
    which turns the kernels' commit / wait_group pipelining into one MMA latency per instruction;
  - nonzero spill stores or loads in any k_conv_*_wgmma kernel: the accumulators live in registers, and a spill puts
    local-memory traffic between the MMAs and the epilogue."""
import os
import re
import shutil
import subprocess

import pytest

import __graft_entry__ as graft

SOURCE = os.path.join(graft.CSRC, 'twg_conv_tc.cu')
# every template instantiation the dispatch can launch: forward / dgrad per tap and column-box, CC x BN = 3 x 4 each;
# weight gradient CN x BNW = 8
EXPECTED = {'k_conv_fwd_wgmma': 12, 'k_conv_fwd_cols_wgmma': 12, 'k_conv_wgrad_wgmma': 8}


def _nvcc():
  nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
  return nvcc if os.path.exists(nvcc) else shutil.which('nvcc')


@pytest.fixture(scope='module')
def report(tmp_path_factory):
  nvcc = _nvcc()
  if not nvcc:
    pytest.skip('nvcc not found')
  out = tmp_path_factory.mktemp('ptxas')
  cmd = [nvcc] + graft.NVCC_FLAGS + ['-Xptxas', '-v', '-c', '-o', str(out / 'twg_conv_tc.o'), SOURCE]
  r = subprocess.run(cmd, cwd=str(out), capture_output=True, text=True)
  assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
  return r.stdout + r.stderr


def _functions(text):
  """{mangled name: (spill store bytes, spill load bytes)} of every entry function in the ptxas report."""
  res, fn = {}, None
  for line in text.splitlines():
    m = re.search(r"Compiling entry function '(\w+)'", line) or re.search(r'Function properties for (\w+)', line)
    if m:
      fn = m.group(1)
      continue
    m = re.search(r'(\d+) bytes spill stores, (\d+) bytes spill loads', line)
    if m and fn:
      res[fn] = (int(m.group(1)), int(m.group(2)))
  return res


def _kernel(mangled):
  m = re.match(r'_ZN3twg\d+(k_conv_\w+?_wgmma)I', mangled)
  return m.group(1) if m else None


def test_no_wgmma_is_serialised(report):
  serialised = [l.strip() for l in report.splitlines() if 'C7518' in l]
  assert not serialised, '%d serialised kernels:\n%s' % (len(serialised), '\n'.join(serialised))


def test_no_wgmma_kernel_spills(report):
  fns = {f: s for f, s in _functions(report).items() if _kernel(f)}
  counts = {k: sum(_kernel(f) == k for f in fns) for k in EXPECTED}
  assert counts == EXPECTED, counts
  spilling = {f: s for f, s in fns.items() if s != (0, 0)}
  assert not spilling, spilling
