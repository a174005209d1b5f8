"""CPU test: the resident-weight instantiations of the column-box forward / dgrad (GEMM K <= 32, BN <= 64, six keys) compile without a spill and without a serialised wgmma.  test_cpu_ptxas checks every kernel of the file the same way; this
names the keys whose consumers keep two 128-row accumulators (BN <= 32) or issue whole tap chains without a wait, where
registers are tightest."""
import re

from tests.test_cpu_ptxas import _functions, _kernel, report  # noqa: F401  (report: the module's ptxas fixture)

RESIDENT = {(16, 16), (16, 32), (16, 64), (32, 16), (32, 32), (32, 64)}


def _key(mangled):
  m = re.search(r'ILi(\d+)ELi(\d+)E', mangled)
  return (int(m.group(1)), int(m.group(2))) if m else None


def test_cols_resident_instantiations(report):
  fns = {_key(f): s for f, s in _functions(report).items() if _kernel(f) == 'k_conv_fwd_cols_wgmma'}
  assert RESIDENT <= set(fns), sorted(fns)
  spilling = {k: fns[k] for k in RESIDENT if fns[k] != (0, 0)}
  assert not spilling, spilling
  assert not [l for l in report.splitlines() if 'C7518' in l and 'k_conv_fwd_cols_wgmma' in l]
