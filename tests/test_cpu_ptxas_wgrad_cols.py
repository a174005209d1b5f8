"""CPU test: every column-box weight-gradient instantiation the dispatch can launch (CN x BNW = 8) is compiled, with no spill.
The serialisation check (C7518) and the spill check of test_cpu_ptxas cover these kernels as well; this adds their count."""
from tests.test_cpu_ptxas import _functions, _kernel, report  # noqa: F401  (report: the module's ptxas fixture)


def test_wgrad_cols_instantiations(report):
  fns = {f: s for f, s in _functions(report).items() if _kernel(f) == 'k_conv_wgrad_cols_wgmma'}
  assert len(fns) == 8, sorted(fns)
  assert all(s == (0, 0) for s in fns.values()), fns
