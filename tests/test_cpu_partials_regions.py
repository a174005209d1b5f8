"""CPU tests: the library's partial-sum scratch is a fixed set of disjoint regions, one per stream that may run the
cross-block reductions at the same time as another (the training step's two discriminator domains), and a region is
never handed to a second stream.  The bindings are process state, so the checks run in a fresh interpreter."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_CHECK = r'''
import sys
sys.path.insert(0, sys.argv[1])
from twingan_b200._lib import lib
L = lib()
c = L.cdll
assert c.twg_partials_regions() == 2
assert c.twg_partials_region_floats() == 8 << 20
assert c.twg_partials_region_uses(0) == 0 and c.twg_partials_region_uses(1) == 0     # nothing reduced yet
assert c.twg_partials_region_uses(-1) == -1 and c.twg_partials_region_uses(2) == -1
a, b = 0x1000, 0x2000                                   # stream handles: binding only compares them
assert c.twg_partials_region(a) == 0 and c.twg_partials_region(None) == 0
assert L.try_call('twg_partials_bind', a, 1) == 0
assert c.twg_partials_region(a) == 1 and c.twg_partials_region(b) == 0
assert L.try_call('twg_partials_bind', a, 1) == 0      # again: no change
assert L.try_call('twg_partials_bind', b, 1) != 0 and 'another stream' in L.last_error()
assert c.twg_partials_region(b) == 0
for bad in (-1, 2):
  assert L.try_call('twg_partials_bind', b, bad) != 0
assert L.try_call('twg_partials_bind', None, 1) != 0   # the default stream keeps region 0
assert L.try_call('twg_partials_bind', a, 0) == 0      # give it back
assert c.twg_partials_region(a) == 0
assert L.try_call('twg_partials_bind', b, 1) == 0 and c.twg_partials_region(b) == 1
print('ok')
'''


def test_partial_regions_are_fixed_disjoint_and_owned_by_one_stream(built_lib):
  out = subprocess.run([sys.executable, '-c', _CHECK, ROOT], capture_output=True, text=True, timeout=120)
  assert out.returncode == 0 and out.stdout.strip() == 'ok', out.stderr
