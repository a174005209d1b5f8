"""Every kernel-launching entry point of include/twg.h has an owner: a GPU suite that holds it to a reference, or a
line here saying why the product never launches it.  A new entry point fails this test until someone decides which."""
from twingan_b200._lib import parse_header

# kernel-launching entry points (they take a stream) that the product does not launch, and why
NOT_LAUNCHED = {}


def _launching_entries():
  return {name for name, (_, args) in parse_header().items() if 'twg_stream_t' in args}


def test_every_launching_entry_has_one_owner_or_a_reason():
  from tests.test_gpu_elementwise_conformance import _owners
  claims = {}
  for suite, entries in _owners().items():
    for e in entries:
      claims.setdefault(e, []).append(suite)
  launching = _launching_entries()
  assert not {e: s for e, s in claims.items() if len(s) > 1}, 'owned twice'
  assert set(claims) <= launching, ('owners name entries twg.h does not declare', sorted(set(claims) - launching))
  assert not set(claims) & set(NOT_LAUNCHED), sorted(set(claims) & set(NOT_LAUNCHED))
  assert set(NOT_LAUNCHED) <= launching, sorted(set(NOT_LAUNCHED) - launching)
  assert all(NOT_LAUNCHED.values())
  unowned = launching - set(claims) - set(NOT_LAUNCHED)
  assert not unowned, ('neither owned by a GPU suite nor listed as not launched', sorted(unowned))
