"""Every status the C boundary returns before a launch, for one lowered level of every
step program (tests/boundary_sweep.py), against tests/golden/boundary_statuses.json.
No GPU: device -1, made-up addresses, nothing launched."""

import ctypes as C
import json
import os

import boundary_sweep
from pycolab_b200 import _lib

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden',
                      'boundary_statuses.json')


def test_boundary_statuses_of_the_lowered_levels_and_their_refusals():
  """The statuses of the golden file, case for case.  Among them, warehouse,
  better_scrolly and marauders refuse a board whose block of four staged backdrop tiles
  (and, for better_scrolly, coin bit rows; for marauders, its static records) would
  exceed the 227 KB of shared memory a block can opt in to (rows or pitch 32768, or
  better_scrolly's bits_words 32768): such a spec could never launch."""
  with open(GOLDEN) as f:
    encoded = json.load(f)
  got = boundary_sweep.sweep()
  assert {level: len(chars) for level, chars in boundary_sweep.encode(got).items()} == \
      {level: len(chars) for level, chars in encoded.items()}, \
      'the sweep no longer makes the cases of the golden file'
  want = boundary_sweep.decode(encoded, list(got))
  differ = ['%s: want %d, got %d' % (k, want[k], got[k]) for k in want if got[k] != want[k]]
  assert not differ, '%d of %d cases differ, first: %s' % (len(differ), len(want),
                                                          '; '.join(differ[:10]))
  for level in encoded:
    assert want[level + '/create'] == want[level + '/bind'] == _lib.OK, level
  for case in ('warehouse/spec.rows=32768', 'warehouse/spec.pitch=32768',
               'better_scrolly/spec.rows=32768', 'better_scrolly/spec.pitch=32768',
               'better_scrolly/spec.bits_words=32768', 'marauders/spec.pitch=32768'):
    assert want[case] == got[case] == _lib.ERR_UNSUPPORTED, case
  programs = set(spec.program for _, spec in boundary_sweep.lowered_specs())
  assert programs == set(range(1, 13))


def test_fixture_refuses_more_update_groups_than_entity_slots():
  """The group lengths are summed over n_groups: a count beyond group_len's slots is
  refused before any of them is read."""
  specs = dict(boundary_sweep.lowered_specs())
  lib = _lib.load()
  for n_groups in (_lib.MAX_SPRITES + _lib.MAX_DRAPES + 1, 129, 32768, 2 ** 31 - 1):
    spec = _lib.Spec.from_buffer_copy(specs['fixture_walkers'])
    spec.n_groups = n_groups
    h = C.c_void_p()
    assert lib.pcl_create(C.byref(spec), 4, -1, C.byref(h)) == _lib.ERR_INVALID, n_groups
