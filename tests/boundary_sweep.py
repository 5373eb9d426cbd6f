"""The C boundary's verdicts on one lowered level of every step program, as named cases.

Every case is a call that returns before anything reaches a device (device -1, made-up
non-null addresses), so the sweep runs on any machine with the library built:
  create            pcl_create on the lowered spec;
  spec.<f>=<v>      pcl_create after setting one spec field (or array element) to v;
  program=<id>      pcl_create with the program id changed;
  bind              pcl_bind_state from a state with every pointer set, every bstride > 0;
  bind.<f>=0        the same state with one pointer nulled or one bstride zeroed;
  bind.null         pcl_bind_state from the all-null state;
  attach.<name>     pcl_attach_cropper on the handle bound from the full state.
`tests/golden/boundary_statuses.json` holds the statuses in `encode`'s form;
test_program_table.py replays them.
"""

import ctypes as C
import importlib
import random

import numpy as np

from pycolab_b200 import _lib
from pycolab_b200 import levels
from pycolab_b200 import lowering

FAKE = 0x10000
STRIDE = 64
PROGRAM_IDS = list(range(0, 13)) + [13, 99, -1]

SCALARS = ('abi_version', 'rows', 'cols', 'pitch', 'n_sprites', 'n_drapes', 'auto_reset',
           'pattern_rows', 'pattern_cols', 'pattern_words', 'bits_words', 'n_groups',
           'n_scroll_groups')
SCALAR_CODES = (0, -1, 1, 2, 10, 17, 33, 65, 129, 32768)
INT_CODES = (0, 1, -1, 2, 3, 9, 11, 1025, 32768)
CHAR_CODES = (0, 1, 255, 32, ord('#'), ord('P'), 128)
# n_groups is tried only up to the number of group_len slots; test_program_table.py checks
# the larger counts on their own.
N_GROUP_SLOTS = _lib.MAX_SPRITES + _lib.MAX_DRAPES


def _fixture(name):
  import golden_cases as gc
  from pycolab_b200.games import fixtures
  kw, _ = gc.fixture_kwargs(gc.load(name))
  return fixtures.make_game(kw['art'], kw['what_lies_beneath'], kw['walkers'], kw['scrollys'],
                            kw['drapes'], kw['update_schedule'], kw['z_order'])


def _t_maze():
  from pycolab_b200.games import t_maze
  random.seed(0)
  np.random.seed(0)
  return t_maze.make_game(1, False)


def _games():
  """(name, facade game) for one level of every program; ordeal's three chapters as
  tests/test_ordeal.py builds them."""
  import golden_cases as gc
  import trajectory as tj
  from pycolab_b200.games import (aperture, apprehend, better_scrolly_maze, fluvial_natation,
                                  hello_world, ordeal, scrolly_maze, shockwave,
                                  warehouse_manager)
  from pycolab_b200.games import extraterrestrial_marauders as marauders
  four_rooms = importlib.import_module('pycolab_b200.games.classics.four_rooms')
  return [
      ('scrolly_maze', lambda: scrolly_maze.make_game(*levels.scrolly_maze_level(
          0, world_shape=(33, 33), board_shape=(16, 16)))),
      ('warehouse', lambda: warehouse_manager.make_game(levels.warehouse_level(1), ' ')),
      ('marauders', lambda: marauders.make_game(levels.marauders_level())),
      ('fixture_walkers', lambda: _fixture('fixture_walkers_0')),
      ('fixture_scrolly', lambda: _fixture('fixture_scrolly_0')),
      ('better_scrolly', lambda: better_scrolly_maze.make_game(
          tj.u8_to_art(gc.load('better_stock_L0')['art']))),
      ('fluvial', fluvial_natation.make_game),
      ('four_rooms', four_rooms.make_game),
      ('aperture', lambda: aperture.make_game(levels.aperture_level())),
      ('ordeal_castle', ordeal.make_castle),
      ('ordeal_cavern', ordeal.make_cavern),
      ('ordeal_kansas', ordeal.make_kansas),
      ('hello', hello_world.make_game),
      ('apprehend', apprehend.make_game),
      ('shockwave', lambda: shockwave.make_game(0)),
      ('t_maze', _t_maze),
  ]


def _elements(spec):
  """(label, array, index, codes) for every spec array element the level uses."""
  ns, nd = spec.n_sprites, spec.n_drapes
  n = ns + nd
  out = []

  def add(name, arr, count, codes, sub=None):
    for i in range(count):
      if sub is None:
        out.append(('%s[%d]' % (name, i), arr, i, codes))
      else:
        for j in range(sub):
          out.append(('%s[%d][%d]' % (name, i, j), arr[i], j, codes))
  add('sprite_char', spec.sprite_char, ns, CHAR_CODES)
  add('drape_char', spec.drape_char, nd, CHAR_CODES)
  add('impassable', spec.impassable, ns, (0, 1, 0xffffffff, 1 << 3, 1 << 2), sub=4)
  add('sprite_confined', spec.sprite_confined, ns, INT_CODES)
  add('sprite_egocentric', spec.sprite_egocentric, ns, INT_CODES)
  add('margins', spec.margins, nd, INT_CODES, sub=2)
  add('z_order', spec.z_order, n, CHAR_CODES)
  add('group_len', spec.group_len, max(spec.n_groups, 1), INT_CODES)
  add('group_chars', spec.group_chars, n, CHAR_CODES)
  add('drape_kind', spec.drape_kind, nd, INT_CODES)
  add('program_arg', spec.program_arg, 8, INT_CODES)
  add('sprite_group', spec.sprite_group, ns, INT_CODES)
  add('drape_group', spec.drape_group, nd, INT_CODES)
  return out


def _create(lib, spec):
  h = C.c_void_p()
  status = lib.pcl_create(C.byref(spec), 4, -1, C.byref(h))
  if status == _lib.OK:
    lib.pcl_destroy(h)
  return status


def _copy(spec):
  return _lib.Spec.from_buffer_copy(spec)


def _state_slots():
  """(label, setter(state, value)) for every pointer and every bstride of pcl_state."""
  ptrs, strides = [], []
  for name, ctype in _lib.State._fields_:
    arr = getattr(ctype, '_length_', None)
    kind = ctype._type_ if arr else ctype
    bucket = strides if kind is C.c_int64 else ptrs
    if arr:
      for i in range(arr):
        bucket.append(('%s[%d]' % (name, i),
                       lambda st, v, name=name, i=i: getattr(st, name).__setitem__(i, v)))
    else:
      bucket.append((name, lambda st, v, name=name: setattr(st, name, v)))
  return ptrs, strides


def _full_state():
  ptrs, strides = _state_slots()
  st = _lib.State()
  for _, put in ptrs:
    put(st, FAKE)
  for _, put in strides:
    put(st, STRIDE)
  return st


def _crop(rows, cols, track=None):
  spec = _lib.CropSpec(rows, cols, 0, ord(' '), rows // 2, cols // 2, 0, 0, 1)
  for i, code in enumerate(track or ()):
    spec.track[i] = code
  return spec


def level_cases(lib, name, spec):
  """{case name: status} for one lowered spec."""
  out = {}
  key = lambda case: '%s/%s' % (name, case)
  out[key('create')] = _create(lib, spec)
  for field in SCALARS:
    v = getattr(spec, field)
    for code in sorted(set((v - 1, v + 1) + SCALAR_CODES)):
      if field == 'n_groups' and code > N_GROUP_SLOTS:
        continue
      s = _copy(spec)
      setattr(s, field, code)
      out[key('spec.%s=%d' % (field, code))] = _create(lib, s)
  for k, (label, _, _, codes) in enumerate(_elements(spec)):
    for code in codes:
      s = _copy(spec)
      _, arr, i, _ = _elements(s)[k]
      arr[i] = code
      out[key('spec.%s=%d' % (label, code))] = _create(lib, s)
  for prog in PROGRAM_IDS:
    if prog == spec.program:
      continue
    s = _copy(spec)
    s.program = prog
    out[key('program=%d' % prog)] = _create(lib, s)

  h = C.c_void_p()
  assert lib.pcl_create(C.byref(spec), 4, -1, C.byref(h)) == _lib.OK, name
  try:
    ptrs, strides = _state_slots()
    for label, put in ptrs + strides:
      st = _full_state()
      put(st, 0)
      out[key('bind.%s=0' % label)] = lib.pcl_bind_state(h, C.byref(st))
    out[key('bind.null')] = lib.pcl_bind_state(h, C.byref(_lib.State()))
    st = _full_state()
    out[key('bind')] = lib.pcl_bind_state(h, C.byref(st))
    crops = [('detach', None, None), ('no_out', _crop(5, 5), None),
             ('sprite', _crop(5, 5), FAKE), ('wide', _crop(255, 257), FAKE),
             ('too_wide', _crop(257, 257), FAKE),
             ('drape', _crop(5, 5, [-1]), FAKE)]
    for label, crop, d_crop in crops:
      got = lib.pcl_attach_cropper(h, C.byref(crop) if crop is not None else None, d_crop, FAKE)
      out[key('attach.%s' % label)] = got
  finally:
    lib.pcl_destroy(h)
  return out


def lowered_specs():
  """(name, spec) of every level, in a fixed order."""
  return [(name, lowering.lower(make()).make_spec(True)) for name, make in _games()]


def sweep():
  """{case name: status} over every level, with the library `_lib` loads."""
  lib = _lib.load()
  out = {}
  for name, spec in lowered_specs():
    out.update(level_cases(lib, name, spec))
  return out


# The golden file's form: per level, one character per case, in sweep order.
STATUS_CHARS = {_lib.OK: '.', _lib.ERR_INVALID: 'i', _lib.ERR_UNSUPPORTED: 'u',
                _lib.ERR_CUDA: 'c', _lib.ERR_UNBOUND: 'b', _lib.ERR_NOMEM: 'm'}


def encode(statuses):
  """{level: status characters} of a {case name: status} sweep."""
  out = {}
  for case, status in statuses.items():
    level = case.split('/')[0]
    out[level] = out.get(level, '') + STATUS_CHARS[status]
  return out


def decode(encoded, names):
  """{case name: status} of `encode`'s form, naming each level's cases by `names`, the
  case names of a sweep in its order."""
  status_of = dict((c, s) for s, c in STATUS_CHARS.items())
  rest = dict((level, list(chars)) for level, chars in encoded.items())
  return dict((name, status_of[rest[name.split('/')[0]].pop(0)]) for name in names)
