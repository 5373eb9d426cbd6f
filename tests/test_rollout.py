"""Rollouts (`pcl_rollout`, `BatchedEngine.rollout`) without a GPU.

- The ctypes mirror of `pcl_rollout_rec` against include/pcl.h: the same fields in the
  same order, and the size the library reports.
- C-boundary refusals on handles that reach no device (device -1, made-up addresses):
  each is refused, with the status of the single entry point, before anything is enqueued.
- The facade's refusals that need no device: a rollout before its_showtime(), observers
  that are not post-processors, and feature planes of games whose layers are not the
  occluded board.
"""

import ctypes as C
import os
import re

import pytest

import boundary_sweep
from pycolab_b200 import _lib

FAKE = boundary_sweep.FAKE
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_ctypes_mirror_matches_the_header():
  with open(os.path.join(ROOT, 'include', 'pcl.h')) as f:
    header = f.read()
  body = re.search(r'typedef struct pcl_rollout_rec \{(.*?)\} pcl_rollout_rec;', header, re.S)
  names = re.findall(r'(\w+);', body.group(1))
  assert names == [name for name, _ in _lib.RolloutRec._fields_]
  lib = _lib.load()
  assert lib.pcl_rollout_rec_size() == C.sizeof(_lib.RolloutRec) == 17 * 8


def _handle(program=_lib.PROG_NONE, spec=None, bind=True):
  lib = _lib.load()
  if spec is None:
    spec = _lib.Spec()
    spec.abi_version, spec.program = _lib.ABI_VERSION, program
    spec.rows, spec.cols, spec.pitch = 16, 16, 16
    spec.n_sprites, spec.n_drapes = 2, 2
  h = C.c_void_p()
  assert lib.pcl_create(C.byref(spec), 4, -1, C.byref(h)) == _lib.OK
  if bind:
    assert lib.pcl_bind_state(h, C.byref(boundary_sweep._full_state())) == _lib.OK
  return lib, h


def _outputs():
  return _lib.Outputs(FAKE, FAKE, FAKE, FAKE, FAKE, FAKE)


def _crop(rows=5, cols=7, track=None, sprite=0):
  spec = _lib.CropSpec(rows, cols, sprite, ord(' '), 1, 1, 0, 0, 1)
  for i, code in enumerate(track or ()):
    spec.track[i] = code
  return spec


def _observing(depth=3, dtype=2, crop=None, view=FAKE, table=FAKE):
  """A record with an observer; the specs are kept alive by the record's owner dict."""
  spec = _lib.ObserveSpec(depth, dtype, 3 * 35, 35, 7, 1)
  rec = _lib.RolloutRec()
  rec.observe = C.pointer(spec)
  if crop is not None:
    rec.observe_crop = C.pointer(crop)
  rec.d_table, rec.d_view, rec.view_stride_t = table, view, 4 * 3 * 35
  return rec, (spec, crop)


def _call(lib, h, rec=None, actions=FAKE, steps=3, out=None):
  out = _outputs() if out is None else out
  return lib.pcl_rollout(h, actions, steps, C.byref(out), None if rec is None else C.byref(rec),
                         None)


def test_refuses_nulls_and_negative_steps():
  lib, h = _handle()
  try:
    assert _call(lib, h, actions=None) == _lib.ERR_INVALID
    assert _call(lib, h, steps=-1) == _lib.ERR_INVALID
    assert _call(lib, h, rec=_lib.RolloutRec(), steps=-1) == _lib.ERR_INVALID
    assert lib.pcl_rollout(None, FAKE, 1, C.byref(_outputs()), None, None) == _lib.ERR_INVALID
    assert lib.pcl_rollout(h, FAKE, 1, None, None, None) == _lib.ERR_INVALID
    partial = _outputs()
    partial.d_done = None
    assert _call(lib, h, out=partial) == _lib.ERR_INVALID
  finally:
    lib.pcl_destroy(h)


def test_refuses_an_unbound_handle():
  lib, h = _handle(bind=False)
  try:
    assert _call(lib, h) == _lib.ERR_UNBOUND
    assert _call(lib, h, rec=_lib.RolloutRec()) == _lib.ERR_UNBOUND
  finally:
    lib.pcl_destroy(h)


def test_refuses_observers_pcl_observe_and_pcl_crop_observe_refuse():
  lib, h = _handle()
  try:
    for depth in (0, -1):
      rec, keep = _observing(depth=depth)
      assert _call(lib, h, rec) == _lib.ERR_INVALID, depth
    for dtype in (-1, 6):
      rec, keep = _observing(dtype=dtype)
      assert _call(lib, h, rec) == _lib.ERR_INVALID, dtype
    rec, keep = _observing(table=None)
    assert _call(lib, h, rec) == _lib.ERR_INVALID
    rec, keep = _observing(view=None)
    assert _call(lib, h, rec) == _lib.ERR_INVALID
    for dtype, size in ((1, 4), (2, 4), (3, 8), (4, 8), (5, 2)):    # a view off its elements
      rec, keep = _observing(dtype=dtype, view=FAKE + size // 2)
      assert _call(lib, h, rec) == _lib.ERR_INVALID, dtype
    rec, keep = _observing(crop=_crop(4, 6, [3]))                    # no sprite 2
    assert _call(lib, h, rec) == _lib.ERR_INVALID
    rec, keep = _observing(crop=_crop(256, 256))                     # past the cell limit
    assert _call(lib, h, rec) == _lib.ERR_UNSUPPORTED
    for track in ([-1], [1, -2]):                                    # curtains per step
      rec, keep = _observing(crop=_crop(5, 7, track))
      assert _call(lib, h, rec) == _lib.ERR_UNSUPPORTED, track
  finally:
    lib.pcl_destroy(h)


def test_refuses_croppers_after_the_step():
  lib, h = _handle()
  try:
    rec = _lib.RolloutRec()
    rec.d_attached = FAKE                                            # no cropper at all
    assert _call(lib, h, rec) == _lib.ERR_INVALID
    for track in ([-1], [2, -1]):
      spec = _crop(5, 7, track)
      rec = _lib.RolloutRec()
      rec.crop, rec.d_crop = C.pointer(spec), FAKE
      assert _call(lib, h, rec) == _lib.ERR_UNSUPPORTED, track
    spec = _crop()
    rec = _lib.RolloutRec()
    rec.crop = C.pointer(spec)                                       # no view buffer
    assert _call(lib, h, rec) == _lib.ERR_INVALID
    wide = _crop(300, 300)
    rec.crop, rec.d_crop = C.pointer(wide), FAKE
    assert _call(lib, h, rec) == _lib.ERR_UNSUPPORTED
  finally:
    lib.pcl_destroy(h)


def _t_maze_spec():
  from pycolab_b200 import lowering
  return lowering.lower(boundary_sweep._t_maze()).make_spec(True)


def test_float_rewards_need_the_float64_slots():
  lib = _lib.load()
  h = C.c_void_p()
  assert lib.pcl_create(C.byref(_t_maze_spec()), 4, -1, C.byref(h)) == _lib.OK
  try:
    status = lib.pcl_bind_state(h, C.byref(boundary_sweep._full_state()))
    assert status == _lib.OK
    rec = _lib.RolloutRec()
    rec.d_reward = FAKE                                  # kept, but as int32
    assert _call(lib, h, rec) == _lib.ERR_INVALID
    out = _outputs()
    out.d_reward_f64 = None                              # as pcl_step refuses it
    assert _call(lib, h, out=out) == _lib.ERR_INVALID
  finally:
    lib.pcl_destroy(h)


# ---- facade --------------------------------------------------------------------------

def _bare_engine(game):
  """A BatchedEngine with the attributes the refusals read, built without a device."""
  from pycolab_b200 import batched, lowering
  eng = batched.BatchedEngine.__new__(batched.BatchedEngine)
  eng.game = lowering.lower(game)
  eng.chars = ''.join(sorted(set(eng.game.sprite_chars + eng.game.drape_chars +
                                 eng.game.backdrop_chars)))
  eng._showtime, eng._tables, eng._h = False, None, C.c_void_p()
  return eng


def test_rollout_before_its_showtime_raises():
  from pycolab_b200.games.classics import four_rooms
  eng = _bare_engine(four_rooms.make_game())
  with pytest.raises(RuntimeError, match='its_showtime'):
    eng.rollout(None)


def test_observer_must_be_a_post_processor():
  from pycolab_b200.games.classics import four_rooms
  eng = _bare_engine(four_rooms.make_game())
  with pytest.raises(TypeError):
    eng._rollout_observer(lambda observation: observation, None)


def test_feature_planes_need_occluded_board_layers():
  from pycolab_b200 import rendering
  from pycolab_b200.errors import NotLoweredError
  from pycolab_b200.games import fixtures
  walkers = {'P': dict(impassable='', confined=False, egocentric=False)}
  art = ['.....', '.P.%.', '.....']
  unoccluded = _bare_engine(fixtures.make_game(art, '.', walkers, drapes='%',
                                               occlusion_in_layers=False))
  hooked = _bare_engine(boundary_sweep._t_maze())
  for eng in (unoccluded, hooked):
    assert not eng.game.occlusion_in_layers or eng.game.layers is not None
    for crop in (None, _crop()):
      with pytest.raises(NotLoweredError):
        eng._rollout_observer(rendering.ObservationToFeatureArray('P.'), crop)
