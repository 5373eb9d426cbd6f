"""The croppers without a GPU.

- The oracle's ScrollingCrop / crop_window against the reference's own
  `cropping.ScrollingCropper` / `FixedCropper`, driven over every case of
  `crop_cases.CASES` on a duck-typed engine: board, every layer (un-occluded, so the pad
  fill of each layer counts) and the window corner, every frame.
- Constructor and set_engine refusals of the facade classes and of
  `batched.scrolling_crop_spec` against the reference's.
- C-boundary statuses of every cropper entry point for windows of more than
  PCL_MAX_CROP_CELLS cells and for drape tracking past 128 rows or columns, on handles
  that reach no device (device -1, made-up addresses): each is refused before anything
  is enqueued, pcl_step_host_async included.
"""

import ctypes as C

import numpy as np
import pytest

import boundary_sweep
import crop_cases as cc
import refdriver
from pycolab_b200 import _lib
from pycolab_b200.errors import NotLoweredError

_Engine = cc.RefEngine


@pytest.mark.skipif(not refdriver.available(), reason='needs the reference pycolab')
@pytest.mark.parametrize('name', [c['name'] for c in cc.CASES])
def test_oracle_matches_the_reference(name):
  cropping = refdriver._import()['cropping']
  c = cc.BY_NAME[name]
  seq = cc.frames(c)
  envs = range(min(c['B'], 5))
  for k, cropper in enumerate(c['croppers']):
    want = cc.oracle(c, cropper, seq, envs, with_layers=True)
    got = cc.reference(cropping, c, cropper, seq, envs)
    _same(want, got, '%s cropper %d' % (name, k), corners=cropper['kind'] == 'scroll')


def _same(want, got, what, corners=True):
  for t, (w, g) in enumerate(zip(want, got)):
    msg = '%s t=%d' % (what, t)
    np.testing.assert_array_equal(g[0], w[0], err_msg=msg)
    if corners:
      np.testing.assert_array_equal(g[1], w[1], err_msg=msg + ' corner')
    for e, (wl, gl) in enumerate(zip(w[2], g[2])):
      assert set(wl) == set(gl), msg
      for ch in wl:
        np.testing.assert_array_equal(gl[ch], wl[ch], err_msg='%s env %d %s' % (msg, e, ch))


@pytest.mark.parametrize('name', cc.golden_names())
def test_oracle_matches_the_reference_goldens(name):
  """The reference's own crops, frozen: the oracle must give them on any machine."""
  c, seq, want = cc.load_golden(name)
  for k, cropper in enumerate(c['croppers']):
    got = cc.oracle(c, cropper, seq, with_layers=True)
    _same(want[k], got, '%s cropper %d' % (name, k))


def test_the_grid_covers_its_axes():
  """Every value of every axis the grid promises is in some case."""
  boards = set((c['H'], c['W']) for c in cc.CASES)
  assert boards >= {(1, 1), (1, 37), (37, 1), (5, 7), (8, 14), (31, 33), (32, 32), (33, 65),
                    (64, 64), (100, 127), (128, 128)}
  crops = [(c, k) for c in cc.CASES for k in c['croppers']]
  windows = set((k['rows'], k['cols']) for _, k in crops)
  assert windows >= {(1, 1), (1, 5), (3, 5), (4, 6), (5, 7), (9, 9), (255, 257)}
  assert any((k['rows'], k['cols']) == (c['H'], c['W']) for c, k in crops)
  assert any(k['rows'] > c['H'] and k['cols'] > c['W'] for c, k in crops)
  scrolls = [(c, k) for c, k in crops if k['kind'] == 'scroll']
  assert any(k['margins'] == (0, 0) for _, k in scrolls)
  assert any(None in k['margins'] and k['margins'] != (None, None) for _, k in scrolls)
  assert any(k['margins'] == (None, None) for _, k in scrolls)
  assert any(k['margins'] == ((k['rows'] - 1) // 2, (k['cols'] - 1) // 2) and k['rows'] > 1
             for _, k in scrolls)
  assert set(str(k['offset']) for _, k in scrolls) >= {'None', '(2, -3)', '(-45, 0)'}
  assert set(k['saccade'] for _, k in scrolls) == {True, False}
  assert set(k['pad'] for _, k in crops) == {None, 'backdrop', 'sprite'}
  tracks = [k['track'] for _, k in scrolls]
  assert ['s0'] in tracks and ['d0'] in tracks and ['s0', 'd0'] in tracks
  assert any(len(t) == 4 and {n[0] for n in t} == {'s', 'd'} for t in tracks)
  assert set(c['B'] for c in cc.CASES) >= {1, 5, 4099}
  assert set(k['state'] for _, k in scrolls) == {'own', 'plot'}
  assert any(c['bump'] for c in cc.CASES) and any(len(c['croppers']) > 1 for c in cc.CASES)
  assert any(c['bump'] and k['state'] == 'plot' for c, k in scrolls)


# ---- constructor refusals --------------------------------------------------------

@pytest.mark.skipif(not refdriver.available(), reason='needs the reference pycolab')
@pytest.mark.parametrize('rows,cols,margins', [
    (4, 5, (None, 2)), (5, 6, (1, None)), (4, 6, (None, None)),     # even window, None margin
    (5, 7, (2, 3)), (5, 7, (3, 2)), (4, 6, (2, 1)), (1, 1, (0, 0)),  # margins at the centre
    (1, 1, (1, 0)), (3, 5, (1, 2)), (9, 9, (None, None)), (6, 8, (2, 3)), (2, 2, (0, 0))])
def test_spec_refusals_match_the_reference(rows, cols, margins):
  from pycolab_b200 import batched, cropping
  ref = refdriver._import()['cropping']
  try:
    ref.ScrollingCropper(rows, cols, ['A'], scroll_margins=margins)
    refused = False
  except ValueError:
    refused = True
  if refused:
    with pytest.raises(ValueError):
      batched.scrolling_crop_spec(rows, cols, 0, scroll_margins=margins)
    with pytest.raises(ValueError):
      cropping.ScrollingCropper(rows, cols, ['A'], scroll_margins=margins)
  else:
    spec = batched.scrolling_crop_spec(rows, cols, 0, scroll_margins=margins)
    assert (spec.margin_rows, spec.margin_cols) == tuple(ref.ScrollingCropper(
        rows, cols, ['A'], scroll_margins=margins)._scroll_margins)
    cropping.ScrollingCropper(rows, cols, ['A'], scroll_margins=margins)


@pytest.mark.skipif(not refdriver.available(), reason='needs the reference pycolab')
@pytest.mark.parametrize('window,pad', [((9, 9), None), ((9, 9), '.'), ((5, 15), None),
                                        ((8, 14), None), ((9, 14), '.')])
def test_window_larger_than_the_board_needs_a_pad(window, pad):
  from pycolab_b200 import cropping
  ref = refdriver._import()['cropping']
  c = dict(H=8, W=14)
  mine = cropping.ScrollingCropper(window[0], window[1], ['A'], pad_char=pad,
                                   scroll_margins=(0, 0))
  theirs = ref.ScrollingCropper(window[0], window[1], ['A'], pad_char=pad,
                                scroll_margins=(0, 0))
  try:
    theirs.set_engine(_Engine(c))
    refused = False
  except ValueError:
    refused = True
  if refused:
    with pytest.raises(ValueError):
      mine.set_engine(_Engine(c))
  else:
    mine.set_engine(_Engine(c))


class _Batched(object):
  sprite_chars, drape_chars = 'A', 'x'


@pytest.mark.parametrize('make', ['fixed', 'scroll'])
def test_illegal_pad_character_raises_at_crop(make):
  """Upstream's _do_crop raises ValueError for a pad character the engine does not use,
  before anything is cropped; so does the facade, before it reaches the device."""
  from pycolab_b200 import cropping
  c = cc.BY_NAME['b8x14_w4x6']
  eng = _Engine(c)
  eng.show(c, cc.frames(c)[0], 0)
  eng.batched = _Batched()
  crop = (cropping.FixedCropper((0, 0), 3, 5, pad_char='~') if make == 'fixed' else
          cropping.ScrollingCropper(3, 5, ['A'], pad_char='~', scroll_margins=(0, 0)))
  crop.set_engine(eng)
  with pytest.raises(ValueError):
    crop.crop(None)


def test_tracking_an_object_character_is_not_lowered():
  """A character the engine has that is neither a sprite nor a drape of the device
  handle (e.g. a box_world key) raises NotLoweredError naming it, not list.index's
  ValueError."""
  from pycolab_b200 import cropping
  c = cc.BY_NAME['b8x14_w4x6']
  eng = _Engine(c)
  eng.show(c, cc.frames(c)[0], 0)
  eng.things['k'] = object()
  eng.batched = _Batched()
  crop = cropping.ScrollingCropper(3, 5, ['k', 'A'], scroll_margins=(0, 0))
  crop.set_engine(eng)
  with pytest.raises(NotLoweredError, match="'k'"):
    crop.crop(None)


# ---- C boundary --------------------------------------------------------------------

def _none_handle(H, W, S=2, D=2):
  lib = _lib.load()
  spec = _lib.Spec()
  spec.abi_version, spec.program = _lib.ABI_VERSION, _lib.PROG_NONE
  spec.rows, spec.cols, spec.pitch = H, W, cc.pitch(W)
  spec.n_sprites, spec.n_drapes = S, D
  h = C.c_void_p()
  assert lib.pcl_create(C.byref(spec), 4, -1, C.byref(h)) == _lib.OK
  assert lib.pcl_bind_state(h, C.byref(boundary_sweep._full_state())) == _lib.OK
  return lib, h


def _scrolly_handle():
  from pycolab_b200 import levels, lowering
  from pycolab_b200.games import scrolly_maze
  art = levels.scrolly_maze_level(3, world_shape=(33, 33), board_shape=(16, 16))
  spec = lowering.lower(scrolly_maze.make_game(*art)).make_spec(True)
  lib = _lib.load()
  h = C.c_void_p()
  assert lib.pcl_create(C.byref(spec), 4, -1, C.byref(h)) == _lib.OK
  assert lib.pcl_bind_state(h, C.byref(boundary_sweep._full_state())) == _lib.OK
  return lib, h


def _spec(rows, cols, track=None, pad='.'):
  from pycolab_b200 import batched
  return batched.scrolling_crop_spec(rows, cols, 0, pad_char=pad, scroll_margins=(0, 0),
                                     track=track)


FAKE = boundary_sweep.FAKE


def _step_host_async(lib, h, spec):
  out = _lib.Outputs(FAKE, FAKE, FAKE, FAKE, FAKE)
  return lib.pcl_step_host_async(h, FAKE, FAKE, C.byref(out), C.byref(spec), FAKE, FAKE, FAKE,
                                 FAKE, FAKE, FAKE, FAKE, 0, None)


def _calls(lib, h, spec):
  """{entry point: status} of every cropper entry point for `spec`, which every one of them
  must refuse: a spec one of them accepts would launch on the made-up addresses (device -1
  only means the handle selects no device; where a GPU is present the launch runs on the
  current one)."""
  curtains = (C.c_void_p * _lib.MAX_TRACK)(*([FAKE] * _lib.MAX_TRACK))
  out = _lib.Outputs(FAKE, FAKE, FAKE, FAKE, FAKE)
  x = _lib.HandoffState()
  x.n_peers, x.rank, x.record_bytes, x.rows, x.first_row = 1, 0, 256, 4, 0
  x.d_peer_base[0], x.d_peer_flags[0], x.d_local = FAKE, FAKE, FAKE
  got = {}
  if not any(code < 0 for code in spec.track):
    got['pcl_crop'] = lib.pcl_crop(h, C.byref(spec), FAKE, FAKE, FAKE, None)
  got['pcl_crop_tracking'] = lib.pcl_crop_tracking(h, C.byref(spec), FAKE, FAKE, FAKE,
                                                   curtains, None)
  got['pcl_crop_handoff'] = lib.pcl_crop_handoff(h, C.byref(spec), FAKE, FAKE, C.byref(out),
                                                 C.byref(x), None)
  got['pcl_step_host_async'] = _step_host_async(lib, h, spec)
  return got


@pytest.mark.parametrize('window', [(256, 256), (257, 256), (65536, 1), (1, 65536),
                                    (300, 300)], ids=str)
def test_windows_past_the_cell_limit_are_unsupported_everywhere(window):
  """More than PCL_MAX_CROP_CELLS cells: PCL_ERR_UNSUPPORTED from every entry point,
  before any launch (a launch would fail with a CUDA error instead)."""
  for track in (None, [1], [-1, 2]):
    lib, h = _none_handle(16, 16)
    try:
      got = _calls(lib, h, _spec(window[0], window[1], track))
    finally:
      lib.pcl_destroy(h)
    assert set(got.values()) == {_lib.ERR_UNSUPPORTED}, (track, got)
  lib, h = _scrolly_handle()
  try:
    spec = _spec(window[0], window[1])
    assert lib.pcl_attach_cropper(h, C.byref(spec), FAKE, FAKE) == _lib.ERR_UNSUPPORTED
    spec = _spec(255, 257)                          # 65 535 cells: the largest accepted
    assert lib.pcl_attach_cropper(h, C.byref(spec), FAKE, FAKE) == _lib.OK
  finally:
    lib.pcl_destroy(h)


@pytest.mark.parametrize('shape', [(129, 8), (8, 129), (129, 129)], ids=str)
def test_drape_tracking_past_128_rows_or_columns_is_unsupported(shape):
  lib, h = _none_handle(*shape)
  try:
    for track in ([-1], [1, -2], [-2, 1, -1, 2]):
      spec = _spec(5, 7, track)
      got = lib.pcl_crop_tracking(h, C.byref(spec), FAKE, FAKE, FAKE,
                                  (C.c_void_p * _lib.MAX_TRACK)(*([FAKE] * 4)), None)
      assert got == _lib.ERR_UNSUPPORTED, track
  finally:
    lib.pcl_destroy(h)


@pytest.mark.parametrize('track', [[-1], [1, -1], [2, 1, -2, -1]], ids=str)
def test_step_host_async_refuses_drape_tracking_before_the_step(track):
  """pcl_step_host_async passes no curtains: a tracking list naming a drape is refused
  with PCL_ERR_UNSUPPORTED before the step is enqueued (here: before the device -1
  handle would fail to create its copy stream).  pcl_crop_tracking accepts the same spec,
  so it is not called here: it would launch on the made-up addresses."""
  lib, h = _none_handle(16, 16)
  try:
    assert _step_host_async(lib, h, _spec(5, 7, track)) == _lib.ERR_UNSUPPORTED
    bad = _spec(5, 7, [3])                                      # no sprite 2
    assert set(_calls(lib, h, bad).values()) == {_lib.ERR_INVALID}
  finally:
    lib.pcl_destroy(h)
