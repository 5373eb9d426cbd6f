"""examples/shockwave.py (SURVEY.md §8f-4): a walker, two static drapes and a ring of
fire around `np.random.randint` impact points whose update() reads the STALE board.
Goldens are the reference's own trajectories (tests/golden/shockwave_*: the stock level
and generated ones, policy-driven so that some episodes are won), replayed in
test_example_goldens.py and test_gpu_example_goldens.py.  Here: lowering, and the oracle
in lock-step with the live reference on the scripted rim cases (shockwave_cases.RIM) and
on open levels at every width and board shape the GPU sweep steps."""

import os

import numpy as np
import pytest

import golden_cases as gc
import refdriver
import rim_sweep as rsw
import shockwave_cases as sc
from oracle import games as ogames
from test_oracle_vs_reference import _lockstep

needs_ref = pytest.mark.skipif(not refdriver.available(), reason='/root/reference not present')


@pytest.mark.parametrize('name', gc.names('shockwave_'))
def test_goldens_hold_a_win(name):
  assert int((gc.load(name)['reward'] == 1).sum()) >= 1          # the safe-zone path


def test_shockwave_lowers_and_validates_on_cpu():
  import ctypes as C
  from pycolab_b200 import _lib, errors, levels, lowering
  from pycolab_b200.games import shockwave
  game = lowering.lower(shockwave.make_game(0))
  assert game.program == _lib.PROG_SHOCKWAVE and game.drape_chars == '@ ^'
  assert game.needs_rng and game.rng_streams == ('numpy',) and game.program_arg[0] == 2
  lib = _lib.load()
  handle = C.c_void_p()
  spec = game.make_spec(True)
  assert lib.pcl_create(C.byref(spec), 4, -1, C.byref(handle)) == _lib.OK
  lib.pcl_destroy(handle)
  spec.rows = 40                                   # one curtain row per lane: 32 rows at most
  assert lib.pcl_create(C.byref(spec), 4, -1, C.byref(handle)) != _lib.OK
  with pytest.raises(errors.NotLoweredError):
    lowering.lower(shockwave.make_game(levels.shockwave_level(0, 40, 20)))


@pytest.mark.skipif(not refdriver.available(), reason='/root/reference not present')
def test_reference_shockwave_file_lowers_like_the_twin():
  import sys
  from pycolab_b200 import compat, lowering
  from pycolab_b200.games import shockwave
  saved = {k: v for k, v in sys.modules.items() if k == 'pycolab' or k.startswith('pycolab.')}
  compat.uninstall()
  try:
    mod = compat.load_example(os.path.join(refdriver.REFERENCE_ROOT, 'pycolab', 'examples',
                                           'shockwave.py'))
    a, b = lowering.lower(mod.make_game(0)), lowering.lower(shockwave.make_game(0))
    assert a.signature() == b.signature()
    for field in ('backdrop', 'sprites', 'drapes', 'plot'):
      np.testing.assert_array_equal(getattr(a, field), getattr(b, field), err_msg=field)
    for d in range(3):
      np.testing.assert_array_equal(a.bits[d], b.bits[d])
  finally:
    compat.uninstall()
    sys.modules.update(saved)


def test_a_level_without_walls_is_not_lowered():
  """The wave's update() reads layers['='], and layers holds only the characters on the
  board: the reference raises KeyError at its_showtime() on a level with no '='.  Such a
  level is refused, with the reason."""
  from pycolab_b200 import errors, lowering
  from pycolab_b200.games import shockwave
  art = ['^^^^^', '     ', '  P  ']
  with pytest.raises(errors.NotLoweredError, match="KeyError"):
    lowering.lower(shockwave.make_game(art))
  with pytest.raises(KeyError):
    ogames.make_shockwave(art, np.random.RandomState(0)).its_showtime()
  lowering.lower(shockwave.make_game(['^^^^^', '  =  ', '  P  ']))


@needs_ref
def test_reference_raises_on_a_level_without_walls():
  with pytest.raises(KeyError):
    refdriver.ref_shockwave(['^^^^^', '     ', '  P  ']).its_showtime()


# ------------------------------------------------- the oracle against the reference

def _wave(ref, ora, t):
  """The ring's curtain and its step count."""
  np.testing.assert_array_equal(ref.things['@'].curtain, ora.things['@'].curtain,
                                err_msg='t=%d' % t)
  assert ref.things['@']._steps_since_impact == ora.things['@'].aux['steps'], t


def _pair(art, width, seed):
  """A reference game and an oracle world on one MT19937 stream from `seed`."""
  return rsw.seeded_pair(lambda: refdriver.ref_shockwave(art, width),
                         lambda rng: sc.make_world(art, rng, width), seed)


@needs_ref
@pytest.mark.parametrize('name', sorted(sc.RIM))
def test_rim_case_oracle_vs_reference(name):
  """Boards, rewards, discounts, game over, P's position and the ring, at every step of
  the scripted case and of 40 more steps of random play."""
  art, width, seed, script, edges = sc.RIM[name]
  actions = script + sc.random_actions(np.random.RandomState(len(name)), 40, 1)[:, 0].tolist()
  _lockstep(*_pair(art, width, seed), actions, check=_wave)
  rng = np.random.RandomState(seed)
  seen, _, _ = rsw.oracle_run(lambda: sc.make_world(art, rng, width), sc.Edges(), script)
  assert edges <= seen, (name, sorted(edges - seen))


@needs_ref
@pytest.mark.parametrize('shape', sc.SHAPES, ids=['%dx%d' % s for s in sc.SHAPES])
def test_open_levels_oracle_vs_reference(shape):
  """Open levels of every shape the GPU sweep steps, at every width, the first impact on
  each corner and side of the board in turn."""
  cells = sc.rim_cells(shape)
  restarts = 0
  for i, width in enumerate(sc.WIDTHS):
    art = sc.sweep_level(shape, i)
    seed = sc.impact_seed(shape, cells[i % len(cells)])
    actions = sc.random_actions(np.random.RandomState(i), 80, 1)[:, 0].tolist()
    restarts += _lockstep(*_pair(art, width, seed), actions, check=_wave)
  assert restarts > 0 or shape[0] * shape[1] == 2     # P and a wall: no episode ends


@needs_ref
@pytest.mark.parametrize('rows,cols', [(32, 64), (31, 33), (32, 15)])
def test_generated_level_board_shapes(rows, cols):
  """Generated levels up to 32 x 64 (H * W = 2048 is a power of two)."""
  from pycolab_b200 import levels
  art = levels.shockwave_level(rows + cols, rows, cols, 0.5)
  steps = 0
  for seed in range(12):
    np.random.seed(seed)
    ref = refdriver.ref_shockwave(art)
    ora = ogames.make_shockwave(art, np.random.RandomState(seed))
    r_out, o_out = ref.its_showtime(), ora.its_showtime()
    rs = np.random.RandomState(200 + seed)
    for _ in range(150):
      np.testing.assert_array_equal(r_out[0].board, o_out[0])
      np.testing.assert_array_equal(ref.things['@'].curtain, ora.things['@'].curtain)
      assert r_out[1] == o_out[1] and type(r_out[1]) is type(o_out[1])
      assert r_out[2] == o_out[2] and ref.game_over == ora.game_over
      if ref.game_over:
        break
      a = int(rs.choice([0, 1, 2, 3, 4], p=[.55, .15, .15, .1, .05]))
      r_out, o_out = ref.play(a), ora.play(a)
      steps += 1
  assert steps > 100
