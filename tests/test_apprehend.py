"""examples/apprehend.py (SURVEY.md §8f-4): two MazeWalkers, a float64 accumulator and
one draw from Python's `random` per episode.  The replays of its goldens
(tests/golden/apprehend_stock_*: 30 episodes each, `random.seed` fixed) are in
test_example_goldens.py and test_gpu_example_goldens.py; here a batched lock-step whose
slopes are drawn ON THE DEVICE from per-env MT19937 states, and lowering."""

import os
import random

import numpy as np
import pytest

import refdriver
from oracle import games as ogames
from oracle import sampled_check


@pytest.mark.gpu
def test_batched_apprehend_device_rng_vs_oracle():
  """Auto-resetting batch: env e's slopes come from random.Random(seed + e), drawn by
  the kernel at every restart; boards, rewards, float registers bit-exact."""
  from pycolab_b200 import _lib, batched
  from pycolab_b200.games import apprehend
  art = apprehend.GAME_ART
  B, T, seed = 21, 160, 40
  eng = batched.BatchedEngine([apprehend.make_game(art)], batch=B, rng_seed=seed)
  assert eng.rng is not None
  rngs = [random.Random(seed + e) for e in range(B)]
  eng.its_showtime()
  rs = np.random.RandomState(3)
  actions = np.stack([rs.randint(0, 3, size=B) for _ in range(T)]).astype(np.int32)
  episodes = [0]

  def same_floats(t, eng, worlds, outs):
    spr, plot = eng.sprites.cpu().numpy(), eng.plot.cpu().numpy()
    for e, w in worlds.items():
      ball = w.things['b']
      dx = np.array([spr[e, 1, _lib.S_AUX0], spr[e, 1, _lib.S_AUX1]], dtype='<i4').view('<f8')[0]
      acc = np.array([plot[e, _lib.P_AUX0], plot[e, _lib.P_AUX1]], dtype='<i4').view('<f8')[0]
      assert dx == ball.aux['dx'] and acc == ball.aux['acc'], (t, e, dx, ball.aux)
      episodes[0] += int(t < T and w.game_over)
  sampled_check.lockstep(eng, lambda e: ogames.make_apprehend(art, rngs[e]), range(B), actions,
                         on_step=same_floats)
  assert episodes[0] > 2 * B
  assert int(eng.error_codes().abs().max()) == 0


def test_apprehend_lowers_and_validates_on_cpu():
  from pycolab_b200 import _lib, lowering
  from pycolab_b200.games import apprehend
  random.seed(5)
  want_dx = random.Random(5).uniform(-2.499, 2.499) / 9.0
  game = lowering.lower(apprehend.make_game())
  assert game.program == _lib.PROG_APPREHEND and game.sprite_chars == 'Pb'
  assert game.needs_rng and game.rng_streams == ('python',)
  words = game.sprites[1, [_lib.S_AUX0, _lib.S_AUX1]].astype('<i4')
  assert words.view('<f8')[0] == want_dx
  import ctypes as C
  lib = _lib.load()
  handle = C.c_void_p()
  spec = game.make_spec(True)
  assert lib.pcl_create(C.byref(spec), 4, -1, C.byref(handle)) == _lib.OK
  lib.pcl_destroy(handle)
  spec.sprite_confined[0] = 0                     # a catcher that may leave the board
  assert lib.pcl_create(C.byref(spec), 4, -1, C.byref(handle)) != _lib.OK


@pytest.mark.skipif(not refdriver.available(), reason='/root/reference not present')
def test_reference_apprehend_file_lowers_like_the_twin():
  import sys
  from pycolab_b200 import compat, lowering
  from pycolab_b200.games import apprehend
  saved = {k: v for k, v in sys.modules.items() if k == 'pycolab' or k.startswith('pycolab.')}
  compat.uninstall()
  try:
    mod = compat.load_example(os.path.join(refdriver.REFERENCE_ROOT, 'pycolab', 'examples',
                                           'apprehend.py'))
    random.seed(11)
    a = lowering.lower(mod.make_game())
    random.seed(11)
    b = lowering.lower(apprehend.make_game())
    assert a.signature() == b.signature()
    for field in ('backdrop', 'sprites', 'drapes', 'plot'):
      np.testing.assert_array_equal(getattr(a, field), getattr(b, field), err_msg=field)
  finally:
    compat.uninstall()
    sys.modules.update(saved)
