"""examples/shockwave.py (SURVEY.md §8f-4): a walker, two static drapes and a ring of
fire around `np.random.randint` impact points whose update() reads the STALE board.
Goldens are the reference's own trajectories (tests/golden/shockwave_*: the stock level
and generated ones, policy-driven so that some episodes are won), replayed in
test_example_goldens.py and test_gpu_example_goldens.py; here a batched lock-step with
per-env generators, and lowering."""

import os

import numpy as np
import pytest

import golden_cases as gc
import refdriver
from oracle import games as ogames
from oracle import sampled_check


@pytest.mark.parametrize('name', gc.names('shockwave_'))
def test_goldens_hold_a_win(name):
  assert int((gc.load(name)['reward'] == 1).sum()) >= 1          # the safe-zone path


@pytest.mark.gpu
@pytest.mark.parametrize('shape', [(12, 15), (32, 64), (9, 33)])
def test_batched_shockwave_vs_oracle(shape):
  """Auto-resetting batch over several generated levels, one NumPy generator per env
  (RandomState(seed + e)), boards / curtains / rewards / discounts every step."""
  from pycolab_b200 import batched, levels
  from pycolab_b200.games import shockwave
  arts = [levels.shockwave_level(30 + i, shape[0], shape[1], 0.45) for i in range(3)]
  B, T, seed = 13, 220, 9
  eng = batched.BatchedEngine([shockwave.make_game(a) for a in arts], batch=B, rng_seed=seed)
  rngs = [np.random.RandomState(seed + e) for e in range(B)]
  eng.its_showtime()
  rs = np.random.RandomState(4)
  actions = np.stack([rs.choice([0, 1, 2, 3, 4], size=B, p=[.6, .12, .12, .12, .04])
                      for _ in range(T)]).astype(np.int32)
  episodes = [0]

  def count(t, eng, worlds, outs):
    episodes[0] += sum(w.game_over for w in worlds.values()) if t < T else 0
  sampled_check.lockstep(eng, lambda e: ogames.make_shockwave(arts[e % len(arts)], rngs[e]),
                         range(B), actions, curtains='@', on_step=count)
  assert episodes[0] > B
  assert int(eng.error_codes().abs().max()) == 0


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
