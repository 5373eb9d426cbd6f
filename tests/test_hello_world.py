"""examples/hello_world.py (SURVEY.md §8f-4): plain wrapping Sprites + a rolling
Drape.  The replays of its goldens (tests/golden/hello_stock_*) are in
test_example_goldens.py and test_gpu_example_goldens.py; here a batched lockstep and
lowering."""

import os

import numpy as np
import pytest

import refdriver
from oracle import games as ogames
from oracle import sampled_check


@pytest.mark.gpu
def test_batched_hello_vs_oracle():
  from pycolab_b200 import batched
  from pycolab_b200.games import hello_world
  art = hello_world.HELLO_ART
  B, T = 19, 200
  eng = batched.BatchedEngine([hello_world.make_game(art)], batch=B)
  eng.its_showtime()
  rs = np.random.RandomState(8)
  actions = np.stack([rs.choice([0, 1, 2, 3, 4, 5], size=B, p=[.23, .23, .23, .23, .03, .05])
                      for _ in range(T)]).astype(np.int32)
  sampled_check.lockstep(eng, lambda e: ogames.make_hello(art), range(B), actions, curtains='@')
  assert int(eng.error_codes().abs().max()) == 0


@pytest.mark.skipif(not refdriver.available(), reason='/root/reference not present')
def test_reference_hello_world_file_lowers_like_the_twin():
  import sys
  from pycolab_b200 import compat, lowering
  from pycolab_b200.games import hello_world
  saved = {k: v for k, v in sys.modules.items() if k == 'pycolab' or k.startswith('pycolab.')}
  compat.uninstall()
  try:
    mod = compat.load_example(os.path.join(refdriver.REFERENCE_ROOT, 'pycolab', 'examples',
                                           'hello_world.py'))
    a, b = lowering.lower(mod.make_game()), lowering.lower(hello_world.make_game())
    assert a.signature() == b.signature()
    for field in ('backdrop', 'sprites', 'drapes', 'plot'):
      np.testing.assert_array_equal(getattr(a, field), getattr(b, field), err_msg=field)
    np.testing.assert_array_equal(a.bits[0], b.bits[0])
  finally:
    compat.uninstall()
    sys.modules.update(saved)
