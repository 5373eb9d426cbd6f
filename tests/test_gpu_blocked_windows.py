"""scrolly_maze_step's wall and coin windows come from row-blocked copies of the wall
pattern and the coin template, which the handle builds from the bound state before its
first launch after each pcl_bind_state (scrolly_maze.cu, "Row-blocked windows").

Every board shape is stepped against the oracle in test_gpu_shapes.py; these cases cover
what only the copies add: copies per env when nothing is shared, and static data that
the host rewrites and binds again.
"""

import ctypes as C

import pytest

import scrolly_shapes as ss
from oracle import sampled_check
from test_gpu_shapes import _walk

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('name', ['20x20', '33x63', '65x64', '12x24_walls_only'])
def test_share_levels_false(name):
  """Every array per env and no level index: one blocked copy per env."""
  from pycolab_b200 import batched
  board, world, margins = ss.SHAPE[name]
  arts = [ss.open_level(60 + i, board, world, coin_density=0.4) for i in range(3)]
  games = [ss.lowered(ss.facade_game(*a, margins=margins)) for a in arts]
  B = 9
  eng = batched.BatchedEngine(games, batch=B, share_levels=False)
  assert eng.level is None
  eng.its_showtime()
  sampled_check.lockstep(eng, lambda e: ss.oracle_world(*arts[e % 3], margins=margins), range(B),
                         _walk(len(name), 80, B), curtains='#@', sprites='Pabc', pad_columns=True)
  assert int(eng.error_codes().abs().max()) == 0


def test_rewritten_wall_pattern_is_read_again_after_rebinding():
  """A host that rewrites the static wall pattern and binds the state again: the next
  step paints the new walls; binding the original back brings the old board back."""
  import torch
  from pycolab_b200 import _lib, batched
  board, world, margins = ss.SHAPE['11x33']
  arts = [ss.open_level(70 + i, board, world) for i in range(2)]
  games = [ss.lowered(ss.facade_game(*a, margins=margins)) for a in arts]
  B = 6
  eng = batched.BatchedEngine(games, batch=B)
  eng.its_showtime()
  torch.cuda.synchronize()
  first = eng._board.clone()
  assert int((first == ord('#')).sum()) > 0
  walls = eng.patterns[0]
  original = walls.clone()

  def rebind_and_repaint():
    _lib.check(eng._lib.pcl_bind_state(eng._h, C.byref(eng._state)), 'pcl_bind_state')
    eng.reset()
    torch.cuda.synchronize()
    return eng._board.clone()

  walls.zero_()
  bare = rebind_and_repaint()
  assert int((bare == ord('#')).sum()) == 0
  walls.copy_(original)
  assert torch.equal(rebind_and_repaint(), first)
