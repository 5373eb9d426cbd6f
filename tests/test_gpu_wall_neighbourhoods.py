"""scrolly_maze_step reads each walker's 5x5 wall patch as one word of a per-level table
that the handle builds from the bound wall pattern before its first launch after each
pcl_bind_state (scrolly_maze.cu, "Wall neighbourhoods").

The table is held against a NumPy statement of its rule at every centre, margins
included; a lock-step after the host rewrites the walls around the walkers and binds
again shows that the kernel reads the rebuilt table.
"""

import ctypes as C

import numpy as np
import pytest

import scrolly_shapes as ss
from oracle import sampled_check
from test_gpu_shapes import _walk

pytestmark = pytest.mark.gpu


def _table_rule(words, PH, PW):
  """Word (pr + 2, pc + 2), bit (dr + 2) * 5 + dc + 2 = the wall at (pr + dr, pc + dc),
  for pr in [-2, PH + 2), pc in [-2, PW + 2): rows outside the pattern, negative
  columns and columns past the row's words read 0; columns in [PW, 32 PWW) read the
  row's words as they are."""
  PWW = words.shape[1]
  bits = np.unpackbits(np.ascontiguousarray(words, dtype='<u4').view(np.uint8),
                       bitorder='little').reshape(PH, 32 * PWW)
  padded = np.zeros((PH + 8, 32 * PWW + 8), dtype=np.uint32)
  padded[4:4 + PH, 4:4 + 32 * PWW] = bits
  table = np.zeros((PH + 4, PW + 4), dtype=np.uint32)
  for dr in range(5):
    for dc in range(5):
      table |= padded[dr:dr + PH + 4, dc:dc + PW + 4] << np.uint32(dr * 5 + dc)
  return table


def _device_table(patterns, PW):
  """pcl_scrolly_wall_neighbourhoods over u32 [copies, PH, PWW] patterns."""
  import torch
  from pycolab_b200 import _lib
  lib = _lib.load()
  fn = lib.pcl_scrolly_wall_neighbourhoods
  fn.argtypes = [C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_int64, C.c_void_p]
  fn.restype = C.c_int
  copies, PH, PWW = patterns.shape
  src = torch.from_numpy(patterns.view(np.int32)).cuda()
  dst = torch.full((copies, PH + 4, PW + 4), -1, dtype=torch.int32, device='cuda')
  assert fn(src.data_ptr(), PH * PWW, PH, PW, PWW, copies, dst.data_ptr()) == 0
  return dst.cpu().numpy().view(np.uint32)


def _level_walls(board, world, seed):
  low = ss.lowered(ss.facade_game(*ss.open_level(seed, board, world, wall_density=0.3),
                                  margins=ss.NO_MARGINS))
  return low.patterns[0], low.pattern_cols


# (board, world): a pattern width that is no multiple of 32, the one-column board, a
# board wider than 64 columns (12 words per pattern row), and a 32-column pattern.
LEVEL_CASES = {
    '11x33': ((11, 33), (25, 81)),
    '9x1': ((9, 1), (25, 41)),
    '6x80': ((6, 80), (14, 131)),
    '4x6_pw32': ((4, 6), (15, 32)),
}


@pytest.mark.parametrize('name', sorted(LEVEL_CASES))
def test_table_matches_rule_for_level_walls(name):
  """Three levels' walls, as a handle without shared levels holds them: one copy each."""
  board, world = LEVEL_CASES[name]
  levels = [_level_walls(board, world, 90 + i) for i in range(3)]
  PW = levels[0][1]
  patterns = np.stack([w for w, _ in levels])
  got = _device_table(patterns, PW)
  for i in range(3):
    np.testing.assert_array_equal(got[i], _table_rule(patterns[i], patterns.shape[1], PW))


@pytest.mark.parametrize('PH,PW,PWW', [(7, 45, 4), (5, 3, 2), (9, 130, 6), (3, 64, 4)])
def test_table_matches_rule_with_set_padding(PH, PW, PWW):
  """Random words, padding bits included: columns in [PW, 32 PWW) are read as stored."""
  rs = np.random.RandomState(PH * 1000 + PW)
  patterns = rs.randint(0, 2 ** 32, size=(2, PH, PWW), dtype=np.uint64).astype(np.uint32)
  got = _device_table(patterns, PW)
  for i in range(2):
    np.testing.assert_array_equal(got[i], _table_rule(patterns[i], PH, PW))


def _walls_changed_around_walkers(art, seed):
  """The maze art with floor and wall swapped in about half of the inner cells within 2
  of each walker's start (no sprite, coin or corner cell changes)."""
  maze, board, beneath = art
  grid = np.array([list(row) for row in maze])
  rs = np.random.RandomState(seed)
  H, W = grid.shape
  flipped = 0
  for ch in 'Pabc':
    (r0,), (c0,) = np.nonzero(grid == ch)
    for r in range(max(1, r0 - 2), min(H - 1, r0 + 3)):
      for c in range(max(1, c0 - 2), min(W - 1, c0 + 3)):
        if grid[r, c] in ' #' and rs.random_sample() < 0.5:
          grid[r, c] = '#' if grid[r, c] == ' ' else ' '
          flipped += 1
  assert flipped > 0
  return [''.join(row) for row in grid], board, beneath


def test_lockstep_after_walls_rewritten_around_walkers_and_rebound():
  """A host that rewrites the wall pattern where the walkers test it and binds again: the
  kernel steps with the new walls, in lock-step with an oracle built from them."""
  import torch
  from pycolab_b200 import _lib, batched
  board, world, margins = ss.SHAPE['11x33']
  arts = [ss.open_level(80 + i, board, world) for i in range(2)]
  changed = [_walls_changed_around_walkers(a, 7 + i) for i, a in enumerate(arts)]
  B = 8
  eng = batched.BatchedEngine([ss.lowered(ss.facade_game(*a, margins=margins)) for a in arts],
                              batch=B)
  eng.its_showtime()
  rs = np.random.RandomState(3)
  for _ in range(5):                         # step on the old walls first
    eng.play(torch.from_numpy(rs.randint(0, 5, size=B).astype(np.int32)).cuda())
  new = batched.BatchedEngine([ss.lowered(ss.facade_game(*a, margins=margins)) for a in changed],
                              batch=2)
  assert not torch.equal(eng.patterns[0], new.patterns[0])
  eng.patterns[0].copy_(new.patterns[0])
  _lib.check(eng._lib.pcl_bind_state(eng._h, C.byref(eng._state)), 'pcl_bind_state')
  eng.reset()
  sampled_check.lockstep(eng, lambda e: ss.oracle_world(*changed[e % 2], margins=margins), range(B),
                         _walk(11, 60, B), curtains='#@', sprites='Pabc')
  assert int(eng.error_codes().abs().max()) == 0
