"""scrolly_maze_step against the oracle at every board shape it branches on.

scrolly_maze_step lays out shared memory by board shape (segments per row, W against 32
and 64, H against 32 and 64, pitch against ceil16(W), where the window corner falls in
a 64-bit word pair).  The board shapes of marauders_step and shockwave_step are swept in
test_gpu_marauders.py and test_gpu_shockwave.py.  Each case steps a BatchedEngine with auto-reset beside B
oracle worlds and compares, every step, the whole [B, H, pitch] board (pad columns must
stay 0), rewards, discounts, done flags, curtains, sprite registers and, at the end, the
error codes.  Several levels and B not a multiple of 4 give a ragged last block whose
warps hold different state, so a write into a neighbouring warp's shared memory shows
up as a wrong board.
"""

import numpy as np
import pytest

import scrolly_shapes as ss
from oracle import engine_model as em
from oracle import games as ogames
from oracle import sampled_check

pytestmark = pytest.mark.gpu


def _torch():
  import torch
  return torch


def _step_vs_oracle(games, make_oracle, actions, check_curtains, sprite_chars, rng_seed=0,
                    on_step=None, crop=None):
  """Step a BatchedEngine (auto-reset) and B oracle worlds in lockstep; compare everything.

  games: lowered games or facade Engines (env e plays games[e % len(games)]).
  on_step: sampled_check.lockstep's hook.  crop: (spec, make_crop()) to attach a cropper
  to the step kernel and compare its view every step too."""
  from pycolab_b200 import batched
  B = actions.shape[1]
  eng = batched.BatchedEngine(games, batch=B, rng_seed=rng_seed)
  assert eng._board.shape == (B, eng.rows, eng.pitch)
  if crop is not None:
    view = eng.attach_cropper(crop[0])
    assert eng._attached[3], 'the cropper runs inside the step kernel'
    crop = (view, None, crop[1])
  eng.its_showtime()
  sampled_check.lockstep(eng, make_oracle, range(B), actions, crop=crop, curtains=check_curtains,
                         sprites=sprite_chars, pad_columns=True, on_step=on_step)
  assert int(eng.error_codes().abs().max()) == 0
  return eng


def _walk(seed, T, B):
  """Walks that drift east in even envs and west in odd ones, so windows scroll far."""
  rs = np.random.RandomState(seed)
  east = rs.choice(5, size=(T, B), p=[.15, .15, .15, .45, .1])
  west = rs.choice(5, size=(T, B), p=[.15, .15, .45, .15, .1])
  return np.where(np.arange(B) % 2 == 0, east, west)


def _scrolly_case(name, B=10, T=150, n_levels=3, pitch=None, min_pattern_words=False,
                  corners=None, on_step=None, crop=None, shape=None):
  """shape: (board, world, margins) for a case not in scrolly_shapes.SHAPES."""
  board, world, margins = shape or ss.SHAPE[name]
  arts = [ss.open_level(40 + i, board, world, corner=None if corners is None else corners[i])
          for i in range(n_levels)]
  games = [ss.lowered(ss.facade_game(*a, margins=margins), pitch, min_pattern_words) for a in arts]
  return _step_vs_oracle(
      games, lambda e: ss.oracle_world(*arts[e % n_levels], margins=margins),
      _walk(len(name), T, B), '#@', 'Pabc', on_step=on_step, crop=crop)


@pytest.mark.parametrize('name', ['4x6', '5x16', '7x17', '11x33', '12x48', '13x49', '9x63',
                                  '33x63', '65x64', '33x33', '11x33_nomargins'])
def test_scrolly_board_shapes(name):
  """1, 2, 3 and 4 segments per row; partial high halves (W = 49..63); narrow boards
  with a ragged last round of rows and a third round; margins None on both drapes."""
  _scrolly_case(name, B=10 if ss.SHAPE[name][0][0] < 40 else 6)


def _dirty_shared_memory():
  """Shared memory is not cleared between launches: step one full wave of 64x64 boards
  first, so words a kernel forgets to write hold stale non-zero bytes, not zeros."""
  from pycolab_b200 import batched, levels
  from pycolab_b200.games import scrolly_maze
  torch = _torch()
  eng = batched.BatchedEngine([scrolly_maze.make_game(*levels.scrolly_maze_level(0))], batch=4096)
  eng.its_showtime()
  eng.play(torch.full((4096,), 3, dtype=torch.int32, device='cuda'))
  torch.cuda.synchronize()


@pytest.mark.parametrize('name,pitch', [('20x20', 80), ('64x64', 80), ('33x33', 64)])
def test_scrolly_pitch_wider_than_the_board(name, pitch):
  """pitch > ceil16(W): the general path on a narrow board (its pad segments are
  written as 0) and spare segments on the narrow path."""
  _dirty_shared_memory()
  if name == '64x64':
    from pycolab_b200 import levels
    from pycolab_b200.games import scrolly_maze
    arts = [levels.scrolly_maze_level(60 + i, world_shape=(97, 97)) for i in range(2)]
    games = [ss.lowered(scrolly_maze.make_game(*a), pitch) for a in arts]
    _step_vs_oracle(games, lambda e: ogames.make_scrolly_maze(arts[e % 2][0], arts[e % 2][1], '+',
                                                              arts[e % 2][2]),
                    _walk(64, 100, 6), '#@', 'Pabc')
  else:
    _scrolly_case(name, pitch=pitch)


def test_scrolly_window_corner_crosses_word_boundaries():
  """Windows whose corner starts left of columns 32, 64 and 96 and walks across them:
  both halves of the staged 64-bit word pair (wsh & 32) and many shifts within it."""
  seen = set()

  def record(t, eng, worlds, outs):
    seen.update((eng.drapes[:, 0, 1].cpu().numpy() & 63).tolist())
  _scrolly_case('12x20_sweep', B=10, T=150, corners=[(5, 20), (5, 56), (5, 84)], on_step=record,
                shape=((12, 20), (22, 161), ss.DEFAULT_MARGINS))
  assert any(v < 32 for v in seen) and any(v >= 32 for v in seen), sorted(seen)
  assert len(seen) >= 16, sorted(seen)


@pytest.mark.parametrize('name', ['12x24_walls_only', '12x24_coins_only'])
def test_scrolly_different_margins_per_drape(name):
  """'#' and '@' with different margins (one of them None).  In the reference the '@'
  drape never issues an order of its own here: it runs after the player, whose motion
  permits are by then for the next frame.  So both corners stay equal, and the kernel's
  restage of the coin window never runs; the registers must say so."""
  def same_corners(t, eng, worlds, outs):
    d = eng.drapes.cpu().numpy()
    np.testing.assert_array_equal(d[:, 0, :2], d[:, 1, :2])
    for e, w in worlds.items():
      assert tuple(d[e, 0, :2]) == w.things['#'].corner == w.things['@'].corner
  _scrolly_case(name, corners=[(5, 52), (5, 60), (5, 20)], on_step=same_corners)


def test_scrolly_one_column_board():
  """W = 1 with margins None, pattern_words at the minimum pcl_create accepts (6 words for
  a 41-column world: the narrow path stages 4 words per row from an even word)."""
  _scrolly_case('9x1_nomargins', min_pattern_words=True)


@pytest.mark.parametrize('name,pitch,rows,cols,pad', [
    ('5x16', None, 9, 22, ' '), ('5x16', None, 5, 16, None),
    ('11x33', None, 15, 39, ' '), ('11x33', None, 11, 33, None),
    ('20x20', 80, 24, 26, ' '), ('20x20', 80, 20, 20, None)])
def test_scrolly_attached_cropper_board_shapes(name, pitch, rows, cols, pad):
  """pcl_attach_cropper vs the oracle's ScrollingCropper: a crop larger than the board
  with a pad character, and one equal to the board without one."""
  from pycolab_b200 import batched
  margins = (1, 1)
  spec = batched.scrolling_crop_spec(rows, cols, 0, pad_char=pad, scroll_margins=margins)

  def make_crop():
    return em.ScrollingCrop(rows, cols, ['P'], pad_char=pad, scroll_margins=margins)
  _scrolly_case(name, B=7, T=100, pitch=pitch, crop=(spec, make_crop))
