"""GPU tests of scrolly_maze_step's delta rendering (scrolly_maze.cu, "Delta rendering").

A step in which neither window moves stores only the cells that can have changed, into
the board the same handle drew last.  Every case here steps two engines over the same
levels and calls: one as a user would (delta rendering wherever it applies), and a twin
whose board buffer alternates between two tensors, so that each of its steps paints the
whole board.  After every call the boards, outputs, records and coin patterns of the two
must be equal byte for byte; where the envs still follow the game, sampled envs are
stepped against the oracle as well.
"""

import ctypes as C

import numpy as np
import pytest

import scrolly_shapes as ss
from oracle import games as ogames
from oracle import sampled_check
from test_gpu_shapes import _walk

pytestmark = pytest.mark.gpu


class Pair:
  """A delta-rendering engine and its full-paint twin over the same games."""

  def __init__(self, games, B, crop=None, **kw):
    import torch
    from pycolab_b200 import batched
    self.delta = batched.BatchedEngine(games, batch=B, **kw)
    self.full = batched.BatchedEngine(games, batch=B, **kw)
    self.spare = torch.zeros_like(self.full._board)
    self.views = None
    if crop is not None:
      self.views = (self.delta.attach_cropper(crop), self.full.attach_cropper(crop))
      assert self.delta._attached[3], 'the cropper runs inside the step kernel'

  def flip(self):
    """The twin's next launch writes the other buffer: a new board epoch, a full paint.
    The other buffer gets a copy of the current boards first, for envs that do not paint
    (frozen, or left out of a masked reset)."""
    f = self.full
    self.spare.copy_(f._board)
    f._board, self.spare = self.spare, f._board
    f._out.d_board = f._board.data_ptr()

  def call(self, name, *args):
    self.flip()
    getattr(self.full, name)(*args)
    getattr(self.delta, name)(*args)
    self.check(name)

  def check(self, what):
    import torch
    torch.cuda.synchronize()
    for attr in ('_board', 'reward', 'has_reward', 'discount', 'done', 'sprites', 'drapes',
                 'plot'):
      assert torch.equal(getattr(self.delta, attr), getattr(self.full, attr)), (attr, what)
    assert torch.equal(self.delta.patterns[1], self.full.patterns[1]), ('coin pattern', what)
    if self.views is not None:
      assert torch.equal(*self.views), ('cropper view', what)

  def lockstep(self, make_world, actions, env_ids, **kw):
    """sampled_check.lockstep of the delta engine; the twin plays the same actions and
    is compared after every step.  Returns (pick-ups, restarts) of the delta engine."""
    import torch
    acts = torch.from_numpy(np.ascontiguousarray(actions, dtype=np.int32)).cuda()
    seen = {'pickups': 0, 'restarts': 0}

    def on_step(t, engine, worlds, outs):
      if t > 0:
        self.flip()
        self.full.play(acts[t - 1])
        seen['pickups'] += int(engine.has_reward.sum())
      self.check(t)
      seen['restarts'] += int(engine.done.sum())

    self.call('its_showtime')
    sampled_check.lockstep(self.delta, make_world, env_ids, actions, on_step=on_step, **kw)
    return seen


def _levels(n, world, board, density, seed0):
  from pycolab_b200 import levels
  return [levels.scrolly_maze_level(seed0 + i, world_shape=world, board_shape=board,
                                    coin_density=density) for i in range(n)]


def _games(arts):
  from pycolab_b200.games import scrolly_maze
  return [scrolly_maze.make_game(*a) for a in arts]


def _oracle(arts):
  n = len(arts)
  return lambda e: ogames.make_scrolly_maze(arts[e % n][0], arts[e % n][1], '+', arts[e % n][2])


def _random_actions(seed, T, B):
  """Mostly moves; 6 (no motion) keeps a picked-up coin stale, 5 quits and restarts."""
  p = [.19, .19, .19, .19, .16, .02, .06]
  return np.random.RandomState(seed).choice(7, size=(T, B), p=p).astype(np.int32)


@pytest.mark.parametrize('world,board,T', [((129, 129), (64, 64), 300),
                                           ((25, 25), (9, 9), 400)], ids=['bench', 'small'])
def test_random_trajectories(world, board, T):
  """Long random trajectories with pick-ups, stale coins, quits and restarts."""
  arts = _levels(4, world, board, density=0.5, seed0=1200)
  B = 64
  pair = Pair(_games(arts), B)
  seen = pair.lockstep(_oracle(arts), _random_actions(len(arts) + T, T, B), range(0, B, 5),
                       curtains='#@', sprites='Pabc')
  assert seen['pickups'] > 0 and seen['restarts'] > 0, seen


def test_share_levels_false():
  arts = _levels(3, (25, 25), (9, 9), density=0.5, seed0=1300)
  B = 9
  pair = Pair(_games(arts), B, share_levels=False)
  assert pair.delta.level is None
  seen = pair.lockstep(_oracle(arts), _random_actions(7, 300, B), range(B), curtains='#@',
                       sprites='Pabc')
  assert seen['pickups'] > 0 and seen['restarts'] > 0, seen


WIDE = ((20, 80), (34, 141), ss.DEFAULT_MARGINS)


@pytest.mark.parametrize('name', ['4x6', '20x20', '65x64', '12x24_walls_only', '12x24_coins_only',
                                  'wide_20x80'])
def test_scripted_walks_scroll_both_windows(name):
  """Walks that drift east or west, so that both windows scroll far; with margins on '#'
  only, '@' issues orders of its own (the fall-back after group 2).  20x80 is wider than
  the 4-word fast paths."""
  board, world, margins = WIDE if name == 'wide_20x80' else ss.SHAPE[name]
  arts = [ss.open_level(80 + i, board, world, coin_density=0.3) for i in range(3)]
  games = [ss.lowered(ss.facade_game(*a, margins=margins)) for a in arts]
  B = 10
  pair = Pair(games, B)
  pair.lockstep(lambda e: ss.oracle_world(*arts[e % 3], margins=margins),
                _walk(len(name), 150, B), range(B), curtains='#@', sprites='Pabc',
                pad_columns=True)


def test_crop_epilogue():
  """The cropper the step kernel runs reads the board delta rendering left behind."""
  from pycolab_b200 import batched
  arts = _levels(2, (65, 65), (32, 32), density=0.4, seed0=1400)
  B = 16
  pair = Pair(_games(arts), B, crop=batched.scrolling_crop_spec(9, 9, 0))
  pair.lockstep(_oracle(arts), _random_actions(3, 200, B), range(0, B, 3), curtains='#@',
                sprites='Pabc')


def test_frozen_envs_and_masked_reset():
  """auto_reset=False: game-over envs stay frozen, board and key untouched; pcl_reset with
  a mask restarts the selected envs only."""
  import torch
  arts = _levels(2, (25, 25), (9, 9), density=0.5, seed0=1500)
  B = 16
  pair = Pair(_games(arts), B, auto_reset=False)
  pair.call('its_showtime')
  acts = torch.from_numpy(_random_actions(11, 240, B)).cuda()
  for t in range(120):
    pair.call('play', acts[t])
  frozen = pair.delta.done.clone()
  assert bool(frozen.any()), 'no env reached game over'
  mask = torch.zeros(B, dtype=torch.uint8, device='cuda')
  mask[::2] = 1
  pair.call('reset', mask)
  for t in range(120, 240):
    pair.call('play', acts[t])


def test_host_edits_of_records_and_coin_patterns():
  """A host that edits sprite records (the key no longer matches) or an env's coin pattern
  (and sets the '@' record's AUX2 to -1, which makes every later step a full paint)."""
  import torch
  from pycolab_b200 import _lib
  arts = _levels(2, (65, 65), (32, 32), density=0.4, seed0=1600)
  B = 8
  pair = Pair(_games(arts), B)
  pair.call('its_showtime')
  acts = torch.from_numpy(_random_actions(13, 90, B)).cuda()
  for t in range(30):
    pair.call('play', acts[t])

  def both(edit):
    torch.cuda.synchronize()
    for eng in (pair.delta, pair.full):
      edit(eng)
    torch.cuda.synchronize()

  def hide_and_move(eng):
    eng.sprites[0, 3, _lib.S_FLAGS] = 0                 # 'c' hidden
    eng.sprites[1, 1, _lib.S_ROW] += 1                  # 'a' drawn one row lower
    eng.sprites[1, 1, _lib.S_VROW] += 1

  def clear_coins(eng):
    eng.patterns[1].view(B, -1)[2:4] = 0               # every coin of envs 2 and 3 gone
    eng.drapes[2:4, 1, _lib.D_AUX2] = -1

  both(hide_and_move)
  for t in range(30, 60):
    pair.call('play', acts[t])
  both(clear_coins)
  for t in range(60, 90):
    pair.call('play', acts[t])


def test_host_board_write_stays_until_a_rebind():
  """Delta rendering repaints only changed cells: a byte the host writes into the board
  buffer survives steps that do not touch it (which also shows that delta rendering
  ran), until pcl_bind_state again, or another board buffer, brings a full paint."""
  import torch
  arts = _levels(2, (129, 129), (64, 64), density=0.1, seed0=1700)
  B = 32
  pair = Pair(_games(arts), B)
  pair.call('its_showtime')
  still = torch.full((B,), 4, dtype=torch.int32, device='cuda')   # 4 = stay: no scroll
  pair.call('play', still)
  board = pair.delta._board
  live = (pair.delta.done == 0).cpu().numpy()        # envs that will not restart next step
  assert live.any()
  # a cell no sprite of any env stands on or next to
  rows, cols = pair.delta.sprites[:, :, 0].cpu().numpy(), pair.delta.sprites[:, :, 1].cpu().numpy()
  cell = next((r, c) for r in range(64) for c in range(64)
              if ((np.abs(rows - r) > 1) | (np.abs(cols - c) > 1)).all())
  saved = board[:, cell[0], cell[1]].clone()
  board[:, cell[0], cell[1]] = ord('X')
  pair.delta.play(still)
  torch.cuda.synchronize()
  assert bool((board[:, cell[0], cell[1]].cpu().numpy()[live] == ord('X')).all())
  board[:, cell[0], cell[1]] = saved
  pair.flip()
  pair.full.play(still)
  pair.check('restored')
  board[:, cell[0], cell[1]] = ord('X')
  from pycolab_b200 import _lib
  _lib.check(pair.delta._lib.pcl_bind_state(pair.delta._h, C.byref(pair.delta._state)),
             'pcl_bind_state')
  pair.call('play', still)
  acts = torch.from_numpy(_random_actions(17, 60, B)).cuda()
  for t in range(60):
    pair.call('play', acts[t])
