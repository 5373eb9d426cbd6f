"""GPU tests of scrolling games on the compiled step program (csrc/compiled.cu): the games
of tests/scrolling_games.py on the H100, against the reference's trajectories
(tests/golden/scrolly_*.npz; the sampler's replay in test_gpu_registered_goldens.py), the
hand-written scrolly_maze kernel and the
oracle interpreter (oracle/compiled.py)."""

import numpy as np
import pytest

import example_games as eg
import golden_cases as gc
import registered_games as rg
import scrolly_shapes
from oracle import compiled as ocompiled
from oracle import sampled_check
from pycolab_b200 import _lib, levels, lowering

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def games():
  yield from rg.registered('scrolling_games.py')


def _margins(name):
  if name.startswith('scrolly_shape'):
    return scrolly_shapes.SHAPE[name[len('scrolly_shape'):]][2]
  return scrolly_shapes.DEFAULT_MARGINS


@pytest.mark.parametrize('name', gc.names('scrolly_'))
def test_facade_replays_scrolly_golden(games, name):
  maze, board, beneath = gc.scrolly_art(gc.load(name))
  eg.assert_replays('facade', name,
                    make_env=lambda: games.make_maze(maze, board, beneath, margins=_margins(name)))


def test_facade_raises_on_postscroll_before_the_move(games):
  engine = games.make_early()
  engine.its_showtime()
  engine.play(0)
  with pytest.raises(RuntimeError, match='pattern_position_postscroll'):
    engine.play(1)


B, T = 4096, 300


def _levels(n):
  return [levels.scrolly_maze_level(100 + i, world_shape=(129, 129), board_shape=(64, 64))
          for i in range(n)]


def test_compiled_maze_matches_the_hand_written_kernel(games):
  """B = 4096 over four generated 64 x 64 levels, auto-reset, 300 steps: every output and
  every sprite and corner word byte for byte against PCL_PROG_SCROLLY_MAZE."""
  import torch
  from pycolab_b200 import batched
  from pycolab_b200.games import scrolly_maze
  arts = _levels(4)
  theirs = batched.BatchedEngine([scrolly_maze.make_game(*a) for a in arts], batch=B)
  ours = batched.BatchedEngine([games.make_maze(*a) for a in arts], batch=B)
  assert theirs.game.program == _lib.PROG_SCROLLY_MAZE
  assert ours.game.program == _lib.PROG_COMPILED
  rs = np.random.RandomState(5)
  actions = torch.from_numpy(rs.randint(0, 6, size=(T, B)).astype(np.int32)).cuda()
  # the compiled program keeps its sprites in update order (abcP), the kernel in PAbc
  order = torch.tensor([ours.sprite_chars.index(ch) for ch in theirs.sprite_chars]).cuda()
  assert theirs.drape_chars == ours.drape_chars == '#@'

  def same(t):
    torch.cuda.synchronize()
    for name in ('_board', 'reward', 'has_reward', 'discount', 'done'):
      a, b = getattr(theirs, name), getattr(ours, name)
      assert torch.equal(a, b), (name, t)
    assert torch.equal(theirs.sprites[:, :, :5], ours.sprites[:, order, :5]), ('sprites', t)
    assert torch.equal(theirs.drapes[:, :, :2], ours.drapes[:, :, :2]), ('corners', t)
  theirs.its_showtime()
  ours.its_showtime()
  same(0)
  dones = 0
  for t in range(T):
    theirs.play(actions[t])
    ours.play(actions[t])
    same(t + 1)
    dones += int(ours.done.sum())
  assert dones > 0                            # episodes end and restart on the way
  assert int(ours.error_codes().abs().sum()) == 0


def test_batched_lockstep_against_the_oracle(games):
  """B = 4096 over two levels: sampled envs against the oracle every step, curtains,
  sprite words and pad columns included, then the coins' final whole_pattern."""
  import torch
  from pycolab_b200 import batched, lowering as low
  arts = _levels(2)
  lowered = [low.lower(games.make_maze(*a)) for a in arts]
  engine = batched.BatchedEngine(lowered, batch=B)
  engine.its_showtime()
  rs = np.random.RandomState(9)
  actions = rs.randint(0, 6, size=(T, B)).astype(np.int32)
  env_ids = [0, 1, 2, 3, 1000, 2049, 4094, 4095]
  worlds = {}

  def make_world(e):
    worlds[e] = ocompiled.make_world(lowered[e % 2])
    return worlds[e]
  n = sampled_check.lockstep(engine, make_world, env_ids, actions, curtains='#@',
                             sprites='Pabc', pad_columns=True)
  assert n == len(env_ids) * (T + 1)
  coins = engine.patterns[1].index_select(
      0, torch.as_tensor(env_ids, device=engine.device)).cpu().numpy().view(np.uint32)
  for k, e in enumerate(env_ids):
    world = worlds[e]
    got = lowering.unpack_rows(coins[k], lowered[0].pattern_cols)
    np.testing.assert_array_equal(got, world.things['@'].pattern, err_msg=str(e))


def test_batched_sampler_lockstep_against_the_oracle(games):
  """The sampler (kept Scrolly curtains, two levels) at B = 4096 against the oracle."""
  from pycolab_b200 import batched, lowering as low
  lowered = [low.lower(games.make_sampler(level)) for level in (0, 1)]
  engine = batched.BatchedEngine(lowered, batch=B)
  engine.its_showtime()
  rs = np.random.RandomState(3)
  actions = rs.randint(0, games.N_ACTIONS['sampler'], size=(T, B)).astype(np.int32)
  env_ids = [0, 1, 7, 2048, 4095]
  n = sampled_check.lockstep(engine, lambda e: ocompiled.make_world(lowered[e % 2]),
                             env_ids, actions, curtains='#*', sprites='Pe', pad_columns=True)
  assert n == len(env_ids) * (T + 1)
