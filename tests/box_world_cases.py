"""Box-World test helpers: the reference module, the golden cases and a scripted player.

The scripted player reads the board (and the level's distractor cells) and walks, by
breadth-first search over free cells, to the object its mode wants: 'solve' opens correct
locks and takes the gem, 'distract' opens a distractor lock, 'dither' steps back and forth and
plays invalid actions until the step limit ends the episode, 'random' draws from -1 .. 5.
"""

import collections
import importlib.util
import os

import numpy as np

import refdriver
from pycolab_b200 import levels

KEYS, LOCKS = levels.BOX_WORLD_KEYS, levels.BOX_WORLD_LOCKS
MODES = ('solve', 'distract', 'dither', 'random')
ARGS = ((1, 2, 3, 4), (0, 1, 2, 3, 4), (0,), 1)     # make_game's arguments after grid_size
# The goldens: (name, seed, grid_size, max_num_steps, modes, T)
CASES = (
    ('box_world_g12_s3_solve', 3, 12, 120, ('solve', 'distract', 'random'), 400),
    ('box_world_g12_s10_mixed', 10, 12, 120, ('solve', 'dither', 'distract'), 500),
    ('box_world_g12_s7_distract', 7, 12, 60, ('distract', 'solve', 'random'), 400),
    ('box_world_g6_s1', 1, 6, 40, ('solve', 'random', 'distract'), 300),
    ('box_world_g20_s2', 2, 20, 150, ('solve', 'dither'), 400),
    ('box_world_g30_s5', 5, 30, 200, ('solve', 'distract'), 400),
)
_STEPS = ((-1, 0, 0), (1, 0, 1), (0, -1, 2), (0, 1, 3))     # (dr, dc, action)


def ref_path():
  return os.path.join(refdriver.REFERENCE_ROOT, 'pycolab', 'examples', 'research', 'box_world',
                      'box_world.py')


def ref_module(name='ref_box_world'):
  """The reference's research/box_world/box_world.py, loaded by path.  Its imports spell
  `collections.Mapping` (gone since Python 3.10); the alias is an environment shim, the
  reference source is untouched."""
  refdriver._import()
  import collections.abc
  for attr in ('Mapping', 'Sequence'):
    if not hasattr(collections, attr):
      setattr(collections, attr, getattr(collections.abc, attr))
  spec = importlib.util.spec_from_file_location(name, ref_path())
  module = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(module)
  return module


def object_grid(things, shape):
  """u8 [rows, cols]: the character of the object drape whose curtain holds each cell, 0 =
  none, from the `things` of a reference Engine, a facade Engine or an oracle World.  Asserts
  that no two curtains share a cell."""
  grid = np.zeros(shape, dtype=np.uint8)
  for ch, thing in things.items():
    if ch == '.':
      continue
    cells = np.asarray(thing.curtain, dtype=bool)
    assert not grid[cells].any(), 'two objects on one cell'
    grid[cells] = ord(ch)
  return grid


def over_words(over):
  """the_plot['over_this'] as [char code, row, col], [0, 0, 0] when unset."""
  return [0, 0, 0] if not over else [ord(over[0]), int(over[1][0]), int(over[1][1])]


def _objects(board):
  out = []
  for y, x in zip(*np.nonzero((board != ord(' ')) & (board != ord('#')) & (board != ord('.')))):
    if y == 0 and x == 0:
      continue                                    # the held key
    out.append(((int(y), int(x)), chr(board[y, x])))
  return out


def _first_step(board, goals):
  """Action of the first step of a shortest walk over free cells that ends by stepping onto
  one of `goals` (cells), or None."""
  start = tuple(int(v) for v in np.argwhere(board == ord('.'))[0])
  goals = set(goals)
  seen = {start: None}
  queue = collections.deque([start])
  while queue:
    cell = queue.popleft()
    for dr, dc, action in _STEPS:
      nxt = (cell[0] + dr, cell[1] + dc)
      first = action if seen[cell] is None else seen[cell]
      if nxt in goals:
        return first
      if nxt not in seen and board[nxt] == ord(' '):
        seen[nxt] = first
        queue.append(nxt)
  return None


def scripted_action(board, distractors, mode, rs, noise=0.05):
  """One action of the scripted player in `mode` on `board` (u8 [H, W])."""
  board = np.asarray(board)
  if mode == 'random' or rs.random_sample() < noise:
    return int(rs.randint(-1, 6))
  if mode == 'dither':
    return int(rs.choice([0, 1, 2, 3, -1, 4, 7]))
  held = chr(board[0, 0])
  wrong = {(int(y), int(x)) for x, y in distractors}
  tiers = [[], [], []]
  for (y, x), c in _objects(board):
    locked = chr(board[y, x + 1]) in LOCKS
    if c in LOCKS:
      if held == c.lower():
        tiers[0 if ((y, x) in wrong) == (mode == 'distract') else 2].append((y, x))
    elif not locked:
      if c == '*':
        tiers[0 if mode == 'solve' else 2].append((y, x))
      else:
        opens = [(yy, xx) for (yy, xx), cc in _objects(board) if cc == c.upper()]
        good = any((cell in wrong) == (mode == 'distract') for cell in opens)
        tiers[1 if good else 2].append((y, x))
  for goals in tiers:
    action = _first_step(board, goals) if goals else None
    if action is not None:
      return action
  return int(rs.randint(0, 4))


def drive(make_env, distractors, modes, T, seed):
  """T actions of the scripted player on envs from make_env() under the auto-reset rule of
  tests/trajectory.py (a restart step stores 0); episode k plays modes[k % len(modes)]."""
  rs = np.random.RandomState(seed)
  env = make_env()
  board = env.its_showtime()[0].board
  episode, actions = 0, []
  for _ in range(T):
    if env.game_over:
      episode += 1
      actions.append(0)
      env = make_env()
      board = env.its_showtime()[0].board
    else:
      actions.append(scripted_action(board, distractors, modes[episode % len(modes)], rs))
      board = env.play(actions[-1])[0].board
  return actions
