"""Box-World set-up (reference `pycolab/examples/research/box_world/box_world.py`): keys open
locks of their colour, a chain of boxes leads to the gem, and opening a distractor lock ends
the episode.

Set-up only; per-step logic is csrc/box_world.cu.  Levels come from
`levels.box_world_level`, which makes upstream's draws, so `random_state=RandomState(s)`
builds the same game here and there.  On the device the keys, locks and the gem are cells of
one per-env object grid, not drapes of their own (programs/box_world.py).
"""

import numpy as np

from pycolab_b200 import ascii_art
from pycolab_b200 import levels
from pycolab_b200 import things as plab_things
from pycolab_b200.prefab_parts import sprites as prefab_sprites

GEM, PLAYER, BACKGROUND, BORDER = '*', '.', ' ', '#'
KEYS, LOCKS = levels.BOX_WORLD_KEYS, levels.BOX_WORLD_LOCKS


def make_game(grid_size, solution_length, num_forward, num_backward, branch_length,
              random_state=None, max_num_steps=120):
  """box_world.py:418-445: a generated level, every object a drape in one update group
  [player, sorted objects], objects behind the player."""
  if random_state is None:
    random_state = np.random.RandomState(None)
  art, distractors = levels.box_world_level(random_state, grid_size, solution_length,
                                            num_forward, num_backward, branch_length)
  return game_from_level(art, distractors, max_num_steps)


def game_from_level(art, distractors, max_num_steps=120):
  """The game of one `levels.box_world_level` result."""
  drapes = {}
  for ch in sorted(set(''.join(art)) - set(PLAYER + BACKGROUND + BORDER)):
    drapes[ch] = GemDrape if ch == GEM else KeyDrape if ch in KEYS else LockDrape
  order = sorted(drapes)
  return ascii_art.ascii_art_to_game(
      art, what_lies_beneath=BACKGROUND,
      sprites={PLAYER: ascii_art.Partial(PlayerSprite, list(distractors), max_num_steps)},
      drapes=drapes, update_schedule=[PLAYER] + order, z_order=order + [PLAYER])


def _device(self, *unused_args, **unused_kwargs):
  raise NotImplementedError('runs on the device: csrc/box_world.cu')


class PlayerSprite(prefab_sprites.MazeWalker):
  """Moves N S W E (actions 0-3) onto free cells, unlocked keys and the gem, and onto a lock
  while holding its key; episodes last max_num_steps + 1 valid actions (:127-202)."""

  def __init__(self, corner, position, character, distractors, max_num_steps):
    super(PlayerSprite, self).__init__(
        corner, position, character, impassable=BORDER, confined_to_board=True)
    self.distractors = distractors
    self._max_num_steps = max_num_steps
    self._step_counter = 0

  update = _device


class BoxThing(plab_things.Drape):
  """A key, lock or gem: its cells are its curtain (:205-229)."""

  update = _device


class GemDrape(BoxThing):
  """+10 and the end of the episode when the player steps on it (:232-238)."""


class KeyDrape(BoxThing):
  """Picked up into the corner cell (0, 0), replacing the key held before (:241-251)."""


class LockDrape(BoxThing):
  """Opened with the held key: +1, or -1 and the end for a distractor (:254-271)."""
