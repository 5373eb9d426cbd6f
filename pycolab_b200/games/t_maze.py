"""T-maze set-up (reference `pycolab/examples/research/lp-rnn/t_maze.py:180-505`): a cue
shows which goal to seek, the player walks onto a teleporter, waits in limbo, lands in the
hallway of the level's T-maze and must pick the cued goal pad.

Set-up only; per-step logic is csrc/t_maze.cu.  As upstream, the cue side is drawn from
Python's global `random` (:262) and the speckle from NumPy's global RandomState (:365) when
the drapes are BUILT, so seeding both and calling make_game() builds the same game here and
there.  A batched engine with auto-reset redraws both at every restart on the device from
per-env `random.Random(seed)` and `RandomState(seed)` states instead.

No level art ships with this module: `levels.t_maze_level()` generates the maze and the
cue, keeping the constants the drapes hard-code (limbo cell (4, 140), hallway of level L
11 * L + 9 rows below it, goal corridors 46 columns left of the limbo cell).
"""

import random

import numpy as np

from pycolab_b200 import ascii_art
from pycolab_b200 import levels
from pycolab_b200 import things as plab_things
from pycolab_b200.prefab_parts import drapes as prefab_drapes
from pycolab_b200.prefab_parts import sprites as prefab_sprites

# The teleporter and the goals look alike, and so do the dirt and the walls (:169).
REPAINT_MAPPING = {'t': '~', 'l': '~', 'r': '~', '*': '#'}


def make_game(level, cue_after_teleport, timeout_frames=-1, teleport_delay=0, limbo_time=10,
              maze_art=None, cue_art=None):
  """t_maze.py:180-217; `maze_art` / `cue_art` default to `levels.t_maze_level()`."""
  if maze_art is None or cue_art is None:
    gen_maze, gen_cue = levels.t_maze_level()
    maze_art = gen_maze if maze_art is None else maze_art
    cue_art = gen_cue if cue_art is None else cue_art
  scrolly_info = prefab_drapes.Scrolly.PatternInfo(
      maze_art, cue_art, board_northwest_corner_mark='+', what_lies_beneath=' ')
  engine = ascii_art.ascii_art_to_game(
      cue_art, what_lies_beneath=' ',
      sprites={'P': ascii_art.Partial(PlayerSprite, scrolly_info.virtual_position('P'))},
      drapes={
          'Q': ascii_art.Partial(CueDrape, cue_after_teleport),
          '#': ascii_art.Partial(MazeDrape, **scrolly_info.kwargs('#')),
          '*': ascii_art.Partial(SpeckleDrape, **scrolly_info.kwargs('*')),
          't': ascii_art.Partial(TeleporterDrape, level, teleport_delay, limbo_time,
                                 **scrolly_info.kwargs('t')),
          'l': ascii_art.Partial(GoalDrape, 'left', **scrolly_info.kwargs('l')),
          'r': ascii_art.Partial(GoalDrape, 'right', **scrolly_info.kwargs('r'))},
      update_schedule=[['Q', '#', '*'], ['P'], ['l', 't', 'r']],
      z_order='*#ltrQP')
  engine.the_plot['timeout_frames'] = float('inf') if timeout_frames < 0 else timeout_frames
  return engine


def _device(self, *unused_args, **unused_kwargs):
  raise NotImplementedError('runs on the device: csrc/t_maze.cu')


class PlayerSprite(prefab_sprites.MazeWalker):
  """Egocentric walker that cannot cross '#' (:220-245)."""

  def __init__(self, corner, position, character, virtual_position):
    super(PlayerSprite, self).__init__(
        corner, position, character, egocentric_scroller=True, impassable='#')
    self._teleport(virtual_position)

  update = _device


class CueDrape(plab_things.Drape):
  """Half of the cue blocks show which goal to seek; -0.001 per frame (:248-283)."""

  def __init__(self, curtain, character, cue_after_teleport):
    super(CueDrape, self).__init__(curtain, character)
    self.which_goal = 'left' if random.random() < 0.5 else 'right'
    if self.which_goal == 'left':
      self.curtain[:, 6:] = False
    else:
      self.curtain[:, :6] = False
    self._cue_after_teleport = cue_after_teleport

  update = _device


class PseudoTeleportingScrolly(prefab_drapes.Scrolly):
  """A Scrolly that teleports by rolling its whole pattern (:286-331)."""

  update = _device


class MazeDrape(PseudoTeleportingScrolly):
  """Maze walls (:334-356)."""

  def __init__(self, *args, **kwargs):
    super(MazeDrape, self).__init__(*args, scroll_margins=None, **kwargs)


class SpeckleDrape(PseudoTeleportingScrolly):
  """Speckled dirt: 40% of the cells cleared at random (:359-382)."""

  def __init__(self, *args, **kwargs):
    super(SpeckleDrape, self).__init__(*args, scroll_margins=None, **kwargs)
    self.whole_pattern[np.random.rand(*self.whole_pattern.shape) < 0.4] = False


class TeleporterDrape(PseudoTeleportingScrolly):
  """Teleporter into limbo, then into the level's hallway (:385-468)."""

  def __init__(self, curtain, character, level, teleport_delay, limbo_time, *args, **kwargs):
    super(TeleporterDrape, self).__init__(
        curtain, character, *args, scroll_margins=None, **kwargs)
    self._teleport_delay = teleport_delay
    if self._teleport_delay > 0:
      self._saved_whole_pattern = self.whole_pattern.copy()
      self.whole_pattern[:] = False
    self._limbo_countdown = limbo_time
    self._in_limbo = False
    self._limbo_row = 4
    self._limbo_col = 140
    self._dx = -46
    self._dy = 11 * level + 9
    if (self._dy + 5) > self.whole_pattern.shape[0]:
      raise ValueError('There is no {} difficulty level.'.format(level))


class GoalDrape(PseudoTeleportingScrolly):
  """A goal pad, matched against the cue drape's `which_goal` (:471-505)."""

  def __init__(self, curtain, character, name, *args, **kwargs):
    super(GoalDrape, self).__init__(
        curtain, character, *args, scroll_margins=None, **kwargs)
    self._name = name
