"""Scrolling games for the compiled step program: ordinary pycolab code, whose entity
classes the tests register with `pycolab_b200.compiler`.

This module imports `pycolab.*` only, so it runs unchanged on the reference (the golden
maker, tests/golden/make_registered_golden.py) and on this package (loaded through
`compat.load_example`).  Three games:

  maze     a scrolly maze in this project's own words: an egocentric player, patrollers
           that turn by reading the walls' pattern, scrolling walls and coins that clear
           their own pattern.  Same arguments, schedule and z-order as
           `pycolab_b200.games.scrolly_maze.make_game`, so it plays the scrolly_* goldens
           and runs beside the hand-written kernel.
  sampler  everything the maze does not use: a Scrolly without margins beside one with
           margins, diagonal helpers, `_stay`, a Scrolly that calls no helper in some
           frames (its curtain lags its pattern until the next one), postscroll queries
           after a move, a walker reading a Scrolly's curtain and `.curtain.any()`,
           Scrolly registers, an egocentric walker's register, a Plot key, two levels.
  early    a Scrolly asking for postscroll coordinates before it moved: RuntimeError.
"""

from pycolab import ascii_art
from pycolab.prefab_parts import drapes as prefab_drapes
from pycolab.prefab_parts import sprites as prefab_sprites


# ----------------------------------------------------------------------- maze --
# Actions 0-3 N S W E, 4 stay, 5 quit.

def make_maze(maze_art, board_art, what_lies_beneath, corner_mark='+',
              margins=((2, 3), (2, 3))):
  info = prefab_drapes.Scrolly.PatternInfo(
      maze_art, board_art, board_northwest_corner_mark=corner_mark,
      what_lies_beneath=what_lies_beneath)
  sprites = {'P': ascii_art.Partial(MazePlayer, info.virtual_position('P'))}
  for ch in 'abc':
    sprites[ch] = ascii_art.Partial(MazePatroller, info.virtual_position(ch))
  return ascii_art.ascii_art_to_game(
      board_art, what_lies_beneath=' ', sprites=sprites,
      drapes={'#': ascii_art.Partial(MazeWalls, scroll_margins=margins[0], **info.kwargs('#')),
              '@': ascii_art.Partial(MazeCoins, scroll_margins=margins[1], **info.kwargs('@'))},
      update_schedule=[['#'], ['a', 'b', 'c', 'P'], ['@']],
      z_order='abc@#P')


class MazePlayer(prefab_sprites.MazeWalker):
  """Egocentric explorer; walls stop it."""

  def __init__(self, corner, position, character, virtual_position):
    super(MazePlayer, self).__init__(
        corner, position, character, egocentric_scroller=True, impassable='#')
    self._teleport(virtual_position)

  def update(self, actions, board, layers, backdrop, things, the_plot):
    if actions == 0:
      self._north(board, the_plot)
    elif actions == 1:
      self._south(board, the_plot)
    elif actions == 2:
      self._west(board, the_plot)
    elif actions == 3:
      self._east(board, the_plot)
    elif actions == 4:
      self._stay(board, the_plot)


class MazePatroller(prefab_sprites.MazeWalker):
  """Paces east and west every other frame, turning at walls it finds in the walls'
  pattern (it may be off the board); meeting the player ends the episode."""

  def __init__(self, corner, position, character, virtual_position):
    super(MazePatroller, self).__init__(corner, position, character, '#')
    self._teleport(virtual_position)
    self.heading_east = bool(ord(character) % 2)

  def update(self, actions, board, layers, backdrop, things, the_plot):
    if the_plot.frame % 2:
      self._stay(board, the_plot)
      return
    row, col = things['#'].pattern_position_prescroll(self.virtual_position, the_plot)
    if things['#'].whole_pattern[row, col + (1 if self.heading_east else -1)]:
      self.heading_east = not self.heading_east
    (self._east if self.heading_east else self._west)(board, the_plot)
    if self.virtual_position == things['P'].virtual_position:
      the_plot.terminate_episode()


class MazeWalls(prefab_drapes.Scrolly):
  """Scrolls with the player's motion."""

  def update(self, actions, board, layers, backdrop, things, the_plot):
    if actions == 0:
      self._north(the_plot)
    elif actions == 1:
      self._south(the_plot)
    elif actions == 2:
      self._west(the_plot)
    elif actions == 3:
      self._east(the_plot)
    elif actions == 4:
      self._stay(the_plot)


class MazeCoins(prefab_drapes.Scrolly):
  """+100 per coin the player stands on; the last coin ends the episode."""

  def update(self, actions, board, layers, backdrop, things, the_plot):
    at = self.pattern_position_prescroll(things['P'].position, the_plot)
    if self.whole_pattern[at]:
      the_plot.add_reward(100)
      self.whole_pattern[at] = False
      if not self.whole_pattern.any():
        the_plot.terminate_episode()
    if actions == 0:
      self._north(the_plot)
    elif actions == 1:
      self._south(the_plot)
    elif actions == 2:
      self._west(the_plot)
    elif actions == 3:
      self._east(the_plot)
    elif actions == 4:
      self._stay(the_plot)
    elif actions == 5:
      the_plot.terminate_episode()


# -------------------------------------------------------------------- sampler --
# Actions 0-7 N NE E SE S SW W NW, 8 stay, 9 quit (discount 0.5).  The board is 6 x 8 over
# a 12 x 20 world; '#' scrolls whenever it can (no margins), '*' only for the margins.

SAMPLER_ART = [
    ['####################',
     '#  *   #     *     #',
     '#  +    *  #   *   #',
     '#   #  *    e   #  #',
     '#  *  P   #    *   #',
     '#     #  *    #    #',
     '#  #    *   #   *  #',
     '#    *    #   *    #',
     '#  #   #   *   #   #',
     '#   *    #    *  # #',
     '#     *    #    *  #',
     '####################'],
    ['####################',
     '#    *   #   *     #',
     '# *   #     *   #  #',
     '#   *   *  #   *   #',
     '#  #  *  +   #  *  #',
     '#   *    # *   *   #',
     '# e   #   * P  #   #',
     '#  *    *    #  *  #',
     '#     #   *    *   #',
     '#  *    #   *  #   #',
     '#    *     #    *  #',
     '####################'],
]
SAMPLER_BOARD = (6, 8)


def make_sampler(level):
  info = prefab_drapes.Scrolly.PatternInfo(
      SAMPLER_ART[level], SAMPLER_BOARD, board_northwest_corner_mark='+',
      what_lies_beneath=' ')
  game = ascii_art.ascii_art_to_game(
      [' ' * SAMPLER_BOARD[1]] * SAMPLER_BOARD[0], what_lies_beneath=' ',
      sprites={'P': ascii_art.Partial(SamplerPlayer, info.virtual_position('P')),
               'e': ascii_art.Partial(Watcher, info.virtual_position('e'))},
      drapes={'#': ascii_art.Partial(SamplerWalls, scroll_margins=None, **info.kwargs('#')),
              '*': ascii_art.Partial(Gems, scroll_margins=(2, 2), **info.kwargs('*'))},
      update_schedule=[['#', '*'], ['P', 'e']],
      z_order='*#eP')
  game.the_plot['gems'] = 0
  return game


class SamplerPlayer(prefab_sprites.MazeWalker):
  """Egocentric, eight directions; counts the moves that went through."""

  def __init__(self, corner, position, character, virtual_position):
    super(SamplerPlayer, self).__init__(
        corner, position, character, egocentric_scroller=True, impassable='#')
    self._teleport(virtual_position)
    self.steps = 0

  def update(self, actions, board, layers, backdrop, things, the_plot):
    if actions == 9:
      the_plot.terminate_episode(0.5)
    elif actions is not None:
      if actions == 0:
        blocked = self._north(board, the_plot)
      elif actions == 1:
        blocked = self._northeast(board, the_plot)
      elif actions == 2:
        blocked = self._east(board, the_plot)
      elif actions == 3:
        blocked = self._southeast(board, the_plot)
      elif actions == 4:
        blocked = self._south(board, the_plot)
      elif actions == 5:
        blocked = self._southwest(board, the_plot)
      elif actions == 6:
        blocked = self._west(board, the_plot)
      elif actions == 7:
        blocked = self._northwest(board, the_plot)
      else:
        blocked = self._stay(board, the_plot)
      if blocked is None:
        self.steps += 1


class Watcher(prefab_sprites.MazeWalker):
  """Not egocentric: scrolls with the world.  Counts the frames it stands on a gem's cell
  of the gems' curtain, and notes whether that curtain shows any gem."""

  def __init__(self, corner, position, character, virtual_position):
    super(Watcher, self).__init__(corner, position, character, impassable='#')
    self._teleport(virtual_position)
    self.on_gem = 0
    self.sees_gems = False

  def update(self, actions, board, layers, backdrop, things, the_plot):
    if self.visible and things['*'].curtain[self.position]:
      self.on_gem += 1
    self.sees_gems = things['*'].curtain.any()
    if the_plot.frame % 3 == 0:
      self._southwest(board, the_plot)
    else:
      self._northeast(board, the_plot)


class SamplerWalls(prefab_drapes.Scrolly):
  """Scrolls whenever the player's permits allow; counts its helper calls."""

  def __init__(self, curtain, character, **kwargs):
    super(SamplerWalls, self).__init__(curtain, character, **kwargs)
    self.calls = 0

  def update(self, actions, board, layers, backdrop, things, the_plot):
    if actions is None or actions == 9:
      return
    self.calls += 1
    if actions == 0:
      self._north(the_plot)
    elif actions == 1:
      self._northeast(the_plot)
    elif actions == 2:
      self._east(the_plot)
    elif actions == 3:
      self._southeast(the_plot)
    elif actions == 4:
      self._south(the_plot)
    elif actions == 5:
      self._southwest(the_plot)
    elif actions == 6:
      self._west(the_plot)
    elif actions == 7:
      self._northwest(the_plot)
    else:
      self._stay(the_plot)


class Gems(prefab_drapes.Scrolly):
  """Calls no helper when the player stays in an odd frame (so nothing scrolls; its curtain
  keeps showing a gem taken in an earlier frame); else moves, then takes the gem under the
  player's post-scroll cell (+10 and the_plot['gems']), which stays on its curtain until its
  next helper call."""

  def __init__(self, curtain, character, **kwargs):
    super(Gems, self).__init__(curtain, character, **kwargs)
    self.taken = 0

  def update(self, actions, board, layers, backdrop, things, the_plot):
    if actions is None or actions == 9 or (actions == 8 and the_plot.frame % 2):
      return
    if actions in (0, 4):
      (self._north if actions == 0 else self._south)(the_plot)
    elif actions in (2, 6):
      (self._east if actions == 2 else self._west)(the_plot)
    elif actions in (1, 3, 5, 7):
      if actions == 1:
        self._northeast(the_plot)
      elif actions == 3:
        self._southeast(the_plot)
      elif actions == 5:
        self._southwest(the_plot)
      else:
        self._northwest(the_plot)
    else:
      self._stay(the_plot)
    r, c = self.pattern_position_postscroll(things['P'].virtual_position, the_plot)
    if self.whole_pattern[r, c]:
      self.whole_pattern[r, c] = False
      self.taken += 1
      the_plot['gems'] += 1
      the_plot.add_reward(10)
    if not self.whole_pattern.any():
      the_plot.terminate_episode()


# ---------------------------------------------------------------------- early --
# Action 1 asks for postscroll coordinates before the Scrolly's helper: RuntimeError.

EARLY_ART = ['#######',
             '#  +  #',
             '#     #',
             '#  #  #',
             '#     #',
             '#######']


def make_early():
  info = prefab_drapes.Scrolly.PatternInfo(EARLY_ART, (3, 3), board_northwest_corner_mark='+',
                                           what_lies_beneath=' ')
  return ascii_art.ascii_art_to_game(
      ['   '] * 3, what_lies_beneath=' ',
      drapes={'#': ascii_art.Partial(EarlyAsker, scroll_margins=None, **info.kwargs('#'))},
      update_schedule=[['#']], z_order='#')


class EarlyAsker(prefab_drapes.Scrolly):

  def update(self, actions, board, layers, backdrop, things, the_plot):
    if actions == 1:
      r, c = self.pattern_position_postscroll((0, 0), the_plot)
    self._stay(the_plot)


# The classes a test registers, and the tables of the golden maker and the replays
# (tests/registered_games.py).
CLASSES = (MazePlayer, MazePatroller, MazeWalls, MazeCoins, SamplerPlayer, Watcher,
           SamplerWalls, Gems, EarlyAsker)

# (golden name, game, level, action seed, generator seed, steps)
CASES = [('scrolling_sampler_0', 'sampler', 0, 11, None, 400),
         ('scrolling_sampler_1', 'sampler', 1, 12, None, 400)]
GAMES = {'sampler': make_sampler}
N_ACTIONS = {'sampler': 10}         # the last quits
SPRITES = {'sampler': 'Pe'}
REGISTERS = {'sampler': [('P', 'steps'), ('e', 'on_gem'), ('e', 'sees_gems'), ('#', 'calls'),
                         ('*', 'taken')]}
PLOT_KEYS = {'sampler': ['gems']}
GENERATORS = ()
RAISES = {}
# Each Scrolly's corner every frame, and its whole_pattern at the end, under 'pattern_' + name.
SCROLLYS = {'sampler': '#*'}
PATTERNS = {'sampler': {'walls': '#', 'gems': '*'}}
FIELDS = ('level', 'actions', 'sprites', 'registers', 'corners', 'reward_type',
          'pattern_walls', 'pattern_gems')
