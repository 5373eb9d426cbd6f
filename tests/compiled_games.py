"""Games for the compiled step program: ordinary pycolab code, whose entity classes the
tests register with `pycolab_b200.compiler`.

This module imports `pycolab.*` only, so it runs unchanged on the reference (the golden
maker, tests/golden/make_registered_golden.py) and on this package (loaded through
`compat.load_example`).  Between them the games use every kind of construct the compiler
accepts: curtain reads and writes, `.any()`, registers flipped by blocked moves, Plot keys,
a float reward stream, backdrop and layer reads, diagonal moves, leaving the board,
`_teleport`, negative indices, floor division and modulo of negative numbers, and a quit
action.
"""

from pycolab import ascii_art
from pycolab import things as plab_things
from pycolab.prefab_parts import sprites as prefab_sprites


# ---------------------------------------------------------------------- coins --
# A player collects coins in a maze while a patroller paces a corridor.  Int rewards; the
# episode ends when every coin is taken, when the player walks where the patroller was,
# on the quit action (5), or when the_plot['countdown'] runs out (discount 0.5).

COINS_ART = [
    ['#########',
     '#P c   c#',
     '# ### # #',
     '#c  e  c#',
     '# # ### #',
     '#c     c#',
     '#########'],
    ['#########',
     '#c  #  c#',
     '# #   # #',
     '#  e  P #',
     '# # # # #',
     '#c  c  c#',
     '#########'],
]


class CoinPlayer(prefab_sprites.MazeWalker):
  """Walks N S W E (0-3), stays (4), quits (5)."""

  def __init__(self, corner, position, character):
    super(CoinPlayer, self).__init__(corner, position, character, impassable='#')
    self.bumps = 0

  def update(self, actions, board, layers, backdrop, things, the_plot):
    del backdrop, things    # unused
    if actions == 0:
      blocked = self._north(board, the_plot)
    elif actions == 1:
      blocked = self._south(board, the_plot)
    elif actions == 2:
      blocked = self._west(board, the_plot)
    elif actions == 3:
      blocked = self._east(board, the_plot)
    else:
      blocked = self._stay(board, the_plot)
    if blocked is not None:
      self.bumps += 1
    if actions == 5:
      the_plot.terminate_episode()
    if layers['e'][self.position]:
      the_plot['caught'] = True
      the_plot.add_reward(-5)
      the_plot.terminate_episode()
    the_plot['countdown'] -= 1
    if the_plot.get('countdown') <= 0 and not the_plot['caught']:
      the_plot.terminate_episode(discount=0.5)


class Patroller(prefab_sprites.MazeWalker):
  """Moves east until blocked, then west until blocked, every other frame."""

  def __init__(self, corner, position, character):
    super(Patroller, self).__init__(corner, position, character, impassable='#c')
    self.eastward = True

  def update(self, actions, board, layers, backdrop, things, the_plot):
    if actions is None or the_plot.frame % 2 == 1:
      self._stay(board, the_plot)
      return
    if self.eastward:
      if self._east(board, the_plot):
        self.eastward = False
    elif self._west(board, the_plot) is not None:
      self.eastward = True


class CoinDrape(plab_things.Drape):
  """Pays 10 per coin under the player; ends the episode when none are left."""

  def __init__(self, curtain, character):
    super(CoinDrape, self).__init__(curtain, character)
    self.collected = 0

  def update(self, actions, board, layers, backdrop, things, the_plot):
    player = things['P'].position
    if self.curtain[player]:
      self.curtain[player] = False
      self.collected += 1
      the_plot.add_reward(10 if self.collected > 1 else 12)
    if not self.curtain.any():
      the_plot.terminate_episode()


def make_coins(level):
  game = ascii_art.ascii_art_to_game(
      COINS_ART[level], what_lies_beneath=' ',
      sprites={'P': CoinPlayer, 'e': Patroller}, drapes={'c': CoinDrape},
      update_schedule=[['P', 'e'], ['c']], z_order='ceP')
  game.the_plot['countdown'] = 40 + 5 * level
  game.the_plot['caught'] = False
  return game


# ----------------------------------------------------------------------- lava --
# A walker that moves diagonally (0-3), north (4, off the top edge: it is not confined),
# home by teleport (5) or quits (6), paying -0.01 a step.  Lava 'L' in the backdrop ends
# the episode, the goal 'g' pays 1.5, a gem 'x' hops around by floor arithmetic on
# negative numbers and pays 0.25 where it lands on the walker.

LAVA_ART = [
    ['..........',
     '.#..LL..g.',
     '..........',
     '..L...#...',
     '....P.....',
     '.LL.......',
     '..........'],
    ['..........',
     '..g....#..',
     '...L......',
     '......LL..',
     '.#....P...',
     '...L....g.',
     '.....L....'],
]


class LavaWalker(prefab_sprites.MazeWalker):

  def __init__(self, corner, position, character):
    super(LavaWalker, self).__init__(corner, position, character, impassable='#',
                                     confined_to_board=False)
    self.home_row = position[0]
    self.home_col = position[1]
    self.steps = 0

  def update(self, actions, board, layers, backdrop, things, the_plot):
    del layers    # unused
    if actions is None:
      return
    if actions == 0:
      self._northwest(board, the_plot)
    elif actions == 1:
      self._northeast(board, the_plot)
    elif actions == 2:
      self._southwest(board, the_plot)
    elif actions == 3:
      self._southeast(board, the_plot)
    elif actions == 4:
      self._north(board, the_plot)
    elif actions == 5:
      self._teleport((self.home_row, self.home_col))
    self.steps += 1
    the_plot.add_reward(-0.01)
    if actions == 6:
      the_plot.terminate_episode()
    if not self.visible:
      if self.virtual_position[0] < -1 or things['x'].curtain[-1, -1]:
        the_plot.add_reward(-0.5)
        the_plot.terminate_episode(0.5)
      return
    here = backdrop.curtain[self.position]
    if chr(here) == 'L' or board[self.position.row, self.position.col - 10] == ord('#'):
      the_plot.add_reward(-1.0)
      the_plot.terminate_episode()
    elif chr(here) in 'gG':
      the_plot.add_reward(1.5)
      the_plot.terminate_episode(0.0)


class GemDrape(plab_things.Drape):

  def __init__(self, curtain, character):
    super(GemDrape, self).__init__(curtain, character)
    self.phase = 3

  def update(self, actions, board, layers, backdrop, things, the_plot):
    self.phase = (self.phase * 5 - 13) % 11 - 6          # -6 .. 4
    row = self.phase // 3                                 # -2 .. 1
    col = (the_plot.frame - 17) // 4 % -5                 # -4 .. 0
    self.curtain[:] = False
    self.curtain[row, col] = True
    if things['P'].visible and self.curtain[things['P'].position]:
      the_plot.add_reward(0.25)


def make_lava(level):
  return ascii_art.ascii_art_to_game(
      LAVA_ART[level], what_lies_beneath='.',
      sprites={'P': LavaWalker}, drapes={'x': GemDrape},
      update_schedule=['x', 'P'], z_order='xP')


# -------------------------------------------------------------------- faults --
# Games whose update() faults: an index off the board, a division by zero.

class OffBoardDrape(plab_things.Drape):

  def update(self, actions, board, layers, backdrop, things, the_plot):
    if actions == 1:
      self.curtain[0, 40] = True


class DivideDrape(plab_things.Drape):

  def __init__(self, curtain, character):
    super(DivideDrape, self).__init__(curtain, character)
    self.divisor = 3

  def update(self, actions, board, layers, backdrop, things, the_plot):
    if actions == 1:
      self.divisor = 0
    self.divisor = 7 // self.divisor if self.divisor else 0 // self.divisor


def make_fault(drape_class):
  return ascii_art.ascii_art_to_game(['....', '.x..'], what_lies_beneath='.',
                                     drapes={'x': drape_class})


# The classes a test registers, and the tables of the golden maker and the replays
# (tests/registered_games.py).
CLASSES = (CoinPlayer, Patroller, CoinDrape, LavaWalker, GemDrape)
GAMES = {'coins': make_coins, 'lava': make_lava}
SPRITES = {'coins': 'Pe', 'lava': 'P'}
REGISTERS = {'coins': (('P', 'bumps'), ('e', 'eastward'), ('c', 'collected')),
             'lava': (('P', 'home_row'), ('P', 'home_col'), ('P', 'steps'), ('x', 'phase'))}
PLOT_KEYS = {'coins': ('countdown', 'caught'), 'lava': ()}
N_ACTIONS = {'coins': 6, 'lava': 7}
GENERATORS = ()
RAISES = {}
FIELDS = ('game', 'level', 'actions', 'sprites', 'registers', 'reward_type', 'reward_f64')

# (golden name, game, level, action seed, generator seed, steps)
CASES = (
    ('compiled_coins_0', 'coins', 0, 1, None, 320),
    ('compiled_coins_1', 'coins', 1, 2, None, 320),
    ('compiled_lava_0', 'lava', 0, 3, None, 320),
    ('compiled_lava_1', 'lava', 1, 4, None, 320),
)
