"""Games with plain Sprites for the compiled step program: ordinary pycolab code, whose entity
classes the tests register with `pycolab_b200.compiler`.

This module imports `pycolab.*` only, so it runs unchanged on the reference (the golden
maker, tests/golden/make_registered_golden.py) and on this package (loaded through
`compat.load_example`).  Three games:

  bounce   a breakout-like game on two levels: the ball is a plain Sprite with dy / dx
           registers that bounces by reading `layers['#']` and `board`; the paddle is a
           MazeWalker the ball blocks; the bricks are a plain Drape that clears the cell the
           ball enters and pays for it.  The ball stays hidden until the first action;
           after a miss it re-serves from a stored position attribute, in a direction drawn
           by `np.random.randint`.  Lives are a Plot key.
  sampler  the other forms, in a scrolling world with an egocentric player: keyword and
           `Sprite.Position` constructors, `self._position = things['P'].position`,
           blinking, a visible sprite at row -1 and at column -1 (painted on the last row
           or column), a hidden sprite far off the board, two sprites of one class, position
           attributes in a walker and in a drape, a drape above a sprite; two levels.
  fallen   a visible sprite that walks off the bottom of the board: IndexError.
"""

import numpy as np

from pycolab import ascii_art
from pycolab import things as plab_things
from pycolab.prefab_parts import drapes as prefab_drapes
from pycolab.prefab_parts import sprites as prefab_sprites
from pycolab.things import Sprite


# --------------------------------------------------------------------- bounce --
# Actions 0 left, 1 right, 2 stay, 3 quit.

BOUNCE_ART = [
    ['##########',
     '#        #',
     '# ====== #',
     '#        #',
     '#   o    #',
     '#        #',
     '#        #',
     '#   P    #'],
    ['##########',
     '#        #',
     '# == = = #',
     '#  == == #',
     '#        #',
     '#     o  #',
     '#        #',
     '#     P  #'],
]


def make_bounce(level):
  game = ascii_art.ascii_art_to_game(
      BOUNCE_ART[level], what_lies_beneath=' ',
      sprites={'P': Paddle, 'o': Ball},
      drapes={'=': Bricks},
      update_schedule=[['P'], ['o'], ['=']],
      z_order='=Po')
  game.the_plot['lives'] = 3
  return game


class Paddle(prefab_sprites.MazeWalker):
  """Slides along the bottom row; walls and the ball stop it."""

  def __init__(self, corner, position, character):
    super(Paddle, self).__init__(corner, position, character, impassable='#o')

  def update(self, actions, board, layers, backdrop, things, the_plot):
    if actions == 0:
      self._west(board, the_plot)
    elif actions == 1:
      self._east(board, the_plot)
    elif actions == 3:
      the_plot.terminate_episode()


class Ball(plab_things.Sprite):
  """Hidden until the first action, then one diagonal cell per frame.  It turns at walls,
  at the paddle and inside a brick; in the paddle's row it has missed: a life is lost and
  it re-serves from where it started."""

  def __init__(self, corner, position, character):
    super(Ball, self).__init__(corner, position, character)
    self._visible = False
    self._serve = self.position
    self.dy = 1
    self.dx = 1

  def update(self, actions, board, layers, backdrop, things, the_plot):
    if actions is None:
      return
    if not self._visible:
      self._visible = True
      return
    r, c = self._position
    if r == self.corner.row - 1:
      the_plot['lives'] -= 1
      if the_plot['lives'] == 0:
        the_plot.terminate_episode()
      self._position = self._serve
      self.dx = np.random.randint(2) * 2 - 1
      self.dy = 1
      return
    if layers['#'][r + self.dy, c]:
      self.dy = -self.dy
    if layers['#'][r, c + self.dx]:
      self.dx = -self.dx
    if board[r + self.dy, c + self.dx] == ord('P'):
      self.dy = -self.dy
    self._position = self.Position(r + self.dy, c + self.dx)
    if layers['='][self._position]:
      self.dy = -self.dy


class Bricks(plab_things.Drape):
  """Clears the brick the ball stands in, +5; the last brick ends the episode."""

  def update(self, actions, board, layers, backdrop, things, the_plot):
    at = things['o'].position
    if things['o'].visible and self.curtain[at]:
      self.curtain[at] = False
      the_plot.add_reward(5)
      if not self.curtain.any():
        the_plot.terminate_episode()


# -------------------------------------------------------------------- sampler --
# Actions 0-3 N S W E, 4 stay, 5 the ghost jumps to the player, 6 marks (the drape's and the
# walker's position attributes), 7 the walker goes home, 8 quit.

SAMPLER_ART = [
    ['##############',
     '#   #    #   #',
     '# +    #     #',
     '#   #  P  w  #',
     '#        #   #',
     '#  #   #     #',
     '#     #   #  #',
     '##############'],
    ['##############',
     '#     #   #  #',
     '#  +  #      #',
     '#   w   #    #',
     '# #   P    # #',
     '#    #    #  #',
     '#  #    #    #',
     '##############'],
]
SAMPLER_BOARD = (5, 8)


def make_sampler(level):
  info = prefab_drapes.Scrolly.PatternInfo(
      SAMPLER_ART[level], SAMPLER_BOARD, board_northwest_corner_mark='+',
      what_lies_beneath=' ')
  board = [' ' * SAMPLER_BOARD[1]] * SAMPLER_BOARD[0]
  board[1] = ' b     c'
  board[3] = '  e   g '
  board[4] = 'x       '
  game = ascii_art.ascii_art_to_game(
      board, what_lies_beneath=' ',
      sprites={'P': ascii_art.Partial(Player, info.virtual_position('P')),
               'w': ascii_art.Partial(Wanderer, info.virtual_position('w')),
               'b': Blinker, 'c': Blinker, 'e': Edge, 'g': Ghost},
      drapes={'#': ascii_art.Partial(Walls, scroll_margins=None, **info.kwargs('#')),
              'x': Marker},
      update_schedule=[['#'], ['P', 'w', 'b', 'c'], ['e', 'g', 'x']],
      z_order='#bceg' + 'xwP')
  game.the_plot['marks'] = 0
  return game


class Player(prefab_sprites.MazeWalker):
  """Egocentric; walls stop it."""

  def __init__(self, corner, position, character, virtual_position):
    super(Player, self).__init__(
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
    elif actions == 8:
      the_plot.terminate_episode(0.5)
    else:
      self._stay(board, the_plot)


class Walls(prefab_drapes.Scrolly):

  def update(self, actions, board, layers, backdrop, things, the_plot):
    if actions == 0:
      self._north(the_plot)
    elif actions == 1:
      self._south(the_plot)
    elif actions == 2:
      self._west(the_plot)
    elif actions == 3:
      self._east(the_plot)
    else:
      self._stay(the_plot)


class Wanderer(prefab_sprites.MazeWalker):
  """Scrolls with the world and paces; a position attribute holds its home."""

  def __init__(self, corner, position, character, virtual_position):
    super(Wanderer, self).__init__(corner, position, character, impassable='#')
    self._teleport(virtual_position)
    self._home = self.virtual_position
    self.seen = 0

  def update(self, actions, board, layers, backdrop, things, the_plot):
    if actions == 7:
      self._teleport(self._home)
    elif actions == 6:
      self._home = self.virtual_position
    elif the_plot.frame % 3 == 0:
      self._west(board, the_plot)
    else:
      self._east(board, the_plot)
    if things['b'].visible and things['c'].visible:
      self.seen += 1


class Blinker(plab_things.Sprite):
  """Two of them: each walks along its row in its own direction, wrapping at the edge with
  `%`, and shows itself in every other frame."""

  def __init__(self, corner, position, character):
    super(Blinker, self).__init__(corner, position, character)
    self.step = 1 if character == 'b' else -1
    self.walked = 0

  def update(self, actions, board, layers, backdrop, things, the_plot):
    if actions is None:
      return
    self._visible = not self._visible
    self._position = self.Position(row=self._position.row,
                                   col=(self.position.col + self.step) % self.corner.col)
    self.walked += 1


class Edge(plab_things.Sprite):
  """Visible at row -1 and at column -1 by turns: the board shows it on the last row or
  column."""

  def update(self, actions, board, layers, backdrop, things, the_plot):
    if actions is None:
      return
    if the_plot.frame % 2:
      self._position = plab_things.Sprite.Position(-1, the_plot.frame % 8)
    else:
      self._position = Sprite.Position(row=the_plot.frame % 5, col=-1)


class Ghost(plab_things.Sprite):
  """Hidden, far off the board; action 5 takes it to the player, still hidden."""

  def __init__(self, corner, position, character):
    super(Ghost, self).__init__(corner, position, character)
    self._visible = False

  def update(self, actions, board, layers, backdrop, things, the_plot):
    if actions == 5:
      self._position = things['P'].position
    elif actions is not None:
      self._position = self.Position(100000, -7 * the_plot.frame)


class Marker(plab_things.Drape):
  """One marked cell, held in a position attribute (a tuple); action 6 moves it to the
  player.  Drawn above the blinkers."""

  def __init__(self, curtain, character):
    super(Marker, self).__init__(curtain, character)
    self._mark = (4, 0)

  def update(self, actions, board, layers, backdrop, things, the_plot):
    if actions == 6:
      self.curtain[self._mark] = False
      self._mark = things['P'].position
      self.curtain[self._mark] = True
      the_plot['marks'] += 1
    if things['b'].position == self._mark:
      the_plot.add_reward(1)


# --------------------------------------------------------------------- fallen --

def make_fallen():
  return ascii_art.ascii_art_to_game(
      [' f ', '   ', '   ', '   '], what_lies_beneath=' ',
      sprites={'f': Faller}, update_schedule=[['f']], z_order='f')


class Faller(plab_things.Sprite):
  """One row down at action 0, visible all the way: off the bottom row, upstream's render
  raises IndexError."""

  def update(self, actions, board, layers, backdrop, things, the_plot):
    if actions == 0:
      self._position = self.Position(self._position.row + 1, self._position.col)


# The classes a test registers, and the tables of the golden maker and the replays
# (tests/registered_games.py).
CLASSES = (Paddle, Ball, Bricks, Player, Walls, Wanderer, Blinker, Edge, Ghost, Marker, Faller)

# (golden name, game, level, action seed, generator seed, steps)
CASES = [('sprite_bounce_0', 'bounce', 0, 21, 5, 400), ('sprite_bounce_1', 'bounce', 1, 22, 6, 400),
         ('sprite_sampler_0', 'sampler', 0, 23, 0, 300),
         ('sprite_sampler_1', 'sampler', 1, 24, 0, 300),
         ('sprite_fallen', 'fallen', 0, 25, 0, 8)]
GAMES = {'bounce': make_bounce, 'sampler': lambda level: make_sampler(level),
         'fallen': lambda level: make_fallen()}
N_ACTIONS = {'bounce': 4, 'sampler': 9, 'fallen': 2}
SPRITES = {'bounce': 'Po', 'sampler': 'Pwbceg', 'fallen': 'f'}
# Registers as ints; a position attribute as its row and column.
REGISTERS = {'bounce': [('o', 'dy'), ('o', 'dx'), ('o', '_serve')],
             'sampler': [('w', '_home'), ('w', 'seen'), ('b', 'step'), ('b', 'walked'),
                         ('c', 'step'), ('c', 'walked'), ('x', '_mark')],
             'fallen': []}
PLOT_KEYS = {'bounce': ['lives'], 'sampler': ['marks'], 'fallen': []}
GENERATORS = ('numpy',)
RAISES = {'fallen': IndexError}
FIELDS = ('game', 'level', 'rng_seed', 'actions', 'sprites', 'registers', 'reward_type',
          'numpy_words', 'raised_at')
