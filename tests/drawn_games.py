"""Games whose update() code draws from NumPy's and Python's global generators: ordinary
pycolab code, whose entity classes the tests register with `pycolab_b200.compiler`.

This module imports `pycolab.*`, `numpy` and `random` only, the way a game author would
(with aliases and `from` imports too), so it runs unchanged on the reference (the golden
maker, tests/golden/make_registered_golden.py) and on this package (loaded through
`compat.load_example`).  No constructor draws.
"""

import random
from random import randint

import numpy as np
from numpy import random as npr

from pycolab import ascii_art
from pycolab import things as plab_things
from pycolab.prefab_parts import sprites as prefab_sprites


# ------------------------------------------------------------------- monsters --
# A player (N S W E 0-3, stay 4, quit 5) eats a fruit 'f' that respawns at a random cell,
# while two monsters wander: 'a' by NumPy's generator, 'b' by Python's.  A monster on the
# player ends the episode; every step pays a bonus with probability 0.1 (NumPy) and
# springs a trap with probability 0.05 (Python) that ends the episode at discount 0.5.

MONSTERS_ART = [
    ['##########',
     '#P   f   #',
     '#  ##    #',
     '#  a   b #',
     '#    ##  #',
     '##########'],
    ['##########',
     '#   #   b#',
     '# a    # #',
     '#   P    #',
     '#f #   # #',
     '##########'],
]


class Player(prefab_sprites.MazeWalker):

  def __init__(self, corner, position, character):
    super(Player, self).__init__(corner, position, character, impassable='#')
    self.bonuses = 0

  def update(self, actions, board, layers, backdrop, things, the_plot):
    if actions == 0:
      self._north(board, the_plot)
    elif actions == 1:
      self._south(board, the_plot)
    elif actions == 2:
      self._west(board, the_plot)
    elif actions == 3:
      self._east(board, the_plot)
    elif actions == 5:
      the_plot.terminate_episode()
    if np.random.rand() < 0.1:
      self.bonuses += 1
      the_plot.add_reward(1)
    if random.random() >= 0.95:
      the_plot.terminate_episode(0.5)
    if self.position == things['a'].position or self.position == things['b'].position:
      the_plot.add_reward(-3)
      the_plot.terminate_episode()


class NumpyMonster(prefab_sprites.MazeWalker):

  def __init__(self, corner, position, character):
    super(NumpyMonster, self).__init__(corner, position, character, impassable='#f')

  def update(self, actions, board, layers, backdrop, things, the_plot):
    move = np.random.randint(4)
    if move == 0:
      self._north(board, the_plot)
    elif move == 1:
      self._south(board, the_plot)
    elif move == 2:
      self._west(board, the_plot)
    else:
      self._east(board, the_plot)


class PythonMonster(prefab_sprites.MazeWalker):

  def __init__(self, corner, position, character):
    super(PythonMonster, self).__init__(corner, position, character, impassable='#f')

  def update(self, actions, board, layers, backdrop, things, the_plot):
    move = random.choice((0, 1, 2, 3))
    if move == 0:
      self._north(board, the_plot)
    elif move == 1:
      self._south(board, the_plot)
    elif move == 2:
      self._west(board, the_plot)
    elif move == 3:
      self._east(board, the_plot)


class Fruit(plab_things.Drape):

  def __init__(self, curtain, character):
    super(Fruit, self).__init__(curtain, character)
    self.eaten = 0

  def update(self, actions, board, layers, backdrop, things, the_plot):
    player = things['P'].position
    if self.curtain[player]:
      self.curtain[player] = False
      self.eaten += 1
      the_plot.add_reward(5)
      row = randint(1, 4)
      col = npr.randint(1, 9)
      self.curtain[row, col] = True


def make_monsters(level):
  return ascii_art.ascii_art_to_game(
      MONSTERS_ART[level], what_lies_beneath=' ',
      sprites={'P': Player, 'a': NumpyMonster, 'b': PythonMonster}, drapes={'f': Fruit},
      update_schedule=[['P', 'a', 'b'], ['f']], z_order='fabP')


# ---------------------------------------------------------------------- edges --
# One draw per frame, cycling through the boundary cases of both generators with
# operands held in registers: widths 1 (NumPy consumes nothing, Python does), 2^k and
# 2^k + 1 for k = 1, 16, 30, 31, negative bounds and the whole int32 range (Python's
# 33-bit getrandbits).  Each result lands in `out`.

class Edges(plab_things.Drape):

  def __init__(self, curtain, character):
    super(Edges, self).__init__(curtain, character)
    self.lo = -2 ** 31
    self.hi = 2 ** 31 - 1
    self.p16 = 2 ** 16
    self.p30 = 2 ** 30
    self.one = 1
    self.case = 0
    self.out = 0

  def update(self, actions, board, layers, backdrop, things, the_plot):
    c = self.case
    self.case = (self.case + 1) % 24
    if c == 0:
      self.out = np.random.randint(0, self.one)
    elif c == 1:
      self.out = np.random.choice(self.one)
    elif c == 2:
      self.out = random.randrange(self.one)
    elif c == 3:
      self.out = np.random.randint(self.one + 1)
    elif c == 4:
      self.out = random.randrange(self.one + 2)
    elif c == 5:
      self.out = np.random.randint(-self.p16, 0)
    elif c == 6:
      self.out = random.randint(-self.p16, 0)
    elif c == 7:
      self.out = np.random.randint(self.p30)
    elif c == 8:
      self.out = random.randrange(-self.p30, self.one)
    elif c == 9:
      self.out = np.random.randint(self.lo, 0)
    elif c == 10:
      self.out = random.randrange(self.lo, 0)
    elif c == 11:
      self.out = np.random.randint(self.lo, self.one)
    elif c == 12:
      self.out = random.randint(self.lo, 0)
    elif c == 13:
      self.out = np.random.randint(self.lo, self.hi)
    elif c == 14:
      self.out = random.randint(self.lo, self.hi)
    elif c == 15:
      self.out = np.random.randint(-7, -2)
    elif c == 16:
      self.out = random.randrange(-7, -2)
    elif c == 17:
      self.out = random.randint(-3, -3)
    elif c == 18:
      self.out = np.random.choice((-5, 9, 2147483647))
    elif c == 19:
      self.out = random.choice([-2147483648, 4])
    elif c == 20:
      self.out = np.random.choice(self.p16 + 1)
    elif c == 21:
      self.out = random.randrange(self.p30 + 1)
    elif c == 22:
      self.out = int(0.5 > np.random.random_sample()) + 2 * int(random.random() == 0.25)
    else:
      self.out = np.random.randint(self.hi - 1, self.hi)


def make_edges(level):
  del level    # one level
  return ascii_art.ascii_art_to_game(['....', '.x..'], what_lies_beneath='.',
                                     drapes={'x': Edges})


# ----------------------------------------------------------------- thresholds --
# Twelve float draws from each generator every frame, each against a literal with one of the
# six comparisons: against 0.5 with the draw on the left, then against 0.25 with the literal
# on the left.  Bit k of `hits` is draw k's outcome, NumPy's draws first.

class Thresholds(plab_things.Drape):

  def __init__(self, curtain, character):
    super(Thresholds, self).__init__(curtain, character)
    self.hits = 0

  def update(self, actions, board, layers, backdrop, things, the_plot):
    self.hits = 0
    if np.random.rand() < 0.5:
      self.hits += 1
    if np.random.rand() <= 0.5:
      self.hits += 2
    if np.random.rand() > 0.5:
      self.hits += 4
    if np.random.rand() >= 0.5:
      self.hits += 8
    if np.random.rand() == 0.5:
      self.hits += 16
    if np.random.rand() != 0.5:
      self.hits += 32
    if 0.25 < np.random.rand():
      self.hits += 64
    if 0.25 <= np.random.rand():
      self.hits += 128
    if 0.25 > np.random.rand():
      self.hits += 256
    if 0.25 >= np.random.rand():
      self.hits += 512
    if 0.25 == np.random.rand():
      self.hits += 1024
    if 0.25 != np.random.rand():
      self.hits += 2048
    if random.random() < 0.5:
      self.hits += 4096
    if random.random() <= 0.5:
      self.hits += 8192
    if random.random() > 0.5:
      self.hits += 16384
    if random.random() >= 0.5:
      self.hits += 32768
    if random.random() == 0.5:
      self.hits += 65536
    if random.random() != 0.5:
      self.hits += 131072
    if 0.25 < random.random():
      self.hits += 262144
    if 0.25 <= random.random():
      self.hits += 524288
    if 0.25 > random.random():
      self.hits += 1048576
    if 0.25 >= random.random():
      self.hits += 2097152
    if 0.25 == random.random():
      self.hits += 4194304
    if 0.25 != random.random():
      self.hits += 8388608
    if actions == 1:
      the_plot.terminate_episode()


# The literal each generator's draws of Thresholds.update are compared with, in order.
THRESHOLDS = (0.5,) * 6 + (0.25,) * 6


def make_thresholds(level):
  del level    # one level
  return ascii_art.ascii_art_to_game(['....', '.t..'], what_lies_beneath='.',
                                     drapes={'t': Thresholds})


# ---------------------------------------------------------------------- empty --
# Draws from an empty range on action 1: NumPy's randint, Python's randrange, choice(0).

class EmptyRange(plab_things.Drape):

  def __init__(self, curtain, character):
    super(EmptyRange, self).__init__(curtain, character)
    self.n = 3
    self.which = 0

  def update(self, actions, board, layers, backdrop, things, the_plot):
    if actions != 1:
      return
    if self.which == 0:
      self.n = np.random.randint(self.n, self.n)
    elif self.which == 1:
      self.n = random.randrange(self.n, self.n - 1)
    else:
      self.n = np.random.choice(self.n - self.n)


def make_empty(which):
  game = ascii_art.ascii_art_to_game(['....', '.x..'], what_lies_beneath='.',
                                     drapes={'x': EmptyRange})
  game.things['x'].which = which
  return game


# The classes a test registers, and the tables of the golden maker and the replays
# (tests/registered_games.py).
CLASSES = (Player, NumpyMonster, PythonMonster, Fruit, Edges, Thresholds, EmptyRange)
GAMES = {'monsters': make_monsters, 'edges': make_edges, 'thresholds': make_thresholds}
SPRITES = {'monsters': 'Pab', 'edges': '', 'thresholds': ''}
REGISTERS = {'monsters': (('P', 'bonuses'), ('f', 'eaten')),
             'edges': (('x', 'case'), ('x', 'out')), 'thresholds': (('t', 'hits'),)}
PLOT_KEYS = {'monsters': (), 'edges': (), 'thresholds': ()}
N_ACTIONS = {'monsters': 6, 'edges': 2, 'thresholds': 2}
GENERATORS = ('numpy', 'python')
RAISES = {}
FIELDS = ('game', 'level', 'rng_seed', 'actions', 'sprites', 'registers', 'reward_type',
          'numpy_words', 'python_words')

# (golden name, game, level, action seed, generator seed, steps)
CASES = (
    ('drawn_monsters_0', 'monsters', 0, 1, 7, 320),
    ('drawn_monsters_1', 'monsters', 1, 2, 8, 320),
    ('drawn_edges_0', 'edges', 0, 3, 9, 320),
    ('drawn_thresholds_0', 'thresholds', 0, 4, 10, 120),
)
