"""Games whose update() code calls the game's own helpers, for the compiled step program:
ordinary pycolab code, whose entity classes the tests register with `pycolab_b200.compiler`
(which inlines each helper call).

This module imports `pycolab.*` only, so it runs unchanged on the reference (the golden
maker, tests/golden/make_registered_golden.py) and on this package (loaded through
`compat.load_example`).  Three games:

  bolts    marauders-like: the bolts share one registered `Bolt` base whose update() calls
           `self._ready`, `self._fly` and `self._fire`, which the upward and downward bolt
           classes override as the reference's extraterrestrial_marauders.py writes them
           (`return self._teleport((-1, -1))`, `the_plot.get(...)`), a downward bolt drawing
           its column from np.random; a stray bolt class overrides nothing.  The marauders
           are a plain drape whose helper erases a hit cell, counts hits in a register and
           writes a Plot key that the upward bolt reads.  Two levels.
  chaser   level 0: module-level functions returning ints and positions (`_sign`, `_gap`,
           `_dist`, `_toward`, `_ahead`), keyword arguments and defaults, value-returning
           helpers in conditions and arithmetic, a helper three calls deep, a motion-result
           helper shared through a user base class, a plain drape whose helper takes a
           character constant (`things[who]`), and a registered Backdrop whose helpers paint
           its curtain with a palette character passed as an argument.  Level 1: a scrolling
           maze, where an egocentric walker's helper and a Scrolly's helper call the motion
           helpers.
  divzero  a helper that divides by a register the actions count down: upstream raises
           ZeroDivisionError.
"""

import numpy as np

from pycolab import ascii_art
from pycolab import things as plab_things
from pycolab.prefab_parts import drapes as prefab_drapes
from pycolab.prefab_parts import sprites as prefab_sprites


# ---------------------------------------------------------------------- bolts --
# Actions 0 left, 1 right, 2 fire, 3 fire the stray bolt, 4 quit.

BOLTS_ART = [
    ['!:;^      ',
     ' XXX  XXX ',
     ' X X  XX  ',
     '          ',
     '          ',
     '          ',
     '    P     '],
    ['!:;^        ',
     '  XX XX XX  ',
     ' XXXXXXXXXX ',
     '            ',
     '            ',
     '      P     '],
]


def make_bolts(level):
  game = ascii_art.ascii_art_to_game(
      BOLTS_ART[level], what_lies_beneath=' ',
      sprites={'P': Cannon, '!': UpBolt, ':': DownBolt, ';': DownBolt, '^': StrayBolt},
      drapes={'X': Marauders},
      update_schedule=[['P', 'X'], ['!', ':', ';', '^']],
      z_order='X!:;^P')
  game.the_plot['hit_frame'] = -1
  game.the_plot['last_player_shot'] = -1
  game.the_plot['last_marauder_shot'] = -1
  return game


class Cannon(prefab_sprites.MazeWalker):
  """Slides along the bottom row."""

  def __init__(self, corner, position, character):
    super(Cannon, self).__init__(corner, position, character, impassable='',
                                 confined_to_board=True)

  def update(self, actions, board, layers, backdrop, things, the_plot):
    if actions == 0:
      self._west(board, the_plot)
    elif actions == 1:
      self._east(board, the_plot)
    elif actions == 4:
      the_plot.terminate_episode()


class Marauders(plab_things.Drape):
  """A visible upward bolt inside a marauder erases it, pays 10 and leaves the frame in
  the Plot, where the bolt looks for it."""

  def __init__(self, curtain, character):
    super(Marauders, self).__init__(curtain, character)
    self.hits = 0

  def update(self, actions, board, layers, backdrop, things, the_plot):
    if things['!'].visible and self.curtain[things['!'].position]:
      self._hit(things['!'].position, the_plot)

  def _hit(self, at, the_plot):
    self.curtain[at] = False
    self.hits += 1
    the_plot['hit_frame'] = the_plot.frame
    the_plot.add_reward(10)
    if not self.curtain.any():
      return the_plot.terminate_episode()


class Bolt(prefab_sprites.MazeWalker):
  """Starts off the board; flies while visible, else fires when it is ready."""

  def __init__(self, corner, position, character):
    super(Bolt, self).__init__(corner, position, character, impassable='')
    self._teleport((-1, -1))

  def update(self, actions, board, layers, backdrop, things, the_plot):
    if self.visible:
      self._fly(board, layers, things, the_plot)
    elif self._ready(actions, the_plot):
      self._fire(layers, things, the_plot)

  def _ready(self, actions, the_plot):
    return actions == 3

  def _fly(self, board, layers, things, the_plot):
    self._north(board, the_plot)

  def _fire(self, layers, things, the_plot):
    row, col = things['P'].position
    self._teleport((row - 2, col))


class UpBolt(Bolt):
  """The player's bolt."""

  def _ready(self, actions, the_plot):
    return actions == 2

  def _fly(self, board, layers, things, the_plot):
    """Disappears where it hit a marauder, else flies north."""
    if the_plot['hit_frame'] == the_plot.frame:
      return self._teleport((-1, -1))
    self._north(board, the_plot)

  def _fire(self, layers, things, the_plot):
    """Launches from just above the player, once per frame."""
    if the_plot.get('last_player_shot') == the_plot.frame: return
    the_plot['last_player_shot'] = the_plot.frame
    row, col = things['P'].position
    self._teleport((row-1, col))


class DownBolt(Bolt):
  """The marauders' bolts: two of them, one launched per frame from a random column."""

  def _ready(self, actions, the_plot):
    return True

  def _fly(self, board, layers, things, the_plot):
    if self.position == things['P'].position: the_plot.terminate_episode()
    if self.position.row == self.corner.row - 1:
      return self._teleport((-1, -1))
    self._south(board, the_plot)

  def _fire(self, layers, things, the_plot):
    if the_plot.get('last_marauder_shot') == the_plot.frame: return
    the_plot['last_marauder_shot'] = the_plot.frame
    col = np.random.randint(10)
    if layers['X'][1, col] or layers['X'][2, col]:
      self._teleport((3, col))


class StrayBolt(Bolt):
  """Overrides nothing: runs Bolt's helpers."""


# --------------------------------------------------------------------- chaser --
# Actions 0-3 N S W E, 4 stay, 5 quit.

CHASER_ART = ['#########',
              '#P   . +#',
              '#  ##   #',
              '# .   c #',
              '#    .  #',
              '#########']

SCROLL_ART = ['##############',
              '#   #    #   #',
              '# +    #     #',
              '#   #  P     #',
              '#        #   #',
              '#  #   #     #',
              '#     #   #  #',
              '##############']
SCROLL_BOARD = (5, 8)


def make_chaser(level):
  if level == 1:
    return make_scrolling()
  return ascii_art.ascii_art_to_game(
      CHASER_ART, what_lies_beneath=' ', sprites={'P': Runner, 'c': Chaser},
      drapes={'.': Coins}, backdrop=Trail, update_schedule=[['P', 'c'], ['.']],
      z_order='.cP')


def make_scrolling():
  info = prefab_drapes.Scrolly.PatternInfo(
      SCROLL_ART, SCROLL_BOARD, board_northwest_corner_mark='+', what_lies_beneath=' ')
  board = [' ' * SCROLL_BOARD[1]] * SCROLL_BOARD[0]
  return ascii_art.ascii_art_to_game(
      board, what_lies_beneath=' ',
      sprites={'P': ascii_art.Partial(Scout, info.virtual_position('P'))},
      drapes={'#': ascii_art.Partial(Maze, scroll_margins=None, **info.kwargs('#'))},
      update_schedule=[['#'], ['P']], z_order='#P')


def _sign(x):
  if x > 0:
    return 1
  if x < 0:
    return -1
  return 0


def _gap(a, b):
  return a - b if a > b else b - a


def _dist(p, q, scale=1):
  return scale * (_gap(p.row, q.row) + _gap(p.col, q.col))


def _toward(pos, target, vertical=True):
  """A direction 0-3 (N S W E) from `pos` toward `target`."""
  dr = _sign(target.row - pos.row)
  dc = _sign(target.col - pos.col)
  if vertical and dr != 0:
    return 0 if dr < 0 else 1
  if dc != 0:
    return 2 if dc < 0 else 3
  return 0 if dr < 0 else 1


def _ahead(pos, direction):
  """The cell one step from `pos` in `direction`."""
  if direction == 0:
    return (pos.row - 1, pos.col)
  if direction == 1:
    return (pos.row + 1, pos.col)
  if direction == 2:
    return (pos.row, pos.col - 1)
  return (pos.row, pos.col + 1)


class Mover(prefab_sprites.MazeWalker):
  """Walls stop it; `_go` steps in a direction 0-3 and returns the motion's result."""

  def __init__(self, corner, position, character):
    super(Mover, self).__init__(corner, position, character, impassable='#')
    self.bumps = 0

  def _go(self, board, the_plot, d):
    if d == 0:
      return self._north(board, the_plot)
    if d == 1:
      return self._south(board, the_plot)
    if d == 2:
      return self._west(board, the_plot)
    if d == 3:
      return self._east(board, the_plot)


class Runner(Mover):

  def update(self, actions, board, layers, backdrop, things, the_plot):
    if actions == 5:
      the_plot.terminate_episode()
    elif self._go(board, the_plot, actions) is not None:
      self._bump()

  def _bump(self):
    self.bumps += 1


class Chaser(Mover):
  """Every other frame, one step toward the runner, turning where a wall is ahead; close
  to the runner it ends the episode."""

  def update(self, actions, board, layers, backdrop, things, the_plot):
    if actions is None:
      return
    if the_plot.frame % 2 == 0:
      self._chase(board, things, the_plot)

  def _chase(self, board, things, the_plot):
    target = things['P'].position
    if _dist(self.position, target, scale=2) <= 2:
      the_plot.add_reward(-1)
      the_plot.terminate_episode()
      return
    d = _toward(self.position, target, vertical=the_plot.frame % 4 == 0)
    if board[_ahead(self.position, d)] == ord('#'):
      d = _toward(self.position, target, vertical=the_plot.frame % 4 != 0)
    if self._go(board, the_plot, d=d) is not None:
      self.bumps += 1 + _gap(d, 1)


class Coins(plab_things.Drape):
  """The runner collects a coin for 3, the chaser eats one for -1; the last ends the
  episode."""

  def __init__(self, curtain, character):
    super(Coins, self).__init__(curtain, character)
    self.eaten = 0

  def update(self, actions, board, layers, backdrop, things, the_plot):
    if self._under(things, 'P'):
      self._collect(things['P'].position, the_plot, reward=3)
    if self._under(things, 'c'):
      self._collect(things['c'].position, the_plot)

  def _under(self, things, who):
    return things[who].visible and self.curtain[things[who].position]

  def _collect(self, at, the_plot, reward=-1):
    self.curtain[at] = False
    self.eaten += 1
    the_plot.add_reward(reward)
    if not self.curtain.any():
      the_plot.terminate_episode()


class Trail(plab_things.Backdrop):
  """Marks the chaser's cell with '+' on frames divisible by 3 and clears it otherwise,
  never over a wall."""

  def update(self, actions, board, layers, things, the_plot):
    if the_plot.frame % 3 == 0:
      self._mark(things['c'].position, '+')
    else:
      self._mark(things['c'].position, ' ')

  def _mark(self, at, ch):
    if self._open(at):
      self.curtain[at] = self.palette[ch]

  def _open(self, at):
    return self.curtain[at] != self.palette['#']


class Scout(prefab_sprites.MazeWalker):
  """Egocentric; walls stop it."""

  def __init__(self, corner, position, character, virtual_position):
    super(Scout, self).__init__(
        corner, position, character, egocentric_scroller=True, impassable='#')
    self._teleport(virtual_position)
    self.bumps = 0

  def update(self, actions, board, layers, backdrop, things, the_plot):
    if actions == 5:
      the_plot.terminate_episode(0.5)
    else:
      self._walk(actions, board, the_plot)

  def _walk(self, action, board, the_plot):
    if action == 0:
      self._north(board, the_plot)
    elif action == 1:
      self._south(board, the_plot)
    elif action == 2:
      self._west(board, the_plot)
    elif action == 3:
      self._east(board, the_plot)
    else:
      self._stay(board, the_plot)
    self.bumps += the_plot.frame % 2


class Maze(prefab_drapes.Scrolly):

  def update(self, actions, board, layers, backdrop, things, the_plot):
    self._follow(actions, the_plot)

  def _follow(self, action, the_plot):
    if action == 0:
      self._north(the_plot)
    elif action == 1:
      self._south(the_plot)
    elif action == 2:
      self._west(the_plot)
    elif action == 3:
      self._east(the_plot)
    else:
      self._stay(the_plot)


# -------------------------------------------------------------------- divzero --
# Actions 0 west, 1 east, 2 count down, 3 quit.

def make_divzero():
  return ascii_art.ascii_art_to_game(
      ['#######', '#  P  #', '#######'], what_lies_beneath=' ',
      sprites={'P': Divider}, update_schedule=[['P']], z_order='P')


class Divider(prefab_sprites.MazeWalker):
  """Shares 12 among `left` parts; the third count-down divides by zero."""

  def __init__(self, corner, position, character):
    super(Divider, self).__init__(corner, position, character, impassable='#')
    self.left = 3
    self.share = 0

  def update(self, actions, board, layers, backdrop, things, the_plot):
    if actions == 0:
      self._west(board, the_plot)
    elif actions == 1:
      self._east(board, the_plot)
    elif actions == 2:
      self.left -= 1
    elif actions == 3:
      the_plot.terminate_episode()
    self.share = self._ratio(12, self.left)

  def _ratio(self, total, parts):
    return total // parts


# The classes a test registers, and the tables of the golden maker and the replays
# (tests/registered_games.py).
CLASSES = (Cannon, Marauders, Bolt, Runner, Chaser, Coins, Trail, Scout, Maze, Divider)

# (golden name, game, level, action seed, generator seed, steps)
CASES = [('helper_bolts_0', 'bolts', 0, 41, 3, 400), ('helper_bolts_1', 'bolts', 1, 42, 4, 400),
         ('helper_chaser_0', 'chaser', 0, 43, 0, 300),
         ('helper_chaser_1', 'chaser', 1, 44, 0, 300),
         ('helper_divzero', 'divzero', 0, 45, 0, 40)]
GAMES = {'bolts': make_bolts, 'chaser': make_chaser, 'divzero': lambda level: make_divzero()}
N_ACTIONS = {'bolts': 5, 'chaser': 6, 'divzero': 4}
SPRITES = {'bolts': 'P!:;^', 'chaser': 'P', 'divzero': 'P'}
# Registers as ints; a position attribute as its row and column.
REGISTERS = {'bolts': [('X', 'hits')], 'chaser': [('P', 'bumps')],
             'divzero': [('P', 'left'), ('P', 'share')]}
PLOT_KEYS = {'bolts': ['hit_frame', 'last_player_shot', 'last_marauder_shot'], 'chaser': [],
             'divzero': []}
GENERATORS = ('numpy',)
RAISES = {'divzero': ZeroDivisionError}
FIELDS = ('game', 'level', 'rng_seed', 'actions', 'sprites', 'registers', 'reward_type',
          'numpy_words', 'raised_at')
