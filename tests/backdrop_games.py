"""Games whose Backdrop has update() code, for the compiled step program: ordinary pycolab
code, whose classes the tests register with `pycolab_b200.compiler`.

This module imports `pycolab.*` only, so it runs unchanged on the reference (the golden
maker, tests/golden/make_registered_golden.py) and on this package (loaded through
`compat.load_example`).  Three games:

  fluvial  a swimmer in a river whose middle rows flow one cell west on even frames: the
           logic of the reference's examples/fluvial_natation.py, so that the reference's
           goldens (tests/golden/fluvial_*.npz) and the hand-written PCL_PROG_CLASSICS kernel
           check it.  `make_fluvial(art)` takes the level's art.
  trail    a walker whose Backdrop paints the cell it just left, with palette look-ups, reads
           of its own curtain and the walker's position: a cell left twice becomes a wall
           '+', which the walker cannot enter, but it still sees the board of the last
           render, so it may step back onto a wall painted in the same frame.  A drape reads
           the updated curtain under the walker in the same frame.  Two levels of one shape.
  flow     bands of the Backdrop rolled on both axes, by shifts drawn from np.random and
           taken from a Plot key, negative ones too; the whole curtain filled when the
           player floods it; a walker confined to the board.  Two levels of one shape.
"""

import numpy as np

from pycolab import ascii_art
from pycolab import things as plab_things
from pycolab.prefab_parts import sprites as prefab_sprites


# -------------------------------------------------------------------- fluvial --
# Actions 0 swim west, 1 swim east, 2 float.

def make_fluvial(art):
  return ascii_art.ascii_art_to_game(art, what_lies_beneath=' ', sprites={'P': Swimmer},
                                     backdrop=River)


class Swimmer(prefab_sprites.MazeWalker):
  """Carried one cell west on even frames; leaving the board east wins, west loses."""

  def __init__(self, corner, position, character):
    super(Swimmer, self).__init__(corner, position, character, impassable='')

  def update(self, actions, board, layers, backdrop, things, the_plot):
    if the_plot.frame % 2 == 0:
      self._west(board, the_plot)
    if actions == 0:
      self._west(board, the_plot)
    elif actions == 1:
      self._east(board, the_plot)
    if self.virtual_position[1] < 0:
      the_plot.add_reward(-1)
      the_plot.terminate_episode()
    elif self.virtual_position[1] >= board.shape[1]:
      the_plot.add_reward(1)
      the_plot.terminate_episode()


class River(plab_things.Backdrop):
  """Rows 1 to 3 flow one cell west on even frames."""

  def update(self, actions, board, layers, things, the_plot):
    if the_plot.frame % 2 == 0:
      self.curtain[1:4, :] = np.roll(self.curtain[1:4, :], shift=-1, axis=1)


# ---------------------------------------------------------------------- trail --
# Actions 0-3 N S W E, 4 stay, 5 quit.

TRAIL_ART = [
    ['##########',
     '#P     $ #',
     '#  ..    #',
     '# $    + #',
     '#     $  #',
     '##########'],
    ['##########',
     '#  $  .  #',
     '# +   P  #',
     '#   $    #',
     '#  .   $ #',
     '##########'],
]


def make_trail(level):
  game = ascii_art.ascii_art_to_game(
      TRAIL_ART[level], what_lies_beneath=' ', sprites={'P': Walker}, drapes={'$': Purse},
      backdrop=Trail, update_schedule=[['P'], ['$']], z_order='$P')
  row, col = game.things['P'].position
  game.the_plot['prev_row'] = int(row)
  game.the_plot['prev_col'] = int(col)
  game.the_plot['dots'] = 0
  return game


class Walker(prefab_sprites.MazeWalker):
  """Walls and painted walls stop it."""

  def __init__(self, corner, position, character):
    super(Walker, self).__init__(corner, position, character, impassable='#+')

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


class Trail(plab_things.Backdrop):
  """Paints the cell the walker left: a dot, or a wall where a dot already was."""

  def update(self, actions, board, layers, things, the_plot):
    del actions, layers
    row, col = things['P'].position
    prev_row = the_plot['prev_row']
    prev_col = the_plot['prev_col']
    if prev_row != row or prev_col != col:
      if self.curtain[prev_row, prev_col] == self.palette.period:
        self.curtain[prev_row, prev_col] = self.palette['+']
      elif board[prev_row, prev_col] == ord('$'):
        self.curtain[prev_row, prev_col] = self.palette.plus if things['P'].visible else 0
      else:
        self.curtain[prev_row, prev_col] = ord('.')
      the_plot['prev_row'] = row
      the_plot['prev_col'] = col
    if row == self.curtain.shape[0] - 2 and col == board.shape[1] - 2:
      self.curtain[1, -2] = self.curtain[row - 1, col]


class Purse(plab_things.Drape):
  """Coins: +10 each, the last ends the episode; -1 for standing on a painted wall, and a
  count of the dots the walker stands on, read from the Backdrop's curtain of this frame."""

  def update(self, actions, board, layers, backdrop, things, the_plot):
    at = things['P'].position
    if self.curtain[at]:
      self.curtain[at] = False
      the_plot.add_reward(10)
      if not self.curtain.any():
        the_plot.terminate_episode()
    if backdrop.curtain[at] == ord('+'):
      the_plot.add_reward(-1)
    if chr(backdrop.curtain[at]) == '.':
      the_plot['dots'] += 1


# ----------------------------------------------------------------------- flow --
# Actions 0-3 N S W E, 4 flood, 5 quit.

FLOW_ART = [
    ['###########',
     '~ .  ~~ . .',
     ' .~   .  ~ ',
     '   ~ P  .  ',
     '.  ~  . ~ .',
     '###########'],
    ['###########',
     '. ~ ~ . . ~',
     '~ .  ~   . ',
     ' ~ . P ~ . ',
     '  .   ~ .~ ',
     '###########'],
]


def make_flow(level):
  game = ascii_art.ascii_art_to_game(FLOW_ART[level], what_lies_beneath=' ',
                                     sprites={'P': Rower}, backdrop=Flow)
  game.the_plot['tide'] = -2
  return game


class Rower(prefab_sprites.MazeWalker):
  """Walls stop it, the board's edge too; +1 for each dot it ends a frame on."""

  def __init__(self, corner, position, character):
    super(Rower, self).__init__(corner, position, character, impassable='#',
                                confined_to_board=True)

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
    if backdrop.curtain[self.position] == ord('.'):
      the_plot.add_reward(1)


class Flow(plab_things.Backdrop):
  """A flood on action 4 in every sixth frame; every frame, the two top water rows drift by the tide less a
  draw, the lower rows move up by one or two, the whole curtain east every ninth frame."""

  def update(self, actions, board, layers, things, the_plot):
    if actions == 4 and the_plot.frame % 6 == 0:
      self.curtain[:] = self.curtain[1, 1] if the_plot['tide'] > 0 else self.palette.tilde
      the_plot.add_reward(-3)
    drift = the_plot['tide'] - np.random.randint(3)
    self.curtain[1:3, :] = np.roll(self.curtain[1:3, :], drift, axis=1)
    self.curtain[2:-1] = np.roll(self.curtain[2:-1], shift=-1 - np.random.randint(2), axis=0)
    self.curtain[:] = np.roll(self.curtain, 1 if the_plot.frame % 9 == 0 else 0, 1)
    if the_plot.frame % 4 == 0:
      the_plot['tide'] = (the_plot['tide'] + 2) % 5 - 2
    self.curtain[0, the_plot.frame % self.curtain.shape[1]] = board[3, 3]
    self.curtain[-1, 0] = self.palette['#'] if layers['P'][3, 5] else self.palette.tilde


# The classes a test registers, and the tables of the golden maker and the replays
# (tests/registered_games.py).
CLASSES = (Swimmer, River, Walker, Trail, Purse, Rower, Flow)

# (golden name, game, level, action seed, generator seed, steps)
CASES = [('backdrop_trail_0', 'trail', 0, 41, 3, 300), ('backdrop_trail_1', 'trail', 1, 42, 4, 300),
         ('backdrop_flow_0', 'flow', 0, 43, 5, 300), ('backdrop_flow_1', 'flow', 1, 44, 6, 300)]
GAMES = {'trail': make_trail, 'flow': make_flow}
N_ACTIONS = {'trail': 6, 'flow': 6}
SPRITES = {'trail': 'P', 'flow': 'P'}
REGISTERS = {'trail': [], 'flow': []}
PLOT_KEYS = {'trail': ['prev_row', 'prev_col', 'dots'], 'flow': ['tide']}
GENERATORS = ('numpy',)
RAISES = {}
FIELDS = ('game', 'level', 'rng_seed', 'actions', 'sprites', 'backdrops', 'plot_keys',
          'reward_type', 'numpy_words')
