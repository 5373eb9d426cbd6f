"""The Story goldens of tests/golden/make_golden.py (story_classics_*), and oracle
worlds dressed as the Engines a Story chains (shared by the story tests and
tests/example_games.py)."""

import importlib

import numpy as np

from oracle import games as ogames
from pycolab_b200 import engine as engine_lib
from pycolab_b200 import plot as plot_lib
from pycolab_b200 import rendering
from pycolab_b200 import things

# Same-shape (4x12) chapters of the list-style story.  (A list-story of scrolly_maze
# levels is not a usable case: the reference copies the old Plot's scrolling-protocol
# entries into the next game, whose Scrollys then reject the stale order.)
LIST_CHAPTERS = (
    ('cliff_walk', None),
    ('chain_walk', ['............', '.....P......', '............', '............']),
    ('cliff_walk', ['............', '............', '........P...', '............']),
)


class _Walker(things.Sprite):
  def update(self, *args, **kwargs):
    raise AssertionError('never called')


class OracleEngine(object):
  """An oracle World with the attributes Story reads from an Engine."""

  def __init__(self, world, palette):
    self._world = world
    self.the_plot = plot_lib.Plot()
    self.rows, self.cols = world.rows, world.cols
    self._palette = palette

  def _obs(self, out):
    board = np.asarray(out[0], dtype=np.uint8)
    chars = set(self._palette) | set(self._world.things)
    return rendering.Observation(board=board, layers=rendering.LazyLayers(board, chars)), out[1], out[2]

  def its_showtime(self):
    return self._obs(self._world.its_showtime())

  def play(self, actions):
    return self._obs(self._world.play(actions))

  @property
  def game_over(self):
    return self._world.game_over

  @property
  def z_order(self):
    return list(self._world.things)

  @property
  def backdrop(self):
    return things.Backdrop(curtain=self._world.backdrop, palette=engine_lib.Palette(self._palette))

  @property
  def things(self):
    return {ch: _Walker(things.Sprite.Position(self.rows, self.cols),
                        things.Sprite.Position(w.row, w.col), ch)
            for ch, w in self._world.things.items()}


def oracle_chapter(kind, art):
  """A Story chapter: makes an OracleEngine of a classics game on `art` (None: its stock
  art)."""
  stock = importlib.import_module('pycolab_b200.games.classics.' + kind).GAME_ART
  palette = ' #' if kind == 'four_rooms' else '.'
  return lambda: OracleEngine(ogames.make_classic(kind, art or list(stock)), palette)
