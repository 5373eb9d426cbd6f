"""The example-game goldens of tests/golden/make_golden.py: one table keyed by family, the
recorder of each side and the one replay.

A golden `<family>_*` belongs to FAMILIES[family], which says:
  keys       the arrays its goldens hold before the trajectory, in file order;
  inputs     those of `keys` a replay plays from; every other key is recorded per frame;
  sprites    the chars of its `sprites` rows (None: the golden's own `sprite_chars`);
  curtain    the drape whose curtain its `curtains` hold;
  seed       (generator, key): the global generator, 'numpy' or 'python', that the
             reference and the facade draw from, seeded from golden key `key`; the oracle
             builds its own generator from the same key;
  reference, oracle, facade
             build(name, g) -> (make_env, croppers) of each side: make_env() makes one env
             and sets the croppers' engine to it; `croppers` holds the croppers whose views
             the golden records, keyed as it holds them;
  frames     how many of a golden's actions the facade plays (None: all of them);
  checks     {side: check(env, out)}: more per-frame checks of that side's env.
The rest of a golden is its trajectory (trajectory.run_trajectory).  make_golden.py plays
the reference; test_example_goldens replays the oracle, test_gpu_example_goldens the facade.
"""

import collections
import importlib
import random

import numpy as np

import golden_cases as gc
import refdriver
import story_cases
import trajectory as tj
from oracle import engine_model as em
from oracle import games as ogames

Family = collections.namedtuple(
    'Family', 'keys inputs reference oracle facade sprites curtain seed frames checks',
    defaults=('', None, None, None, {}))


def family_of(name):
  return FAMILIES[name.split('_')[0]]


# ------------------------------------------------------------------ builders --

def _with(make, croppers=None):
  """(make_env, croppers): each env make() builds is the croppers' engine."""
  croppers = croppers or {}

  def make_env():
    env = make()
    for c in croppers.values():
      c.set_engine(env)
    return env
  return make_env, croppers


def _art(g):
  return tj.u8_to_art(g['art'])


def _seed(g, key):
  return int(g[key][0])


class _FixedCrop(object):
  """The oracle's FixedCropper (cropping.py:229-310): one window that never moves."""

  def __init__(self, top_left_corner, rows, cols, pad_char=None):
    self.corner, self.rows, self.cols, self.pad = top_left_corner, rows, cols, pad_char

  def set_engine(self, world):
    pass

  def crop(self, board):
    return em.crop_window(board, self.corner, self.rows, self.cols, self.pad)


def _better_croppers(g, scrolling, fixed):
  """The three views of better_scrolly_maze.py:224-251: the player's, patroller c's and a
  fixed teaser window."""
  return {'view_player': scrolling(rows=10, cols=30, to_track=['P'],
                                   initial_offset=tuple(int(x) for x in g['starter_offset'])),
          'view_patroller': scrolling(rows=7, cols=10, to_track=['c'], pad_char=' ',
                                      scroll_margins=(None, 3)),
          'view_teaser': fixed(top_left_corner=tuple(int(x) for x in g['teaser_corner']),
                               rows=12, cols=20, pad_char=' ')}


def _facade_better_croppers(g):
  from pycolab_b200.games import better_scrolly_maze as bsm
  views = bsm.make_croppers(tuple(int(x) for x in g['starter_offset']),
                            tuple(int(x) for x in g['teaser_corner']))
  return dict(zip(('view_player', 'view_patroller', 'view_teaser'), views))


def _crop_croppers(g, scrolling):
  """The one ScrollingCropper of a crop_* golden, as its config says."""
  cfg = gc.config_of(g)
  return {'crops': scrolling(cfg['rows'], cfg['cols'], ['P'], pad_char=cfg['pad'],
                             scroll_margins=tuple(cfg['margins']),
                             initial_offset=None if cfg['offset'] is None else tuple(cfg['offset']),
                             saccade=cfg['saccade'])}


def _reference_cropping():
  return refdriver._import()['cropping']


def _reference_example(module):
  refdriver._import()
  return importlib.import_module('pycolab.examples.' + module)


def _reference_shockwave(art):
  """A reference Shockwave game of `art`: make_game() takes a LEVELS index."""
  m = _reference_example('shockwave')
  m.LEVELS.append(art)
  try:
    return m.make_game(len(m.LEVELS) - 1)
  finally:
    m.LEVELS.pop()


def _classic(kind, art=None):
  return importlib.import_module('pycolab_b200.games.classics.' + kind).make_game(art)


class OracleOrdeal(object):
  """The three oracle worlds of examples/ordeal.py chained the way Story chains Engines
  (storytelling.py:391-474): crop, start successors until one survives its first
  frame, sum the rewards, keep the last discount."""

  def __init__(self):
    from pycolab_b200.games import ordeal
    self._arts = ordeal.ARTS
    self._crop = em.ScrollingCrop(8, 15, ['P'], scroll_margins=(2, 3))
    self.game_over = False
    self._enter('kansas', None)

  def _enter(self, chapter, story_plot):
    self.world = ogames.make_ordeal(chapter, self._arts[chapter], story_plot)
    self.chapter = chapter
    if chapter == 'kansas':
      self._crop.set_engine(self.world)

  def _view(self, board):
    return self._crop.crop(board) if self.chapter == 'kansas' else board

  def _deliver(self, out):
    board, reward, discount = out
    view = self._view(board)
    while self.world.game_over:
      store = self.world.plot.store
      if store['next_chapter'] is None:
        self.game_over = True
        break
      self._enter(store['next_chapter'], dict(has_sword=store['has_sword'],
                                              last_position=store['last_position'],
                                              prior_chapter=store['this_chapter']))
      board, more, discount = self.world.its_showtime()
      view = self._view(board)
      if more is not None:
        reward = more if reward is None else reward + more
    return view, reward, discount

  def its_showtime(self):
    return self._deliver(self.world.its_showtime())

  def play(self, action):
    return self._deliver(self.world.play(action))


def _oracle_list_story():
  from pycolab_b200 import storytelling

  class Story(storytelling.Story):
    @property
    def chapter(self):                    # as OracleOrdeal names its chapter
      return self.the_plot.this_chapter
  return Story([story_cases.oracle_chapter(k, a) for k, a in story_cases.LIST_CHAPTERS])


def _story(name, reference):
  """The Story of golden `name`, on the reference's classes or on the facade's."""
  if reference:
    storytelling, cropping = refdriver.ref_storytelling(), _reference_cropping()
    game = refdriver.ref_classic
  else:
    from pycolab_b200 import cropping, storytelling
    game = _classic
  if name == 'story_classics_list':
    return storytelling.Story([lambda k=k, a=a: game(k, a) for k, a in story_cases.LIST_CHAPTERS])

  def then(kind, target):
    def build():
      chapter = game(kind)
      chapter.the_plot.next_chapter = target
      return chapter
    return build
  return storytelling.Story(
      {'rooms': then('four_rooms', 'cliff'), 'cliff': then('cliff_walk', 'chain'),
       'chain': lambda: game('chain_walk')},
      first_chapter='rooms',
      croppers={'rooms': cropping.FixedCropper((1, 0), 4, 12), 'cliff': None,
                'chain': cropping.FixedCropper((0, 0), 4, 12, pad_char='.')})


def _apertures_follow_the_curtain(env, out):
  drape = env.things['X']
  assert sorted(drape.apertures) == sorted(zip(*np.nonzero(drape.curtain)))


def _int_rewards(env, out):
  assert out[1] is None or type(out[1]) is int


def _facade(module):
  return importlib.import_module('pycolab_b200.games.' + module).make_game


def _oracle_maze(g):
  maze, board, beneath = gc.scrolly_art(g)
  return ogames.make_scrolly_maze(maze, board, '+', beneath)


FAMILIES = {
    'scrolly': Family(
        ('maze_art', 'board_art', 'beneath', 'actions', 'sprites'),
        ('maze_art', 'board_art', 'beneath', 'actions'), sprites='Pabc',
        reference=lambda name, g: _with(lambda: refdriver.ref_scrolly_maze(*gc.scrolly_art(g))),
        oracle=lambda name, g: _with(lambda: _oracle_maze(g)),
        facade=lambda name, g: _with(lambda: _facade('scrolly_maze')(*gc.scrolly_art(g)))),
    'warehouse': Family(
        ('art', 'what_lies_beneath', 'sprite_chars', 'actions', 'sprites'),
        ('art', 'what_lies_beneath', 'sprite_chars', 'actions'), sprites=None,
        reference=lambda name, g: _with(lambda: refdriver.ref_warehouse(*gc.warehouse_art(g))),
        oracle=lambda name, g: _with(lambda: ogames.make_warehouse(*gc.warehouse_art(g))),
        facade=lambda name, g: _with(
            lambda: _facade('warehouse_manager')(*gc.warehouse_art(g)))),
    'marauders': Family(
        ('art', 'rng_seed', 'actions', 'sprites'), ('art', 'rng_seed', 'actions'),
        sprites='Pabcdyz', seed=('numpy', 'rng_seed'),
        reference=lambda name, g: _with(lambda: refdriver.ref_marauders(_art(g))),
        oracle=lambda name, g: (lambda rng: _with(lambda: ogames.make_marauders(_art(g), rng)))(
            np.random.RandomState(_seed(g, 'rng_seed'))),
        facade=lambda name, g: _with(lambda: _facade('extraterrestrial_marauders')(_art(g)))),
    'better': Family(
        ('art', 'starter_offset', 'teaser_corner', 'actions', 'sprites', 'view_player',
         'view_patroller', 'view_teaser'),
        ('art', 'starter_offset', 'teaser_corner', 'actions'), sprites='Pabc', frames=250,
        reference=lambda name, g: _with(
            lambda: refdriver.ref_better_scrolly(_art(g)),
            _better_croppers(g, _reference_cropping().ScrollingCropper,
                             _reference_cropping().FixedCropper)),
        oracle=lambda name, g: _with(lambda: ogames.make_better_scrolly(_art(g)),
                                     _better_croppers(g, em.ScrollingCrop, _FixedCrop)),
        facade=lambda name, g: _with(lambda: _facade('better_scrolly_maze')(_art(g)),
                                     _facade_better_croppers(g))),
    'crop': Family(
        ('maze_art', 'board_art', 'beneath', 'config', 'actions', 'crops', 'corners'),
        ('maze_art', 'board_art', 'beneath', 'config', 'actions'), frames=150,
        reference=lambda name, g: _with(
            lambda: refdriver.ref_scrolly_maze(*gc.scrolly_art(g)),
            _crop_croppers(g, _reference_cropping().ScrollingCropper)),
        oracle=lambda name, g: _with(
            lambda: _oracle_maze(g),
            _crop_croppers(g, em.ScrollingCrop)),
        facade=lambda name, g: _with(
            lambda: _facade('scrolly_maze')(*gc.scrolly_art(g)),
            _crop_croppers(g, importlib.import_module('pycolab_b200.cropping').ScrollingCropper))),
    'classic': Family(
        ('art', 'kind', 'actions', 'sprites', 'reward_type'), ('art', 'kind', 'actions'),
        sprites='P', frames=400,
        reference=lambda name, g: _with(
            lambda: refdriver.ref_classic(bytes(g['kind']).decode(), _art(g))),
        oracle=lambda name, g: _with(
            lambda: ogames.make_classic(bytes(g['kind']).decode(), _art(g))),
        facade=lambda name, g: _with(lambda: _classic(bytes(g['kind']).decode(), _art(g)))),
    'fluvial': Family(
        ('art', 'actions', 'sprites', 'backdrops'), ('art', 'actions'), sprites='P', frames=400,
        checks={'facade': _int_rewards},
        reference=lambda name, g: _with(lambda: refdriver.ref_fluvial(_art(g))),
        oracle=lambda name, g: _with(lambda: ogames.make_fluvial(_art(g))),
        facade=lambda name, g: _with(lambda: _facade('fluvial_natation')(_art(g)))),
    'aperture': Family(
        ('art', 'actions', 'sprites', 'curtains'), ('art', 'actions'), sprites='A', curtain='X',
        frames=350, checks={'facade': _apertures_follow_the_curtain},
        reference=lambda name, g: _with(lambda: refdriver.ref_aperture(art=_art(g))),
        oracle=lambda name, g: _with(lambda: ogames.make_aperture(_art(g))),
        facade=lambda name, g: _with(lambda: _facade('aperture')(_art(g)))),
    # The reference's hello_world and apprehend build their stock art, which `art` holds.
    'hello': Family(
        ('art', 'actions', 'sprites', 'curtains'), ('art', 'actions'), sprites='1234',
        curtain='@',
        reference=lambda name, g: _with(_reference_example('hello_world').make_game),
        oracle=lambda name, g: _with(lambda: ogames.make_hello(_art(g))),
        facade=lambda name, g: _with(lambda: _facade('hello_world')(_art(g)))),
    'apprehend': Family(
        ('art', 'actions', 'sprites', 'floats', 'random_seed'), ('art', 'actions', 'random_seed'),
        sprites='Pb', seed=('python', 'random_seed'),
        reference=lambda name, g: _with(_reference_example('apprehend').make_game),
        oracle=lambda name, g: (lambda rng: _with(lambda: ogames.make_apprehend(_art(g), rng)))(
            random.Random(_seed(g, 'random_seed'))),
        facade=lambda name, g: _with(lambda: _facade('apprehend')(_art(g)))),
    'shockwave': Family(
        ('art', 'actions', 'sprites', 'curtains', 'numpy_seed'), ('art', 'actions', 'numpy_seed'),
        sprites='P', curtain='@', seed=('numpy', 'numpy_seed'),
        reference=lambda name, g: _with(lambda: _reference_shockwave(_art(g))),
        oracle=lambda name, g: (lambda rng: _with(lambda: ogames.make_shockwave(_art(g), rng)))(
            np.random.RandomState(_seed(g, 'numpy_seed'))),
        facade=lambda name, g: _with(lambda: _facade('shockwave')(_art(g)))),
    'ordeal': Family(
        ('actions', 'chapters', 'has_sword'), ('actions',),
        reference=lambda name, g: _with(
            (refdriver.ref_storytelling(), _reference_example('ordeal'))[1].make_game),
        oracle=lambda name, g: _with(OracleOrdeal),
        facade=lambda name, g: _with(_facade('ordeal'))),
    'story': Family(
        ('actions', 'chapters'), ('actions',),
        reference=lambda name, g: _with(lambda: _story(name, reference=True)),
        oracle=lambda name, g: _with(_oracle_list_story),
        facade=lambda name, g: _with(lambda: _story(name, reference=False))),
}

# The goldens the parametrised replays cover: every one of FAMILIES but the Story goldens,
# whose replays are the story tests' own (test_story, test_gpu_story).
# story_classics_cropped crops on the device: the oracle has no replay of it.
REPLAYS = [name for fam in FAMILIES if fam != 'story' for name in gc.names(fam + '_')]


# ----------------------------------------------------------------- recorders --

class _Recorder(object):
  """on_frame for trajectory.run_trajectory: the fields golden `g`'s family records, frame
  by frame, the views from `croppers`; `arrays()` returns them as the goldens hold them.
  `check(env, out)`, if given, runs at every frame."""

  DTYPES = dict(sprites=np.int32, curtains=np.uint8, backdrops=np.uint8, reward_type=np.uint8,
                corners=np.int32, has_sword=np.uint8, floats=np.float64)

  def __init__(self, fam, g, croppers, check=None):
    self.chars = bytes(g['sprite_chars']).decode() if fam.sprites is None else fam.sprites
    self.curtain, self.croppers, self.check = fam.curtain, croppers, check
    self.rows = {k: [] for k in fam.keys if k not in fam.inputs}

  def __call__(self, env, out):
    for key, rows in self.rows.items():   # in file order: a frame's corner after its crop
      if key in self.croppers:
        rows.append(tj.board_of(self.croppers[key].crop(out[0])).copy())
      else:
        rows.append(getattr(self, key)(env, out))
    if self.check is not None:
      self.check(env, out)

  def arrays(self):
    # `chapters` is as wide as its longest chapter name, as in the goldens.
    return {k: np.array(rows, dtype=self.DTYPES.get(k)) for k, rows in self.rows.items()}

  def curtains(self, env, out):
    return np.array(env.things[self.curtain].curtain, dtype=np.uint8)

  def reward_type(self, env, out):
    return tj.reward_type(out[1])

  def corners(self, env, out):
    return self.corner(self.croppers['crops'])


class EngineRecorder(_Recorder):
  """The recorder of an Engine with the pycolab API: the reference's, or the facade's."""

  def sprites(self, env, out):
    return tj.sprite_rows(env, self.chars)

  def backdrops(self, env, out):
    return np.array(env.backdrop.curtain, dtype=np.uint8)

  def chapters(self, env, out):
    return str(env.the_plot.this_chapter)

  def has_sword(self, env, out):
    return 1 if env.the_plot.get('has_sword') else 0

  def floats(self, env, out):
    """Apprehend's ball: its slope and the accumulator of its drift.  The facade's ball
    drifts on the device, which holds them as float64 words of the ball's sprite record
    and of the Plot record."""
    ball, engine = env.things['b'], getattr(env, 'batched', None)
    if engine is None:
      return [ball._dx, ball._x_accumulator]
    from pycolab_b200 import _lib
    s = engine.sprite_chars.index('b')
    words = np.concatenate([engine.sprites[0, s, _lib.S_AUX0:_lib.S_AUX0 + 2].cpu().numpy(),
                            engine.plot[0, _lib.P_AUX0:_lib.P_AUX0 + 2].cpu().numpy()])
    return list(words.astype('<i4').view('<f8'))

  def corner(self, cropper):
    state = getattr(cropper, '_state', None)     # the facade's window is device state
    return list(cropper._corner) if state is None else [int(v) for v in state[0, :2].cpu()]


class WorldRecorder(_Recorder):
  """The recorder of oracle worlds (oracle/games.py, oracle/compiled.py) and of
  OracleOrdeal."""

  def sprites(self, world, out):
    return tj.world_sprite_rows(world, self.chars)

  def backdrops(self, world, out):
    return np.array(world.backdrop, dtype=np.uint8)

  def chapters(self, env, out):
    return str(env.chapter)

  def has_sword(self, env, out):
    return 1 if env.world.plot.store.get('has_sword') else 0

  def floats(self, world, out):
    ball = world.things['b']
    return [ball.aux['dx'], ball.aux['acc']]

  def corner(self, cropper):
    return list(cropper.corner)


# -------------------------------------------------------------------- replay --

def play(side, name, g, frames=None, make_env=None, check=None):
  """Plays the first `frames` of golden `g`'s actions (None: all of them) on `side`'s env
  of golden `name` under the trajectory protocol, the family's global generator seeded
  from `g` on the reference and the facade.  Returns the trajectory and every field the
  family records.  A `make_env` replaces the table's env and its croppers."""
  fam = family_of(name)
  croppers = {}
  if make_env is None:
    make_env, croppers = getattr(fam, side)(name, g)
  if fam.seed is not None and side != 'oracle':
    stream, key = fam.seed
    (random if stream == 'python' else np.random).seed(_seed(g, key))
  rec = (WorldRecorder if side == 'oracle' else EngineRecorder)(fam, g, croppers, check)
  got = tj.run_trajectory(make_env, g['actions'].tolist()[:frames], on_frame=rec)
  got.update(rec.arrays())
  return got


def assert_replays(side, name, make_env=None, check=None):
  """`side`'s env ('oracle' or 'facade') reproduces every array golden `name` holds apart
  from its inputs, dtype and shape included, up to the frames it plays: all of them, or the
  family's facade limit.  A field the replay did not record fails, naming the field.  The
  family's checks of `side` run at every frame.  A caller's `make_env` replaces the table's
  env, its frame limit and its checks by `check`; it replays the whole golden.  Run the
  facade under the global_generators fixture: it seeds the global generators."""
  g = gc.load(name)
  fam = family_of(name)
  if make_env is None:
    frames, check = (fam.frames if side == 'facade' else None), fam.checks.get(side)
  else:
    frames = None
  got = play(side, name, g, frames, make_env, check)
  n = len(got['boards'])
  want = {k: v if k in fam.inputs else v[:n] for k, v in g.items()}
  tj.assert_golden_arrays(name, want, got, fam.inputs)
