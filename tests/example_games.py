"""The example-game and research-game goldens of tests/golden/make_golden.py: one table keyed
by family, the recorder of each side and the one replay.

A golden `<family>_*` belongs to FAMILIES[family], which says:
  keys       the arrays its goldens hold, in file order; the trajectory's arrays
             (trajectory.TRAJECTORY) follow them unless `keys` places them;
  inputs     those of `keys` a replay plays from; every other key is recorded per frame;
  sprites    the chars of its `sprites` rows (None: the golden's own `sprite_chars`);
  curtain    the drape whose curtain its `curtains` hold;
  seed       (generator, key): the global generator, 'numpy', 'python' or 'both', that the
             reference and the facade draw from, seeded from golden key `key` ('config':
             the seed its config holds); the oracle builds its own generators from it;
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

import box_world_cases as bwc
import golden_cases as gc
import lp_rnn_cases as lc
import refdriver
import story_cases
import trajectory as tj
from oracle import box_world as obw
from oracle import cued_catch as occ
from oracle import engine_model as em
from oracle import games as ogames
from oracle import sequence_recall as osr
from oracle import t_maze as otm

Family = collections.namedtuple(
    'Family', 'keys inputs reference oracle facade sprites curtain seed frames checks',
    defaults=('', None, None, None, {}))


def family_of(name):
  return next(fam for key, fam in FAMILIES.items() if name.startswith(key + '_'))


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
  return gc.config_of(g)['seed'] if key == 'config' else int(g[key][0])


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


def _float_rewards(env, out):
  assert out[1] is None or isinstance(out[1], float)


def _t_maze_windows(env, out):
  """Float rewards, and each Scrolly's curtain the window of its rolled whole_pattern
  (drapes.py:689-695)."""
  _float_rewards(env, out)
  for ch in '#*ltr':
    d = env.things[ch]
    r, c = d._northwest_corner
    np.testing.assert_array_equal(d.curtain, d.whole_pattern[r:r + env.rows, c:c + env.cols], ch)


def _box_world_plot(env, out):
  """Float rewards, and the_plot['over_this'] holding a Position, as the reference's does."""
  _float_rewards(env, out)
  over = env.the_plot.get('over_this')
  assert not over or type(over[1]).__name__ == 'Position'


def _facade(module):
  return importlib.import_module('pycolab_b200.games.' + module).make_game


def _oracle_maze(g):
  maze, board, beneath = gc.scrolly_art(g)
  return ogames.make_scrolly_maze(maze, board, '+', beneath)


def _t_maze(g):
  """t_maze's maze and cue art and make_game's arguments after them."""
  cfg = gc.config_of(g)
  return (tj.u8_to_art(g['maze_art']), tj.u8_to_art(g['cue_art']), cfg['level'],
          cfg['cue_after_teleport'], cfg['timeout_frames'], cfg['teleport_delay'],
          cfg['limbo_time'])


def _reference_t_maze(name, g):
  ref, args = lc.ref_module('t_maze'), _t_maze(g)[2:]    # on its own art, as `maze_art` holds
  return _with(lambda: ref.make_game(*args))


def _oracle_t_maze(name, g):
  seed = _seed(g, 'config')
  rng, np_rng = random.Random(seed), np.random.RandomState(seed)
  return _with(lambda: otm.make_t_maze(*_t_maze(g), rng=rng, np_rng=np_rng))


def _facade_t_maze(name, g):
  maze, cue, *args = _t_maze(g)
  return _with(lambda: _facade('t_maze')(*args, maze_art=maze, cue_art=cue))


def _reference_lp_rnn(game, shim):
  """The build of a Cued Catch or Sequence Recall golden's reference env: the reference's
  module, shimmed, on the golden's art."""
  def build(name, g):
    ref, args = lc.ref_module(game), gc.config_of(g)['args']
    return _with(lambda: shim(lc.with_art(ref, _art(g), lambda: ref.make_game(*args))))
  return build


def _box_level(g):
  """(art, distractors, max_num_steps) of a box_world golden."""
  return (_art(g), [tuple(int(v) for v in xy) for xy in g['distractors']],
          gc.config_of(g)['max_num_steps'])


def _reference_box_world(name, g):
  ref, cfg = bwc.ref_module(), gc.config_of(g)
  return _with(lambda: ref.make_game(cfg['grid_size'], *bwc.ARGS,
                                     random_state=np.random.RandomState(cfg['seed']),
                                     max_num_steps=cfg['max_num_steps']))


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
    't_maze': Family(
        ('maze_art', 'cue_art', 'actions', 'sprites', 'reward_f64', 'which_goal', 'config'),
        ('maze_art', 'cue_art', 'actions', 'config'), sprites='P', seed=('both', 'config'),
        checks={'facade': _t_maze_windows},
        reference=_reference_t_maze, oracle=_oracle_t_maze, facade=_facade_t_maze),
    'cued_catch': Family(
        ('art', 'actions', 'sprites', 'reward_f64', 'reward_type', 'state', 'config'),
        ('art', 'actions', 'config'), sprites='Pab', seed=('python', 'config'),
        reference=_reference_lp_rnn('cued_catch', lc.shim_cued_catch),
        oracle=lambda name, g: (lambda rng: _with(lambda: occ.make_cued_catch(
            _art(g), *gc.config_of(g)['args'], rng=rng)))(random.Random(_seed(g, 'config'))),
        facade=lambda name, g: _with(lambda: _facade('cued_catch')(
            *gc.config_of(g)['args'], art=_art(g)))),
    'sequence_recall': Family(
        ('art', 'actions', 'sprites', 'reward_f64', 'state', 'config'),
        ('art', 'actions', 'config'), sprites='P', seed=('python', 'config'),
        checks={'facade': _float_rewards},
        reference=_reference_lp_rnn('sequence_recall', lc.shim_sequence_recall),
        oracle=lambda name, g: (lambda rng: _with(lambda: osr.make_sequence_recall(
            _art(g), *gc.config_of(g)['args'], rng=rng)))(random.Random(_seed(g, 'config'))),
        facade=lambda name, g: _with(lambda: _facade('sequence_recall')(
            *gc.config_of(g)['args'], art=_art(g)))),
    # Its files hold reward_f64 among the trajectory's arrays.
    'box_world': Family(
        ('art', 'distractors', 'config', 'actions', 'boards', 'reward', 'has_reward',
         'reward_f64', 'discount', 'game_over', 'grid', 'over_this', 'steps'),
        ('art', 'distractors', 'config', 'actions'),
        checks={'oracle': _float_rewards, 'facade': _box_world_plot},
        reference=_reference_box_world,
        oracle=lambda name, g: _with(lambda: obw.make_box_world(*_box_level(g))),
        facade=lambda name, g: _with(lambda: importlib.import_module(
            'pycolab_b200.games.box_world').game_from_level(*_box_level(g)))),
}

# The goldens the parametrised replays cover: every one of FAMILIES but the Story goldens,
# whose replays are the story tests' own (test_story, test_gpu_story).
# story_classics_cropped crops on the device: the oracle has no replay of it.
REPLAYS = [name for fam in FAMILIES if fam != 'story' for name in gc.names(fam + '_')]
# test_cued_catch replays its goldens on the facade itself, then checks where the global
# generator ends.
FACADE_REPLAYS = [name for name in REPLAYS if not name.startswith('cued_catch_')]


# ----------------------------------------------------------------- recorders --

class _Recorder(object):
  """on_frame for trajectory.run_trajectory: the fields golden `g`'s family records, frame
  by frame, the views from `croppers`; `arrays()` returns them as the goldens hold them.
  `check(env, out)`, if given, runs at every frame."""

  DTYPES = dict(sprites=np.int32, curtains=np.uint8, backdrops=np.uint8, reward_type=np.uint8,
                corners=np.int32, has_sword=np.uint8, floats=np.float64, reward_f64=np.float64,
                state=np.int64, which_goal=np.uint8, grid=np.uint8, over_this=np.int32,
                steps=np.int32)

  def __init__(self, fam, g, croppers, check=None):
    self.chars = bytes(g['sprite_chars']).decode() if fam.sprites is None else fam.sprites
    self.curtain, self.croppers, self.check = fam.curtain, croppers, check
    self.rows = {k: [] for k in fam.keys if k not in fam.inputs + tj.TRAJECTORY}

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

  def reward_f64(self, env, out):
    return np.nan if out[1] is None else float(out[1])

  def grid(self, env, out):
    return bwc.object_grid(env.things, (env.rows, env.cols))

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

  def state(self, env, out):
    """Sequence Recall's program state, or else Cued Catch's."""
    if 'program' in env.the_plot:
      return lc.sequence_recall_state(env)
    return lc.cued_catch_state(env)

  def which_goal(self, env, out):
    return 0 if env.things['Q'].which_goal == 'left' else 1

  def over_this(self, env, out):
    return bwc.over_words(env.the_plot.get('over_this'))

  def steps(self, env, out):
    return env.things['.']._step_counter


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

  def state(self, world, out):
    if 'program' in world.plot.store:
      return lc.sequence_recall_state(world)
    return lc.oracle_cued_catch_state(world)

  def which_goal(self, world, out):
    return 0 if world.things['Q'].aux['which_goal'] == 'left' else 1

  def over_this(self, world, out):
    return bwc.over_words(obw.over_this(world))

  def steps(self, world, out):
    return world.things['.'].aux['steps']


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
    if stream != 'numpy':
      random.seed(_seed(g, key))
    if stream != 'python':
      np.random.seed(_seed(g, key))
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
