"""Scaffolding shared by the compiled program's tests: game modules loaded through `compat`
with their classes registered, handles that reach no device, and the recorders and replay
of the registered-game goldens.

Each module of MODULES exports the same tables, keyed by game: GAMES, N_ACTIONS, SPRITES,
REGISTERS (entity attributes; a position takes its row and column), PLOT_KEYS, RAISES (the
exception a game's golden ends at); and GENERATORS (the global generators a case seeds),
FIELDS (what its goldens hold before the trajectory, in order) and CASES rows of (golden
name, game, level, action seed, generator seed or None, steps).
tests/golden/make_registered_golden.py plays them on the reference; test_registered_goldens
replays them on the oracle, test_gpu_registered_goldens through the facade.
"""

import ctypes as C
import inspect
import os
import random
import sys

import numpy as np
import pytest

import golden_cases as gc
import trajectory as tj
from pycolab_b200 import _lib, compat, compiler, lowering
from pycolab_b200.prefab_parts import sprites as b_sprites

HERE = os.path.dirname(os.path.abspath(__file__))

MODULES = ('compiled_games', 'drawn_games', 'sprite_games', 'scrolling_games',
           'backdrop_games', 'helper_games')
# Every golden of MODULES as (module file, golden name): `<family>_games`' are `<family>_*`.
GOLDENS = [(m + '.py', name) for m in MODULES for name in gc.names(m.split('_')[0] + '_')]
# What a golden holds as the replay's input rather than as an output to compare.
INPUTS = ('game', 'level', 'actions', 'rng_seed')


def load(path):
  """Import a pycolab module through compat, leaving sys.modules as it was.  A relative
  `path` names a file under tests/."""
  saved = {k: v for k, v in sys.modules.items() if k == 'pycolab' or k.startswith('pycolab.')}
  compat.uninstall()
  try:
    return compat.load_example(os.path.join(HERE, path))
  finally:
    compat.uninstall()
    sys.modules.update(saved)


def registered(name, *extra):
  """Body of a module-scoped fixture: tests/`name` loaded, its CLASSES and the classes it
  names `extra` registered, and unregistered again at teardown."""
  mod = load(name)
  classes = list(mod.CLASSES) + [getattr(mod, k) for k in extra]
  compiler.register(*classes)
  yield mod
  compiler.unregister(*classes)


def handle(lib, spec):
  h = C.c_void_p()
  assert lib.pcl_create(C.byref(spec), 4, -1, C.byref(h)) == _lib.OK
  return h


def bind(lib, h, words):
  words = np.ascontiguousarray(words, dtype=np.int32)
  return lib.pcl_bind_code(h, words.ctypes.data, len(words))


class _Walker(b_sprites.MazeWalker):
  def __init__(self, corner, position, character):
    super(_Walker, self).__init__(corner, position, character, impassable='#')
    self.n = 0


def walker(update):
  """A MazeWalker class `Case` with one register `n`, whose update() is `update`."""
  return type('Case', (_Walker,), {'update': update, '__module__': update.__module__})


def assert_refused(klass, what):
  """Compiling `klass` is refused with a message naming its update()'s line marked
  `# REFUSED`, as `<class>.update, line <n>:`, and `what`.  Returns the message."""
  lines, first = inspect.getsourcelines(klass.update)
  line = first + [i for i, l in enumerate(lines) if '# REFUSED' in l][0]
  with pytest.raises(compiler.NotLoweredError) as e:
    compiler.compile_class(klass)
  msg = str(e.value)
  assert '%s.update, line %d:' % (klass.__name__, line) in msg and what in msg, msg
  return msg


def sample_envs(rs, B):
  """The first two and last two of B envs, and 28 others drawn by `rs`."""
  return [int(e) for e in np.unique(np.concatenate(
      [[0, 1, B - 2, B - 1], rs.choice(np.arange(2, B - 2), 28, replace=False)]))]


def register_check(lowered_by_env, layers=False, extra=None):
  """on_step for sampled_check.lockstep: every register word of the sampled envs' entities
  and the Plot against the oracle worlds; a plain Sprite's row, col and visible bit (the
  sprites of program_arg[3]); with `layers`, the un-occluded layers too; then `extra`."""
  from oracle import engine_model as em

  def on_step(t, engine, worlds, outs):
    import torch
    ids = sorted(worlds)
    idx = torch.as_tensor(ids, device=engine.device)
    sprites = engine.sprites.index_select(0, idx).cpu().numpy()
    drapes = engine.drapes.index_select(0, idx).cpu().numpy()
    plot = engine.plot.index_select(0, idx).cpu().numpy()
    if layers:
      planes = engine.unoccluded_layers(engine.chars).index_select(0, idx).cpu().numpy()
    for k, e in enumerate(ids):
      w, game = worlds[e], lowered_by_env(e)
      assert w.error == 0
      for s, ch in enumerate(engine.sprite_chars):
        ent, rec = w.things[ch], sprites[k, s]
        if (game.program_arg[3] >> s) & 1:
          assert [rec[0], rec[1], rec[4] & 1] == [ent.row, ent.col, int(bool(ent.visible))], (t, e, ch)
          words = list(rec[2:4]) + list(rec[5:])
        else:
          words = list(rec[_lib.S_AUX2 if game.egocentric[s] else _lib.S_AUX0:])
        assert words[:len(ent.regs)] == ent.regs[:len(words)], (t, e, ch)
      for d, ch in enumerate(engine.drape_chars):
        if not game.drape_kind[d]:
          assert list(drapes[k, d]) == w.things[ch].regs, (t, e, ch)
      assert list(plot[k, _lib.P_AUX0:_lib.P_AUX0 + 4]) == w.plot.regs, (t, e)
      if layers:
        want = em.unoccluded_layers_of(w.backdrop, w.things, engine.chars)
        for c, ch in enumerate(engine.chars):
          np.testing.assert_array_equal(planes[k, c], want[ch], err_msg=str((t, e, ch)))
    if extra is not None:
      extra(t, engine, worlds, outs)
  return on_step


# --------------------------------------------------------- global generators --

def global_words(stream):
  """The words (624 key words + position) of a global generator now."""
  if stream == 'python':
    return [int(w) for w in random.getstate()[1]]
  _, key, pos = np.random.get_state()[:3]
  return [int(w) for w in key] + [int(pos)]


def seed_generators(games, seed):
  for stream in games.GENERATORS:
    (random if stream == 'python' else np.random).seed(seed)


def seeded_words(games, seed):
  """{stream: words} of the module's GENERATORS seeded with `seed`, as the mutable lists an
  oracle world draws from."""
  from pycolab_b200 import batched
  return {s: [int(w) for w in batched._mt_state(s, seed)] for s in games.GENERATORS}


@pytest.fixture
def global_generators():
  """Leave NumPy's and Python's global generators as the test found them."""
  np_state, py_state = np.random.get_state(), random.getstate()
  yield
  np.random.set_state(np_state)
  random.setstate(py_state)


# ----------------------------------------------------------------- recorders --

def value_types(games, game, env):
  """The Python types of a game's registers and Plot keys in an Engine."""
  return ([type(getattr(env.things[ch], name)) for ch, name in games.REGISTERS[game]] +
          [type(env.the_plot[key]) for key in games.PLOT_KEYS[game]])


class _Recorder(object):
  """on_frame for trajectory.run_trajectory: every field a registered game's goldens may
  hold, frame by frame; `arrays()` returns them as the goldens hold them."""

  def __init__(self, games, game):
    self.games, self.game = games, game
    self.env = None                       # the env of the last frame
    self.rows = {k: [] for k in ('sprites', 'registers', 'plot_keys', 'reward_type',
                                 'reward_f64', 'corners', 'backdrops')}

  def __call__(self, env, out):
    games, game, rows = self.games, self.game, self.rows
    self.env = env
    plot = self.plot(env, games.PLOT_KEYS[game])
    rows['sprites'].append(self.sprites(env, games.SPRITES[game]))
    rows['registers'].append(self.registers(env, games.REGISTERS[game]) + plot)
    rows['plot_keys'].append(plot)
    rows['reward_type'].append(tj.reward_type(out[1]))
    rows['reward_f64'].append(np.nan if out[1] is None else float(out[1]))
    rows['corners'].append([self.corner(env, ch)
                            for ch in getattr(games, 'SCROLLYS', {}).get(game, '')])
    rows['backdrops'].append(self.backdrop(env))

  def arrays(self):
    rows, n = self.rows, len(self.rows['reward_type'])
    out = dict(sprites=np.array(rows['sprites'], dtype=np.int32).reshape(n, -1, 5),
               registers=np.array(rows['registers'], dtype=np.int64).reshape(n, -1),
               plot_keys=np.array(rows['plot_keys'], dtype=np.int64).reshape(n, -1),
               reward_type=np.array(rows['reward_type'], dtype=np.uint8),
               reward_f64=np.array(rows['reward_f64'], dtype=np.float64),
               corners=np.array(rows['corners'], dtype=np.int32).reshape(n, -1, 2),
               backdrops=np.stack(rows['backdrops']))
    for name, ch in getattr(self.games, 'PATTERNS', {}).get(self.game, {}).items():
      out['pattern_' + name] = self.pattern(self.env, ch)
    for stream, words in self.words().items():
      out[stream + '_words'] = np.array(words, dtype=np.uint32)
    return out


class EngineRecorder(_Recorder):
  """The recorder of an Engine with the pycolab API: the reference's, or the facade's.  The
  final words are the global generators'.  `types` holds each frame's value_types()."""

  def __init__(self, games, game):
    super(EngineRecorder, self).__init__(games, game)
    self.types = []

  def __call__(self, env, out):
    super(EngineRecorder, self).__call__(env, out)
    self.types.append(value_types(self.games, self.game, env))

  def sprites(self, env, chars):
    return tj.sprite_rows(env, chars)

  def registers(self, env, regs):
    out = []
    for ch, name in regs:
      value = getattr(env.things[ch], name)
      out += [int(x) for x in value] if isinstance(value, tuple) else [int(value)]
    return out

  def plot(self, env, keys):
    return [int(env.the_plot[key]) for key in keys]

  def corner(self, env, ch):
    return [int(x) for x in env.things[ch]._northwest_corner]

  def backdrop(self, env):
    return np.array(env.backdrop.curtain, dtype=np.uint8)

  def pattern(self, env, ch):
    return np.array(env.things[ch].whole_pattern, dtype=bool)

  def words(self):
    return {stream: global_words(stream) for stream in self.games.GENERATORS}


class WorldRecorder(_Recorder):
  """The recorder of oracle worlds (oracle/compiled.py) of `lowered`, the lowering of
  `engine`, drawing from `words` (seeded_words()).  Registers are read through the compiled
  classes' slots, so a position takes two words.  Every frame must have latched no error."""

  def __init__(self, games, game, engine, lowered, words):
    super(WorldRecorder, self).__init__(games, game)
    self.engine, self.lowered, self.streams = engine, lowered, words
    self.keys = [key for key, _ in lowered.plot_keys]

  def make_world(self):
    from oracle import compiled as ocompiled
    words = [self.streams[s] for s in self.lowered.rng_streams]
    return ocompiled.make_world(self.lowered, words or None)

  def __call__(self, world, out):
    assert world.error == 0
    super(WorldRecorder, self).__call__(world, out)

  def sprites(self, world, chars):
    lowered = self.lowered
    plain = [ch for s, ch in enumerate(lowered.sprite_chars) if (lowered.program_arg[3] >> s) & 1]
    return tj.world_sprite_rows(world, chars, plain)

  def registers(self, world, regs):
    out = []
    for ch, name in regs:
      comp = compiler.registered(type(self.engine.things[ch]))
      slot = comp.slot(name)
      out += world.things[ch].regs[slot:slot + comp.width(name)]
    return out

  def plot(self, world, keys):
    return [world.plot.regs[self.keys.index(key)] for key in keys]

  def corner(self, world, ch):
    return list(world.things[ch].corner)

  def backdrop(self, world):
    return np.array(world.backdrop, dtype=np.uint8)

  def pattern(self, world, ch):
    return np.array(world.things[ch].pattern, dtype=bool)

  def words(self):
    return self.streams


# -------------------------------------------------------------------- replay --

def case(games, name):
  """(game, level, generator seed) of golden `name` in its module's CASES."""
  row = [row for row in games.CASES if row[0] == name][0]
  return row[1], row[2], row[4]


def _assert_replays(games, name, g, make_env, recorder, check_raise):
  """Plays golden `g`'s actions on envs from `make_env` under the auto-reset protocol,
  recording every frame; for a game of RAISES, only the actions before `raised_at`, and
  then `check_raise(env, action, exception)` with the action that raised.  Then every
  array `g` holds, apart from its inputs, must equal the replay's, dtype and shape
  included; a field the replay did not record fails."""
  game = case(games, name)[0]
  actions = g['actions'].tolist()
  at = int(g['raised_at'][0]) if game in games.RAISES else -1
  got = tj.run_trajectory(make_env, actions[:at] if at >= 0 else actions, on_frame=recorder)
  if at >= 0:
    check_raise(recorder.env, actions[at], games.RAISES[game])
  got.update(recorder.arrays(), raised_at=np.array([at], dtype=np.int32))
  tj.assert_golden_arrays(name, g, got, INPUTS)


def _oracle_raise(world, action, exception):
  if exception is ZeroDivisionError:
    world.play(action)
    assert world.error & _lib.ENV_ERR_ARITH
  else:
    assert exception is IndexError
    with pytest.raises(IndexError):
      world.play(action)


def assert_oracle_replays(games, name):
  """The oracle interpreter (oracle/compiled.py), running the compiled words of golden
  `name` of `games` (its classes registered), reproduces every array the golden holds.
  Where the reference raised IndexError the oracle raises it too; for a ZeroDivisionError
  it latches PCL_ENV_ERR_ARITH, as the device does."""
  g = gc.load(name)
  game, level, seed = case(games, name)
  engine = games.GAMES[game](level)
  lowered = lowering.lower(engine)
  assert lowered.program == _lib.PROG_COMPILED
  assert lowered.float_reward == bool((g['reward_type'] == 2).any())
  rec = WorldRecorder(games, game, engine, lowered, seeded_words(games, seed))
  _assert_replays(games, name, g, rec.make_world, rec, _oracle_raise)


def _facade_raise(env, action, exception):
  with pytest.raises(exception):
    env.play(action)


def assert_facade_replays(games, name):
  """The facade Engine reproduces every array golden `name` of `games` (its classes
  registered) holds, with the global generators seeded as the reference's were (run it
  under the global_generators fixture).  Every register and Plot key keeps, at every
  frame, the Python type it has in a freshly made game; where the reference raised, the
  facade raises the same exception."""
  g = gc.load(name)
  game, level, seed = case(games, name)
  want = value_types(games, game, games.GAMES[game](level))
  seed_generators(games, seed)
  rec = EngineRecorder(games, game)
  _assert_replays(games, name, g, lambda: games.GAMES[game](level), rec, _facade_raise)
  for t, types in enumerate(rec.types):
    assert types == want, (name, t, types, want)
