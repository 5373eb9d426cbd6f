"""research/box_world: keys, locks and the gem as one per-env object grid (csrc/box_world.cu).

CPU: the level generator against the reference's `make_game`, the oracle (oracle/box_world.py)
in lock-step with the live reference, lowering, the C boundary's statuses and the kernel's
resources.  The goldens the reference made (tests/golden/box_world_*, by
tests/golden/make_golden.py) replay on the oracle and the facade through
tests/example_games.py."""

import ctypes as C
import os
import sys

import numpy as np
import pytest

import box_world_cases as bwc
import golden_cases as gc
import refdriver
import trajectory as tj
from oracle import box_world as obw

NAMES = gc.names('box_world_')
ARGS = bwc.ARGS
needs_ref = pytest.mark.skipif(not refdriver.available(), reason='/root/reference not present')


def oracle_grid(world):
  return bwc.object_grid(world.things, (world.rows, world.cols))


def oracle_over(world):
  return bwc.over_words(obw.over_this(world))


def golden_level(g):
  return tj.u8_to_art(g['art']), [tuple(int(v) for v in xy) for xy in g['distractors']]


# ----------------------------------------------------------------------------- generator --

@needs_ref
def test_generator_makes_the_references_levels():
  """RandomState(s) gives the reference's art, drape set, per-cell distractors and step limit:
  1000 seeds at grid_size 12 and a few at 6, 20 and 30."""
  from pycolab_b200 import levels
  from pycolab_b200.games import box_world
  ref = bwc.ref_module()
  cases = [(12, s) for s in range(1000)] + [(g, s) for g in (6, 20, 30) for s in range(8)]
  for grid_size, seed in cases:
    steps = 120 if seed % 3 else 37
    want = ref.make_game(grid_size, *ARGS, random_state=np.random.RandomState(seed),
                         max_num_steps=steps)
    art, distractors = levels.box_world_level(seed, grid_size)
    assert art == [bytes(r).decode() for r in want.its_showtime()[0].board], (grid_size, seed)
    assert sorted(distractors) == sorted(want.things['.'].distractors), (grid_size, seed)
    got = box_world.make_game(grid_size, *ARGS, random_state=np.random.RandomState(seed),
                              max_num_steps=steps)
    assert set(got.things) == set(want.things), (grid_size, seed)
    assert got.things['.'].distractors == want.things['.'].distractors
    assert got.things['.']._max_num_steps == want.things['.']._max_num_steps == steps
    for ch in want.things:
      if ch != '.':
        np.testing.assert_array_equal(got.things[ch].curtain, want.things[ch].curtain)


def test_generator_continues_a_random_state():
  from pycolab_b200 import levels
  rs, want = np.random.RandomState(4), np.random.RandomState(4)
  a, b = levels.box_world_level(rs), levels.box_world_level(rs)
  assert a == levels.box_world_level(want) and b == levels.box_world_level(want) and a != b


# ----------------------------------------------------------------------------- oracle --

def _frame_state(env, is_ref):
  if is_ref:
    return (bwc.object_grid(env.things, (env.rows, env.cols)),
            bwc.over_words(env.the_plot.get('over_this')), env.things['.']._step_counter)
  return oracle_grid(env), oracle_over(env), env.things['.'].aux['steps']


# (seed, grid_size, max_num_steps, the scripted player's modes, outcomes the run must reach)
LOCKSTEP = [(3, 12, 120, ('solve', 'random'), {'correct', 'gem'}),
            (10, 12, 120, ('distract', 'solve'), {'correct', 'distractor', 'gem'}),
            (7, 12, 25, ('dither', 'solve', 'distract'), {'correct', 'distractor', 'timeout'}),
            (1, 6, 30, ('random', 'solve'), {'correct', 'gem', 'timeout'}),
            (2, 20, 150, ('solve', 'distract'), {'correct', 'gem'}),
            (5, 30, 200, ('solve', 'dither'), {'correct', 'gem', 'timeout'})]


def _twin_key_seeds(n):
  """The first n seeds whose levels put one key character on two cells."""
  from pycolab_b200 import levels
  out = []
  for seed in range(400):
    art, _ = levels.box_world_level(seed)
    cells = ''.join(art)
    if any(cells.count(k) > 1 for k in bwc.KEYS):
      out.append(seed)
    if len(out) == n:
      return out
  return out


def _outcome(reward, over, steps, max_steps):
  """What ended or paid in one frame: 'correct', 'distractor', 'gem', 'timeout' or None."""
  if reward == 1.0:
    return 'correct'
  if over and reward == -1.0:
    return 'distractor'
  if over and reward == 10.0:
    return 'gem'
  if over and steps > max_steps:
    return 'timeout'
  return None


@needs_ref
@pytest.mark.parametrize('case', LOCKSTEP + [(s, 12, 120, ('solve', 'distract', 'random'),
                                              {'correct'}) for s in _twin_key_seeds(3)])
def test_oracle_lockstep_with_reference(case):
  """Every frame: board, reward (value, type, None), discount, game over, every object
  curtain, the_plot['over_this'] and the step counter; the scripted player opens correct and
  distractor locks, takes the gem, times out and plays invalid actions, and each run reaches
  the outcomes its case names."""
  seed, grid_size, steps, modes, outcomes = case
  ref = bwc.ref_module()
  make_ref = lambda: ref.make_game(grid_size, *ARGS, random_state=np.random.RandomState(seed),
                                   max_num_steps=steps)
  first = make_ref()
  art = [bytes(r).decode() for r in first.its_showtime()[0].board]
  distractors = first.things['.'].distractors
  make_or = lambda: obw.make_box_world(art, distractors, steps)
  rs = np.random.RandomState(seed)
  a_env, b_env = make_ref(), make_or()
  a, b = a_env.its_showtime(), b_env.its_showtime()
  episode, seen, invalid = 0, set(), 0
  for t in range(700):
    assert np.array_equal(a[0].board, b[0]), t
    assert type(a[1]) is type(b[1]) and a[1] == b[1], (t, a[1], b[1])
    assert a[2] == b[2] and a_env.game_over == b_env.game_over, t
    ga, oa, sa = _frame_state(a_env, True)
    gb, ob, sb = _frame_state(b_env, False)
    assert np.array_equal(ga, gb) and oa == ob and sa == sb, (t, oa, ob, sa, sb)
    seen.add(_outcome(a[1], a_env.game_over, sa, steps))
    if a_env.game_over:
      episode += 1
      a_env, b_env = make_ref(), make_or()
      a, b = a_env.its_showtime(), b_env.its_showtime()
      continue
    act = bwc.scripted_action(a[0].board, distractors, modes[episode % len(modes)], rs)
    invalid += act not in range(4)
    a, b = a_env.play(act), b_env.play(act)
  assert outcomes <= seen, (outcomes, seen)
  assert episode >= 1 and invalid >= 1


def test_goldens_cover_every_outcome():
  assert len(NAMES) >= 6
  rewards = np.concatenate([gc.load(n)['reward_f64'] for n in NAMES])
  assert {0.0, 1.0, -1.0, 10.0} <= set(rewards[~np.isnan(rewards)].tolist())
  timeouts = 0
  for n in NAMES:
    g = gc.load(n)
    cfg = gc.config_of(g)
    timeouts += int(((g['steps'] > cfg['max_num_steps']) & (g['game_over'] == 1)).sum())
  assert timeouts >= 1
  assert any(((gc.load(n)['actions'] < 0) | (gc.load(n)['actions'] > 3)).any() for n in NAMES)
  assert {gc.config_of(gc.load(n))['grid_size'] for n in NAMES} >= {6, 12, 20, 30}


# ----------------------------------------------------------------------------- lowering --

def _lower(seed, grid_size=12, steps=120):
  from pycolab_b200 import lowering
  from pycolab_b200.games import box_world
  return lowering.lower(box_world.make_game(grid_size, *ARGS,
                                            random_state=np.random.RandomState(seed),
                                            max_num_steps=steps))


def test_levels_with_different_keys_share_one_signature():
  from pycolab_b200 import _lib
  games = [_lower(s) for s in range(40)]
  assert len({g.object_chars for g in games}) > 10
  assert len({g.signature() for g in games}) == 1
  g = games[0]
  assert g.program == _lib.PROG_BOX_WORLD and g.drape_chars == '' and g.sprite_chars == '.'
  assert g.z_order == '.' and g.groups == ['.'] and g.program_arg[0] == 120
  assert g.bits_words * 4 == g.pitch and g.bits[0].shape == (14, g.bits_words)
  assert _lower(0, steps=99).signature() != g.signature()
  assert _lower(0, grid_size=13).signature() != g.signature()


def test_lowered_grid_holds_objects_and_distractor_flags():
  from pycolab_b200 import levels
  for seed in range(30):
    game = _lower(seed)
    art, distractors = levels.box_world_level(seed)
    grid = game.bits[0].view(np.uint8).reshape(game.rows, game.pitch)
    want = np.array([[ord(c) if c not in ' #.' else 0 for c in row] for row in art], np.uint8)
    np.testing.assert_array_equal(grid[:, :game.cols] & 0x7f, want)
    flagged = {(int(x), int(y)) for y, x in zip(*np.nonzero(grid & 0x80))}
    assert flagged == set(distractors)
    assert not grid[:, game.cols:].any()


def test_boards_over_32_rows_are_refused():
  from pycolab_b200.errors import NotLoweredError
  _lower(1, grid_size=30)
  with pytest.raises(NotLoweredError):
    _lower(1, grid_size=31)


@needs_ref
def test_reference_box_world_file_lowers_like_the_twin():
  from pycolab_b200 import compat, lowering
  from pycolab_b200.games import box_world
  saved = {k: v for k, v in sys.modules.items() if k == 'pycolab' or k.startswith('pycolab.')}
  compat.uninstall()
  try:
    mod = compat.load_example(bwc.ref_path())
    for seed, grid_size in ((0, 12), (5, 12), (11, 6), (3, 30)):
      a = lowering.lower(mod.make_game(grid_size, *ARGS, random_state=np.random.RandomState(seed)))
      b = lowering.lower(box_world.make_game(grid_size, *ARGS,
                                             random_state=np.random.RandomState(seed)))
      assert a.signature() == b.signature() and a.object_chars == b.object_chars
      for field in ('backdrop', 'sprites', 'drapes', 'plot'):
        np.testing.assert_array_equal(getattr(a, field), getattr(b, field), err_msg=field)
      np.testing.assert_array_equal(a.bits[0], b.bits[0])
  finally:
    compat.uninstall()
    sys.modules.update(saved)


@needs_ref
@pytest.mark.parametrize('edit', [
    ('if lock_chr in LOCKS and things[lock_chr].curtain[y][x + 1]:',
     'if lock_chr in LOCKS and things[lock_chr].curtain[y][x - 1]:'),
    ('      if character == self.character and self.curtain[y][x]:',
     '      if character == self.character:'),
    ('REWARD_OPEN_WRONG)', 'REWARD_OPEN_CORRECT)')])
def test_edited_box_world_copy_is_refused(tmp_path, edit):
  """Edits to BoxThing (which every object drape runs) or to a drape's update() are refused:
  the source differs from what the kernel restates."""
  from pycolab_b200 import compat, lowering
  from pycolab_b200.errors import NotLoweredError
  src = open(bwc.ref_path()).read()
  edited = src.replace(*edit)
  assert edited != src
  path = tmp_path / 'box_world.py'
  path.write_text(edited)
  saved = {k: v for k, v in sys.modules.items() if k == 'pycolab' or k.startswith('pycolab.')}
  compat.uninstall()
  try:
    mod = compat.load_example(str(path))
    with pytest.raises(NotLoweredError, match='source differs'):
      lowering.lower(mod.make_game(12, *ARGS, random_state=np.random.RandomState(3)))
  finally:
    compat.uninstall()
    sys.modules.update(saved)


# ----------------------------------------------------------------------------- C boundary --

def test_boundary_statuses():
  """pcl_create / pcl_bind_state for the box_world program, device -1 (nothing touches a GPU)."""
  from pycolab_b200 import _lib
  lib = _lib.load()
  game = _lower(2)

  def create(spec):
    handle = C.c_void_p()
    status = lib.pcl_create(C.byref(spec), 4, -1, C.byref(handle))
    if status == _lib.OK:
      lib.pcl_destroy(handle)
    return status
  assert create(game.make_spec(True)) == _lib.OK
  assert create(_lower(2, grid_size=30).make_spec(True)) == _lib.OK
  bad = {}
  for name, edit in (('rows', lambda s: setattr(s, 'rows', 33)),
                     ('pitch', lambda s: setattr(s, 'pitch', 48)),
                     ('bits_words', lambda s: setattr(s, 'bits_words', 5)),
                     ('max_steps', lambda s: s.program_arg.__setitem__(0, -1)),
                     ('egocentric', lambda s: s.sprite_egocentric.__setitem__(0, 1)),
                     ('confined', lambda s: s.sprite_confined.__setitem__(0, 0)),
                     ('impassable', lambda s: s.impassable[0].__setitem__(1, 0)),   # drop '#'
                     ('drape', lambda s: setattr(s, 'n_drapes', 1)),
                     ('tiny', lambda s: (setattr(s, 'rows', 2), setattr(s, 'cols', 2)))):
    spec = game.make_spec(True)
    edit(spec)
    bad[name] = create(spec)
  assert bad == {'rows': _lib.ERR_UNSUPPORTED, 'pitch': _lib.ERR_UNSUPPORTED,
                 'bits_words': _lib.ERR_INVALID, 'max_steps': _lib.ERR_INVALID,
                 'egocentric': _lib.ERR_UNSUPPORTED, 'confined': _lib.ERR_UNSUPPORTED,
                 'impassable': _lib.ERR_UNSUPPORTED, 'drape': _lib.ERR_UNSUPPORTED,
                 'tiny': _lib.ERR_INVALID}
  spec = game.make_spec(True)
  handle = C.c_void_p()
  assert lib.pcl_create(C.byref(spec), 4, -1, C.byref(handle)) == _lib.OK
  fake = 0x1000
  try:
    st = _lib.State()
    st.d_backdrop = st.d_plot = st.d_plot_init = st.d_sprites = st.d_sprites_init = fake
    assert lib.pcl_bind_state(handle, C.byref(st)) == _lib.ERR_INVALID       # no grid
    st.d_bits[0] = st.d_bits_init[0] = fake
    st.bits_bstride[0] = game.rows * game.bits_words - 1
    assert lib.pcl_bind_state(handle, C.byref(st)) == _lib.ERR_INVALID       # grids overlap
    st.bits_bstride[0] = game.rows * game.bits_words
    assert lib.pcl_bind_state(handle, C.byref(st)) == _lib.OK
  finally:
    lib.pcl_destroy(handle)


def test_kernel_has_no_stack():
  import shutil
  import subprocess
  from pycolab_b200 import _lib
  tool = shutil.which('cuobjdump') or os.path.join(os.environ.get('CUDA_HOME', '/usr/local/cuda'),
                                                   'bin', 'cuobjdump')
  if not os.access(tool, os.X_OK):
    pytest.skip('cuobjdump not found')
  out = subprocess.run([tool, '--dump-resource-usage', _lib.LIB_PATH], check=True,
                       capture_output=True, text=True).stdout
  lines = out.splitlines()
  found = [lines[i + 1] for i, line in enumerate(lines[:-1]) if 'box_world_step' in line]
  assert found, 'no box_world_step in %s' % _lib.LIB_PATH
  for line in found:
    assert 'STACK:0' in line.replace(' ', ''), line


# ------------------------------------------------------------------ facade hooks on the CPU --

class _StubBatched(object):
  """The parts of a batch-1 `BatchedEngine` that `Engine._sync_things` and the box_world sync
  hook read, as CPU tensors the test writes."""

  def __init__(self, lowered):
    import torch
    self.game, self.batch = lowered, 1
    self.rows, self.cols, self.pitch = lowered.rows, lowered.cols, lowered.pitch
    self.sprite_chars, self.drape_chars = lowered.sprite_chars, lowered.drape_chars
    self.object_chars = lowered.object_chars
    self.z_order = None
    self.template = lowered.bits[0].view(np.uint8).reshape(self.rows, self.pitch)
    self.bits = {0: torch.zeros((1, self.rows, self.pitch // 4), dtype=torch.int32)}
    self.sprites = torch.from_numpy(lowered.sprites.copy())[None]
    self.drapes = torch.zeros((1, 0, 8), dtype=torch.int32)
    self.plot = torch.from_numpy(lowered.plot.copy())[None]

  def load(self, world):
    """Write an oracle world's state as the device keeps it."""
    import torch
    from pycolab_b200 import _lib
    grid = np.zeros((self.rows, self.pitch), dtype=np.uint8)
    grid[:, :self.cols] = oracle_grid(world)
    grid |= self.template & 0x80 & np.where(grid != 0, 0xff, 0).astype(np.uint8)
    self.bits[0][0] = torch.from_numpy(grid.view(np.int32).copy())
    p = world.things['.']
    self.sprites[0, 0, :5] = torch.tensor([p.row, p.col, p.row, p.col, 1])
    self.sprites[0, 0, _lib.S_AUX0] = p.aux['steps']
    over = oracle_over(world)
    self.plot[0, _lib.P_FRAME] = world.plot.frame
    self.plot[0, _lib.P_AUX0] = over[0]
    self.plot[0, _lib.P_AUX1] = over[1] << 16 | over[2]


def _sync_replay(engine, name):
  """Replay golden `name` on the oracle and mirror every frame into `engine` (an un-started
  facade Engine of the same level) through Engine._sync_things and the program's sync hook:
  Drape curtains, the player's position and step counter and the_plot['over_this'] must be
  the golden's."""
  from pycolab_b200 import lowering, programs
  g = gc.load(name)
  cfg = gc.config_of(g)
  art, distractors = golden_level(g)
  lowered = lowering.lower(engine)
  assert lowered.sync is programs.box_world.sync
  assert lowered.curtain is programs.box_world.curtain
  assert lowered.layers is programs.box_world.layers
  stub = _StubBatched(lowered)
  engine._batched = stub
  world = obw.make_box_world(art, distractors, cfg['max_num_steps'])
  world.its_showtime()
  for t, act in enumerate([None] + g['actions'].tolist()):
    if t:
      if world.game_over:
        world = obw.make_box_world(art, distractors, cfg['max_num_steps'])
        world.its_showtime()
      else:
        world.play(act)
    stub.load(world)
    engine._sync_things()
    np.testing.assert_array_equal(bwc.object_grid(engine.things, (engine.rows, engine.cols)),
                                  g['grid'][t], '%s frame %d' % (name, t))
    over = engine.the_plot.get('over_this')
    assert bwc.over_words(over) == g['over_this'][t].tolist(), (name, t)
    assert over is None or type(over[1]).__name__ == 'Position'
    assert engine.things['.']._step_counter == g['steps'][t]
    where = np.argwhere(g['boards'][t] == ord('.'))[0]
    assert tuple(engine.things['.'].position) == tuple(int(v) for v in where)


@pytest.mark.parametrize('name', NAMES[:2])
def test_facade_sync_of_the_twin(name):
  from pycolab_b200.games import box_world
  g = gc.load(name)
  art, distractors = golden_level(g)
  _sync_replay(box_world.game_from_level(art, distractors, gc.config_of(g)['max_num_steps']),
               name)


@needs_ref
@pytest.mark.parametrize('name', NAMES[:2])
def test_facade_sync_of_the_reference_module(name):
  """The reference's file through compat: its lowered game carries the twin's hooks,
  object_chars and templates, and the sync hook mirrors the device state into its own
  Drapes, player and Plot.  (On the device the facade runs with the twin's classes; the
  reference file is not on the GPU machines.)"""
  from pycolab_b200 import compat, lowering
  from pycolab_b200.games import box_world
  g = gc.load(name)
  cfg = gc.config_of(g)
  saved = {k: v for k, v in sys.modules.items() if k == 'pycolab' or k.startswith('pycolab.')}
  compat.uninstall()
  try:
    mod = compat.load_example(bwc.ref_path())
    make = lambda m: m.make_game(cfg['grid_size'], *ARGS,
                                 random_state=np.random.RandomState(cfg['seed']),
                                 max_num_steps=cfg['max_num_steps'])
    a, b = lowering.lower(make(mod)), lowering.lower(make(box_world))
    assert a.object_chars == b.object_chars and a.signature() == b.signature()
    assert (a.curtain, a.layers, a.sync) == (b.curtain, b.layers, b.sync)
    for field in ('backdrop', 'sprites', 'drapes', 'plot'):
      np.testing.assert_array_equal(getattr(a, field), getattr(b, field), err_msg=field)
    np.testing.assert_array_equal(a.bits[0], b.bits[0])
    _sync_replay(make(mod), name)
  finally:
    compat.uninstall()
    sys.modules.update(saved)
