"""The per-env protocol every step program shares (include/pcl.h, csrc/pcl_device.cuh
env_run, plot_carry, store_outputs), byte for byte, with guard bytes around every buffer a
step touches:

  * an env past the batch does nothing, and a skipped env (frozen without auto_reset, or
    left out of a masked pcl_reset) writes nothing, outputs included;
  * a restart rebuilds the env from the *_init templates at its level as a fresh Engine's
    its_showtime() does, keeps the episode count (+1) and the error word, and continues
    the env's random streams, whether a step or a masked reset starts it;
  * no step writes the static arrays (backdrop, read-only patterns, every *_init template,
    d_level), nor the reward array its program does not use (d_reward_f64 of an int-reward
    program, d_reward of a float-reward one).

Every engine here is rebound by `Guarded` onto copies of its arrays that sit in the middle
of larger allocations filled with a sentinel byte, and an unguarded twin plays the same
calls: after every call the guards, the static arrays and the unused reward array are as
they were, and the guarded engine equals its twin byte for byte.

What these checks need not carve out, and why:
  * scrolly_maze's render key (csrc/scrolly_maze.cu, "Delta rendering") lives in the
    handle's own derived buffer, which no test can see; a rebind invalidates it, so the
    guarded engine paints in full where its twin takes the delta path, and the boards
    must still agree.
  * scrolly_maze's dirty-group mask ('@' record AUX2, "Coin groups") is part of the '@'
    record: a restart reloads the record from its template, so the mask is 0 again on
    both paths, while the restart copies back only the dirty coin groups and a host reset
    every group; the coin pattern must come out the same either way.
"""

import collections
import ctypes as C
import functools
import random

import numpy as np
import pytest

import golden_cases as gc
import registered_games as rg
import trajectory as tj

pytestmark = pytest.mark.gpu

SENTINEL = 0xA5          # guard bytes
UNUSED = 0x3C            # the bytes of the reward array a program does not use
POISON = 0x5A            # outputs a skipped env must leave as they are
ALIGN = 512              # every guarded array starts 512 bytes into a fresh allocation
WARPS_PER_BLOCK = 4      # the most envs one thread block of any step kernel covers


def _torch():
  import torch
  return torch


# ------------------------------------------------------------------------- the programs
# Per program: the game factory, draw(rs, shape) -> random action words, and the action
# row that ends an episode at once (None: the drawn actions end episodes on their own).

def _fixture_game():
  from pycolab_b200.games import fixtures
  kw, _ = gc.fixture_kwargs(gc.load('fixture_walkers_0'))
  return fixtures.make_game(kw['art'], kw['what_lies_beneath'], kw['walkers'], kw['scrollys'],
                            kw['drapes'], kw['update_schedule'], kw['z_order'])


def _protocol_program(name):
  from pycolab_b200 import _lib, levels, lowering
  from pycolab_b200.games import (aperture, apprehend, better_scrolly_maze, hello_world, ordeal,
                                  scrolly_maze, shockwave, warehouse_manager)
  from pycolab_b200.games import extraterrestrial_marauders as marauders
  from pycolab_b200.games.classics import cliff_walk
  below = lambda n: (lambda rs, shape: rs.randint(0, n, size=shape))
  if name == 'fixture':
    low = lowering.lower(_fixture_game())
    n_ent, n_dir = len(low.sprite_chars) + len(low.drape_chars), _lib.FIXTURE_DIRECTIVES

    def draw(rs, shape):                      # a motion per entity, no Plot directives
      rows = np.zeros(tuple(shape) + (n_ent + 2 * n_dir,), dtype=np.int64)
      rows[..., :n_ent] = rs.randint(0, 9, size=tuple(shape) + (n_ent,))
      return rows
    quit_row = np.zeros(n_ent + 2 * n_dir, dtype=np.int64)
    quit_row[:n_ent] = 8
    quit_row[n_ent] = _lib.DIR_TERMINATE      # terminate_episode(discount 0.0)
    return _fixture_game, draw, quit_row
  return {
      'scrolly_maze': (lambda: scrolly_maze.make_game(*levels.scrolly_maze_level(
          4, world_shape=(65, 65), board_shape=(32, 32))), below(4), 5),
      'warehouse': (lambda: warehouse_manager.make_game(levels.warehouse_level(3)), below(5), 5),
      'marauders': (lambda: marauders.make_game(levels.marauders_level()), below(4), 4),
      'better_scrolly': (lambda: better_scrolly_maze.make_game(
          tj.u8_to_art(gc.load('better_stock_L1')['art'])), below(5), 5),
      'classics': (lambda: cliff_walk.make_game(), below(4), 3),   # east off the start: the cliff
      'aperture': (lambda: aperture.make_game(
          tj.u8_to_art(gc.load('aperture_stock_L1')['art'])), below(9), 9),
      'ordeal': (ordeal.make_castle, below(4), 4),
      'hello': (hello_world.make_game, below(4), 4),
      'apprehend': (apprehend.make_game, below(3), None),   # the ball lands within a board height
      'shockwave': (lambda: shockwave.make_game(levels.shockwave_level(30, 12, 15, 0.45)),
                    lambda rs, shape: rs.choice(5, size=shape, p=[.6, .12, .12, .12, .04]), None),
  }[name]


PROTOCOL_PROGRAMS = ['scrolly_maze', 'warehouse', 'marauders', 'better_scrolly', 'fixture',
                     'classics', 'aperture', 'ordeal', 'hello', 'apprehend', 'shockwave']


# Levels beyond the first one of _protocol_program, for the programs with a level generator
# whose levels share one structure: they make the kernels read the static arrays through
# d_level.
def _more_levels(name):
  from pycolab_b200 import levels
  from pycolab_b200.games import scrolly_maze, shockwave, warehouse_manager
  return {
      'scrolly_maze': [lambda: scrolly_maze.make_game(*levels.scrolly_maze_level(
          5, world_shape=(65, 65), board_shape=(32, 32)))],
      'warehouse': [lambda: warehouse_manager.make_game(levels.warehouse_level(4))],
      'shockwave': [lambda: shockwave.make_game(levels.shockwave_level(31, 12, 15, 0.45))],
  }.get(name, [])


Case = collections.namedtuple('Case', 'games draw quit')


def _choice(options):
  return lambda rs, shape: rs.choice(options, size=shape)


def _lp_rnn_case(name):
  """t_maze, cued_catch and sequence_recall with the quit actions of lp_rnn_cases' policies
  (cued_catch_policy quits with 4, the t_maze and sequence_recall oracles with 0 and 6)."""
  from pycolab_b200 import levels
  from pycolab_b200.games import cued_catch, sequence_recall, t_maze
  random.seed(0)                 # the facades draw their templates from the global `random`
  if name == 't_maze':
    arts = [levels.t_maze_level(i) for i in range(2)]
    return ([t_maze.make_game(1, True, 40, 5, 4, maze_art=m, cue_art=c) for m, c in arts],
            _choice([1, 2, 3, 4, 5]), 6)
  if name in ('cued_catch', 'cued_catch_sigma'):
    args = (2, 2, 6, False, 0.0, 1) if name == 'cued_catch' else (3, 2, 5, False, 0.8, 2)
    art = levels.cued_catch_art()
    return [cued_catch.make_game(*args, art=art)], _choice([1, 2, 3]), 4
  art = levels.sequence_recall_art(9, 13)
  return [sequence_recall.make_game(2, 1, 2, 1, 30, art=art)], _choice([1, 2, 3, 4, 5]), 6


def _compiled_case(name, mods):
  """The compiled program on a plain game (lava: float rewards, quit 6) and on a game with
  a registered Backdrop (flow: a live curtain per env, np.random draws, quit 5)."""
  compiled_games, backdrop_games = mods
  if name == 'compiled':
    return [compiled_games.make_lava(k) for k in range(2)], _choice(range(6)), 6
  return [backdrop_games.make_flow(k) for k in range(2)], _choice(range(5)), 5


def _box_world_case():
  """A pool of three generated levels; the step limit ends every episode (the box_world_cases
  drivers' 'dither' mode), so there is no quit row."""
  from pycolab_b200 import levels
  from pycolab_b200.games import box_world
  pool = [levels.box_world_level(i, 8) for i in range(3)]
  return ([box_world.game_from_level(art, d, 7) for art, d in pool],
          _choice([-1, 0, 1, 2, 3, 4]), None)


CASES = PROTOCOL_PROGRAMS + ['t_maze', 'compiled', 'compiled_backdrop', 'box_world', 'cued_catch',
                             'cued_catch_sigma', 'sequence_recall']


@pytest.fixture(scope='module')
def compiled_modules():
  from pycolab_b200 import compiler
  mods = [rg.load('compiled_games.py'), rg.load('backdrop_games.py')]
  classes = [c for m in mods for c in m.CLASSES]
  compiler.register(*classes)
  yield mods
  compiler.unregister(*classes)


@functools.lru_cache(maxsize=None)
def _lowered(name, mods):
  from pycolab_b200 import lowering
  if name in PROTOCOL_PROGRAMS:
    make, draw, quit_row = _protocol_program(name)
    games, case = [make()] + [f() for f in _more_levels(name)], (draw, quit_row)
  else:
    if name in ('compiled', 'compiled_backdrop'):
      games, draw, quit_row = _compiled_case(name, mods)
    elif name == 'box_world':
      games, draw, quit_row = _box_world_case()
    else:
      games, draw, quit_row = _lp_rnn_case(name)
    case = (draw, quit_row)
  return Case(tuple(lowering.lower(g) for g in games), *case)


@pytest.fixture(params=CASES)
def case(request, compiled_modules):
  return _lowered(request.param, tuple(compiled_modules))


# Batch sizes: one env; a last block that is ragged for 2 and 4 warps per block; several
# blocks, the last ragged.
BATCHES = [1, 3, 11]


# ---------------------------------------------------------------------- guarded binding

def _rows(t):
  """u8 [B, bytes] view of a tensor with one row per env."""
  return t.reshape(t.shape[0], t.numel() // t.shape[0]).view(_torch().uint8)


def _held(eng):
  """(container, key, tensor) of every tensor an engine holds, in attributes, dicts, lists."""
  torch = _torch()
  for k, v in list(vars(eng).items()):
    if torch.is_tensor(v):
      yield vars(eng), k, v
    elif isinstance(v, (dict, list)):
      for kk, vv in list(v.items() if isinstance(v, dict) else enumerate(v)):
        if torch.is_tensor(vv):
          yield v, kk, vv


def _round(n):
  return (n + ALIGN - 1) // ALIGN * ALIGN


class Guarded(object):
  """A built BatchedEngine rebound onto guarded copies of every array its handle sees.

  Each array moves, contents and all, to offset `pad` of a sentinel-filled allocation of
  pad + nbytes + pad bytes (pad a multiple of 512 and at least WARPS_PER_BLOCK env slices
  plus 4 KB), so a 16-byte vector access, a cp.async or a bulk copy that strays into a
  neighbour's slot, or past either end of the array, lands on a guard byte.  The engine's
  tensor attributes, `_state` and `_out` follow the copies; int-reward programs get an
  unused d_reward_f64 as well.  check() asserts the guards, the static arrays and the
  unused reward array after a call."""

  def __init__(self, eng):
    from pycolab_b200 import _lib
    torch = _torch()
    self.eng = eng
    self.guards, self.frozen = [], []            # (name, tensor that must stay as it is)
    moved = {}                                   # old data_ptr -> guarded copy
    held = list(_held(eng))

    def guard(ptr, name, static):
      if not ptr:
        return ptr
      if ptr not in moved:
        owners = [t for _, _, t in held if t.data_ptr() == ptr and t.numel()]
        assert owners, 'the engine holds no tensor at %s' % name
        t = owners[0]
        nbytes = t.numel() * t.element_size()
        pad = _round(WARPS_PER_BLOCK * nbytes // t.shape[0] + 4096)
        buf = torch.full((2 * pad + nbytes,), SENTINEL, dtype=torch.uint8, device=eng.device)
        copy = buf[pad:pad + nbytes].view(t.dtype).view(t.shape)
        copy.copy_(t)
        self.guards += [(name + ' guard', buf[:pad]), (name + ' guard', buf[pad + nbytes:])]
        if static:
          self.frozen.append((name, copy.clone().reshape(-1).view(torch.uint8), copy))
        moved[ptr] = copy
      return moved[ptr].data_ptr()

    st, out, game = eng._state, eng._out, eng.game
    for f in ('d_backdrop', 'd_sprites_init', 'd_drapes_init', 'd_plot_init', 'd_z_order_init',
              'd_groups_init', 'd_level'):
      setattr(st, f, guard(getattr(st, f), f, True))
    for f in ('d_sprites', 'd_drapes', 'd_plot', 'd_rng', 'd_z_order', 'd_groups'):
      setattr(st, f, guard(getattr(st, f), f, False))
    for d in range(_lib.MAX_DRAPES):
      mutable = d in game.pattern_mutable and game.pattern_mutable[d]
      st.d_pattern[d] = guard(st.d_pattern[d], 'd_pattern[%d]' % d, not mutable)
      st.d_pattern_init[d] = guard(st.d_pattern_init[d], 'd_pattern_init[%d]' % d, True)
      st.d_bits[d] = guard(st.d_bits[d], 'd_bits[%d]' % d, False)
      st.d_bits_init[d] = guard(st.d_bits_init[d], 'd_bits_init[%d]' % d, True)
    if not game.float_reward:
      # bind d_reward_f64 for every program: the ones with int rewards must ignore it
      eng._reward_f64 = torch.full((eng.batch * 8,), UNUSED, dtype=torch.uint8,
                                   device=eng.device).view(torch.float64)
      held.append((vars(eng), '_reward_f64', eng._reward_f64))
      out.d_reward_f64 = eng._reward_f64.data_ptr()
    unused = 'd_reward' if game.float_reward else 'd_reward_f64'
    for f in ('d_board', 'd_reward', 'd_has_reward', 'd_discount', 'd_done', 'd_reward_f64'):
      setattr(out, f, guard(getattr(out, f), f, f == unused))
    live = eng.backdrop_live
    live_ptr = guard(None if live is None else live.data_ptr(), 'backdrop_live', False)
    for container, key, t in held:
      if t.data_ptr() in moved and tuple(moved[t.data_ptr()].shape) == tuple(t.shape):
        container[key] = moved[t.data_ptr()]
    _lib.check(eng._lib.pcl_bind_state(eng._h, C.byref(st)), 'pcl_bind_state')
    if live_ptr:
      _lib.check(eng._lib.pcl_bind_backdrop(eng._h, live_ptr), 'pcl_bind_backdrop')

  def check(self, what):
    torch = _torch()
    flags = [(name + ' written', (g != SENTINEL).any()) for name, g in self.guards]
    flags += [(name + ' changed', (now.reshape(-1).view(torch.uint8) != snap).any())
              for name, snap, now in self.frozen]
    bad = _failed(flags)
    assert not bad, '%s: %s' % (what, ', '.join(bad))


def _failed(flags):
  """Names of the (name, bool tensor) pairs that are true, with one device round trip."""
  if not flags:
    return []
  got = _torch().stack([f for _, f in flags]).cpu().tolist()
  return [name for (name, _), g in zip(flags, got) if g]


def _state(eng):
  """name -> u8 [B, bytes]: every per-env array a step may write, and every output the
  program defines."""
  per_env = dict(sprites=eng.sprites, drapes=eng.drapes, plot=eng.plot, rng=eng.rng,
                 z_order=eng.z_order, groups=eng.groups, backdrop_live=eng.backdrop_live,
                 board=eng._board, reward=eng.reward, has_reward=eng.has_reward,
                 discount=eng.discount, done=eng.done)
  for d, t in eng.patterns.items():
    if eng.game.pattern_mutable[d]:
      per_env['pattern%d' % d] = t
  for d, t in eng.bits.items():
    per_env['bits%d' % d] = t
  return {k: _rows(t) for k, t in per_env.items() if t is not None and t.numel()}


def _snapshot(eng):
  return {k: v.clone() for k, v in _state(eng).items()}


def _same_rows(got, want, envs, what, skip=()):
  """Every byte of rows `envs` of each array of `got` equals `want`'s."""
  idx = _torch().as_tensor(list(envs), dtype=_torch().long, device=next(iter(got.values())).device)
  if not len(envs):
    return
  bad = _failed([(k, (got[k].index_select(0, idx) != want[k].index_select(0, idx)).any())
                 for k in got if k not in skip])
  assert not bad, '%s, envs %s: %s differ' % (what, list(envs), ', '.join(bad))


class Pair(object):
  """A guarded engine and its unguarded twin, playing the same calls."""

  def __init__(self, case, B, auto_reset):
    from pycolab_b200 import batched
    self.case, self.B = case, B
    self.g = Guarded(batched.BatchedEngine(list(case.games), batch=B, auto_reset=auto_reset))
    self.eng = self.g.eng
    self.twin = batched.BatchedEngine(list(case.games), batch=B, auto_reset=auto_reset)

  def call(self, what, fn):
    fn(self.eng)
    fn(self.twin)
    self.g.check(what)
    _same_rows(_state(self.eng), _state(self.twin), range(self.B),
               what + ': guarded engine vs its twin')


def _device_actions(a):
  torch = _torch()
  return torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32).reshape(-1)).cuda()


def _draw(case, rs, T, B, quit_p):
  """int [T, B(, words)] drawn actions; each env-step quits with probability quit_p."""
  a = case.draw(rs, (T, B))
  if case.quit is not None:
    a[rs.random_sample((T, B)) < quit_p] = case.quit
  return a


def _poison_outputs(*engines):
  """Fill reward, has_reward, discount and done with a byte no step writes, so that a
  skipped env storing even the values it already held shows.  No kernel reads them."""
  for eng in engines:
    for t in (eng.reward, eng.has_reward, eng.discount, eng.done):
      t.view(_torch().uint8).fill_(POISON)


def _episodes(eng):
  from pycolab_b200 import _lib
  return eng.plot[:, _lib.P_EPISODES].cpu().numpy()


# ----------------------------------------------------------------------------- scenarios

@pytest.mark.parametrize('B', BATCHES)
def test_auto_reset_run_keeps_to_its_slices(case, B):
  """~60 steps with quits, so restarts happen mid-batch, then one pcl_run call: no guard
  byte, static array or unused reward word changes, and the guarded engine equals its twin."""
  pair = Pair(case, B, auto_reset=True)
  pair.call('its_showtime', lambda e: e.its_showtime())
  rs = np.random.RandomState(B)
  actions = _draw(case, rs, 60, B, 0.06)
  for t in range(len(actions)):
    a = _device_actions(actions[t])
    pair.call('step %d' % t, lambda e: e.play(a))
  run = _device_actions(_draw(case, rs, 9, B, 0.1)).view(9, -1)
  pair.call('pcl_run', lambda e: e.run(run))
  assert _episodes(pair.eng).sum() > B, 'no env restarted'


@pytest.mark.parametrize('B', BATCHES)
def test_frozen_envs_keep_every_byte(case, B):
  """Without auto_reset an env that is game over is skipped: every byte of its slice of
  every per-env array and every output stays as it was, while the other envs step."""
  pair = Pair(case, B, auto_reset=False)
  pair.call('its_showtime', lambda e: e.its_showtime())
  rs = np.random.RandomState(10 + B)
  T = 2 * B + 24                 # box_world's step limit and shockwave's waves end episodes too
  actions = case.draw(rs, (T, B))
  if case.quit is not None:
    for e in (range(B - 1) if B > 1 else [0]):       # env e quits at step 2e; the last never
      actions[2 * e, e] = case.quit
  frozen_steps = 0
  for t in range(T):
    over = np.flatnonzero(pair.eng.done.cpu().numpy())
    _poison_outputs(pair.eng, pair.twin)
    before = _snapshot(pair.eng)
    a = _device_actions(actions[t])
    pair.call('step %d' % t, lambda e: e.play(a))
    _same_rows(_state(pair.eng), before, over, 'step %d, frozen' % t)
    frozen_steps += len(over)
  assert frozen_steps > 0, 'no env was frozen'


@pytest.mark.parametrize('B', BATCHES)
def test_masked_reset_rebuilds_only_the_selected_envs(case, B):
  """A masked pcl_reset leaves every byte of the unselected envs alone, and the selected
  ones equal a fresh engine's after its_showtime() (built from the same games, drawing from
  where each env's random streams stand), but for the episode count (+1) and the error
  word (carried)."""
  from pycolab_b200 import _lib, batched
  torch = _torch()
  pair = Pair(case, B, auto_reset=False)
  pair.call('its_showtime', lambda e: e.its_showtime())
  rs = np.random.RandomState(20 + B)
  actions = _draw(case, rs, 20, B, 0.05)
  for t in range(len(actions)):
    a = _device_actions(actions[t])
    pair.call('step %d' % t, lambda e: e.play(a))

  _poison_outputs(pair.eng, pair.twin)
  before = _snapshot(pair.eng)
  none = torch.zeros(B, dtype=torch.uint8, device='cuda')
  pair.call('reset of no env', lambda e: e.reset(none))
  _same_rows(_state(pair.eng), before, range(B), 'reset of no env')

  chosen = np.arange(B) % 3 == 0
  mask = torch.from_numpy(chosen.astype(np.uint8)).cuda()
  rng = None if pair.eng.rng is None else pair.eng.rng.cpu().numpy().view(np.uint32).copy()
  plot = pair.eng.plot.cpu().numpy().copy()
  pair.call('masked reset', lambda e: e.reset(mask))
  now = _state(pair.eng)
  _same_rows(now, before, np.flatnonzero(~chosen), 'masked reset, unselected')
  fresh = batched.BatchedEngine(list(case.games), batch=B, auto_reset=False, rng_states=rng)
  fresh.its_showtime()
  want = _state(fresh)
  sel = np.flatnonzero(chosen)
  _same_rows(now, want, sel, 'masked reset vs a fresh engine', skip=('plot',))
  got_plot, fresh_plot = pair.eng.plot.cpu().numpy(), fresh.plot.cpu().numpy()
  carried = [_lib.P_EPISODES, _lib.P_ERROR]
  keep = np.setdiff1d(np.arange(_lib.PLOT_WORDS), carried)
  np.testing.assert_array_equal(got_plot[sel][:, keep], fresh_plot[sel][:, keep])
  np.testing.assert_array_equal(got_plot[sel, _lib.P_EPISODES], plot[sel, _lib.P_EPISODES] + 1)
  np.testing.assert_array_equal(got_plot[sel, _lib.P_ERROR], plot[sel, _lib.P_ERROR])


@pytest.mark.parametrize('B', BATCHES)
def test_restart_equals_masked_reset(case, B):
  """Two engines in the same state, env k game over: (a) one auto-reset step, (b) pcl_reset
  of env k alone.  Env k's slice of every per-env array and output is the same on both."""
  torch = _torch()
  k = B - 1
  a_pair, b_pair = Pair(case, B, auto_reset=True), Pair(case, B, auto_reset=True)
  for p in (a_pair, b_pair):
    p.call('its_showtime', lambda e: e.its_showtime())
  rs = np.random.RandomState(30 + B)
  actions = case.draw(rs, (80, B))
  if case.quit is not None:
    actions[3, k] = case.quit
  for t in range(len(actions)):
    a = _device_actions(actions[t])
    for p in (a_pair, b_pair):
      p.call('step %d' % t, lambda e: e.play(a))
    if pair_done(a_pair, k):
      break
  assert pair_done(a_pair, k), 'env %d never ended its episode' % k
  _same_rows(_state(a_pair.eng), _state(b_pair.eng), range(B), 'the two engines before')
  a = _device_actions(case.draw(rs, (B,)))
  a_pair.call('restart step', lambda e: e.play(a))
  mask = torch.from_numpy((np.arange(B) == k).astype(np.uint8)).cuda()
  b_pair.call('masked reset', lambda e: e.reset(mask))
  _same_rows(_state(a_pair.eng), _state(b_pair.eng), [k], 'restart vs masked reset')


def pair_done(pair, k):
  return bool(pair.eng.done[k].item())


# ------------------------------------------------- the protocol at B = 4 and 6, on boards

@pytest.mark.parametrize('program', PROTOCOL_PROGRAMS)
def test_partial_reset_touches_only_masked_envs(program):
  """A masked reset rebuilds the selected envs as a fresh Engine would (its_showtime,
  frame 0) and leaves every other env's board and frame as they were."""
  from pycolab_b200 import batched
  torch = _torch()
  make, draw, _ = _protocol_program(program)
  B = 6
  eng = batched.BatchedEngine([make()], batch=B, auto_reset=False)
  first = eng.its_showtime().board.clone()
  rs = np.random.RandomState(0)
  for _ in range(25):
    eng.play(draw(rs, (B,)).astype(np.int32).reshape(-1))
  before = eng.board.clone()
  frames = eng.frames().tolist()
  # A fresh Engine draws from where each env's random stream stands now.
  rng = None if eng.rng is None else eng.rng.cpu().numpy().view(np.uint32).copy()
  mask = torch.tensor([1, 0, 0, 1, 0, 0], dtype=torch.uint8, device='cuda')
  eng.reset(mask)
  fresh = batched.BatchedEngine([make()], batch=B, auto_reset=False, rng_states=rng)
  want = fresh.its_showtime().board
  torch.cuda.synchronize()
  if rng is None:
    assert bool((want == first).all())
  assert bool((eng.board[[0, 3]] == want[[0, 3]]).all())
  assert bool((eng.board[[1, 2, 4, 5]] == before[[1, 2, 4, 5]]).all())
  assert eng.frames().tolist() == [0, frames[1], frames[2], 0, frames[4], frames[5]]


@pytest.mark.parametrize('program', PROTOCOL_PROGRAMS)
def test_finished_env_freezes_without_auto_reset(program):
  """Upstream raises on play() after the episode ended (engine.py:622-624); the
  batched engine leaves such an env untouched instead, and steps the others."""
  from pycolab_b200 import batched
  torch = _torch()
  make, draw, quit_row = _protocol_program(program)
  B, T = 4, 12
  eng = batched.BatchedEngine([make()], batch=B, auto_reset=False)
  eng.its_showtime()
  rs = np.random.RandomState(4)
  actions = draw(rs, (T, B))
  if quit_row is not None:
    for e in range(B - 1):                    # env e quits at step 2e, the last env never
      actions[2 * e, e] = quit_row
  frozen_steps = 0
  for t in range(T):
    done = eng.done.cpu().numpy().astype(bool)
    board = eng.board.cpu().numpy()
    frames = eng.frames().cpu().numpy()
    res = eng.play(actions[t].astype(np.int32).reshape(-1))
    torch.cuda.synchronize()
    now = res.done.cpu().numpy().astype(bool)
    assert now[done].all(), (t, done, now)
    np.testing.assert_array_equal(res.board.cpu().numpy()[done], board[done], err_msg='t=%d' % t)
    new_frames = eng.frames().cpu().numpy()
    np.testing.assert_array_equal(new_frames[done], frames[done], err_msg='t=%d' % t)
    np.testing.assert_array_equal(new_frames[~done], frames[~done] + 1, err_msg='t=%d' % t)
    discount = res.discount.cpu().numpy()
    np.testing.assert_array_equal(discount[~done], np.where(now[~done], 0.0, 1.0))
    frozen_steps += int(done.sum())
  assert frozen_steps > 0                     # some env really was frozen
