"""Episode time limits (`pcl_set_time_limit`, `BatchedEngine.set_time_limit`) on the device.

A limit of L is exactly "game over at frame L": an engine with the limit and a twin without
it play the same actions, and wherever the limited engine reports done 2 the twin reports
done 0, with every other byte the same; the test then writes 2 into the twin's plot
game-over word and done, and from there on the two must stay equal byte for byte (records,
patterns, bits, random streams, boards, outputs and error words), restarts and frozen envs
included.  Also: the oracle lock-step with the rule layered on the oracle worlds
(tests/time_limit_lockstep.py), rollouts (eager, captured, with the limit changed between
calls) against play()s, the host-buffer and hand-off paths, shards, launch and chaining
counts, and guard bytes around every array and output slot.
"""

import numpy as np
import pytest

import test_gpu_protocol as gp
import test_gpu_rollout as gr
import time_limit_lockstep as tll
from oracle import games as ogames

pytestmark = pytest.mark.gpu

compiled_modules = gp.compiled_modules      # the fixture the compiled cases need


def _torch():
  import torch
  return torch


@pytest.fixture(params=gp.CASES)
def case(request, compiled_modules):
  return gp._lowered(request.param, tuple(compiled_modules))


def _engine(games, B, **kw):
  from pycolab_b200 import batched
  return batched.BatchedEngine(list(games), batch=B, **kw)


def _game_over(eng):
  from pycolab_b200 import _lib
  return eng.plot[:, _lib.P_GAME_OVER]


def _same_engines(a, b, what, skip=()):
  gp._same_rows(gp._state(a), gp._state(b), range(a.batch), what, skip=skip)
  gr._same(a.error_codes(), b.error_codes(), '%s: error words' % what)


def _mark_cut(eng, twin, live):
  """After a step: the envs the limited `eng` truncated (done 2 where the env was running
  before the step) are running on the unlimited twin; end them there by hand.  Returns how
  many there were."""
  cut = (eng.done == 2) & live
  assert not bool((twin.done[cut] != 0).any()), 'a truncated env is not running on the twin'
  _game_over(twin)[cut] = 2
  twin.done[cut] = 2
  return int(cut.sum())


# ----------------------------------------------------- a limit is game over at frame L

@pytest.mark.parametrize('auto_reset', [True, False], ids=['auto_reset', 'frozen'])
@pytest.mark.parametrize('L', [1, 2, 7])
@pytest.mark.parametrize('B', gp.BATCHES)
def test_limit_is_game_over_at_frame_L(case, B, L, auto_reset):
  eng = _engine(case.games, B, auto_reset=auto_reset, time_limit=L)
  twin = _engine(case.games, B, auto_reset=auto_reset)
  eng.its_showtime(), twin.its_showtime()
  _same_engines(eng, twin, 'its_showtime')
  rs = np.random.RandomState(100 * L + B + (0 if auto_reset else 50))
  T = 3 * L + 12
  actions = gp._draw(case, rs, T, B, 0.08)
  actions[0] = case.draw(rs, (1, B))[0]          # no quit in the first step
  cut = 0
  for t in range(T):
    live = _game_over(eng) == 0
    a = gp._device_actions(actions[t])
    eng.play(a), twin.play(a)
    cut += _mark_cut(eng, twin, live)
    _same_engines(eng, twin, 'L %d, step %d' % (L, t))
  if L == 1:
    assert cut > 0, 'the limit ended no episode'
  assert bool((_game_over(eng) <= 2).all())


# ------------------------------------------------------------ reference semantics

def _lockstep(make_facade_game, make_oracle, actions, L, n_levels=1, rng_seed=0, curtains=''):
  from pycolab_b200 import batched
  B = actions.shape[1]
  eng = batched.BatchedEngine([make_facade_game(i) for i in range(n_levels)], batch=B,
                              rng_seed=rng_seed, time_limit=L)
  eng.its_showtime()
  compared, cut = tll.lockstep(eng, make_oracle, range(B), actions, L, curtains=curtains)
  assert compared == (actions.shape[0] + 1) * B
  assert cut > 0, 'the limit ended no episode'
  assert int(eng.error_codes().max()) == 0


@pytest.mark.parametrize('L', [1, 17])
def test_scrolly_maze_vs_oracle(L):
  import golden_cases as gc
  from pycolab_b200.games import scrolly_maze
  maze, board, beneath = gc.scrolly_art(gc.load('scrolly_stock_L0'))
  rs = np.random.RandomState(42)
  actions = rs.randint(0, 6, size=(120, 24))
  actions[rs.random_sample(actions.shape) < 0.95] %= 5
  _lockstep(lambda i: scrolly_maze.make_game(maze, board, beneath),
            lambda e: ogames.make_scrolly_maze(maze, board, '+', beneath), actions, L,
            curtains='#@')


def test_warehouse_vs_oracle():
  from pycolab_b200 import levels
  from pycolab_b200.games import warehouse_manager
  arts = [levels.warehouse_level(20, shape=(24, 31), num_boxes=4, num_goals=6),
          levels.warehouse_level(77, shape=(24, 31), num_boxes=4, num_goals=6)]
  rs = np.random.RandomState(44)
  actions = rs.randint(0, 6, size=(150, 16))
  actions[rs.random_sample(actions.shape) < 0.97] %= 5
  _lockstep(lambda i: warehouse_manager.make_game(arts[i]),
            lambda e: ogames.make_warehouse(arts[e % 2]), actions, 23, n_levels=2,
            curtains='X')


def test_marauders_vs_oracle():
  from pycolab_b200 import levels
  from pycolab_b200.games import extraterrestrial_marauders as marauders
  art = levels.marauders_level()
  rs = np.random.RandomState(46)
  B = 12
  actions = rs.randint(0, 4, size=(200, B))
  rngs = [np.random.RandomState(900 + e) for e in range(B)]     # one stream per env, kept
  _lockstep(lambda i: marauders.make_game(art), lambda e: ogames.make_marauders(art, rngs[e]),
            actions, 31, rng_seed=900, curtains='BX')


# ------------------------------------------------------------------------ rollouts

def test_rollout_equals_play_for_every_program(case):
  T, B, L = 64, 11, 5
  eng = _engine(case.games, B, time_limit=L)
  twin = _engine(case.games, B, time_limit=L)
  eng.its_showtime(), twin.its_showtime()
  rs = np.random.RandomState(64)
  actions = gr._device(gp._draw(case, rs, T, B, 0.04).reshape(T, B, eng.actions_per_env))
  want = gr._played(twin, actions, observe=lambda e: e.repaint({}))
  traj = eng.rollout(actions, observer=gr._identity())
  gr._check_slots(traj, want, T, 'rollout')
  _same_engines(eng, twin, 'after the rollout')
  assert bool((traj.done == 2).any()), 'the limit ended no episode'


def _scrolly(B, **kw):
  case = gp._lowered('scrolly_maze', ())
  return case, [_engine(case.games, B, **kw) for _ in range(2)]


def test_frozen_envs_after_a_truncation_hold_the_fixed_record():
  """Without auto_reset, a rollout slot shows done 2 at the truncating step and the fixed
  frozen record (done 1, discount 0.0) at every later one."""
  T, B, L = 20, 11, 6
  case, (eng, twin) = _scrolly(B, auto_reset=False, time_limit=L)
  eng.its_showtime(), twin.its_showtime()
  actions = gr._device(case.draw(np.random.RandomState(5), (T, B)))
  want = gr._played(twin, actions)
  traj = eng.rollout(actions)
  done = want['done'].cpu().numpy()
  for e in range(B):
    end = int(np.flatnonzero(done[:, e])[0])        # every env ends by step L - 1
    assert end <= L - 1
    for name in ('reward', 'has_reward', 'discount', 'done'):
      gr._same(getattr(traj, name)[:end + 1, e], want[name][:end + 1, e],
               '%s env %d' % (name, e))
    assert traj.done[end + 1:, e].eq(1).all() and traj.discount[end + 1:, e].eq(0).all()
    assert traj.has_reward[end + 1:, e].eq(0).all() and traj.reward[end + 1:, e].eq(0).all()
  assert (done == 2).any()
  # the rollout leaves the fixed record in the outputs of envs frozen at its last step
  _same_engines(eng, twin, 'after the rollout', skip=('reward', 'has_reward', 'discount', 'done'))


def test_set_time_limit_between_calls():
  """The limit applies from the next launch: rollouts and play()s under the same sequence of
  limits agree, including an env already past a lowered limit, cut at its next step."""
  case, (eng, twin) = _scrolly(B=37, time_limit=9)
  eng.its_showtime(), twin.its_showtime()
  rs = np.random.RandomState(8)
  for k, L in enumerate([9, 3, None, 4, 0, 12]):
    eng.set_time_limit(L), twin.set_time_limit(L)
    actions = gr._device(gp._draw(case, rs, 15, eng.batch, 0.03))
    want = gr._played(twin, actions)
    traj = eng.rollout(actions)
    gr._check_slots(traj, want, 15, 'call %d (limit %r)' % (k, L))
    _same_engines(eng, twin, 'after call %d' % k)
    assert bool((traj.done == 2).any()) == bool(L), (k, L)


def test_captured_rollout_keeps_its_limit():
  """A rollout captured at limit 5 replays at limit 5 whatever the engine's limit is now,
  against an eager twin at limit 5."""
  from pycolab_b200 import batched
  torch = _torch()
  case, (eng, twin) = _scrolly(B=64, time_limit=5)
  crop = batched.scrolling_crop_spec(9, 9, 0)
  views = [e.attach_cropper(crop) for e in (eng, twin)]
  eng.its_showtime(), twin.its_showtime()
  T = 16
  actions = gr._device(gp._draw(case, np.random.RandomState(4), 3 * T, eng.batch, 0.02))
  fixed = actions[:T].clone()
  traj = eng.rollout(fixed, keep_attached=True)
  twin.rollout(actions[:T], keep_attached=True)
  torch.cuda.synchronize()
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g):
    assert eng.rollout(fixed, out=traj, keep_attached=True) is traj
  eng.set_time_limit(2)                        # not seen by the captured launches
  for r in (1, 2):
    fixed.copy_(actions[r * T:(r + 1) * T])
    g.replay()
    want = twin.rollout(actions[r * T:(r + 1) * T], keep_attached=True)
    torch.cuda.synchronize()
    for name in ('reward', 'has_reward', 'discount', 'done', 'attached'):
      gr._same(getattr(traj, name), getattr(want, name), 'replay %d: %s' % (r, name))
    gr._same(views[0], views[1], 'replay %d: attached view' % r)
    _same_engines(eng, twin, 'replay %d' % r)
    assert bool((traj.done == 2).any())


@pytest.mark.parametrize('keep_attached', [False, True])
def test_launches_and_chaining_as_without_a_limit(keep_attached):
  from pycolab_b200 import batched
  case = gp._lowered('scrolly_maze', ())
  counts = []
  for L in (None, 3):
    eng = _engine(case.games, 300, time_limit=L)
    eng.attach_cropper(batched.scrolling_crop_spec(9, 9, 0))
    eng.its_showtime()
    T = 24
    actions = gr._device(gp._draw(case, np.random.RandomState(1), T, eng.batch, 0.05))
    n0, c0 = eng.launch_count(), gr._chained(eng)
    traj = eng.rollout(actions, keep_attached=keep_attached)
    counts.append((eng.launch_count() - n0, gr._chained(eng) - c0))
    assert bool((traj.done == 2).any()) == (L is not None)
  assert counts[0] == counts[1] == (24, 22)


# --------------------------------------------------------- host buffers and hand-off

def test_host_paths_and_handoff_carry_done_2():
  from pycolab_b200 import _lib
  torch = _torch()
  B, L = 11, 4
  case, (eng, twin) = _scrolly(B, time_limit=L)
  eng.its_showtime(), twin.its_showtime()
  rs = np.random.RandomState(12)
  view_bytes = eng.rows * eng.pitch
  off = (view_bytes + 3) & ~3                  # PCL_HANDOFF_RECORD_BYTES: reward, discount, done
  packed = torch.zeros((B, off + 12), dtype=torch.uint8, device='cuda')
  seen = set()
  for t in range(3 * L):
    a = gp._draw(case, rs, 1, B, 0.02)[0].astype(np.int32)
    if t % 2:
      board, reward, has, disc, done = eng.play_host(a)
    else:
      eng.play_host_async(a, slot=t % _lib.HOST_SLOTS)
      board, reward, has, disc, done = eng.host_wait(t % _lib.HOST_SLOTS)
    twin.play(gp._device_actions(a))
    np.testing.assert_array_equal(done, twin.done.cpu().numpy())
    np.testing.assert_array_equal(reward, twin.reward.cpu().numpy())
    np.testing.assert_array_equal(disc, twin.discount.cpu().numpy())
    np.testing.assert_array_equal(has, twin.has_reward.cpu().numpy())
    np.testing.assert_array_equal(board[:, :, :eng.cols], twin.board.cpu().numpy())
    eng.pack_handoff(eng._board.reshape(B, -1), packed)
    rec = packed.cpu().numpy()
    np.testing.assert_array_equal(rec[:, off + 8], done)
    np.testing.assert_array_equal(rec[:, off:off + 4].copy().view(np.int32)[:, 0], reward)
    seen.update(done.tolist())
  assert 2 in seen


def test_shards_reproduce_one_engine():
  from pycolab_b200 import dist
  torch = _torch()
  case = gp._lowered('shockwave', ())
  B, T, L = 22, 40, 6
  game = case.games[0]
  whole = _engine([game], B, time_limit=L)
  shards = [dist.make_shard_engine([game], B, r, 2, 0, time_limit=L) for r in range(2)]
  for e in [whole] + shards:
    e.its_showtime()
  actions = gr._device(gp._draw(case, np.random.RandomState(9), T, B, 0.0))
  want = whole.rollout(actions)
  got = [s.rollout(actions[:, r * 11:(r + 1) * 11].contiguous()) for r, s in enumerate(shards)]
  for name in ('reward', 'has_reward', 'discount', 'done'):
    gr._same(torch.cat([getattr(g, name) for g in got], 1), getattr(want, name), name)
  assert bool((want.done == 2).any())


# ---------------------------------------------------------------------- guard bytes

def test_guarded_arrays_with_a_limit(case):
  """Every array the handle sees sits between guard bytes (gp.Guarded): with a limit,
  play(), run() and a rollout write nothing outside each env's slice, and the guarded
  engine equals its unguarded twin."""
  B, L = 11, 3
  eng = gp.Guarded(_engine(case.games, B, time_limit=L))
  twin = _engine(case.games, B, time_limit=L)
  rs = np.random.RandomState(77)

  def both(what, fn):
    fn(eng.eng), fn(twin)
    eng.check(what)
    _same_engines(eng.eng, twin, what)
  both('its_showtime', lambda e: e.its_showtime())
  for t in range(2 * L + 2):
    a = gp._device_actions(gp._draw(case, rs, 1, B, 0.05)[0])
    both('step %d' % t, lambda e: e.play(a))
  run = gr._device(gp._draw(case, rs, 7, B, 0.05).reshape(7, B, -1))
  both('pcl_run', lambda e: e.run(run))
  roll = gr._device(gp._draw(case, rs, 9, B, 0.05).reshape(9, B, -1))
  both('rollout', lambda e: e.rollout(roll))
  assert int(gp._episodes(twin).sum()) > B, 'no env restarted'


@pytest.mark.parametrize('auto_reset', [True, False])
def test_nothing_outside_the_slots_is_written(auto_reset):
  from pycolab_b200 import batched
  B, T, L = 37, 16, 4
  case, (eng, twin) = _scrolly(B, auto_reset=auto_reset, time_limit=L)
  crop = batched.scrolling_crop_spec(5, 7, 0, pad_char=' ', scroll_margins=(1, 2))
  for e in (eng, twin):
    e.attach_cropper(crop)
    e.its_showtime()
  actions = gr._device(gp._draw(case, np.random.RandomState(2), T, B, 0.05))
  shapes = twin.rollout(actions, observer=gr._identity(), keep_attached=True)
  out, guards = gr._guarded_like(shapes)
  traj = eng.rollout(actions, observer=gr._identity(), keep_attached=True, out=out)
  for name in batched.Trajectory.__slots__:
    if getattr(traj, name) is not None:
      gr._same(getattr(traj, name), getattr(shapes, name), name)
  bad = [name for name, g in guards if bool((g != gr.SENTINEL).any())]
  assert not bad, bad
  assert bool((traj.done == 2).any())
