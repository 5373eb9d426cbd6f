"""Rollouts (`pcl_rollout`, `BatchedEngine.rollout`) against T play()s, on the device.

Twin engines built from the same games and seeds take the same actions: one plays T steps
and clones, after each, the outputs, the attached cropper's view and the observer's result
(to_feature_array / to_array / repaint); the other runs one rollout.  Every slot must be
byte-identical, and afterwards both engines' per-env state (gp._state: boards, records,
patterns, bits, RNG states, outputs) and error words too.  Also: the fixed record of frozen
envs, guard bytes around every destination, launch and chaining counts, capture into a CUDA
graph, and shards that reproduce one engine.
"""

import ctypes as C

import numpy as np
import pytest

import test_gpu_protocol as gp

pytestmark = pytest.mark.gpu

compiled_modules = gp.compiled_modules      # the fixture the compiled cases need

SENTINEL = 0xA5


def _torch():
  import torch
  return torch


@pytest.fixture(params=gp.CASES)
def case(request, compiled_modules):
  return gp._lowered(request.param, tuple(compiled_modules))


def _twins(games, B, **kw):
  from pycolab_b200 import batched
  engs = [batched.BatchedEngine(list(games), batch=B, **kw) for _ in range(2)]
  return engs


def _device(a):
  return _torch().from_numpy(np.ascontiguousarray(a, dtype=np.int32)).cuda()


def _bytes(t):
  return t.contiguous().reshape(-1).view(_torch().uint8)


def _same(got, want, what):
  assert got.shape == want.shape and got.dtype == want.dtype, (what, got.shape, want.shape)
  assert bool(_torch().equal(_bytes(got), _bytes(want))), what


def _played(eng, actions, observe=None, keep_attached=False):
  """T play()s: the per-step outputs, views and attached views, stacked as [T, B, ...]."""
  torch = _torch()
  keep = dict(reward=[], has_reward=[], discount=[], done=[], view=[], attached=[])
  for t in range(actions.shape[0]):
    eng.play(actions[t])
    for name in ('reward', 'has_reward', 'discount', 'done'):
      keep[name].append(getattr(eng, name).clone())
    if observe is not None:
      keep['view'].append(observe(eng).clone())
    if keep_attached:
      keep['attached'].append(eng._attached[2].clone())
  return {k: torch.stack(v) if v else None for k, v in keep.items()}


def _check_slots(traj, want, T, what, envs=None):
  for name in ('reward', 'has_reward', 'discount', 'done', 'view', 'attached'):
    got, exp = getattr(traj, name), want.get(name)
    if exp is None or T == 0:
      continue
    if envs is not None:
      got, exp = got[:, envs], exp[:, envs]
    _same(got, exp, '%s: %s' % (what, name))


def _check_engines(a, b, what, skip=()):
  state_a, state_b = gp._state(a), gp._state(b)
  for k in state_a:
    if k not in skip:
      _same(state_a[k], state_b[k], '%s: engine %s' % (what, k))
  _same(a.error_codes(), b.error_codes(), '%s: error words' % what)


def _identity():
  from pycolab_b200 import rendering
  return rendering.ObservationCharacterRepainter({})


# ------------------------------------------------------------ lock-step, every program

@pytest.mark.parametrize('T,B', [(0, 11), (1, 11), (64, 1), (64, 11), (64, 37)])
def test_rollout_equals_play_for_every_program(case, T, B):
  """The identity repaint keeps every step's board, so every slot, boards included, is
  what play() left after that step."""
  eng, twin = _twins(case.games, B)
  eng.its_showtime(), twin.its_showtime()
  rs = np.random.RandomState(T + B)
  actions = _device(gp._draw(case, rs, T, B, 0.08).reshape(T, B, eng.actions_per_env))
  want = _played(twin, actions, observe=lambda e: e.repaint({}))
  n0 = eng.launch_count()
  traj = eng.rollout(actions, observer=_identity())
  assert eng.launch_count() == n0 + 2 * T                # a step and an observer per step
  assert traj.reward.dtype == eng.reward.dtype and traj.view.shape == (T, B, eng.rows, eng.cols)
  _check_slots(traj, want, T, 'rollout')
  _check_engines(eng, twin, 'after the rollout')
  if T == 64:
    assert gp._episodes(eng).sum() > B, 'no env restarted'
  a = _device(gp._draw(case, rs, 1, B, 0.1).reshape(B, -1))
  eng.play(a), twin.play(a)                              # play() goes on from the rollout
  _check_engines(eng, twin, 'a play() after the rollout')


# ------------------------------------------------------------------ frozen envs

@pytest.mark.parametrize('program', ['scrolly_maze', 'classics', 'fixture', 'warehouse'])
def test_frozen_envs_hold_the_fixed_record(program):
  """Without auto_reset an env that is game over is skipped: its output slots hold done 1,
  has_reward 0, reward 0, discount 0.0, and its view slots the view of its unchanged
  board; the stepping envs' slots are play()'s."""
  torch = _torch()
  case = gp._lowered(program, ())
  B, T = 11, 30
  eng, twin = _twins(case.games, B, auto_reset=False)
  eng.its_showtime(), twin.its_showtime()
  rs = np.random.RandomState(7)
  actions = case.draw(rs, (T, B))
  if case.quit is not None:
    for e in range(B - 1):                         # env e quits at step 2e; the last never
      actions[2 * e, e] = case.quit
  actions = _device(actions.reshape(T, B, -1))
  frozen = []
  want = dict(reward=[], has_reward=[], discount=[], done=[], view=[])
  for t in range(T):
    frozen.append(twin.done.clone().bool())
    got = _played(twin, actions[t:t + 1], observe=lambda e: e.repaint({}))
    for k in want:
      want[k].append(got[k][0])
  want = {k: torch.stack(v) for k, v in want.items()}
  frozen = torch.stack(frozen)
  assert bool(frozen.any()), 'no env was frozen'
  want['done'][frozen] = 1
  want['has_reward'][frozen] = 0
  want['reward'][frozen] = 0
  want['discount'][frozen] = 0.0
  traj = eng.rollout(actions, observer=_identity())
  _check_slots(traj, want, T, 'frozen')
  # the engines' outputs differ only in envs frozen at the last step
  live = (~frozen[-1]).nonzero().flatten().tolist()
  _check_engines(eng, twin, 'after the rollout', skip=('reward', 'has_reward', 'discount', 'done'))
  for name in ('reward', 'has_reward', 'discount', 'done'):
    _same(getattr(eng, name)[live], getattr(twin, name)[live], name)


def test_frozen_envs_keep_their_attached_view():
  """scrolly_maze's in-step cropper skips frozen envs; a rollout that keeps the attached
  view crops after the step instead, and every slot is the view play() leaves."""
  from pycolab_b200 import batched
  case = gp._lowered('scrolly_maze', ())
  B, T = 11, 24
  eng, twin = _twins(case.games, B, auto_reset=False)
  crop = batched.scrolling_crop_spec(7, 9, 0, pad_char=' ', scroll_margins=(2, 3))
  views = [e.attach_cropper(crop) for e in (eng, twin)]
  assert eng._attached[3]
  eng.its_showtime(), twin.its_showtime()
  actions = case.draw(np.random.RandomState(3), (T, B))
  for e in range(B - 1):
    actions[2 * e, e] = case.quit
  actions = _device(actions)
  want = _played(twin, actions, keep_attached=True)
  traj = eng.rollout(actions, keep_attached=True)
  _same(traj.attached, want['attached'], 'attached views')
  _same(views[0], views[1], 'the attached view after the rollout')


# ---------------------------------------------------------------------- observers

def _scrolly(B=11, **kw):
  case = gp._lowered('scrolly_maze', ())
  return case, _twins(case.games, B, **kw)


def _observer(kind, depth, chars, permute):
  """(post-processor, call on an engine) for `kind` of `depth` planes."""
  from pycolab_b200 import rendering
  layers = ''.join(chars[k % len(chars)] for k in range(depth))
  if kind == 'feature':
    return (rendering.ObservationToFeatureArray(layers, permute),
            lambda e, **kw: e.to_feature_array(layers, permute, **kw))
  mapping = dict((ch, tuple((ord(ch) * (d + 1)) % 251 - 100 for d in range(depth)))
                 for ch in chars)
  return (rendering.ObservationToArray(mapping, np.int16, permute),
          lambda e, **kw: e.to_array(mapping, np.int16, permute, **kw))


@pytest.mark.parametrize('window', [False, True], ids=['board', 'window'])
@pytest.mark.parametrize('permute', [None, (1, 2, 0)], ids=['planes', 'channels_last'])
@pytest.mark.parametrize('depth', [1, 32, 33, 70])
@pytest.mark.parametrize('kind', ['feature', 'array'])
def test_observers(kind, depth, permute, window):
  from pycolab_b200 import batched
  case, (eng, twin) = _scrolly()
  crop = batched.scrolling_crop_spec(9, 9, 0, pad_char=' ', scroll_margins=(None, None))
  states = [e.new_crop_state() if window else None for e in (eng, twin)]
  kw = lambda i: dict(crop_spec=crop, state=states[i]) if window else {}
  obs, call = _observer(kind, depth, twin.chars + ' ', permute)
  eng.its_showtime(), twin.its_showtime()
  T, B = 12, eng.batch
  actions = _device(gp._draw(case, np.random.RandomState(depth), T, B, 0.05))
  want = _played(twin, actions, observe=lambda e: call(e, **kw(1)))
  traj = eng.rollout(actions, observer=obs, **kw(0))
  _check_slots(traj, want, T, '%s depth %d' % (kind, depth))
  if window:
    _same(states[0], states[1], 'window corners')
  _check_engines(eng, twin, 'after the rollout')


@pytest.mark.parametrize('window', [False, True], ids=['board', 'window'])
def test_repaint_observer(window):
  from pycolab_b200 import batched, rendering
  case, (eng, twin) = _scrolly()
  crop = batched.scrolling_crop_spec(9, 9, 0, pad_char=' ', scroll_margins=(2, 2))
  mapping = {'#': '+', ' ': '.'}
  kw = dict(crop_spec=crop) if window else {}      # the plot record's cropper slot
  eng.its_showtime(), twin.its_showtime()
  T, B = 12, eng.batch
  actions = _device(gp._draw(case, np.random.RandomState(5), T, B, 0.05))
  want = _played(twin, actions, observe=lambda e: e.repaint(mapping, **kw))
  traj = eng.rollout(actions, observer=rendering.ObservationCharacterRepainter(mapping), **kw)
  assert traj.unknown is None
  _check_slots(traj, want, T, 'repaint')
  _check_engines(eng, twin, 'after the rollout')


@pytest.mark.parametrize('game', ['scrolly_maze', 'four_rooms'])
def test_keep_attached(game):
  """The cropper attached to the step kernel (scrolly_maze) or run after it (four_rooms),
  with an observer over another window."""
  from pycolab_b200 import batched
  from pycolab_b200.games.classics import four_rooms
  if game == 'scrolly_maze':
    case = gp._lowered('scrolly_maze', ())
    games, draw = case.games, lambda rs, T, B: gp._draw(case, rs, T, B, 0.05)
  else:
    games, draw = [four_rooms.make_game()], lambda rs, T, B: rs.randint(0, 4, (T, B))
  B, T = 37, 20
  eng, twin = _twins(games, B)
  crop = batched.scrolling_crop_spec(5, 5, 0, pad_char='~', scroll_margins=(1, 1))
  views = [e.attach_cropper(crop) for e in (eng, twin)]
  assert eng._attached[3] == (game == 'scrolly_maze')
  eng.its_showtime(), twin.its_showtime()
  obs, call = _observer('feature', 5, twin.chars, None)
  window = batched.scrolling_crop_spec(3, 3, 0, pad_char='~', scroll_margins=(None, None))
  states = [e.new_crop_state() for e in (eng, twin)]
  actions = _device(draw(np.random.RandomState(11), T, B))
  want = _played(twin, actions, observe=lambda e: call(e, crop_spec=window, state=states[1]),
                 keep_attached=True)
  traj = eng.rollout(actions, observer=obs, crop_spec=window, state=states[0],
                     keep_attached=True)
  _check_slots(traj, want, T, 'keep_attached')
  _same(views[0], views[1], 'the attached view after the rollout')
  plain = eng.rollout(actions[:3])                 # the cropper follows a rollout that keeps
  for t in range(3):                               # nothing, too
    twin.play(actions[t])
  assert plain.attached is None and plain.view is None
  _same(views[0], views[1], 'the attached view after a rollout that keeps no view')
  _check_engines(eng, twin, 'after the rollouts')


def test_to_array_raises_once_on_an_unmapped_pad():
  """A fixed window past the board shows the pad '~': an ObservationToArray without it
  raises after the rollout; one with it, a repaint and feature planes do not."""
  import torch
  from pycolab_b200 import _lib, batched, rendering
  from pycolab_b200.games.classics import four_rooms
  eng = batched.BatchedEngine([four_rooms.make_game()], batch=5)
  eng.its_showtime()
  fixed = _lib.CropSpec(5, 7, -1, ord('~'), 0, 0, -3, -4, 0)
  mapping = dict((ch, ord(ch)) for ch in eng.chars)
  actions = torch.zeros((6, 5), dtype=torch.int32, device='cuda')
  with pytest.raises(RuntimeError, match='only knows array values'):
    eng.rollout(actions, observer=rendering.ObservationToArray(mapping, np.int32),
                crop_spec=fixed)
  traj = eng.rollout(actions, observer=rendering.ObservationToArray(dict(mapping, **{'~': -1}),
                                                                    np.int32), crop_spec=fixed)
  assert int(traj.unknown[0]) == 0 and bool((traj.view[:, :, :3, :] == -1).all())
  eng.rollout(actions, observer=rendering.ObservationCharacterRepainter({'~': '#'}),
              crop_spec=fixed)
  eng.rollout(actions, observer=rendering.ObservationToFeatureArray('~#'), crop_spec=fixed)
  inner = _lib.CropSpec(3, 3, -1, ord('~'), 0, 0, 1, 1, 0)
  eng.rollout(actions, observer=rendering.ObservationToArray(mapping, np.int32), crop_spec=inner)


# ---------------------------------------------------------------------- guard bytes

def _guarded_like(traj, pad=4096):
  """A Trajectory of `traj`'s shapes whose tensors sit in the middle of sentinel-filled
  allocations, and the guards."""
  from pycolab_b200 import batched
  torch = _torch()
  guards, fields = [], {}
  for name in batched.Trajectory.__slots__:
    t = getattr(traj, name)
    if t is None:
      fields[name] = None
      continue
    nbytes = t.numel() * t.element_size()
    buf = torch.full((2 * pad + nbytes,), SENTINEL, dtype=torch.uint8, device=t.device)
    fields[name] = buf[pad:pad + nbytes].view(t.dtype).view(t.shape)
    guards += [(name, buf[:pad]), (name, buf[pad + nbytes:])]
  return batched.Trajectory(**fields), guards


@pytest.mark.parametrize('auto_reset', [True, False])
@pytest.mark.parametrize('game', ['scrolly_maze', 'four_rooms'])
def test_nothing_outside_the_slots_is_written(game, auto_reset):
  from pycolab_b200 import batched, rendering
  from pycolab_b200.games.classics import four_rooms
  torch = _torch()
  case = gp._lowered('scrolly_maze', ())
  games = case.games if game == 'scrolly_maze' else [four_rooms.make_game()]
  B, T = 37, 16
  rs = np.random.RandomState(2)
  eng, twin = _twins(games, B, auto_reset=auto_reset)
  crop = batched.scrolling_crop_spec(5, 7, 0, pad_char=' ', scroll_margins=(1, 2))
  for e in (eng, twin):
    e.attach_cropper(crop)
    e.its_showtime()
  mapping = dict((ch, (ord(ch), -ord(ch))) for ch in eng.chars + ' ')
  obs = rendering.ObservationToArray(mapping, np.float64, (1, 2, 0))
  window = batched.scrolling_crop_spec(9, 9, 0, pad_char=' ', scroll_margins=(None, None))
  actions = _device(gp._draw(case, rs, T, B, 0.1) if game == 'scrolly_maze' else
                    rs.randint(0, 4, (T, B)))
  shapes = twin.rollout(actions, observer=obs, crop_spec=window, keep_attached=True)
  out, guards = _guarded_like(shapes)
  traj = eng.rollout(actions, observer=obs, crop_spec=window, keep_attached=True, out=out)
  assert traj is out
  for name, t in ((n, getattr(traj, n)) for n in batched.Trajectory.__slots__):
    if t is not None:
      _same(t, getattr(shapes, name), name)
  bad = [name for name, g in guards if bool((g != SENTINEL).any())]
  assert not bad, bad


# ------------------------------------------------------------ launches and chaining

def _chained(e):
  n = C.c_int64()
  assert e._lib.pcl_chained_launch_count(e._h, C.byref(n)) == 0
  return n.value


@pytest.mark.parametrize('keep_attached', [False, True])
def test_launches_and_chaining(keep_attached):
  """scrolly_maze with its cropper in the step kernel and no observer: one launch per step,
  chained as pcl_run's are (the first follows no step launch, the second keeps the full
  wait and starts the counters, every later one is chained); with an observer between
  them, none is chained."""
  from pycolab_b200 import batched
  case, (eng, _) = _scrolly(B=300)
  eng.attach_cropper(batched.scrolling_crop_spec(9, 9, 0))
  eng.its_showtime()
  T = 24
  actions = _device(gp._draw(case, np.random.RandomState(1), T, eng.batch, 0.05))
  n0, c0 = eng.launch_count(), _chained(eng)
  eng.rollout(actions, keep_attached=keep_attached)
  assert eng.launch_count() - n0 == T
  assert _chained(eng) - c0 == T - 2
  n0, c0 = eng.launch_count(), _chained(eng)
  eng.rollout(actions, observer=_identity())
  assert eng.launch_count() - n0 == 2 * T
  assert _chained(eng) == c0


# -------------------------------------------------------------------------- capture

def test_captured_rollout_replays_into_its_trajectory():
  from pycolab_b200 import batched, rendering
  torch = _torch()
  case, (eng, twin) = _scrolly(B=64)
  crop = batched.scrolling_crop_spec(9, 9, 0)
  views = [e.attach_cropper(crop) for e in (eng, twin)]
  for e in (eng, twin):
    e.its_showtime()
  mapping = dict((ch, k) for k, ch in enumerate(eng.chars + ' '))
  obs = rendering.ObservationToArray(mapping, np.int32)
  window = batched.scrolling_crop_spec(7, 7, 0, pad_char=' ', scroll_margins=(None, None))
  T = 16
  actions = _device(gp._draw(case, np.random.RandomState(4), 3 * T, eng.batch, 0.05))
  fixed = actions[:T].clone()
  kw = dict(observer=obs, crop_spec=window, keep_attached=True)
  traj = eng.rollout(fixed, **kw)                 # allocates the trajectory and the tables
  twin.rollout(actions[:T], **kw)
  torch.cuda.synchronize()
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g):
    assert eng.rollout(fixed, out=traj, **kw) is traj
  for r in (1, 2):
    fixed.copy_(actions[r * T:(r + 1) * T])
    g.replay()
    want = twin.rollout(actions[r * T:(r + 1) * T], **kw)
    torch.cuda.synchronize()
    for name in batched.Trajectory.__slots__:
      _same(getattr(traj, name), getattr(want, name), 'replay %d: %s' % (r, name))
    _same(views[0], views[1], 'replay %d: attached view' % r)
    _check_engines(eng, twin, 'replay %d' % r)


# ------------------------------------------------------------------------- sharding

def test_shards_reproduce_one_engine():
  """Two shard engines (env_offset) reproduce one engine's rollout slot for slot: the same
  per-env random streams, levels and outputs."""
  from pycolab_b200 import batched
  torch = _torch()
  case = gp._lowered('shockwave', ())
  B, T, half = 22, 40, 11
  game = case.games[0]                         # one level: shard env e is global env e + offset
  whole = batched.BatchedEngine([game], batch=B)
  shards = [batched.BatchedEngine([game], batch=half, env_offset=r * half)
            for r in range(2)]
  for e in [whole] + shards:
    e.its_showtime()
  obs, _ = _observer('feature', 4, whole.chars, (1, 2, 0))
  window = batched.scrolling_crop_spec(5, 5, 0, pad_char=' ', scroll_margins=(None, None))
  actions = _device(gp._draw(case, np.random.RandomState(9), T, B, 0.0))
  want = whole.rollout(actions, observer=obs, crop_spec=window)
  got = [s.rollout(actions[:, r * half:(r + 1) * half].contiguous(), observer=obs,
                   crop_spec=window) for r, s in enumerate(shards)]
  for name in ('reward', 'has_reward', 'discount', 'done', 'view'):
    _same(torch.cat([getattr(g, name) for g in got], 1), getattr(want, name), name)
