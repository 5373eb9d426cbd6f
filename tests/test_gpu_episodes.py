"""Episode returns (`pcl_bind_episodes`, `pcl_rollout_episodes`, `track_episodes=`) on the
device.

A tracking engine and a non-tracking twin play the same actions: every array the step
writes stays byte-identical between them, and the tracking engine's `episode_return` equals
the host rule (tests/episode_reference.py) applied to the engine's own rewards and plot
frames, bit for bit.  Also: masked resets, rollouts against play()s, guard bytes around the
returns and the kept slots, a captured rollout, a captured graph of play()s at 4096 envs,
launch and chaining counts, the host-buffer paths, shards, C2's 4096-env scrolly_maze, and the
float-reward programs against Python's in-order `+=`.
"""

import ctypes as C

import numpy as np
import pytest

import episode_reference as ref
import test_gpu_protocol as gp
import test_gpu_rollout as gr

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


class Reference(object):
  """The rule of include/pcl.h over what an engine's calls leave in its outputs and plot:
  call after() with the envs the call ran."""

  def __init__(self, eng):
    self.eng = eng
    self.ret = np.zeros(eng.batch, np.float64)

  def after(self, ran):
    from pycolab_b200 import _lib
    eng = self.eng
    frame = eng.plot[:, _lib.P_FRAME].cpu().numpy()
    r = np.where(eng.has_reward.cpu().numpy() != 0,
                 eng.reward.cpu().numpy().astype(np.float64), 0.0)
    ran = np.asarray(ran, bool)
    self.ret = np.where(ran, np.where(frame == 0, r, self.ret + r), self.ret)

  def ran_by_play(self):
    """The envs the next play() steps: all but the frozen ones."""
    from pycolab_b200 import _lib
    over = self.eng.plot[:, _lib.P_GAME_OVER].cpu().numpy() != 0
    return np.ones(self.eng.batch, bool) if self.eng.auto_reset else ~over


def _check(eng, want, what):
  got = eng.episode_return.cpu().numpy()
  assert ref.same_bits(got, want), '%s: returns %s, want %s' % (what, got, want)


# -------------------------------------------------------- twins and the host rule

@pytest.mark.parametrize('L', [None, 5])
@pytest.mark.parametrize('auto_reset', [True, False], ids=['auto_reset', 'frozen'])
@pytest.mark.parametrize('B', gp.BATCHES)
def test_tracking_changes_nothing_and_follows_the_rule(case, B, auto_reset, L):
  eng = _engine(case.games, B, auto_reset=auto_reset, time_limit=L, track_episodes=True)
  twin = _engine(case.games, B, auto_reset=auto_reset, time_limit=L)
  assert twin.episode_return is None
  host = Reference(eng)
  eng.its_showtime(), twin.its_showtime()
  host.after(np.ones(B, bool))
  gp._same_rows(gp._state(eng), gp._state(twin), range(B), 'its_showtime')
  _check(eng, host.ret, 'its_showtime')
  rs = np.random.RandomState(7 * B + (0 if auto_reset else 3) + (L or 0))
  T = 30
  actions = gp._draw(case, rs, T, B, 0.08)
  ended = 0
  for t in range(T):
    ran = host.ran_by_play()
    a = gp._device_actions(actions[t])
    eng.play(a), twin.play(a)
    host.after(ran)
    gp._same_rows(gp._state(eng), gp._state(twin), range(B), 'step %d' % t)
    _check(eng, host.ret, 'step %d' % t)
    ended += int((eng.done != 0).sum())
  gr._same(eng.error_codes(), twin.error_codes(), 'error words')
  assert ended > 0 or L is None, 'the limit ended no episode'


def test_masked_reset_restarts_only_the_masked_returns(case):
  torch = _torch()
  B = 11
  eng = _engine(case.games, B, track_episodes=True)
  host = Reference(eng)
  eng.its_showtime()
  host.after(np.ones(B, bool))
  rs = np.random.RandomState(31)
  for t in range(6):
    eng.play(gp._device_actions(case.draw(rs, (1, B))[0]))
    host.after(np.ones(B, bool))
  before = eng.episode_return.clone()
  mask = np.zeros(B, bool)
  mask[[0, 4, 5, 10]] = True
  eng.reset(torch.from_numpy(mask.astype(np.uint8)).cuda())
  host.after(mask)
  _check(eng, host.ret, 'masked reset')
  keep = torch.from_numpy(~mask).cuda()
  gr._same(eng.episode_return[keep], before[keep], 'unmasked envs')
  # a masked env's return is its showtime reward
  from pycolab_b200 import _lib
  assert bool((eng.plot[torch.from_numpy(mask).cuda(), _lib.P_FRAME] == 0).all())


# ------------------------------------------------------------------------ rollouts

@pytest.mark.parametrize('auto_reset', [True, False], ids=['auto_reset', 'frozen'])
@pytest.mark.parametrize('T', [0, 1, 64])
def test_rollout_keeps_returns_and_lengths_as_play_does(case, T, auto_reset):
  from pycolab_b200 import _lib
  torch = _torch()
  B = 11
  eng = _engine(case.games, B, auto_reset=auto_reset, time_limit=9, track_episodes=True)
  twin = _engine(case.games, B, auto_reset=auto_reset, time_limit=9, track_episodes=True)
  eng.its_showtime(), twin.its_showtime()
  rs = np.random.RandomState(64 + T)
  actions = gr._device(gp._draw(case, rs, T, B, 0.04).reshape(T, B, eng.actions_per_env))
  rets, lens, frozen = [], [], []
  for t in range(T):
    frozen.append((twin.plot[:, _lib.P_GAME_OVER] != 0) & (not auto_reset))
    twin.play(actions[t])
    rets.append(twin.episode_return.clone())
    lens.append(twin.plot[:, _lib.P_FRAME].clone())
  ep = eng.new_episodes(T)
  traj = eng.rollout(actions, episodes=ep)
  if T:
    want_r, want_l, frozen = torch.stack(rets), torch.stack(lens), torch.stack(frozen)
    want_r[frozen], want_l[frozen] = 0.0, 0
    gr._same(ep.episode_return, want_r, 'kept returns')
    gr._same(ep.episode_length, want_l, 'kept lengths')
    assert not auto_reset or not bool(frozen.any())
    assert traj.done.shape == ep.episode_return.shape
  gr._same(eng.episode_return, twin.episode_return, 'returns after the rollout')
  gp._same_rows(gp._state(eng), gp._state(twin), range(B), 'after the rollout',
                skip=() if auto_reset else ('reward', 'has_reward', 'discount', 'done'))
  again = eng.rollout(actions, episodes=ep)     # reused buffers
  assert again.reward.shape[0] == T


def test_rollout_refusals():
  from pycolab_b200 import batched
  torch = _torch()
  case = gp._lowered('classics', ())
  plain = _engine(case.games, 3)
  eng = _engine(case.games, 3, track_episodes=True)
  for e in (plain, eng):
    e.its_showtime()
  actions = gr._device(np.zeros((4, 3)))
  with pytest.raises(ValueError, match='track_episodes=True'):
    plain.rollout(actions, episodes=eng.new_episodes(4))
  with pytest.raises(ValueError, match='track_episodes=True'):
    plain.new_episodes(4)
  bad = [batched.Episodes(torch.zeros((5, 3), dtype=torch.float64, device='cuda'),
                          torch.zeros((4, 3), dtype=torch.int32, device='cuda')),
         batched.Episodes(torch.zeros((4, 3), dtype=torch.float32, device='cuda'),
                          torch.zeros((4, 3), dtype=torch.int32, device='cuda')),
         batched.Episodes(torch.zeros((4, 3), dtype=torch.float64, device='cuda'),
                          torch.zeros((4, 3), dtype=torch.int64, device='cuda')),
         batched.Episodes(torch.zeros((4, 3), dtype=torch.float64),
                          torch.zeros((4, 3), dtype=torch.int32)),
         batched.Episodes(torch.zeros((3, 4), dtype=torch.float64, device='cuda').t(),
                          torch.zeros((4, 3), dtype=torch.int32, device='cuda'))]
  for ep in bad:
    with pytest.raises(ValueError, match='episodes'):
      eng.rollout(actions, episodes=ep)
  with pytest.raises(TypeError, match='Episodes'):
    eng.rollout(actions, episodes=(1, 2))


# ---------------------------------------------------------------------- guard bytes

def _guarded(t, pad=4096):
  """A copy of `t` in the middle of a sentinel-filled allocation, and its two guards."""
  torch = _torch()
  nbytes = t.numel() * t.element_size()
  buf = torch.full((2 * pad + nbytes,), gr.SENTINEL, dtype=torch.uint8, device=t.device)
  copy = buf[pad:pad + nbytes].view(t.dtype).view(t.shape)
  copy.copy_(t)
  return copy, [buf[:pad], buf[pad + nbytes:]]


def test_nothing_outside_the_returns_and_slots_is_written(case):
  from pycolab_b200 import _lib, batched
  B, T = 11, 24
  eng = gp.Guarded(_engine(case.games, B, time_limit=4, track_episodes=True))
  twin = _engine(case.games, B, time_limit=4, track_episodes=True)
  ret, guards = _guarded(eng.eng.episode_return)
  eng.eng.episode_return = ret
  _lib.check(eng.eng._lib.pcl_bind_episodes(eng.eng._h, ret.data_ptr()), 'pcl_bind_episodes')
  rs = np.random.RandomState(5)

  def both(what, fn):
    fn(eng.eng), fn(twin)
    eng.check(what)
    gp._same_rows(gp._state(eng.eng), gp._state(twin), range(B), what)
    gr._same(eng.eng.episode_return, twin.episode_return, what + ': returns')
    assert not any(bool((g != gr.SENTINEL).any()) for g in guards), what
  both('its_showtime', lambda e: e.its_showtime())
  for t in range(6):
    a = gp._device_actions(gp._draw(case, rs, 1, B, 0.05)[0])
    both('step %d' % t, lambda e: e.play(a))
  run = gr._device(gp._draw(case, rs, 7, B, 0.05).reshape(7, B, -1))
  both('pcl_run', lambda e: e.run(run))
  roll = gr._device(gp._draw(case, rs, T, B, 0.05).reshape(T, B, -1))
  r_copy, r_guards = _guarded(eng.eng.new_episodes(T).episode_return)
  l_copy, l_guards = _guarded(eng.eng.new_episodes(T).episode_length)
  mine, want = batched.Episodes(r_copy, l_copy), twin.new_episodes(T)
  both('rollout', lambda e: e.rollout(roll, episodes=mine if e is eng.eng else want))
  gr._same(mine.episode_return, want.episode_return, 'kept returns')
  gr._same(mine.episode_length, want.episode_length, 'kept lengths')
  assert not any(bool((g != gr.SENTINEL).any()) for g in r_guards + l_guards)


# -------------------------------------------------------------------------- capture

def test_captured_rollout_equals_an_eager_twin():
  """A rollout captured with episodes= replays into the same buffers, with returns that
  carry from one replay to the next, as an eager twin's."""
  torch = _torch()
  case = gp._lowered('scrolly_maze', ())
  B, T = 64, 16
  eng = _engine(case.games, B, track_episodes=True)
  twin = _engine(case.games, B, track_episodes=True)
  eng.its_showtime(), twin.its_showtime()
  actions = gr._device(gp._draw(case, np.random.RandomState(4), 3 * T, B, 0.01))
  fixed = actions[:T].clone()
  ep, want = eng.new_episodes(T), twin.new_episodes(T)
  traj = eng.rollout(fixed, episodes=ep)
  twin.rollout(actions[:T], episodes=want)
  torch.cuda.synchronize()
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g):
    eng.rollout(fixed, out=traj, episodes=ep)
  spanned = False
  for r in (1, 2):
    fixed.copy_(actions[r * T:(r + 1) * T])
    g.replay()
    twin_traj = twin.rollout(actions[r * T:(r + 1) * T], episodes=want)
    torch.cuda.synchronize()
    gr._same(ep.episode_return, want.episode_return, 'replay %d: returns' % r)
    gr._same(ep.episode_length, want.episode_length, 'replay %d: lengths' % r)
    gr._same(traj.done, twin_traj.done, 'replay %d: done' % r)
    gr._same(eng.episode_return, twin.episode_return, 'replay %d: [B] returns' % r)
    spanned |= bool((ep.episode_length[0] > 1).any())   # an episode begun in an earlier call
  assert spanned


def test_captured_plays_at_4096_envs_equal_an_eager_twin():
  """A CUDA graph of many play()s on a tracking 4096-env scrolly_maze engine, with quits
  (so envs restart inside the graph), replayed twice against an eager twin."""
  torch = _torch()
  case = gp._lowered('scrolly_maze', ())
  B, T = 4096, 200
  eng = _engine(case.games, B, track_episodes=True)
  twin = _engine(case.games, B, track_episodes=True)
  eng.its_showtime(), twin.its_showtime()
  actions = gr._device(gp._draw(case, np.random.RandomState(21), 3 * T, B, 0.01))
  fixed = actions[:T].clone()
  for t in range(T):                      # the launches the graph holds, eagerly first
    eng.play(fixed[t]), twin.play(actions[t])
  torch.cuda.synchronize()
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g):
    for t in range(T):
      eng.play(fixed[t])
  for r in (1, 2):
    fixed.copy_(actions[r * T:(r + 1) * T])
    g.replay()
    for t in range(r * T, (r + 1) * T):
      twin.play(actions[t])
    torch.cuda.synchronize()
    gr._same(eng.episode_return, twin.episode_return, 'replay %d: returns' % r)
    gp._same_rows(gp._state(eng), gp._state(twin), range(B), 'replay %d' % r)
  assert int(gp._episodes(eng).sum()) > B, 'no env restarted'


# ------------------------------------------------------------------------- launches

def test_launches_and_chaining_as_without_tracking():
  from pycolab_b200 import batched
  case = gp._lowered('scrolly_maze', ())
  counts = []
  for track in (False, True):
    eng = _engine(case.games, 300, time_limit=5, track_episodes=track)
    eng.attach_cropper(batched.scrolling_crop_spec(9, 9, 0))
    eng.its_showtime()
    T = 24
    actions = gr._device(gp._draw(case, np.random.RandomState(1), T, eng.batch, 0.05))
    n0, c0 = eng.launch_count(), gr._chained(eng)
    eng.rollout(actions, episodes=eng.new_episodes(T) if track else None)
    counts.append((eng.launch_count() - n0, gr._chained(eng) - c0))
  assert counts[0] == counts[1] == (24, 22)


def test_run_rotating_over_tracking_handles_chains_as_before():
  from pycolab_b200 import batched
  case = gp._lowered('scrolly_maze', ())
  R, b, T = 2, 512, 30
  chained = []
  for track in (False, True):
    engs = [_engine(case.games, b, env_offset=r * b, track_episodes=track) for r in range(R)]
    twins = [_engine(case.games, b, env_offset=r * b, track_episodes=True) for r in range(R)]
    for e in engs + twins:
      e.its_showtime()
    acts = gr._device(gp._draw(case, np.random.RandomState(5), T, b, 0.02))
    c0 = sum(gr._chained(e) for e in engs)
    batched.run_rotating(engs, [acts[t] for t in range(T)])
    chained.append(sum(gr._chained(e) for e in engs) - c0)
    for t in range(T):
      twins[t % R].play(acts[t])
    for i in range(R):
      gp._same_rows(gp._state(engs[i]), gp._state(twins[i]), range(b), 'batch %d' % i)
      if track:
        gr._same(engs[i].episode_return, twins[i].episode_return, 'batch %d returns' % i)
  assert chained[0] == chained[1] == T - 2


# ------------------------------------------------------------------------ other paths

def test_host_paths_update_returns_as_play_does():
  from pycolab_b200 import _lib
  case = gp._lowered('scrolly_maze', ())
  B = 11
  eng = _engine(case.games, B, time_limit=4, track_episodes=True)
  twin = _engine(case.games, B, time_limit=4, track_episodes=True)
  eng.its_showtime(), twin.its_showtime()
  rs = np.random.RandomState(12)
  for t in range(14):
    a = gp._draw(case, rs, 1, B, 0.02)[0].astype(np.int32)
    if t % 2:
      eng.play_host(a)
    else:
      eng.play_host_async(a, slot=t % _lib.HOST_SLOTS)
      eng.host_wait(t % _lib.HOST_SLOTS)
    twin.play(gp._device_actions(a))
    gr._same(eng.episode_return, twin.episode_return, 'step %d' % t)


def test_shards_reproduce_one_engine():
  from pycolab_b200 import dist
  torch = _torch()
  case = gp._lowered('shockwave', ())
  B, T = 22, 40
  game = case.games[0]
  whole = _engine([game], B, time_limit=6, track_episodes=True)
  shards = [dist.make_shard_engine([game], B, r, 2, 0, time_limit=6, track_episodes=True)
            for r in range(2)]
  for e in [whole] + shards:
    e.its_showtime()
  actions = gr._device(gp._draw(case, np.random.RandomState(9), T, B, 0.0))
  want = whole.new_episodes(T)
  whole.rollout(actions, episodes=want)
  got = [s.new_episodes(T) for s in shards]
  for r, s in enumerate(shards):
    s.rollout(actions[:, r * 11:(r + 1) * 11].contiguous(), episodes=got[r])
  for name in ('episode_return', 'episode_length'):
    gr._same(torch.cat([getattr(g, name) for g in got], 1), getattr(want, name), name)
  gr._same(torch.cat([s.episode_return for s in shards]), whole.episode_return, 'returns')


# ---------------------------------------------------------- scale and float rewards

def test_c2_scrolly_maze_at_4096_envs():
  """The one-wave path, several envs per warp's block: 200 steps with quits."""
  case = gp._lowered('scrolly_maze', ())
  B = 4096
  eng = _engine(case.games, B, track_episodes=True)
  host = Reference(eng)
  eng.its_showtime()
  host.after(np.ones(B, bool))
  rs = np.random.RandomState(2)
  actions = gr._device(gp._draw(case, rs, 200, B, 0.01))
  for t in range(200):
    eng.play(actions[t])
    host.after(np.ones(B, bool))
  _check(eng, host.ret, 'after 200 steps')
  assert int(gp._episodes(eng).sum()) > B, 'no env restarted'


@pytest.mark.parametrize('name', ['t_maze', 'sequence_recall', 'cued_catch_sigma', 'compiled'])
def test_float_rewards_are_pythons_in_order_sum(name, compiled_modules):
  from pycolab_b200 import _lib
  case = gp._lowered(name, tuple(compiled_modules))
  assert case.games[0].float_reward
  B, T = 11, 80
  eng = _engine(case.games, B, track_episodes=True)
  eng.its_showtime()
  rows = []

  def keep():
    rows.append((eng.reward.cpu().numpy().tolist(), eng.has_reward.cpu().numpy().tolist(),
                 eng.plot[:, _lib.P_FRAME].cpu().numpy().tolist(),
                 eng.episode_return.cpu().numpy()))
  keep()
  actions = gp._draw(case, np.random.RandomState(17), T, B, 0.02)
  for t in range(T):
    eng.play(gp._device_actions(actions[t]))
    keep()
  ret = [0.0] * B
  paid = False
  for reward, has, frame, got in rows:
    for e in range(B):
      r = reward[e] if has[e] else 0.0
      paid |= r != 0.0
      if frame[e] == 0:
        ret[e] = r
      else:
        ret[e] += r
    assert ref.same_bits(got, ret)
  assert paid, 'no reward was paid'
