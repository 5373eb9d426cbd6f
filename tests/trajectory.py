"""Shared trajectory protocol for golden fixtures and parity tests.

An "env" is anything with `its_showtime()`, `play(action)` and `game_over`
(a reference Engine, an oracle World, the device facade Engine).  The protocol is
the batched engine's auto-reset rule: an env that reported game over is rebuilt
at the NEXT step (that step's action is ignored) and returns its
`its_showtime()` outputs.
"""

import numpy as np


def board_of(obs):
  return np.asarray(obs.board if hasattr(obs, 'board') else obs, dtype=np.uint8)


class _Frames(object):
  """The frames of one trajectory, recorded at once: the reference renders into one
  buffer."""

  def __init__(self, on_frame):
    self.on_frame = on_frame
    self.boards, self.reward, self.has_reward, self.discount, self.over = [], [], [], [], []

  def record(self, env, out):
    self.boards.append(board_of(out[0]).copy())
    self.reward.append(0 if out[1] is None else int(out[1]))
    self.has_reward.append(0 if out[1] is None else 1)
    self.discount.append(float(out[2]))
    self.over.append(1 if env.game_over else 0)
    if self.on_frame is not None:
      self.on_frame(env, out)

  def arrays(self):
    return dict(boards=np.stack(self.boards), reward=np.array(self.reward, dtype=np.int64),
                has_reward=np.array(self.has_reward, dtype=np.uint8),
                discount=np.array(self.discount, dtype=np.float64),
                game_over=np.array(self.over, dtype=np.uint8))


def run_trajectory(make_env, actions, convert_action=None, on_frame=None):
  """Returns dict(boards[T+1,H,W] u8, reward[T+1] i64, has_reward[T+1] u8,
  discount[T+1] f64, game_over[T+1] u8)."""
  frames = _Frames(on_frame)
  env = make_env()
  frames.record(env, env.its_showtime())
  for a in actions:
    if env.game_over:
      env = make_env()
      out = env.its_showtime()
    else:
      out = env.play(convert_action(a) if convert_action else a)
    frames.record(env, out)
  return frames.arrays()


def run_until_raise(make_env, actions, exception, on_frame=None):
  """One episode, without auto-reset, played until play() raises `exception`.  Returns
  (the trajectory of the frames before it, as run_trajectory's, and the index of the action
  that raised)."""
  frames = _Frames(on_frame)
  env = make_env()
  frames.record(env, env.its_showtime())
  for t, a in enumerate(actions):
    try:
      out = env.play(a)
    except exception:
      return frames.arrays(), t
    frames.record(env, out)
  raise AssertionError('play() never raised %s' % exception.__name__)


def art_to_u8(art):
  return np.vstack([np.frombuffer(l.encode('ascii'), dtype=np.uint8) for l in art])


def u8_to_art(arr):
  return [bytes(row).decode('ascii') for row in np.asarray(arr, dtype=np.uint8)]


def assert_same_trajectory(want, got, label=''):
  for key in ('boards', 'reward', 'has_reward', 'discount', 'game_over'):
    w, g = np.asarray(want[key]), np.asarray(got[key])
    assert w.shape == g.shape, (label, key, w.shape, g.shape)
    if not np.array_equal(w, g):
      bad = np.argwhere(w != g)[0]
      raise AssertionError('%s: %s differs first at %s: want %r got %r' % (
          label, key, tuple(bad), w[tuple(bad)], g[tuple(bad)]))
