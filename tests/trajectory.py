"""Shared trajectory protocol for golden fixtures and parity tests.

An "env" is anything with `its_showtime()`, `play(action)` and `game_over`
(a reference Engine, an oracle World, the device facade Engine).  The protocol is
the batched engine's auto-reset rule: an env that reported game over is rebuilt
at the NEXT step (that step's action is ignored) and returns its
`its_showtime()` outputs.
"""

import numpy as np

# The arrays of every trajectory, as run_trajectory returns them.
TRAJECTORY = ('boards', 'reward', 'has_reward', 'discount', 'game_over')


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


def reward_type(reward):
  """A golden's `reward_type`: 0 for no reward, 1 for an int, 2 for a float."""
  return 0 if reward is None else (2 if isinstance(reward, float) else 1)


def sprite_rows(env, chars):
  """A golden's `sprites` row of an Engine with the pycolab API: (row, col, visible,
  virtual row, virtual col) of each sprite of `chars`.  A plain Sprite has no virtual
  position: its position stands in."""
  rows = []
  for s in (env.things[ch] for ch in chars):
    vp = getattr(s, 'virtual_position', s.position)
    rows.append([int(s.position[0]), int(s.position[1]), int(bool(s.visible)),
                 int(vp[0]), int(vp[1])])
  return rows


def world_sprite_rows(world, chars, plain=''):
  """sprite_rows() of an oracle world.  A plain sprite (oracle.games.PlainSprite) has no
  vrow and vcol, and a compiled plain Sprite, one of `plain`, holds registers there: the
  position stands in for both."""
  rows = []
  for ch in chars:
    w = world.things[ch]
    v = (w.row, w.col) if ch in plain or not hasattr(w, 'vrow') else (w.vrow, w.vcol)
    rows.append([w.row, w.col, int(bool(w.visible)), v[0], v[1]])
  return rows


def assert_golden_arrays(name, g, got, inputs):
  """Every array golden `name`'s `g` holds apart from its `inputs` equals `got`'s, dtype
  and shape included, floats bit for bit.  A key `got` lacks fails, and is named."""
  keys = sorted(set(g) - set(inputs))
  missing = [key for key in keys if key not in got]
  assert not missing, '%s: the replay recorded no %s' % (name, ', '.join(missing))
  for key in keys:
    msg = '%s: %s' % (name, key)
    np.testing.assert_array_equal(got[key], g[key], err_msg=msg, strict=True)
    if g[key].dtype.kind == 'f':
      assert got[key].tobytes() == g[key].tobytes(), msg + ': float bits differ'


def art_to_u8(art):
  return np.vstack([np.frombuffer(l.encode('ascii'), dtype=np.uint8) for l in art])


def u8_to_art(arr):
  return [bytes(row).decode('ascii') for row in np.asarray(arr, dtype=np.uint8)]


def assert_same_trajectory(want, got, label=''):
  for key in TRAJECTORY:
    w, g = np.asarray(want[key]), np.asarray(got[key])
    assert w.shape == g.shape, (label, key, w.shape, g.shape)
    if not np.array_equal(w, g):
      bad = np.argwhere(w != g)[0]
      raise AssertionError('%s: %s differs first at %s: want %r got %r' % (
          label, key, tuple(bad), w[tuple(bad)], g[tuple(bad)]))
