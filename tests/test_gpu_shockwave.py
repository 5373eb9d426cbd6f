"""shockwave_step against the oracle at every board shape, pitch, ring width, level
binding and batch it is launched with, and at the board's rim.

Every case runs through sampled_check.lockstep and compares, at every step, the board,
reward, discount and done, P's record words, the '@' curtain, the pitch padding, and each
env's error word (which must stay 0).  The levels put '^', ' ', '+' and '=' anywhere
(shockwave_cases), and env 0's generator seed puts its first impact on a corner or a side
of the board, so the ring is clipped there.  A pitch past 64 columns puts segments of pad
columns past the 64-bit curtain rows, which must come out 0.  Each case asserts that it
reached the edge it is there for."""

import numpy as np
import pytest

import rim_sweep as rsw
import shockwave_cases as sc
from oracle import games as ogames

pytestmark = pytest.mark.gpu

T = 60
# A pitch of 4096 on the largest board: shockwave stages nothing in shared memory.
WIDEST = ((32, 64), 4096)
# What every run compares, and the edges it tracks.
LOCKSTEP = dict(curtains='@', sprites='P', make_edges=sc.Edges)


def _cases():
  """Every shape at pitch ceil16(W) + 0, 16 and 64, widths, bindings, batches and the
  first impact's cell rotated across them; the widest pitch with 5 envs."""
  out = [(shape, pitch, sc.WIDTHS[k % len(sc.WIDTHS)], binding, B, k)
         for _, _, k, shape, pitch, binding, B in rsw.rotate(sc.SHAPES)]
  out.append(WIDEST + (2, rsw.POOL, 5, 0))
  return [('%dx%d_p%d_w%d_%s_B%d' % (c[0] + c[1:5]),) + c for c in out]


CASES = _cases()


@pytest.mark.parametrize('name,shape,pitch,width,binding,B,k', CASES,
                         ids=[c[0] for c in CASES])
def test_shockwave_cases(name, shape, pitch, width, binding, B, k):
  """Random play on open levels; env 0's first impact on a corner or side of the board,
  whose ring is clipped there.  A pool's levels differ in their '^' and ' ' cells."""
  n, B = rsw.levels_and_batch(binding, B)
  arts = [sc.sweep_level(shape, k + i) for i in range(n)]
  games = [sc.lowered(a, width, pitch=pitch) for a in arts]
  cells = sc.rim_cells(shape)
  seed = sc.impact_seed(shape, cells[k % len(cells)])
  actions = sc.random_actions(np.random.RandomState(k), T, B)
  compared, raised, track = rsw.run(
      games, lambda e, rng: sc.make_world(arts[e % n], rng, width), actions,
      share_levels=binding != rsw.PER_ENV, rng_seed=seed, **LOCKSTEP)
  assert not raised, raised
  assert compared == (T + 1) * B
  first = track.edges[0]
  if width > 0 and shape[0] * shape[1] > 2:   # else P and a wall fill the board
    assert {'clip_n', 'clip_s', 'clip_w', 'clip_e'} & first.seen, (name, sorted(first.seen))
  if width == 0:
    assert 'redraw' in track.seen(), name


@pytest.mark.parametrize('name', sorted(sc.RIM))
@pytest.mark.parametrize('extra', [0, 64])
def test_shockwave_rim(name, extra):
  """The scripted rim cases, 6 envs of one level: env 0 plays the script with the seed
  it was found with and must reach every edge the case names; the others play at
  random."""
  art, width, seed, script, edges = sc.RIM[name]
  game = sc.lowered(art, width, pitch=rsw.ceil16(len(art[0])) + extra)
  actions = sc.random_actions(np.random.RandomState(len(name)), T, 6)
  actions[:len(script), 0] = script
  _, raised, track = rsw.run([game], lambda e, rng: sc.make_world(art, rng, width), actions,
                             rng_seed=seed, **LOCKSTEP)
  assert not raised, raised
  assert edges <= track.seen(0), (name, sorted(edges - track.seen(0)))


@pytest.mark.parametrize('shape', [(32, 64), (31, 33), (32, 15), (20, 63)])
def test_shockwave_generated_levels(shape):
  """One generated level (a '^' row on top, P on the bottom row) up to 32 x 64 (H * W =
  2048, a power of two) over an auto-resetting batch of 10."""
  from pycolab_b200 import levels
  rows, cols = shape
  art = levels.shockwave_level(rows + cols, rows, cols, 0.5)
  actions = np.random.RandomState(rows * cols).choice(
      5, size=(150, 10), p=[.55, .15, .15, .1, .05]).astype(np.int32)
  _, raised, track = rsw.run([sc.lowered(art)], lambda e, rng: ogames.make_shockwave(art, rng),
                             actions, rng_seed=700, **LOCKSTEP)
  assert not raised, raised
  assert track.restarts > 0


@pytest.mark.parametrize('shape', [(12, 15), (32, 64), (9, 33), (16, 48)])
def test_shockwave_generated_level_pools(shape):
  """A pool of three generated levels over an auto-resetting batch of 13, one generator
  per env: more episodes end than there are envs."""
  from pycolab_b200 import levels
  arts = [levels.shockwave_level(30 + i, shape[0], shape[1], 0.45) for i in range(3)]
  B, T = 13, 220
  rs = np.random.RandomState(4)
  actions = np.stack([rs.choice([0, 1, 2, 3, 4], size=B, p=[.6, .12, .12, .12, .04])
                      for _ in range(T)]).astype(np.int32)
  _, raised, track = rsw.run([sc.lowered(a) for a in arts],
                             lambda e, rng: ogames.make_shockwave(arts[e % 3], rng), actions,
                             rng_seed=9, **LOCKSTEP)
  assert not raised, raised
  assert track.restarts > B
