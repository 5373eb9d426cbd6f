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

import shockwave_cases as sc
from oracle import games as ogames
from oracle import sampled_check

pytestmark = pytest.mark.gpu

T = 60
SHARED, POOL, PER_ENV = 'shared', 'pool', 'per_env'
BINDINGS = (SHARED, POOL, PER_ENV)
BATCHES = (1, 5, 37)
# A pitch of 4096 on the largest board: shockwave stages nothing in shared memory.
WIDEST = ((32, 64), 4096)


def _cases():
  """Every shape at pitch ceil16(W) + 0, 16 and 64, widths, bindings, batches and the
  first impact's cell rotated across them; the widest pitch with 5 envs."""
  out = []
  for i, shape in enumerate(sc.SHAPES):
    for j, extra in enumerate((0, 16, 64)):
      k = 3 * i + j
      out.append((shape, sc.ceil16(shape[1]) + extra, sc.WIDTHS[k % len(sc.WIDTHS)],
                  BINDINGS[(i + 2 * j) % 3], BATCHES[(k // 2) % 3], k))
  out.append(WIDEST + (2, POOL, 5, 0))
  return [('%dx%d_p%d_w%d_%s_B%d' % (c[0] + c[1:5]),) + c for c in out]


CASES = _cases()


class _Track(object):
  """on_step hook: the edges each sampled env's oracle world went through, and the
  number of restarts."""

  def __init__(self, actions):
    self.actions = actions
    self.edges, self.worlds, self.restarts = {}, {}, 0

  def __call__(self, t, engine, worlds, outs):
    for e, w in worlds.items():
      if self.worlds.get(e) is not w:
        self.edges.setdefault(e, sc.Edges()).start(w, outs[e])
        self.restarts += t > 0
      else:
        self.edges[e].step(w, outs[e], int(self.actions[t - 1, e]))
      self.worlds[e] = w

  def seen(self, e=None):
    if e is not None:
      return self.edges[e].seen if e in self.edges else set()
    return set().union(*(x.seen for x in self.edges.values()))


def _run(games, make_world, actions, share_levels=True, rng_seed=0):
  """Env e draws from RandomState(rng_seed + e) across its episodes, on the device and
  in its oracle world make_world(e, rng)."""
  from pycolab_b200 import batched
  B = actions.shape[1]
  eng = batched.BatchedEngine(games, batch=B, share_levels=share_levels, rng_seed=rng_seed)
  eng.its_showtime()
  rngs = [np.random.RandomState(rng_seed + e) for e in range(B)]
  raised = {}
  track = _Track(actions)
  compared = sampled_check.lockstep(eng, lambda e: make_world(e, rngs[e]), range(B), actions,
                                    curtains='@', sprites='P', pad_columns=True,
                                    on_step=track, raised=raised)
  assert not raised, raised
  return compared, track


@pytest.mark.parametrize('name,shape,pitch,width,binding,B,k', CASES,
                         ids=[c[0] for c in CASES])
def test_shockwave_cases(name, shape, pitch, width, binding, B, k):
  """Random play on open levels; env 0's first impact on a corner or side of the board,
  whose ring is clipped there.  A pool's levels differ in their '^' and ' ' cells."""
  n = 1 if binding == SHARED else 3 if binding == POOL else 2
  if binding == POOL:
    B = max(B, 5)
  arts = [sc.sweep_level(shape, k + i) for i in range(n)]
  games = [sc.lowered(a, width, pitch=pitch) for a in arts]
  cells = sc.rim_cells(shape)
  seed = sc.impact_seed(shape, cells[k % len(cells)])
  actions = sc.random_actions(np.random.RandomState(k), T, B)
  compared, track = _run(games, lambda e, rng: sc.make_world(arts[e % n], rng, width),
                         actions, share_levels=binding != PER_ENV, rng_seed=seed)
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
  game = sc.lowered(art, width, pitch=sc.ceil16(len(art[0])) + extra)
  actions = sc.random_actions(np.random.RandomState(len(name)), T, 6)
  actions[:len(script), 0] = script
  _, track = _run([game], lambda e, rng: sc.make_world(art, rng, width), actions,
                  rng_seed=seed)
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
  _, track = _run([sc.lowered(art)], lambda e, rng: ogames.make_shockwave(art, rng), actions,
                  rng_seed=700)
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
  _, track = _run([sc.lowered(a) for a in arts],
                  lambda e, rng: ogames.make_shockwave(arts[e % 3], rng), actions, rng_seed=9)
  assert track.restarts > B
