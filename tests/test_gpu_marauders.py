"""marauders_step against the oracle at every board shape, pitch, level binding and batch
it is launched with, and at the board's rim.

Every case runs through sampled_check.lockstep and compares, at every step, the board,
reward, discount and done, the record words of P and of every bolt, the 'B' and 'X'
curtains, the pitch padding, and each env's latched error word.  The levels put X, B and
P anywhere (marauders_cases), so marauders reverse at both sides and roll from the last
row to the first, bolts leave the board at both ends, and a down bolt can find no column
to fire from: that env must latch ENV_ERR_EMPTY_CHOICE at the step where the oracle
raises ValueError, while the others keep a zero word and stay in lock-step.  A pitch past
64 columns puts segments of pad columns past the 64-bit curtain rows, which must come out
0; past 512 columns a warp's 32 lanes cover less than one row per round of the render.
Each case asserts that it reached the edge it is there for."""

import numpy as np
import pytest

import marauders_cases as mc
from oracle import sampled_check

pytestmark = pytest.mark.gpu

T = 60
SHARED, POOL, PER_ENV = 'shared', 'pool', 'per_env'
BINDINGS = (SHARED, POOL, PER_ENV)
BATCHES = (1, 5, 37)
# Pitch 1024 on 12 rows stages exactly 48 KB of tiles per block: with the 1,536 bytes of
# static records, past what a block gets without opting in.
PITCHES = ('+0', '+16', '+64', 544, 1024)
# The widest pitches pcl_create accepts: 4 * 32 * 1792 + 1536 and 4 * 11 * 5248 + 1536
# bytes of shared memory per block, the second exactly 227 KB.
WIDEST = [((32, 64), 1792), ((11, 64), 5248)]


def _pitch(shape, p):
  return mc.ceil16(shape[1]) + int(p[1:]) if isinstance(p, str) else p


def _cases():
  """Every shape at each pitch, bindings and batches rotated across them so that each
  value of every axis meets several of the others; the widest pitches with 5 envs."""
  out = []
  for i, shape in enumerate(mc.SHAPES):
    for j, p in enumerate(PITCHES):
      k = len(PITCHES) * i + j
      binding = BINDINGS[(i + 2 * j) % 3]
      B = BATCHES[(k // 2) % 3]
      out.append((shape, _pitch(shape, p), binding, B))
  out += [(shape, pitch, BINDINGS[i], 5) for i, (shape, pitch) in enumerate(WIDEST)]
  return [('%dx%d_p%d_%s_B%d' % (c[0] + c[1:]),) + c for c in out]


CASES = _cases()


class _Track(object):
  """on_step hook: the edges each sampled env's oracle world went through, and the
  number of restarts."""

  def __init__(self, raised, actions):
    self.raised, self.actions = raised, actions
    self.edges, self.worlds, self.restarts = {}, {}, 0

  def __call__(self, t, engine, worlds, outs):
    for e, w in worlds.items():
      if e in self.raised:
        continue
      if self.worlds.get(e) is not w:
        self.edges.setdefault(e, mc.Edges()).start(w, outs[e])
        self.restarts += t > 0
      else:
        self.edges[e].step(w, outs[e], int(self.actions[t - 1, e]))
      self.worlds[e] = w

  def seen(self, e=None):
    if e is not None:
      return self.edges[e].seen if e in self.edges else set()
    return set().union(*(x.seen for x in self.edges.values()))


def _run(games, arts, actions, share_levels=True, rng_seed=0):
  """Env e plays games[e % len(games)] and draws from RandomState(rng_seed + e) across
  its episodes, on the device and in its oracle world."""
  from pycolab_b200 import batched
  B = actions.shape[1]
  eng = batched.BatchedEngine(games, batch=B, share_levels=share_levels, rng_seed=rng_seed)
  eng.its_showtime()
  rngs = [np.random.RandomState(rng_seed + e) for e in range(B)]
  raised = {}
  track = _Track(raised, actions)
  compared = sampled_check.lockstep(
      eng, lambda e: mc.make_world(arts[e % len(arts)], rngs[e]), range(B), actions,
      curtains='BX', sprites='Pabcdyz', pad_columns=True, on_step=track, raised=raised)
  return compared, raised, track


@pytest.mark.parametrize('name,shape,pitch,binding,B', CASES, ids=[c[0] for c in CASES])
def test_marauders_cases(name, shape, pitch, binding, B):
  """Random play with quits on open levels, env 0 quitting a third of the way in: the
  marauders reverse and the episodes restart.  An env may raise where its oracle does."""
  n = 1 if binding == SHARED else 3 if binding == POOL else 2
  if binding == POOL:
    B = max(B, 5)
  seed = sum(shape) + pitch
  arts = [mc.sweep_level(shape, s) for s in range(n)]
  games = [mc.lowered(a, pitch=pitch) for a in arts]
  actions = mc.random_actions(np.random.RandomState(seed), T, B)
  actions[T // 3, 0] = 4                     # env 0 restarts inside the run
  compared, raised, track = _run(games, arts, actions, share_levels=binding != PER_ENV,
                                 rng_seed=seed)
  assert track.restarts > 0, name
  assert 'reverse' in track.seen(), (name, sorted(track.seen()))
  assert compared >= T * B // 2, (name, compared, raised)


def _rim_actions(name, B):
  """Env 0 plays the script, quits, and plays it again; the others play at random."""
  script = mc.RIM[name][1]
  actions = mc.random_actions(np.random.RandomState(len(name)), T, B)
  first = script + [4] + script
  actions[:, 0] = 3
  actions[:len(first), 0] = first
  return actions


STEADY = sorted(name for name in mc.RIM if name not in mc.RAISES)


@pytest.mark.parametrize('name', STEADY)
@pytest.mark.parametrize('extra', [0, 64])
def test_marauders_rim(name, extra):
  """The scripted rim cases, 6 envs of one level: env 0 (drawing from RandomState(0), as
  the script was found with) must reach every edge the case names, and restart."""
  art, _, edges = mc.RIM[name]
  game = mc.lowered(art, pitch=mc.ceil16(len(art[0])) + extra)
  actions = _rim_actions(name, 6)
  _, raised, track = _run([game], [art], actions)
  assert 0 not in raised, (name, raised)
  assert edges <= track.seen(0), (name, sorted(edges - track.seen(0)))
  assert track.restarts > 0


@pytest.mark.parametrize('name', sorted(mc.RAISES))
@pytest.mark.parametrize('extra', [0, 64])
def test_marauders_rim_raises(name, extra):
  """A raising level in a pool with a steady one of its shape, 6 envs: env 0 plays the
  raising script and latches ENV_ERR_EMPTY_CHOICE at the action that raises; the other
  envs latch it where their oracle raises, and every other env keeps a zero word."""
  art = mc.RIM[name][0]
  steady = mc.open_level(1, (len(art), len(art[0])), 2, x_rows=range(5))
  pitch = mc.ceil16(len(art[0])) + extra
  games = [mc.lowered(art, pitch=pitch), mc.lowered(steady, pitch=pitch)]
  actions = _rim_actions(name, 6)
  _, raised, _ = _run(games, [art, steady], actions)
  assert raised.get(0) == mc.RAISES[name] + 1, raised
  assert len(raised) < 6, raised


@pytest.mark.parametrize('shape', [(32, 64), (32, 39), (16, 64), (20, 63)])
def test_marauders_stock_layout_board_shapes(shape):
  """The stock layout generated up to 32 x 64: the W == 64 mask, wraps by W - 1 and the
  row roll over all 32 lanes."""
  from pycolab_b200 import levels
  art = levels.marauders_level(*shape)
  actions = np.random.RandomState(sum(shape)).randint(0, 4, size=(150, 10)).astype(np.int32)
  _, raised, track = _run([mc.lowered(art)], [art], actions, rng_seed=900)
  assert not raised, raised
  assert 'reverse' in track.seen()


def test_single_env_engine_raises_at_the_same_play():
  """The facade Engine on the 12 x 1 level raises ValueError at the first play(), as the
  oracle does."""
  from pycolab_b200.games import extraterrestrial_marauders as marauders
  art = mc.RIM['raise_hidden'][0]
  world = mc.make_world(art, np.random.RandomState(5))
  world.its_showtime()
  with pytest.raises(ValueError):
    world.play(3)
  np.random.seed(5)
  eng = marauders.make_game(art)
  eng.its_showtime()
  with pytest.raises(ValueError):
    eng.play(3)
