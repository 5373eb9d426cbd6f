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
import rim_sweep as rsw

pytestmark = pytest.mark.gpu

T = 60
# Pitch 1024 on 12 rows stages exactly 48 KB of tiles per block: with the 1,536 bytes of
# static records, past what a block gets without opting in.
PITCHES = ('+0', '+16', '+64', 544, 1024)
# The widest pitches pcl_create accepts: 4 * 32 * 1792 + 1536 and 4 * 11 * 5248 + 1536
# bytes of shared memory per block, the second exactly 227 KB.
WIDEST = [((32, 64), 1792), ((11, 64), 5248)]
# What every run compares, and the edges it tracks.
LOCKSTEP = dict(curtains='BX', sprites='Pabcdyz', make_edges=mc.Edges)


def _cases():
  """Every shape at each pitch, bindings and batches rotated across them so that each
  value of every axis meets several of the others; the widest pitches with 5 envs."""
  out = [(shape, pitch, binding, B)
         for _, _, _, shape, pitch, binding, B in rsw.rotate(mc.SHAPES, PITCHES)]
  out += [(shape, pitch, rsw.BINDINGS[i], 5) for i, (shape, pitch) in enumerate(WIDEST)]
  return [('%dx%d_p%d_%s_B%d' % (c[0] + c[1:]),) + c for c in out]


CASES = _cases()


@pytest.mark.parametrize('name,shape,pitch,binding,B', CASES, ids=[c[0] for c in CASES])
def test_marauders_cases(name, shape, pitch, binding, B):
  """Random play with quits on open levels, env 0 quitting a third of the way in: the
  marauders reverse and the episodes restart.  An env may raise where its oracle does."""
  n, B = rsw.levels_and_batch(binding, B)
  seed = sum(shape) + pitch
  arts = [mc.sweep_level(shape, s) for s in range(n)]
  games = [mc.lowered(a, pitch=pitch) for a in arts]
  actions = mc.random_actions(np.random.RandomState(seed), T, B)
  actions[T // 3, 0] = 4                     # env 0 restarts inside the run
  compared, raised, track = rsw.run(
      games, lambda e, rng: mc.make_world(arts[e % n], rng), actions,
      share_levels=binding != rsw.PER_ENV, rng_seed=seed, **LOCKSTEP)
  assert track.restarts > 0, name
  assert 'reverse' in track.seen(), (name, sorted(track.seen()))
  assert compared >= T * B // 2, (name, compared, raised)


STEADY = sorted(name for name in mc.RIM if name not in mc.RAISES)


@pytest.mark.parametrize('name', STEADY)
@pytest.mark.parametrize('extra', [0, 64])
def test_marauders_rim(name, extra):
  """The scripted rim cases, 6 envs of one level: env 0 (drawing from RandomState(0), as
  the script was found with) plays the script, quits, and plays it again, and must reach
  every edge the case names, and restart; the others play at random."""
  art, script, edges = mc.RIM[name]
  game = mc.lowered(art, pitch=rsw.ceil16(len(art[0])) + extra)
  actions = rsw.rim_actions(script, 4, 3, T, 6, mc.random_actions, len(name))
  _, raised, track = rsw.run([game], lambda e, rng: mc.make_world(art, rng), actions,
                             rng_seed=0, **LOCKSTEP)
  assert 0 not in raised, (name, raised)
  assert edges <= track.seen(0), (name, sorted(edges - track.seen(0)))
  assert track.restarts > 0


@pytest.mark.parametrize('name', sorted(mc.RAISES))
@pytest.mark.parametrize('extra', [0, 64])
def test_marauders_rim_raises(name, extra):
  """A raising level in a pool with a steady one of its shape, 6 envs: env 0 plays the
  raising script and latches ENV_ERR_EMPTY_CHOICE at the action that raises; the other
  envs latch it where their oracle raises, and every other env keeps a zero word."""
  art, script, _ = mc.RIM[name]
  steady = mc.open_level(1, (len(art), len(art[0])), 2, x_rows=range(5))
  pitch = rsw.ceil16(len(art[0])) + extra
  games = [mc.lowered(art, pitch=pitch), mc.lowered(steady, pitch=pitch)]
  actions = rsw.rim_actions(script, 4, 3, T, 6, mc.random_actions, len(name))
  _, raised, _ = rsw.run(games, lambda e, rng: mc.make_world((art, steady)[e % 2], rng),
                         actions, rng_seed=0, **LOCKSTEP)
  assert raised.get(0) == mc.RAISES[name] + 1, raised
  assert len(raised) < 6, raised


@pytest.mark.parametrize('shape', [(32, 64), (32, 39), (16, 64), (20, 63)])
def test_marauders_stock_layout_board_shapes(shape):
  """The stock layout generated up to 32 x 64: the W == 64 mask, wraps by W - 1 and the
  row roll over all 32 lanes."""
  from pycolab_b200 import levels
  art = levels.marauders_level(*shape)
  actions = np.random.RandomState(sum(shape)).randint(0, 4, size=(150, 10)).astype(np.int32)
  _, raised, track = rsw.run([mc.lowered(art)], lambda e, rng: mc.make_world(art, rng),
                             actions, rng_seed=900, **LOCKSTEP)
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
