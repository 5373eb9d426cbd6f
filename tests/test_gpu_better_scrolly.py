"""better_scrolly_step against the oracle at every board shape, pitch, level binding and
batch it is launched with, and at the board's rim.

Every case runs through sampled_check.lockstep and compares, at every step, the board,
reward, discount and done, the record words of P and of every patroller, the '@'
curtain, the pitch padding, and each env's latched error word.  The levels have floor up
to the edge (better_scrolly_cases), so P and the patrollers leave the board, and a
patroller's look-up can raise: that env must latch ENV_ERR_INDEX at the step, or at the
reset launch, where the oracle raises, while the others keep a zero word and stay in
lock-step.  The widened pitches put segments of pad columns past the coin bit rows, which
must come out 0.  Each case asserts that it reached the edge it is there for."""

import numpy as np
import pytest

import better_scrolly_cases as bc
import rim_sweep as rsw

pytestmark = pytest.mark.gpu

T = 60
COINS = (0, 1, 6, 40)
# The largest board pcl_create accepts at its own pitch: 4 * (256 + H*pitch + H*BW*4)
# is exactly 227 KB.  96 x 128 is past the 48 KB a block gets without opting in.
LARGEST = (226, 224)
SHAPES = [(2, 4), (1, 16), (5, 17), (29, 30), (33, 64), (45, 89), (64, 65), (96, 128), LARGEST]
# What every run compares, and the edges it tracks.
LOCKSTEP = dict(curtains='@', sprites='Pabc', make_edges=bc.Edges)


def _cases():
  """Every shape at each pitch, the coin counts, bindings and batches rotated across
  them so that each value of every axis meets several of the others.  The largest board
  runs at its own pitch only, with 5 envs."""
  out = []
  for i, j, k, shape, pitch, binding, B in rsw.rotate(SHAPES):
    if shape == LARGEST:
      if j:
        continue
      B = 5
    coins = min(COINS[k % 4], shape[0] * shape[1] - 5)
    out.append(('%dx%d_p%d_%s_%dc_B%d' % (shape + (pitch, binding, coins, B)),
                shape, pitch - rsw.ceil16(shape[1]), coins, binding, B))
  return out


CASES = _cases()


@pytest.mark.parametrize('name,shape,extra,coins,binding,B', CASES, ids=[c[0] for c in CASES])
def test_better_scrolly_cases(name, shape, extra, coins, binding, B):
  """Random play with quits on fenced open levels (no patroller can reach the last
  column), env 0 quitting a third of the way in: P leaves the board and the episodes
  restart, and no env raises."""
  n, B = rsw.levels_and_batch(binding, B)
  seed = sum(shape) + extra + coins
  arts = [bc.open_level(seed + i, shape, coins) for i in range(n)]
  pitch = rsw.ceil16(shape[1]) + extra
  games = [bc.lowered(a, pitch=pitch) for a in arts]
  actions = bc.random_actions(np.random.RandomState(seed), T, B)
  actions[T // 3, 0] = 5                     # env 0 restarts inside the run
  compared, raised, track = rsw.run(games, lambda e: bc.make_world(arts[e % n]), actions,
                                    share_levels=binding != rsw.PER_ENV, **LOCKSTEP)
  assert not raised, (name, raised)
  assert track.restarts > 0, name
  assert compared >= T * B, (name, compared)
  if shape[0] * shape[1] <= 64:
    assert any(s.startswith('player_off') for s in track.seen()), (name, track.seen())


STEADY = sorted(name for name in bc.RIM if name not in bc.RAISES)


@pytest.mark.parametrize('name', STEADY)
@pytest.mark.parametrize('extra', [0, 64])
def test_better_scrolly_rim(name, extra):
  """The scripted rim cases, 6 envs of one level: env 0 plays the script, quits, and
  plays it again, and must reach every edge the case names, and restart; the others walk
  at random.  No env raises."""
  art, script, edges = bc.RIM[name]
  game = bc.lowered(art, pitch=rsw.ceil16(len(art[0])) + extra)
  actions = rsw.rim_actions(script, 5, 4, T, 6, bc.random_actions, len(name))
  _, raised, track = rsw.run([game], lambda e: bc.make_world(art), actions, **LOCKSTEP)
  assert not raised, (name, raised)
  assert edges <= track.seen(0), (name, sorted(edges - track.seen(0)))
  assert track.restarts > 0


@pytest.mark.parametrize('extra', [0, 64])
def test_better_scrolly_rim_raises(extra):
  """A pool of the two raising levels, 6 envs: the odd envs' patroller starts in the
  last column and latches ENV_ERR_INDEX at the first launch, its_showtime; env 0 plays
  the raising script and latches it at the action that raises, as the even envs do
  where their oracle raises.  Every other env keeps a zero word."""
  (mid, script, _), show = bc.RIM['raise_mid_run'], bc.RIM['raise_at_showtime'][0]
  assert len(mid) == len(show) and len(mid[0]) == len(show[0])
  pitch = rsw.ceil16(len(mid[0])) + extra
  games = [bc.lowered(mid, pitch=pitch), bc.lowered(show, pitch=pitch)]
  actions = rsw.rim_actions(script, 5, 4, T, 6, bc.random_actions, len('raise_mid_run'))
  _, raised, _ = rsw.run(games, lambda e: bc.make_world((mid, show)[e % 2]), actions,
                         **LOCKSTEP)
  assert raised.get(0) == bc.RAISES['raise_mid_run'] + 1, raised
  assert all(raised.get(e) == 0 for e in (1, 3, 5)), raised
  assert all(raised.get(e, 0) > 0 for e in (2, 4)), raised
