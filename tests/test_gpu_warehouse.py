"""warehouse_step against the oracle at every box count, board shape, pitch, level binding
and batch it is launched with, and at the board's rim.

Every case runs through sampled_check.lockstep and compares, at every step, the board,
reward, discount and done, the record words of every box and of P, the 'X' curtain (the
host hook that rebuilds it from the boxes' AUX0 bits), the pitch padding, and each env's
latched error word.  The levels have floor up to the edge (warehouse_cases), so boxes and
P leave the board, and a push can raise: that env must latch ENV_ERR_INDEX at the step
the oracle raises, while the others keep a zero word and stay in lock-step.  Each case
asserts that it reached the edge it is there for."""

import numpy as np
import pytest

import rim_sweep as rsw
import warehouse_cases as wc

pytestmark = pytest.mark.gpu

T = 60
BOX_COUNTS = (1, 2, 7, 10)
# The largest tile pcl_create accepts: 4 * (512 + H * pitch) = 227 KB.
LARGEST = (240, 240)
SHAPES = [(8, 8), (8, 17), (33, 15), (31, 64), (64, 65), (80, 80), (96, 128), LARGEST]


def _cases():
  """Every shape at each pitch, the box counts, bindings and batches rotated across them
  so that each value of every axis meets several of the others.  The largest tile runs at
  its own pitch only, with 5 envs."""
  out = []
  for i, j, k, shape, pitch, binding, B in rsw.rotate(SHAPES):
    if shape == LARGEST:
      if j:
        continue
      B = 5
    boxes = wc.BOX_SETS[BOX_COUNTS[k % 4]]
    out.append(('%dx%d_p%d_%s_%db_B%d' % (shape + (pitch, binding, len(boxes), B)),
                shape, pitch - rsw.ceil16(shape[1]), boxes, binding, B))
  return out


CASES = _cases()


@pytest.mark.parametrize('name,shape,extra,boxes,binding,B', CASES, ids=[c[0] for c in CASES])
def test_warehouse_cases(name, shape, extra, boxes, binding, B):
  n, B = rsw.levels_and_batch(binding, B)
  seed = sum(shape) + extra + len(boxes)
  arts = [wc.open_level(seed + i, shape, boxes) for i in range(n)]
  pitch = rsw.ceil16(shape[1]) + extra
  games = [wc.lowered(a, pitch=pitch) for a in arts]
  actions = wc.random_actions(np.random.RandomState(seed), T, B)
  actions[T // 3, 0] = 5                     # env 0 restarts inside the run
  compared, raised, track = rsw.run(
      games, lambda e: wc.make_world(arts[e % n]), actions, curtains='X', sprites=boxes + 'P',
      make_edges=lambda: wc.Edges(boxes), share_levels=binding != rsw.PER_ENV)
  assert track.restarts > 0, name
  assert compared >= T, (name, compared, raised)


@pytest.mark.parametrize('name', sorted(wc.RIM))
@pytest.mark.parametrize('extra', [0, 64])
def test_warehouse_rim(name, extra):
  """The scripted rim cases, 6 envs of one level: env 0 plays the script, quits, and
  plays it again, and must reach every edge the case names; a raising script latches
  ENV_ERR_INDEX in env 0 at the oracle's step only, while env 1 plays it up to the
  raising action and then idles.  The others walk at random."""
  art, beneath, script, edges = wc.RIM[name]
  boxes = wc.rim_boxes(name)
  game = wc.lowered(art, beneath, pitch=rsw.ceil16(len(art[0])) + extra)
  actions = rsw.rim_actions(script, 5, 4, T, 6, wc.random_actions, len(name))
  if name in wc.RAISES:
    safe = script[:wc.RAISES[name]]
    actions[:, 1] = 4
    actions[:len(safe), 1] = safe
  _, raised, track = rsw.run([game], lambda e: wc.make_world(art, beneath), actions,
                             curtains='X', sprites=boxes + 'P',
                             make_edges=lambda: wc.Edges(boxes))
  if name in wc.RAISES:
    assert raised.get(0) == wc.RAISES[name] + 1, (name, raised)
    assert 1 not in raised
  else:
    assert 0 not in raised, (name, raised)
    assert edges <= track.seen(0), (name, sorted(edges - track.seen(0)))
    assert track.restarts > 0
  assert len(raised) < 6
