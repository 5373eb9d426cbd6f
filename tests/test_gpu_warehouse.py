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

import warehouse_cases as wc
from oracle import sampled_check

pytestmark = pytest.mark.gpu

T = 60
SHARED, POOL, PER_ENV = 'shared', 'pool', 'per_env'
BOX_COUNTS = (1, 2, 7, 10)
BINDINGS = (SHARED, POOL, PER_ENV)
BATCHES = (1, 5, 37)
# The largest tile pcl_create accepts: 4 * (512 + H * pitch) = 227 KB.
LARGEST = (240, 240)
SHAPES = [(8, 8), (8, 17), (33, 15), (31, 64), (64, 65), (80, 80), (96, 128), LARGEST]


def _cases():
  """Every shape at each pitch, the box counts, bindings and batches rotated across them
  so that each value of every axis meets several of the others.  The largest tile runs at
  its own pitch only, with 5 envs."""
  out = []
  for i, shape in enumerate(SHAPES):
    extras = (0,) if shape == LARGEST else (0, 16, 64)
    for j, extra in enumerate(extras):
      k = 3 * i + j
      boxes = wc.BOX_SETS[BOX_COUNTS[k % 4]]
      binding = BINDINGS[(i + 2 * j) % 3]
      B = 5 if shape == LARGEST else BATCHES[(k // 2) % 3]
      out.append(('%dx%d_p%d_%s_%db_B%d' % (shape + (wc.ceil16(shape[1]) + extra, binding,
                                                      len(boxes), B)),
                  shape, extra, boxes, binding, B))
  return out


CASES = _cases()


class _Track(object):
  """on_step hook: the edges each sampled env's oracle world went through, and the
  number of restarts."""

  def __init__(self, actions, boxes, raised):
    self.actions, self.boxes, self.raised = actions, boxes, raised
    self.edges, self.worlds, self.restarts = {}, {}, 0

  def __call__(self, t, engine, worlds, outs):
    for e, w in worlds.items():
      if e in self.raised:
        continue
      if self.worlds.get(e) is not w:
        self.edges.setdefault(e, wc.Edges(self.boxes)).start(w)
        self.restarts += t > 0
      else:
        self.edges[e].step(w, int(self.actions[t - 1, e]))
      self.worlds[e] = w

  def seen(self, e=None):
    if e is not None:
      return self.edges[e].seen
    return set().union(*(x.seen for x in self.edges.values()))


def _run(games, make_world, actions, boxes, share_levels=True):
  from pycolab_b200 import batched
  B = actions.shape[1]
  eng = batched.BatchedEngine(games, batch=B, share_levels=share_levels)
  eng.its_showtime()
  raised = {}
  track = _Track(actions, boxes, raised)
  compared = sampled_check.lockstep(eng, make_world, range(B), actions, curtains='X',
                                    sprites=boxes + 'P', pad_columns=True, on_step=track,
                                    raised=raised)
  return compared, raised, track


@pytest.mark.parametrize('name,shape,extra,boxes,binding,B', CASES, ids=[c[0] for c in CASES])
def test_warehouse_cases(name, shape, extra, boxes, binding, B):
  n = 1 if binding == SHARED else 3 if binding == POOL else 2
  if binding == POOL:
    B = max(B, 5)
  seed = sum(shape) + extra + len(boxes)
  arts = [wc.open_level(seed + i, shape, boxes) for i in range(n)]
  pitch = wc.ceil16(shape[1]) + extra
  games = [wc.lowered(a, pitch=pitch) for a in arts]
  actions = wc.random_actions(np.random.RandomState(seed), T, B)
  actions[T // 3, 0] = 5                     # env 0 restarts inside the run
  compared, raised, track = _run(games, lambda e: wc.make_world(arts[e % n]), actions, boxes,
                                 share_levels=binding != PER_ENV)
  assert track.restarts > 0, name
  assert compared >= T, (name, compared, raised)


def _rim_actions(name, B):
  """Env 0 plays the script, quits, and plays it again; in a raising case env 1 plays it
  up to the raising action and then idles; the others walk at random."""
  script = wc.RIM[name][2]
  actions = wc.random_actions(np.random.RandomState(len(name)), T, B)
  first = script + [5] + script
  actions[:, 0] = 4
  actions[:len(first), 0] = first
  if name in wc.RAISES:
    safe = script[:wc.RAISES[name]]
    actions[:, 1] = 4
    actions[:len(safe), 1] = safe
  return actions


@pytest.mark.parametrize('name', sorted(wc.RIM))
@pytest.mark.parametrize('extra', [0, 64])
def test_warehouse_rim(name, extra):
  """The scripted rim cases, 6 envs of one level: env 0 must reach every edge the case
  names; a raising script latches ENV_ERR_INDEX in env 0 at the oracle's step only."""
  art, beneath, _, edges = wc.RIM[name]
  boxes = wc.rim_boxes(name)
  game = wc.lowered(art, beneath, pitch=wc.ceil16(len(art[0])) + extra)
  actions = _rim_actions(name, 6)
  _, raised, track = _run([game], lambda e: wc.make_world(art, beneath), actions, boxes)
  if name in wc.RAISES:
    assert raised.get(0) == wc.RAISES[name] + 1, (name, raised)
    assert 1 not in raised
  else:
    assert 0 not in raised, (name, raised)
    assert edges <= track.seen(0), (name, sorted(edges - track.seen(0)))
    assert track.restarts > 0
  assert len(raised) < 6
