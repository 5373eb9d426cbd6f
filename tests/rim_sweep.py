"""The parts of a board-rim sweep that do not depend on the step program.  A sweep is a
cases module (levels, scripted rim cases and an `Edges` tracker of one game), a CPU
module (the oracle against the reference) and a GPU module (the device against the
oracle); this module holds what they share:
  * lowered games re-padded to a wider pitch, and the level bindings and batches the
    sweeps rotate across board shapes and pitches;
  * `run`: a BatchedEngine in lock-step with oracle worlds, an `Edges` per env;
  * `oracle_run`: the same auto-reset play on the CPU;
  * pcl_create's answer for a spec at another board shape, and a bisection for the
    largest size it accepts.

Every `Edges` has start(world, out), called on a fresh world with its its_showtime()
output, step(world, out, action), called after each play(action), and the set `seen`
of edges the world went through.
"""

import ctypes as C

import numpy as np

from oracle import sampled_check
from pycolab_b200 import _lib

SHARED, POOL, PER_ENV = 'shared', 'pool', 'per_env'
BINDINGS = (SHARED, POOL, PER_ENV)
BATCHES = (1, 5, 37)
MAX_BLOCK_SMEM = 227 * 1024     # H100: the shared memory one block may opt in to, static included


def ceil16(x):
  return (x + 15) // 16 * 16


def repitch(low, pitch):
  """`low`, a lowered game, with its backdrop re-padded to `pitch` columns (None: as it
  is)."""
  if pitch is not None:
    backdrop = np.zeros((low.rows, pitch), dtype=np.uint8)
    backdrop[:, :low.cols] = low.backdrop[:, :low.cols]
    low.backdrop, low.pitch = backdrop, pitch
  return low


def levels_and_batch(binding, B):
  """How many levels a sweep case binds (one shared, three in a pool, two per env), and
  its batch: at least 5 for a pool, so that its envs read every level."""
  if binding == POOL:
    return 3, max(B, 5)
  return (1 if binding == SHARED else 2), B


def rotate(shapes, pitches=('+0', '+16', '+64')):
  """(i, j, k, shape, pitch, binding, B) for shape i at pitch j, k = len(pitches) * i + j,
  with the bindings and batches rotated across them so that each value of every axis
  meets several of the others.  A pitch '+n' is ceil16(W) + n, an int is itself."""
  for i, shape in enumerate(shapes):
    for j, p in enumerate(pitches):
      k = len(pitches) * i + j
      pitch = ceil16(shape[1]) + int(p[1:]) if isinstance(p, str) else p
      yield i, j, k, shape, pitch, BINDINGS[(i + 2 * j) % 3], BATCHES[(k // 2) % 3]


class Track(object):
  """on_step hook of sampled_check.lockstep: feeds each sampled env's oracle world to its
  own make_edges(), and counts the restarts.  Envs in `raised` are left alone."""

  def __init__(self, make_edges, actions, raised):
    self.make_edges, self.actions, self.raised = make_edges, actions, raised
    self.edges, self.worlds, self.restarts = {}, {}, 0

  def __call__(self, t, engine, worlds, outs):
    for e, w in worlds.items():
      if e in self.raised:
        continue
      if self.worlds.get(e) is not w:
        self.edges.setdefault(e, self.make_edges()).start(w, outs[e])
        self.restarts += t > 0
      else:
        self.edges[e].step(w, outs[e], int(self.actions[t - 1, e]))
      self.worlds[e] = w

  def seen(self, e=None):
    if e is not None:
      return self.edges[e].seen if e in self.edges else set()
    return set().union(*(x.seen for x in self.edges.values()))


def run(games, make_world, actions, *, curtains, sprites, make_edges, share_levels=True,
        rng_seed=None):
  """Step a BatchedEngine of `games` with actions [T, B] in lock-step with make_world(e)
  for every env, comparing the curtains, the sprites' records, the pitch padding and the
  latched error words.  With rng_seed, env e draws from RandomState(rng_seed + e) across
  its episodes, on the device and in its oracle world make_world(e, rng).  Returns (pairs
  compared, {env: step it raised at}, Track)."""
  from pycolab_b200 import batched
  B = actions.shape[1]
  world_of, seeded = make_world, {}
  if rng_seed is not None:
    rngs = [np.random.RandomState(rng_seed + e) for e in range(B)]
    world_of, seeded = (lambda e: make_world(e, rngs[e])), {'rng_seed': rng_seed}
  eng = batched.BatchedEngine(games, batch=B, share_levels=share_levels, **seeded)
  eng.its_showtime()
  raised = {}
  track = Track(make_edges, actions, raised)
  compared = sampled_check.lockstep(eng, world_of, range(B), actions, curtains=curtains,
                                    sprites=sprites, pad_columns=True, on_step=track,
                                    raised=raised)
  return compared, raised, track


def twice(script, quit):
  """The script, a quit, and the script again from a fresh episode."""
  return script + [quit] + script


def rim_actions(script, quit, idle, T, B, draw, seed):
  """Env 0 plays twice(script, quit) and then idles; the others play
  draw(RandomState(seed), T, B)."""
  actions = draw(np.random.RandomState(seed), T, B)
  first = twice(script, quit)
  actions[:, 0] = idle
  actions[:len(first), 0] = first
  return actions


def oracle_run(make_world, edges, actions, raises=()):
  """Play `actions` on make_world() worlds with auto-reset, feeding `edges`.  Returns
  (edges seen, restarts, the step whose action raised one of `raises`, -1 if its_showtime
  did, or None).  A raise adds 'raise' to the edges, and calls edges.on_raise(world) where
  the tracker has it."""
  def raised(world):
    edges.seen.add('raise')
    if hasattr(edges, 'on_raise'):
      edges.on_raise(world)
    return edges.seen

  world = make_world()
  try:
    out = world.its_showtime()
  except raises:
    return raised(world), 0, -1
  edges.start(world, out)
  restarts = 0
  for t, a in enumerate(actions):
    if world.game_over:
      restarts += 1
      world = make_world()
      edges.start(world, world.its_showtime())
      continue
    try:
      out = world.play(int(a))
    except raises:
      return raised(world), restarts, t
    edges.step(world, out, int(a))
  return edges.seen, restarts, None


def seeded_pair(make_ref, make_ora, seed):
  """make_ref, and a maker of make_ora(rng) worlds, drawing from one MT19937 stream: NumPy's
  global generator and rng = RandomState(seed), both seeded here and never again, so that
  later episodes continue the stream on both sides."""
  np.random.seed(seed)
  rng = np.random.RandomState(seed)
  return make_ref, (lambda: make_ora(rng))


# ------------------------------------------------------------ pcl_create's bound

def create_status(game, batch, **fields):
  """pcl_create's answer for the spec of `game` (lowered) with `fields` (rows, cols,
  pitch, ...) set, at `batch` envs on device -1: no CUDA call."""
  spec = game.make_spec(auto_reset=True)
  for name, value in fields.items():
    setattr(spec, name, value)
  lib = _lib.load()
  h = C.c_void_p()
  status = lib.pcl_create(C.byref(spec), batch, -1, C.byref(h))
  if status == _lib.OK:
    lib.pcl_destroy(h)
  return status


def largest_accepted(status, lo, hi, step=1):
  """The largest x below hi, on the grid of `step`, with status(x) OK, by bisection:
  status(lo) must be OK and status(hi) ERR_UNSUPPORTED."""
  assert status(lo) == _lib.OK
  assert status(hi) == _lib.ERR_UNSUPPORTED
  while hi - lo > step:
    mid = (lo + hi) // (2 * step) * step
    lo, hi = (mid, hi) if status(mid) == _lib.OK else (lo, mid)
  return lo
