"""GPU tests of block chaining in scrolly_maze_step (scrolly_maze.cu, "Block chaining").

A step launch that follows another step launch of the library on its stream, inside one
pcl_run / pcl_run_many call or in a captured graph, skips the wait for the whole previous
grid: each block waits only for its own envs' previous step.  Each case checks which
launches chained (pcl_chained_launch_count, counted when a launch is enqueued or
captured), and runs the same
calls on a twin engine stepped eagerly, one pcl_step at a time, where every launch keeps
the full wait, and the two must agree byte for byte: boards, outputs, records, coin
patterns and cropper views.  Sampled envs are replayed on the oracle as well.
"""

import ctypes as C

import numpy as np
import pytest

from oracle import games as ogames
from oracle import sampled_check

pytestmark = pytest.mark.gpu

B = 1024                         # 256 blocks: the chained launches overlap on every SM
ARTS = None


def _arts():
  global ARTS
  if ARTS is None:
    from pycolab_b200 import levels
    ARTS = [levels.scrolly_maze_level(1700 + i, world_shape=(129, 129), board_shape=(64, 64),
                                      coin_density=0.4) for i in range(4)]
  return ARTS


def _engine(batch=B, env_offset=0, **kw):
  from pycolab_b200 import batched
  from pycolab_b200.games import scrolly_maze
  return batched.BatchedEngine([scrolly_maze.make_game(*a) for a in _arts()], batch=batch,
                               env_offset=env_offset, **kw)


def _make_world(e):
  a = _arts()[e % len(_arts())]
  return ogames.make_scrolly_maze(a[0], a[1], '+', a[2])


def _actions(seed, T, batch=B):
  """Mostly moves; 5 quits and restarts, 6 moves nothing."""
  import torch
  p = [.19, .19, .19, .19, .16, .02, .06]
  a = np.random.RandomState(seed).choice(7, size=(T, batch), p=p).astype(np.int32)
  return a, torch.from_numpy(a).cuda()


def _same(a, b, what, views=None):
  import torch
  torch.cuda.synchronize()
  for attr in ('_board', 'reward', 'has_reward', 'discount', 'done', 'sprites', 'drapes', 'plot'):
    assert torch.equal(getattr(a, attr), getattr(b, attr)), (attr, what)
  assert torch.equal(a.patterns[1], b.patterns[1]), ('coin pattern', what)
  if views is not None:
    assert torch.equal(*views), ('cropper view', what)


def _oracle_check(eng, acts_np, ids=range(0, B, 97)):
  streams = {e: [int(x) for x in acts_np[:, e]] for e in ids}
  assert sampled_check.final_state_check(eng, _make_world, ids, streams, 'Pabc') > 0


def _chained(e):
  """The handle's launches enqueued or captured as chained."""
  n = C.c_int64()
  assert e._lib.pcl_chained_launch_count(e._h, C.byref(n)) == 0
  return n.value


def _capture(fn):
  import torch
  torch.cuda.synchronize()
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g):
    fn()
  return g


def test_graph_steps_one_batch():
  """One batch stepped K times per replay, each launch chained to the one before it, with
  the cropper attached to the step kernel."""
  from pycolab_b200 import batched
  eng, twin = _engine(), _engine()
  crop = batched.scrolling_crop_spec(9, 9, 0)
  views = (eng.attach_cropper(crop), twin.attach_cropper(crop))
  assert eng._attached[3]
  eng.its_showtime(), twin.its_showtime()
  K = 40
  acts_np, acts = _actions(1, 2 * K)
  g = _capture(lambda: [eng.play(acts[t]) for t in range(K)])
  # the first step follows no step, the second keeps the full wait and the counters
  assert _chained(eng) == K - 2
  for r in range(2):
    if r:                        # the graph reads rows 0..K-1: give them the next actions
      acts[:K].copy_(acts[K:])
    g.replay()
    for t in range(K):
      twin.play(acts[r * K + t])
    _same(eng, twin, 'replay %d' % r, views)
  assert _chained(twin) == 0        # eager steps keep the full wait
  _oracle_check(eng, acts_np)


def test_graph_six_batch_rotation():
  """bench.py's headline: six batches stepped round-robin in one graph, each launch chained
  to another handle's.  A crop kernel of the first batch ends the graph: it follows only
  the last step launch, and must still see the first batch's last step done."""
  import torch
  from pycolab_b200 import batched
  R, b, K = 6, 256, 48
  engs = [_engine(b, env_offset=r * b) for r in range(R)]
  twins = [_engine(b, env_offset=r * b) for r in range(R)]
  for e in engs + twins:
    e.its_showtime()
  crop = batched.scrolling_crop_spec(9, 9, 0)
  states = (engs[0].new_crop_state(), twins[0].new_crop_state())
  views = [engs[0].crop(crop, state=states[0]), twins[0].crop(crop, state=states[1])]
  acts_np, acts = _actions(2, 2 * K, b)

  def body():
    for t in range(K):
      engs[t % R].play(acts[t])
    engs[0].crop(crop, state=states[0], out=views[0])

  g = _capture(body)
  assert sum(_chained(e) for e in engs) == K - 2
  for r in range(2):
    if r:
      acts[:K].copy_(acts[K:])
    g.replay()
    for t in range(K):
      twins[t % R].play(acts[r * K + t])
    twins[0].crop(crop, state=states[1], out=views[1])
    for i in range(R):
      _same(engs[i], twins[i], 'replay %d batch %d' % (r, i), views if i == 0 else None)
  assert torch.equal(*states), 'crop state'
  streams = {e: [int(acts_np[t, e]) for t in range(0, 2 * K, R)] for e in range(0, b, 31)}
  assert sampled_check.final_state_check(engs[0], _make_world, sorted(streams), streams,
                                         'Pabc') > 0


def test_graph_with_action_kernel_between_steps():
  """A torch kernel writes the actions before every step: no step follows a step, so each
  keeps the full wait, and reads the actions that kernel wrote."""
  import torch
  eng, twin = _engine(), _engine()
  eng.its_showtime(), twin.its_showtime()
  K = 30
  acts_np, acts = _actions(3, 2 * K)
  buf = torch.zeros(B, dtype=torch.int32, device='cuda')

  def body():
    for t in range(K):
      torch.add(acts[t], 0, out=buf)
      eng.play(buf)

  g = _capture(body)
  assert _chained(eng) == 0
  g.replay()
  for t in range(K):
    twin.play(acts[t])
  _same(eng, twin, 'replay 0')
  # the second replay writes other actions into the same source rows
  acts[:K].copy_(acts[K:])
  g.replay()
  for t in range(K):
    twin.play(acts[K + t])
  _same(eng, twin, 'replay 1')
  _oracle_check(eng, acts_np)


def test_run_steps_one_batch():
  """pcl_run over T steps: every launch after the first is chained."""
  eng, twin = _engine(), _engine()
  eng.its_showtime(), twin.its_showtime()
  T = 60
  acts_np, acts = _actions(4, T)
  eng.run(acts)
  assert _chained(eng) == T - 2
  for t in range(T):
    twin.play(acts[t])
  _same(eng, twin, 'pcl_run')
  _oracle_check(eng, acts_np)


def test_run_many_rotation():
  """pcl_run_many over three handles, each chained to another handle's launch."""
  from pycolab_b200 import batched
  R, b, T = 3, 512, 36
  engs = [_engine(b, env_offset=r * b) for r in range(R)]
  twins = [_engine(b, env_offset=r * b) for r in range(R)]
  for e in engs + twins:
    e.its_showtime()
  _, acts = _actions(5, T, b)
  batched.run_rotating(engs, [acts[t] for t in range(T)])
  assert sum(_chained(e) for e in engs) == T - 2
  for t in range(T):
    twins[t % R].play(acts[t])
  for i in range(R):
    _same(engs[i], twins[i], 'batch %d' % i)


def test_bind_state_and_reset_mid_chain():
  """pcl_bind_state starts the block counters afresh, and a host reset lands between two
  chained runs."""
  from pycolab_b200 import _lib
  eng, twin = _engine(), _engine()
  eng.its_showtime(), twin.its_showtime()
  T = 30
  acts_np, acts = _actions(6, 3 * T)
  eng.run(acts[:T])
  for t in range(T):
    twin.play(acts[t])
  _same(eng, twin, 'first run')
  for e in (eng, twin):
    _lib.check(e._lib.pcl_bind_state(e._h, C.byref(e._state)), 'pcl_bind_state')
  eng.run(acts[T:2 * T])
  for t in range(T, 2 * T):
    twin.play(acts[t])
  _same(eng, twin, 'after the rebind')
  eng.reset(), twin.reset()
  eng.run(acts[2 * T:])
  for t in range(2 * T, 3 * T):
    twin.play(acts[t])
  _same(eng, twin, 'after the reset')
  assert _chained(eng) == 3 * (T - 2)     # the reset itself is eager
  _oracle_check(eng, acts_np[2 * T:])


def test_graph_masked_reset_between_steps():
  """MODE_RESET with a mask, chained between steps of a graph: envs outside the mask are
  frozen for that launch and go on from where they were."""
  import torch
  eng, twin = _engine(), _engine()
  eng.its_showtime(), twin.its_showtime()
  K = 20
  _, acts = _actions(7, 2 * K)
  mask = torch.from_numpy((np.arange(B) % 3 == 0).astype(np.uint8)).cuda()

  def calls(e, base):
    for t in range(K):
      e.play(acts[base + t])
      if t % 5 == 4:
        e.reset(mask)

  g = _capture(lambda: calls(eng, 0))
  assert _chained(eng) == K + K // 5 - 2
  g.replay()
  calls(twin, 0)
  _same(eng, twin, 'replay 0')
  acts[:K].copy_(acts[K:])
  g.replay()
  calls(twin, K)
  _same(eng, twin, 'replay 1')


def test_graph_second_dependency():
  """A step whose stream also waits on another stream's kernel has two dependencies in
  the capture: it keeps the full wait, the step after it keeps the counters, and the one
  after that chains again."""
  import torch
  eng, twin = _engine(), _engine()
  eng.its_showtime(), twin.its_showtime()
  _, acts = _actions(8, 4)
  side = torch.cuda.Stream()
  junk = torch.zeros(1 << 20, dtype=torch.int32, device='cuda')

  def body():
    main = torch.cuda.current_stream()
    eng.play(acts[0])
    side.wait_stream(main)
    with torch.cuda.stream(side):
      junk.add_(1)
    main.wait_stream(side)
    eng.play(acts[1])
    eng.play(acts[2])
    eng.play(acts[3])

  g = _capture(body)
  assert _chained(eng) == 1
  g.replay()
  for t in range(4):
    twin.play(acts[t])
  _same(eng, twin, 'replay')
