"""Episode time limits (`pcl_set_time_limit`, `BatchedEngine.set_time_limit`) without a GPU.

- The header's PCL_DONE_TIME_LIMIT and pcl_set_time_limit against the ctypes binding.
- pcl_set_time_limit's refusals on a handle that reaches no device (device -1).
- The facade's argument checks, which run before anything needs CUDA.
- The time-limited lock-step harness (tests/time_limit_lockstep.py) on a CPU stand-in for
  BatchedEngine: it passes on frames recorded with the rule, and names one corrupted done.
"""

import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from oracle import games as ogames
from oracle import sampled_check as sc
from pycolab_b200 import _lib, levels
import time_limit_lockstep as tll

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_constant_and_symbol_match_the_binding():
  with open(os.path.join(ROOT, 'include', 'pcl.h')) as f:
    header = f.read()
  assert int(re.search(r'#define PCL_DONE_TIME_LIMIT (\d+)', header).group(1)) == \
      _lib.DONE_TIME_LIMIT == 2
  assert re.search(r'int pcl_set_time_limit\(pcl_handle\* h, int32_t max_frames\);', header)
  restype, argtypes = _lib.SYMBOLS['pcl_set_time_limit']
  assert restype is C.c_int and argtypes == [C.c_void_p, C.c_int32]
  assert _lib.load().pcl_set_time_limit is not None


def _handle():
  lib = _lib.load()
  spec = _lib.Spec()
  spec.abi_version, spec.program = _lib.ABI_VERSION, _lib.PROG_NONE
  spec.rows, spec.cols, spec.pitch = 16, 16, 16
  h = C.c_void_p()
  assert lib.pcl_create(C.byref(spec), 4, -1, C.byref(h)) == _lib.OK
  return lib, h


def test_set_time_limit_refusals():
  lib, h = _handle()
  try:
    assert lib.pcl_set_time_limit(None, 5) == _lib.ERR_INVALID
    assert lib.pcl_set_time_limit(None, 0) == _lib.ERR_INVALID
    for bad in (-1, -(2 ** 31)):
      assert lib.pcl_set_time_limit(h, bad) == _lib.ERR_INVALID, bad
    for good in (0, 1, 7, 2 ** 31 - 1, 0):
      assert lib.pcl_set_time_limit(h, good) == _lib.OK, good
  finally:
    lib.pcl_destroy(h)


@pytest.mark.parametrize('bad,error', [(True, TypeError), (False, TypeError), (1.0, TypeError),
                                       ('8', TypeError), (-1, ValueError),
                                       (2 ** 31, ValueError)])
def test_facade_refuses_a_bad_limit_before_cuda(bad, error):
  from pycolab_b200 import batched
  from pycolab_b200.games.classics import four_rooms
  with pytest.raises(error, match='time_limit'):
    batched.BatchedEngine([four_rooms.make_game()], batch=2, time_limit=bad)


def test_set_time_limit_on_a_handle_without_a_device():
  from pycolab_b200 import batched
  lib, h = _handle()
  eng = batched.BatchedEngine.__new__(batched.BatchedEngine)
  eng._lib, eng._h, eng.time_limit = lib, h, 0
  try:
    for n, want in ((5, 5), (np.int64(3), 3), (None, 0), (0, 0)):
      eng.set_time_limit(n)
      assert eng.time_limit == want and type(eng.time_limit) is int
    eng.set_time_limit(4)
    for bad, error in ((-2, ValueError), (True, TypeError), (2.5, TypeError)):
      with pytest.raises(error):
        eng.set_time_limit(bad)
      assert eng.time_limit == 4
  finally:
    eng.close()


# ---- the lock-step harness -----------------------------------------------------------

ART = levels.scrolly_maze_level(7, world_shape=(33, 41), board_shape=(12, 20))
B, T, PITCH, LIMIT = 5, 40, 32, 6


def make_world(e):
  return ogames.make_scrolly_maze(ART[0], ART[1], '+', ART[2])


def _actions():
  rs = np.random.RandomState(3)
  return rs.choice(6, size=(T, B), p=[.23, .23, .23, .23, .02, .06]).astype(np.int32)


class StandIn(object):
  """What lockstep reads of a BatchedEngine, replaying frames recorded on the CPU from
  oracle worlds with the time limit applied by hand."""
  device = 'cpu'
  sprite_chars = 'Pabc'

  def __init__(self, actions):
    self.actions, self.t = actions, 0
    frames = [self._record(e, actions[:, e]) for e in range(B)]
    self.frames = {k: torch.from_numpy(np.stack([f[k] for f in frames], axis=1))
                   for k in frames[0]}
    self.cols = len(ART[1][0])

  @staticmethod
  def _record(e, actions):
    rec = {k: [] for k in ('board', 'reward', 'has_reward', 'discount', 'done')}

    def keep(out, done):
      board = np.zeros((out[0].shape[0], PITCH), np.uint8)
      board[:, :out[0].shape[1]] = out[0]
      rec['board'].append(board)
      rec['reward'].append(0 if out[1] is None else out[1])
      rec['has_reward'].append(out[1] is not None)
      rec['discount'].append(out[2])
      rec['done'].append(done)

    world = make_world(e)
    keep(world.its_showtime(), 0)
    done, plays = 0, 0
    for a in actions:
      if done:                               # auto-reset: a fresh world, its_showtime()
        world, done, plays = make_world(e), 0, 0
        keep(world.its_showtime(), 0)
        continue
      out = world.play(int(a))
      plays += 1
      done = 1 if world.game_over else 2 if plays == LIMIT else 0
      keep(out, done)
    dtypes = dict(board=np.uint8, reward=np.int32, has_reward=np.uint8, discount=np.float32,
                  done=np.uint8)
    return {k: np.array(v, dtype=dtypes[k]) for k, v in rec.items()}

  def play(self, actions):
    assert actions.tolist() == self.actions[self.t].tolist()
    self.t += 1

  def _now(self, name):
    return self.frames[name][self.t]

  @property
  def _board(self):
    return self._now('board')

  @property
  def board(self):
    return self._now('board')[:, :, :self.cols]

  reward = property(lambda self: self._now('reward'))
  has_reward = property(lambda self: self._now('has_reward'))
  discount = property(lambda self: self._now('discount'))
  done = property(lambda self: self._now('done'))


def test_stand_in_with_the_rule_passes():
  actions = _actions()
  eng = StandIn(actions)
  done = eng.frames['done'].numpy()
  assert (done == 1).any() and (done == 2).any(), 'the actions end no episode both ways'
  compared, cut = tll.lockstep(eng, make_world, range(B), actions, LIMIT)
  assert compared == (T + 1) * B
  assert cut == int(np.count_nonzero(done == 2))


@pytest.mark.parametrize('was,now', [(2, 1), (2, 0), (1, 2), (0, 2)])
def test_one_corrupted_done_is_named(was, now):
  actions = _actions()
  eng = StandIn(actions)
  t, e = [int(x) for x in np.argwhere(eng.frames['done'].numpy() == was)[-1]]
  eng.frames['done'][t, e] = now
  with pytest.raises(sc.Mismatch, match='step %d env %d' % (t, e)):
    tll.lockstep(eng, make_world, range(B), actions, LIMIT)


def test_without_a_limit_a_truncation_is_a_mismatch():
  actions = _actions()
  with pytest.raises(sc.Mismatch, match='done differs|game_over differs'):
    tll.lockstep(StandIn(actions), make_world, range(B), actions, 0)
