"""tests/layer_cases.py on the CPU: the status each case records is what pcl_create answers
for its spec, and its walk does what test_gpu_layers asserts of it on the device (envs
restart inside the run; a scrolly_maze case of more than one env collects a coin on a quit,
which leaves the coin window's stale slot live), replayed on the oracle."""

import ctypes as C

import numpy as np
import pytest

import layer_cases as lc
from pycolab_b200 import _lib


def _create_status(spec, batch):
  lib = _lib.load()
  h = C.c_void_p()
  status = lib.pcl_create(C.byref(spec), batch, -1, C.byref(h))   # device -1: no CUDA call
  if status == _lib.OK:
    lib.pcl_destroy(h)
  return status


@pytest.mark.parametrize('case', lc.CASES, ids=[c.id for c in lc.CASES])
def test_case_table(case):
  built = case.build()
  assert {_create_status(g.make_spec(auto_reset=True), case.batch) for g in built.games} == {
      {'ok': _lib.OK, 'unsupported': _lib.ERR_UNSUPPORTED}[case.status]}
  assert all((g.rows, g.cols, g.pitch) == case.shape + (case.pitch,) for g in built.games)
  assert case.batch in lc.BATCHES and (case.binding != lc.POOL or case.batch > 1)
  assert (len(built.games) == 1) == (case.binding == lc.SHARED)
  restarts, stale = _replay(built, case.batch, case.batch + case.pitch,
                            case.program == 'scrolly_maze')
  assert restarts > 0
  if case.program == 'scrolly_maze' and case.batch > 1:
    assert stale > 0


@pytest.mark.parametrize('program,hook,build', lc.HOOK_CASES, ids=[c[0] for c in lc.HOOK_CASES])
def test_host_hook_walks_restart(program, hook, build):
  assert _replay(build(), 5, 3, False)[0] > 0


def _replay(built, B, seed, scrolly):
  """(restarts, coins collected on a quit) of the case's walk on the oracle, under
  sampled_check.lockstep's auto-reset rule, with the seed test_gpu_layers draws it with."""
  T = built.steps
  actions = built.draw(np.random.RandomState(seed), T, B)
  restarts = stale = 0
  for e in range(B):
    world = built.make_world(e)
    world.its_showtime()
    for t in range(T):
      if world.game_over:
        world = built.make_world(e)
        world.its_showtime()
        restarts += 1
        continue
      pending = scrolly and lc.coin_under_player(world)
      _, reward, _ = world.play(int(actions[t, e]))
      if pending and actions[t, e] == 5:
        assert reward == 100
        stale += 1
  return restarts, stale
