"""GPU tests of inlined helper calls on the compiled step program (csrc/compiled.cu): the
games of tests/helper_games.py on the H100, against the oracle interpreter
(oracle/compiled.py).  Their goldens replay in test_gpu_registered_goldens.py."""

import numpy as np
import pytest

import registered_games as rg
from registered_games import global_generators  # noqa: F401  (a fixture)
from oracle import compiled as ocompiled
from oracle import sampled_check
from pycolab_b200 import _lib, lowering

pytestmark = pytest.mark.gpu

B, T = 4096, 300


@pytest.fixture(scope='module')
def games():
  yield from rg.registered('helper_games.py')


@pytest.mark.parametrize('level', [0, 1])
def test_bolts_lockstep_against_the_oracle(games, level):
  """B = 4096 with auto-reset (the levels differ in shape: one engine each): each env
  draws its own downward bolts' columns; sampled envs every step, the marauders' curtain,
  the bolts' records, the registers and the generators' words at the end."""
  from pycolab_b200 import batched
  seed = 50 + level
  lowered = lowering.lower(games.make_bolts(level))
  eng = batched.BatchedEngine([lowered], batch=B, rng_seed=seed)
  rs = np.random.RandomState(9 + level)
  actions = rs.randint(0, 5, size=(T, B)).astype(np.int32)
  sample = rg.sample_envs(rs, B)
  words = {e: ocompiled.seeded_words(lowered, seed + e) for e in sample}
  eng.its_showtime()
  n = sampled_check.lockstep(
      eng, lambda e: ocompiled.make_world(lowered, words[e]), sample, actions,
      curtains='X', sprites='P!:;^', pad_columns=True,
      on_step=rg.register_check(lambda e: lowered))
  assert n == len(sample) * (T + 1)
  rng = eng.rng.cpu().numpy().view(np.uint32).reshape(B, 1, _lib.MT_WORDS)
  for e in sample:
    assert rng[e].tolist() == words[e], e
  assert int((eng.error_codes() != 0).sum()) == 0


@pytest.mark.parametrize('level,curtains,sprites', [(0, '.', 'Pc'), (1, '#', 'P')])
def test_chaser_lockstep_against_the_oracle(games, level, curtains, sprites):
  """Each chaser level at B = 4096: module functions, a Backdrop's and a drape's helpers
  (level 0), and helpers issuing scroll orders and egocentric moves (level 1)."""
  from pycolab_b200 import batched
  lowered = lowering.lower(games.make_chaser(level))
  eng = batched.BatchedEngine([lowered], batch=B)
  eng.its_showtime()
  rs = np.random.RandomState(10 + level)
  actions = rs.randint(0, 6, size=(T, B)).astype(np.int32)
  sample = rg.sample_envs(rs, B)
  n = sampled_check.lockstep(
      eng, lambda e: ocompiled.make_world(lowered), sample, actions, curtains=curtains,
      sprites=sprites, pad_columns=True, on_step=rg.register_check(lambda e: lowered))
  assert n == len(sample) * (T + 1)
  assert int((eng.error_codes() != 0).sum()) == 0


def test_facade_raises_zero_division_where_the_reference_did(games, global_generators):  # noqa: F811
  """helper_divzero through the facade: every frame before the reference's
  ZeroDivisionError, then the ZeroDivisionError (a case of test_gpu_registered_goldens
  too)."""
  rg.assert_facade_replays(games, 'helper_divzero')


def test_only_the_envs_that_divide_by_zero_latch_arith_errors(games):
  """Envs that count down three times latch PCL_ENV_ERR_ARITH at that step; the others
  stay in lock-step with the oracle."""
  import torch
  from pycolab_b200 import batched
  n_envs = 256
  lowered = lowering.lower(games.make_divzero())
  eng = batched.BatchedEngine([lowered], batch=n_envs, auto_reset=False)
  divides = np.arange(n_envs) % 3 == 0
  worlds = [ocompiled.make_world(lowered) for _ in range(n_envs)]
  for w in worlds:
    w.its_showtime()
  eng.its_showtime()
  for t in range(6):
    acts = np.where(divides & (t < 3), 2, t % 2).astype(np.int32)
    eng.play(torch.from_numpy(acts).cuda())
    torch.cuda.synchronize()
    errors = eng.error_codes().cpu().numpy()
    boards = eng.board.cpu().numpy()
    for e in range(n_envs):
      if divides[e] and t >= 2:
        assert errors[e] & _lib.ENV_ERR_ARITH, (t, e)
        continue
      assert errors[e] == 0, (t, e)
      board, _, _ = worlds[e].play(int(acts[e]))
      np.testing.assert_array_equal(boards[e], board, err_msg=str((t, e)))
  assert int((eng.error_codes().cpu().numpy() != 0).sum()) == int(divides.sum())
