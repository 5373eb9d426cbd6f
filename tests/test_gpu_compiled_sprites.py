"""GPU tests of plain Sprites on the compiled step program (csrc/compiled.cu): the games of
tests/sprite_games.py on the H100, against the oracle interpreter (oracle/compiled.py).
Their goldens replay in test_gpu_registered_goldens.py."""

import numpy as np
import pytest

import registered_games as rg
from registered_games import global_generators  # noqa: F401  (a fixture)
from oracle import compiled as ocompiled
from oracle import sampled_check
from pycolab_b200 import _lib, lowering, rendering

pytestmark = pytest.mark.gpu

B, T = 4096, 300


@pytest.fixture(scope='module')
def games():
  yield from rg.registered('sprite_games.py')


def test_bounce_lockstep_against_the_oracle(games):
  """B = 4096, both levels, auto-reset: sampled envs every step, the bricks' curtain, the
  ball's words and registers, and the generators' words at the end."""
  from pycolab_b200 import batched
  seed = 30
  lowered = [lowering.lower(games.make_bounce(level)) for level in (0, 1)]
  eng = batched.BatchedEngine(lowered, batch=B, rng_seed=seed)
  rs = np.random.RandomState(7)
  actions = rs.randint(0, 4, size=(T, B)).astype(np.int32)
  sample = rg.sample_envs(rs, B)
  words = {e: ocompiled.seeded_words(lowered[e % 2], seed + e) for e in sample}
  eng.its_showtime()
  n = sampled_check.lockstep(
      eng, lambda e: ocompiled.make_world(lowered[e % 2], words[e]), sample, actions,
      curtains='=', sprites='P', pad_columns=True,
      on_step=rg.register_check(lambda e: lowered[e % 2], layers=True))
  assert n == len(sample) * (T + 1)
  rng = eng.rng.cpu().numpy().view(np.uint32).reshape(B, 1, _lib.MT_WORDS)
  for e in sample:
    assert rng[e].tolist() == words[e], e
  assert int((eng.error_codes() != 0).sum()) == 0


def test_sampler_lockstep_against_the_oracle(games):
  """The sampler at B = 4096 over two levels: plain Sprites beside a Scrolly and an
  egocentric walker, wrapped and far-off positions, every step; and pcl_render painting one
  sampled env's state as the step kernel did."""
  from pycolab_b200 import batched
  lowered = [lowering.lower(games.make_sampler(level)) for level in (0, 1)]
  eng = batched.BatchedEngine(lowered, batch=B)
  eng.its_showtime()
  rs = np.random.RandomState(8)
  actions = rs.randint(0, 9, size=(T, B)).astype(np.int32)
  sample = rg.sample_envs(rs, B)
  seen = {'wrapped': 0, 'far': 0}

  def render_check(t, engine, worlds, outs):
    w = worlds[sample[0]]
    e = w.things['e']
    seen['wrapped'] += int(e.visible and (e.row < 0 or e.col < 0))
    seen['far'] += int(abs(w.things['g'].row) >= 1000)
    if t % 25:
      return
    painted = []
    for ch in w.z_order:
      ent = w.things[ch]
      if not getattr(ent, 'is_sprite', False):
        painted.append(('drape', ch, np.asarray(ent.curtain, dtype=bool)))
      elif ent.visible:
        painted.append(('sprite', ch, (ent.row, ent.col)))
    board = rendering.render_on_device(w.backdrop, painted, device=engine.device.index or 0)
    np.testing.assert_array_equal(board, w.board, err_msg=str(t))
    np.testing.assert_array_equal(engine.board[sample[0]].cpu().numpy(), w.board)
  n = sampled_check.lockstep(
      eng, lambda e: ocompiled.make_world(lowered[e % 2]), sample, actions,
      curtains='#x', sprites='Pw', pad_columns=True,
      on_step=rg.register_check(lambda e: lowered[e % 2], layers=True, extra=render_check))
  assert n == len(sample) * (T + 1)
  assert seen['wrapped'] > 0 and seen['far'] > 0
  assert int((eng.error_codes() != 0).sum()) == 0


def test_facade_raises_index_error_where_the_reference_did(games, global_generators):  # noqa: F811
  """sprite_fallen through the facade: every frame before the reference's IndexError, then
  the IndexError (a case of test_gpu_registered_goldens too)."""
  rg.assert_facade_replays(games, 'sprite_fallen')


def test_only_the_envs_that_fall_latch_index_errors(games):
  """Envs whose sprite walks off the board latch PCL_ENV_ERR_INDEX at the step the
  reference raised; the others stay in lock-step with the oracle."""
  import torch
  from pycolab_b200 import batched
  n_envs = 256
  lowered = lowering.lower(games.make_fallen())
  eng = batched.BatchedEngine([lowered], batch=n_envs, auto_reset=False)
  falls = np.arange(n_envs) % 3 == 0
  worlds = [ocompiled.make_world(lowered) for _ in range(n_envs)]
  outs = [w.its_showtime() for w in worlds]
  eng.its_showtime()
  for t in range(6):
    acts = np.where(falls, 0, 1).astype(np.int32) if t < 3 else np.where(falls, 0, t % 2)
    eng.play(torch.from_numpy(acts.astype(np.int32)).cuda())
    torch.cuda.synchronize()
    errors = eng.error_codes().cpu().numpy()
    boards = eng.board.cpu().numpy()
    for e in range(n_envs):
      if falls[e] and t >= 3:
        assert errors[e] & _lib.ENV_ERR_INDEX, (t, e)
        continue
      assert errors[e] == 0, (t, e)
      board, _, _ = worlds[e].play(int(acts[e]))
      np.testing.assert_array_equal(boards[e], board, err_msg=str((t, e)))
  assert int((eng.error_codes().cpu().numpy() != 0).sum()) == int(falls.sum())


def test_shards_reproduce_one_engine(games):
  """bounce's draws are per env: engines of env_offset 0 and B / 2 step as the two halves
  of one engine of B."""
  import torch
  from pycolab_b200 import batched
  n_envs, steps = 1024, 150
  lowered = [lowering.lower(games.make_bounce(level)) for level in (0, 1)]
  whole = batched.BatchedEngine(lowered, batch=n_envs, rng_seed=5)
  halves = [batched.BatchedEngine(lowered, batch=n_envs // 2, rng_seed=5, env_offset=off)
            for off in (0, n_envs // 2)]
  rs = np.random.RandomState(2)
  outs = [whole.its_showtime()] + [h.its_showtime() for h in halves]
  for t in range(steps + 1):
    if t > 0:
      a = torch.from_numpy(rs.randint(0, 4, size=n_envs).astype(np.int32)).cuda()
      outs = [whole.play(a), halves[0].play(a[:n_envs // 2].contiguous()),
              halves[1].play(a[n_envs // 2:].contiguous())]
    torch.cuda.synchronize()
    for field in ('board', 'reward', 'has_reward', 'discount', 'done'):
      joined = torch.cat([getattr(outs[1], field), getattr(outs[2], field)])
      assert bool((getattr(outs[0], field) == joined).all()), (t, field)
  assert bool((whole.rng == torch.cat([h.rng for h in halves])).all())
  assert bool((whole.sprites == torch.cat([h.sprites for h in halves])).all())
