"""GPU tests of draws from the global generators in compiled code (csrc/compiled.cu
PCL_OP_RANDINT / RANDCMP / PICK): tests/drawn_games.py on the H100, against the oracle
(oracle/compiled.py).  Its goldens replay in test_gpu_registered_goldens.py."""

import numpy as np
import pytest

import registered_games as rg
from registered_games import global_generators  # noqa: F401  (a fixture)
from oracle import compiled as ocompiled
from oracle import sampled_check
from pycolab_b200 import _lib, lowering

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def games():
  yield from rg.registered('drawn_games.py')


def _device_regs(eng, envs):
  S = len(eng.sprite_chars)
  sprites = eng.sprites[envs].cpu().numpy()[:, :, _lib.S_AUX0:].reshape(len(envs), -1)
  drapes = eng.drapes[envs].cpu().numpy().reshape(len(envs), -1)
  plot = eng.plot[envs].cpu().numpy()[:, _lib.P_AUX0:_lib.P_AUX0 + 4]
  assert sprites.shape[1] == 3 * S
  return np.concatenate([sprites, drapes, plot], axis=1).astype(np.int64)


def test_batched_monsters_vs_oracle(games):
  """B = 4096, both levels alternating, auto-reset, 300 steps: 128 sampled envs (the
  first and last of each level among them) against oracle worlds whose generators are
  seeded rng_seed + env, every step, registers included, then their final generator
  words."""
  from pycolab_b200 import batched
  B, T, seed = 4096, 300, 40
  levels = [lowering.lower(games.make_monsters(k)) for k in range(2)]
  eng = batched.BatchedEngine(levels, batch=B, rng_seed=seed)
  rs = np.random.RandomState(13)
  table = rs.randint(0, games.N_ACTIONS['monsters'], size=(T, B)).astype(np.int32)
  sample = [int(e) for e in np.unique(np.concatenate(
      [[0, 1, B - 2, B - 1], rs.choice(np.arange(2, B - 2), 124, replace=False)]))]
  assert len(sample) == 128
  words = {e: ocompiled.seeded_words(levels[e % 2], seed + e) for e in sample}
  eng.its_showtime()
  episodes = [0]

  def same_registers(t, eng, worlds, outs):
    regs = _device_regs(eng, sample)
    for k, e in enumerate(sample):
      w = worlds[e]
      want = ([r for ch in eng.sprite_chars for r in w.things[ch].regs] +
              [r for ch in eng.drape_chars for r in w.things[ch].regs] + list(w.plot.regs))
      assert (regs[k] == want).all(), (t, e, regs[k], want)
      assert w.error == 0
    episodes[0] += int(eng.done.sum())
  sampled_check.lockstep(eng, lambda e: ocompiled.make_world(levels[e % 2], words[e]), sample,
                         table, pad_columns=True, on_step=same_registers)
  assert episodes[0] > B                    # the streams run on across auto-resets
  rng = eng.rng.cpu().numpy().view(np.uint32).reshape(B, 2, _lib.MT_WORDS)
  for e in sample:
    assert rng[e].tolist() == words[e], e
  assert int((eng.error_codes() != 0).sum()) == 0
  assert int(eng._board[:, :, eng.cols:].sum()) == 0        # the pitch padding stays zero


def test_shards_reproduce_one_engine(games):
  """Engines of env_offset 0 and B / 2 step as the two halves of one engine of B."""
  import torch
  from pycolab_b200 import batched
  B, T = 1024, 120
  levels = [lowering.lower(games.make_monsters(k)) for k in range(2)]
  whole = batched.BatchedEngine(levels, batch=B, rng_seed=5)
  halves = [batched.BatchedEngine(levels, batch=B // 2, rng_seed=5, env_offset=off)
            for off in (0, B // 2)]
  rs = np.random.RandomState(2)
  outs = [whole.its_showtime()] + [h.its_showtime() for h in halves]
  for t in range(T + 1):
    if t > 0:
      a = torch.from_numpy(rs.randint(0, 6, size=B).astype(np.int32)).cuda()
      outs = [whole.play(a), halves[0].play(a[:B // 2].contiguous()),
              halves[1].play(a[B // 2:].contiguous())]
    torch.cuda.synchronize()
    for field in ('board', 'reward', 'has_reward', 'discount', 'done'):
      joined = torch.cat([getattr(outs[1], field), getattr(outs[2], field)])
      assert bool((getattr(outs[0], field) == joined).all()), (t, field)
  assert bool((whole.rng == torch.cat([h.rng for h in halves])).all())


@pytest.mark.parametrize('which', [0, 1, 2], ids=['numpy_randint', 'python_randrange',
                                                  'numpy_choice'])
def test_empty_range_raises_value_error(games, global_generators, which):  # noqa: F811
  engine = games.make_empty(which)
  engine.its_showtime()
  before = (rg.global_words('numpy'), rg.global_words('python'))
  engine.play(0)
  with pytest.raises(ValueError):
    engine.play(1)
  assert (rg.global_words('numpy'), rg.global_words('python')) == before  # nothing drawn
