"""GPU tests of Backdrops with registered update() code on the compiled step program
(csrc/compiled.cu backdrop_step): the games of tests/backdrop_games.py on the H100, against
the reference's fluvial trajectories (tests/golden/fluvial_*.npz; the others replay in
test_gpu_registered_goldens.py), the hand-written
PCL_PROG_CLASSICS river and the oracle interpreter (oracle/compiled.py)."""

import numpy as np
import pytest

import example_games as eg
import golden_cases as gc
import registered_games as rg
import trajectory as tj
from oracle import compiled as ocompiled
from oracle import engine_model as em
from oracle import sampled_check
from pycolab_b200 import _lib, levels, lowering

pytestmark = pytest.mark.gpu

B, T = 4096, 300


@pytest.fixture(scope='module')
def games():
  yield from rg.registered('backdrop_games.py')


@pytest.mark.parametrize('name', gc.names('fluvial_'))
def test_facade_replays_fluvial_golden_with_the_compiled_pair(games, name):
  art = tj.u8_to_art(gc.load(name)['art'])
  assert lowering.lower(games.make_fluvial(art)).program == _lib.PROG_COMPILED
  eg.assert_replays('facade', name, make_env=lambda: games.make_fluvial(art))


@pytest.mark.parametrize('which', ['stock', 'other'])
def test_compiled_fluvial_matches_the_classics_kernel(games, which):
  """The registered pair on PCL_PROG_COMPILED and the river on PCL_PROG_CLASSICS, 4096 envs
  through auto-resets: every output byte-identical at every step."""
  import torch
  from pycolab_b200 import batched
  from pycolab_b200.games import fluvial_natation
  art = list(fluvial_natation.GAME_ART) if which == 'stock' else levels.fluvial_level()
  compiled = batched.BatchedEngine([lowering.lower(games.make_fluvial(art))], batch=B)
  classics = batched.BatchedEngine([fluvial_natation.make_game(art)], batch=B)
  assert compiled.game.program == _lib.PROG_COMPILED
  assert classics.game.program == _lib.PROG_CLASSICS
  rs = np.random.RandomState(11)
  outs = [compiled.its_showtime(), classics.its_showtime()]
  dones = 0
  for t in range(T + 1):
    if t:
      a = torch.from_numpy(rs.choice([0, 1, 2], size=B, p=[.2, .6, .2]).astype(np.int32)).cuda()
      outs = [compiled.play(a), classics.play(a)]
    torch.cuda.synchronize()
    for field in ('board', 'reward', 'has_reward', 'discount', 'done'):
      assert bool((getattr(outs[0], field) == getattr(outs[1], field)).all()), (t, field)
    dones += int(outs[0].done.sum())
  assert dones > 0
  assert int((compiled.error_codes() != 0).sum()) == 0


def _backdrop_check(t, engine, worlds, outs):
  """Each sampled env's live curtain and un-occluded layers against its oracle world."""
  import torch
  ids = sorted(worlds)
  idx = torch.as_tensor(ids, device=engine.device)
  live = engine.backdrop_live.index_select(0, idx).cpu().numpy()
  layers = engine.unoccluded_layers(engine.chars).index_select(0, idx).cpu().numpy()
  for k, e in enumerate(ids):
    w = worlds[e]
    assert w.error == 0
    np.testing.assert_array_equal(live[k, :, :engine.cols], w.backdrop, err_msg=str((t, e)))
    assert not live[k, :, engine.cols:].any(), (t, e)
    want = em.unoccluded_layers_of(w.backdrop, w.things, engine.chars)
    for c, ch in enumerate(engine.chars):
      np.testing.assert_array_equal(layers[k, c], want[ch], err_msg=str((t, e, ch)))


@pytest.mark.parametrize('game', ['trail', 'flow'])
def test_backdrop_games_lockstep_against_the_oracle(games, game):
  from pycolab_b200 import batched
  seed = 17
  lowered = [lowering.lower(games.GAMES[game](level)) for level in (0, 1)]
  eng = batched.BatchedEngine(lowered, batch=B, rng_seed=seed)
  rs = np.random.RandomState(9)
  actions = rs.randint(0, games.N_ACTIONS[game], size=(T, B)).astype(np.int32)
  sample = rg.sample_envs(rs, B)
  words = {e: (ocompiled.seeded_words(lowered[e % 2], seed + e) if lowered[0].rng_streams
               else None) for e in sample}
  eng.its_showtime()
  n = sampled_check.lockstep(
      eng, lambda e: ocompiled.make_world(lowered[e % 2], words[e]), sample, actions,
      curtains=lowered[0].drape_chars, sprites='P', pad_columns=True, on_step=_backdrop_check)
  assert n == len(sample) * (T + 1)
  if lowered[0].rng_streams:
    rng = eng.rng.cpu().numpy().view(np.uint32).reshape(B, 1, _lib.MT_WORDS)
    for e in sample:
      assert rng[e].tolist() == words[e], e
  assert int((eng.error_codes() != 0).sum()) == 0


def test_masked_reset_restores_only_the_masked_curtains(games):
  import torch
  from pycolab_b200 import batched
  n_envs = 256
  lowered = [lowering.lower(games.make_trail(level)) for level in (0, 1)]
  eng = batched.BatchedEngine(lowered, batch=n_envs, auto_reset=False)
  eng.its_showtime()
  rs = np.random.RandomState(4)
  for _ in range(20):
    eng.play(torch.from_numpy(rs.randint(0, 4, size=n_envs).astype(np.int32)).cuda())
  before = eng.backdrop_live.clone()
  templates = [torch.from_numpy(g.backdrop).cuda() for g in lowered]
  changed = [e for e in range(n_envs) if not bool((before[e] == templates[e % 2]).all())]
  assert len(changed) > n_envs // 2
  mask = torch.from_numpy((np.arange(n_envs) % 3 == 0).astype(np.uint8)).cuda()
  eng.reset(mask)
  torch.cuda.synchronize()
  after = eng.backdrop_live
  for e in range(n_envs):
    if e % 3 == 0:
      # its_showtime() ran the Backdrop once on the template: the walker has not moved
      assert bool((after[e] == templates[e % 2]).all()), e
    else:
      assert bool((after[e] == before[e]).all()), e


def test_shards_reproduce_one_engine(games):
  import torch
  from pycolab_b200 import batched
  n_envs, steps = 1024, 150
  lowered = [lowering.lower(games.make_flow(level)) for level in (0, 1)]
  whole = batched.BatchedEngine(lowered, batch=n_envs, rng_seed=5)
  halves = [batched.BatchedEngine(lowered, batch=n_envs // 2, rng_seed=5, env_offset=off)
            for off in (0, n_envs // 2)]
  rs = np.random.RandomState(2)
  outs = [whole.its_showtime()] + [h.its_showtime() for h in halves]
  for t in range(steps + 1):
    if t > 0:
      a = torch.from_numpy(rs.randint(0, 6, size=n_envs).astype(np.int32)).cuda()
      outs = [whole.play(a), halves[0].play(a[:n_envs // 2].contiguous()),
              halves[1].play(a[n_envs // 2:].contiguous())]
    torch.cuda.synchronize()
    for field in ('board', 'reward', 'has_reward', 'discount', 'done'):
      joined = torch.cat([getattr(outs[1], field), getattr(outs[2], field)])
      assert bool((getattr(outs[0], field) == joined).all()), (t, field)
  assert bool((whole.backdrop_live == torch.cat([h.backdrop_live for h in halves])).all())
  assert bool((whole.rng == torch.cat([h.rng for h in halves])).all())
