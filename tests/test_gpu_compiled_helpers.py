"""GPU tests of inlined helper calls on the compiled step program (csrc/compiled.cu): the
games of tests/helper_games.py on the H100, against the reference's trajectories
(tests/golden/helper_*.npz) and the oracle interpreter (oracle/compiled.py)."""

import numpy as np
import pytest

import golden_cases as gc
import registered_games as rg
import trajectory as tj
from oracle import compiled as ocompiled
from oracle import sampled_check
from pycolab_b200 import _lib, lowering

pytestmark = pytest.mark.gpu

B, T = 4096, 300


@pytest.fixture(scope='module')
def games():
  yield from rg.registered('helper_games.py')


def _sprite_rows(env, chars):
  rows = []
  for s in (env.things[ch] for ch in chars):
    vp = getattr(s, 'virtual_position', s.position)
    rows.append([s.position[0], s.position[1], int(bool(s.visible)), vp[0], vp[1]])
  return rows


def _register_row(env, regs, keys):
  return ([int(getattr(env.things[ch], name)) for ch, name in regs] +
          [int(env.the_plot[key]) for key in keys])


@pytest.mark.parametrize('name', [n for n in gc.names('helper_') if n != 'helper_divzero'])
def test_facade_replays_helper_golden(games, name):
  g = gc.load(name)
  game, level = bytes(g['game']).decode(), int(g['level'][0])
  np.random.seed(int(g['rng_seed'][0]))
  sprites, registers = [], []

  def on_frame(env, out):
    sprites.append(_sprite_rows(env, games.SPRITES[game]))
    registers.append(_register_row(env, games.REGISTERS[game], games.PLOT_KEYS[game]))
    for ch, attr in games.REGISTERS[game]:       # written back with the type it had: int
      assert type(getattr(env.things[ch], attr)) is int, (ch, attr)
    for key in games.PLOT_KEYS[game]:
      assert type(env.the_plot[key]) is int, key
  got = tj.run_trajectory(lambda: games.GAMES[game](level), g['actions'].tolist(),
                          on_frame=on_frame)
  tj.assert_same_trajectory(g, got, name)
  np.testing.assert_array_equal(g['sprites'], np.array(sprites))
  np.testing.assert_array_equal(g['registers'], np.array(registers).reshape(len(sprites), -1))
  _, key, pos = np.random.get_state()[:3]
  assert np.append(key, pos).astype(np.uint32).tolist() == g['numpy_words'].tolist()


def _register_check(lowered_by_env):
  """on_step for lockstep: every register word of the sampled envs' entities and the Plot
  against the oracle worlds."""
  def on_step(t, engine, worlds, outs):
    import torch
    ids = sorted(worlds)
    idx = torch.as_tensor(ids, device=engine.device)
    sprites = engine.sprites.index_select(0, idx).cpu().numpy()
    drapes = engine.drapes.index_select(0, idx).cpu().numpy()
    plot = engine.plot.index_select(0, idx).cpu().numpy()
    for k, e in enumerate(ids):
      w, game = worlds[e], lowered_by_env(e)
      assert w.error == 0
      for s, ch in enumerate(engine.sprite_chars):
        words = list(sprites[k, s, _lib.S_AUX2 if game.egocentric[s] else _lib.S_AUX0:])
        regs = w.things[ch].regs
        assert words[:len(regs)] == regs[:len(words)], (t, e, ch)
      for d, ch in enumerate(engine.drape_chars):
        if not game.drape_kind[d]:
          assert list(drapes[k, d]) == w.things[ch].regs, (t, e, ch)
      assert list(plot[k, _lib.P_AUX0:_lib.P_AUX0 + 4]) == w.plot.regs, (t, e)
  return on_step


def _sample(rs):
  return [int(e) for e in np.unique(np.concatenate(
      [[0, 1, B - 2, B - 1], rs.choice(np.arange(2, B - 2), 28, replace=False)]))]


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
  sample = _sample(rs)
  words = {e: ocompiled.seeded_words(lowered, seed + e) for e in sample}
  eng.its_showtime()
  n = sampled_check.lockstep(
      eng, lambda e: ocompiled.make_world(lowered, words[e]), sample, actions,
      curtains='X', sprites='P!:;^', pad_columns=True,
      on_step=_register_check(lambda e: lowered))
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
  sample = _sample(rs)
  n = sampled_check.lockstep(
      eng, lambda e: ocompiled.make_world(lowered), sample, actions, curtains=curtains,
      sprites=sprites, pad_columns=True, on_step=_register_check(lambda e: lowered))
  assert n == len(sample) * (T + 1)
  assert int((eng.error_codes() != 0).sum()) == 0


def test_facade_raises_zero_division_where_the_reference_did(games):
  g = gc.load('helper_divzero')
  engine = games.make_divzero()
  boards = [engine.its_showtime()[0].board.copy()]
  at = int(g['raised_at'][0])
  for a in g['actions'][:at].tolist():
    boards.append(engine.play(a)[0].board.copy())
  np.testing.assert_array_equal(g['boards'], np.array(boards))
  with pytest.raises(ZeroDivisionError):
    engine.play(int(g['actions'][at]))


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
