"""GPU tests of plain Sprites on the compiled step program (csrc/compiled.cu): the games of
tests/sprite_games.py on the H100, against the reference's trajectories
(tests/golden/sprite_*.npz) and the oracle interpreter (oracle/compiled.py)."""

import numpy as np
import pytest

import golden_cases as gc
import registered_games as rg
import trajectory as tj
from oracle import compiled as ocompiled
from oracle import engine_model as em
from oracle import sampled_check
from pycolab_b200 import _lib, lowering, rendering
from pycolab_b200 import things as b_things

pytestmark = pytest.mark.gpu

B, T = 4096, 300


@pytest.fixture(scope='module')
def games():
  yield from rg.registered('sprite_games.py')


def _sprite_rows(env, chars):
  rows = []
  for s in (env.things[ch] for ch in chars):
    vp = getattr(s, 'virtual_position', s.position)
    rows.append([s.position[0], s.position[1], int(bool(s.visible)), vp[0], vp[1]])
  return rows


def _register_row(env, regs, keys):
  out = []
  for ch, name in regs:
    value = getattr(env.things[ch], name)
    out += [int(x) for x in value] if isinstance(value, tuple) else [int(value)]
  return out + [int(env.the_plot[key]) for key in keys]


@pytest.mark.parametrize('name', [n for n in gc.names('sprite_') if n != 'sprite_fallen'])
def test_facade_replays_sprite_golden(games, name):
  g = gc.load(name)
  game, level = bytes(g['game']).decode(), int(g['level'][0])
  np.random.seed(int(g['rng_seed'][0]))
  sprites, registers = [], []
  types = {('o', '_serve'): b_things.Sprite.Position, ('w', '_home'): b_things.Sprite.Position,
           ('x', '_mark'): tuple, ('o', 'dy'): int, ('w', 'seen'): int}

  def on_frame(env, out):
    sprites.append(_sprite_rows(env, games.SPRITES[game]))
    registers.append(_register_row(env, games.REGISTERS[game], games.PLOT_KEYS[game]))
    for (ch, name), t in types.items():        # written back with the type it had
      if ch in env.things:
        assert type(getattr(env.things[ch], name)) is t, (ch, name)
  got = tj.run_trajectory(lambda: games.GAMES[game](level), g['actions'].tolist(),
                          on_frame=on_frame)
  tj.assert_same_trajectory(g, got, name)
  np.testing.assert_array_equal(g['sprites'], np.array(sprites))
  np.testing.assert_array_equal(g['registers'], np.array(registers).reshape(len(sprites), -1))
  _, key, pos = np.random.get_state()[:3]
  assert np.append(key, pos).astype(np.uint32).tolist() == g['numpy_words'].tolist()


def test_facade_raises_index_error_where_the_reference_did(games):
  g = gc.load('sprite_fallen')
  engine = games.make_fallen()
  boards = [engine.its_showtime()[0].board.copy()]
  at = int(g['raised_at'][0])
  for a in g['actions'][:at].tolist():
    boards.append(engine.play(a)[0].board.copy())
  np.testing.assert_array_equal(g['boards'], np.array(boards))
  with pytest.raises(IndexError):
    engine.play(int(g['actions'][at]))


def _plain_check(lowered_by_env, extra=None):
  """on_step for lockstep: each plain Sprite's row, col and visible bit, every register
  word, and the un-occluded layers, against the oracle worlds."""
  def on_step(t, engine, worlds, outs):
    import torch
    ids = sorted(worlds)
    idx = torch.as_tensor(ids, device=engine.device)
    sprites = engine.sprites.index_select(0, idx).cpu().numpy()
    drapes = engine.drapes.index_select(0, idx).cpu().numpy()
    plot = engine.plot.index_select(0, idx).cpu().numpy()
    layers = engine.unoccluded_layers(engine.chars).index_select(0, idx).cpu().numpy()
    for k, e in enumerate(ids):
      w, game = worlds[e], lowered_by_env(e)
      assert w.error == 0
      for s, ch in enumerate(engine.sprite_chars):
        ent, rec = w.things[ch], sprites[k, s]
        if (game.program_arg[3] >> s) & 1:
          assert [rec[0], rec[1], rec[4] & 1] == [ent.row, ent.col, int(bool(ent.visible))], (t, e, ch)
          words = list(rec[2:4]) + list(rec[5:])
        else:
          words = list(rec[_lib.S_AUX2 if game.egocentric[s] else _lib.S_AUX0:])
        assert words[:len(ent.regs)] == ent.regs[:len(words)], (t, e, ch)
      for d, ch in enumerate(engine.drape_chars):
        if not game.drape_kind[d]:
          assert list(drapes[k, d]) == w.things[ch].regs, (t, e, ch)
      assert list(plot[k, _lib.P_AUX0:_lib.P_AUX0 + 4]) == w.plot.regs, (t, e)
      want = em.unoccluded_layers_of(w.backdrop, w.things, engine.chars)
      for c, ch in enumerate(engine.chars):
        np.testing.assert_array_equal(layers[k, c], want[ch], err_msg=str((t, e, ch)))
    if extra is not None:
      extra(t, engine, worlds, outs)
  return on_step


def _sample(rs):
  return [int(e) for e in np.unique(np.concatenate(
      [[0, 1, B - 2, B - 1], rs.choice(np.arange(2, B - 2), 28, replace=False)]))]


def test_bounce_lockstep_against_the_oracle(games):
  """B = 4096, both levels, auto-reset: sampled envs every step, the bricks' curtain, the
  ball's words and registers, and the generators' words at the end."""
  from pycolab_b200 import batched
  seed = 30
  lowered = [lowering.lower(games.make_bounce(level)) for level in (0, 1)]
  eng = batched.BatchedEngine(lowered, batch=B, rng_seed=seed)
  rs = np.random.RandomState(7)
  actions = rs.randint(0, 4, size=(T, B)).astype(np.int32)
  sample = _sample(rs)
  words = {e: ocompiled.seeded_words(lowered[e % 2], seed + e) for e in sample}
  eng.its_showtime()
  n = sampled_check.lockstep(
      eng, lambda e: ocompiled.make_world(lowered[e % 2], words[e]), sample, actions,
      curtains='=', sprites='P', pad_columns=True,
      on_step=_plain_check(lambda e: lowered[e % 2]))
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
  sample = _sample(rs)
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
      on_step=_plain_check(lambda e: lowered[e % 2], render_check))
  assert n == len(sample) * (T + 1)
  assert seen['wrapped'] > 0 and seen['far'] > 0
  assert int((eng.error_codes() != 0).sum()) == 0


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
