"""research/lp-rnn/cued_catch.py: a trial cue per episode-drawn pairing, every frame paid, and
reward noise from random.normalvariate.  Goldens are the shimmed reference's own trajectories
(tests/golden/cued_catch_*, made by tests/golden/make_golden.py; tests/example_games.py
replays them on the oracle); CPU: the oracle (oracle/cued_catch.py) in lock-step with the
live reference, lowering, fingerprints and the C boundary's refusals; GPU: the goldens
through the facade, batched auto-reset runs whose pairings, trials and noise are drawn ON
THE DEVICE."""

import ctypes as C
import os
import random
import sys

import numpy as np
import pytest

import example_games as eg
import golden_cases as gc
import lp_rnn_cases as lc
import refdriver
import trajectory as tj
from oracle import cued_catch as occ
from oracle import sampled_check
from registered_games import global_generators  # noqa: F401  (a fixture)

NAMES = gc.names('cued_catch_')
REF = os.path.join(refdriver.REFERENCE_ROOT, 'pycolab', 'examples', 'research', 'lp-rnn',
                   'cued_catch.py')


def test_goldens_cover_the_rules():
  assert len(NAMES) >= 7
  gs = [gc.load(n) for n in NAMES]
  cfgs = [gc.config_of(g)['args'] for g in gs]
  assert any(a[:6] == [10, 10, 100, False, 0.0, 40] for a in cfgs)       # the paper's
  assert any(a[3] for a in cfgs) and any(a[4] > 0 for a in cfgs) and any(a[5] > 0 for a in cfgs)
  types = np.concatenate([g['reward_type'] for g in gs])
  assert (types == 1).any() and (types == 2).any()
  acts = np.concatenate([g['actions'] for g in gs])
  assert (acts == 0).any() and (acts == 4).any()
  small = [g for g in gs if g['art'].shape[0] < 7]
  assert small and small[0]['art'].shape[1] % 4 and (small[0]['art'][0] == ord('Q')).any()


@pytest.mark.skipif(not refdriver.available(), reason='/root/reference not present')
@pytest.mark.parametrize('case', [((4, 3, 6, False, 0.0, 2), 0), ((2, 2, 9, True, 0.7, 1), 4),
                                  ((1, 5, 4, False, 2.0, 0), 0)])
def test_oracle_lockstep_with_reference(case):
  """Every frame: board, float64 reward bits and type, discount, game over and the game's
  state; the shimmed reference draws from the global `random`, the oracle from a
  random.Random with the same seed."""
  args, quit_action = case
  ref = lc.ref_module('cued_catch')
  seed = 31 + args[2]
  random.seed(seed)
  rng = random.Random(seed)
  mk_ref = lambda: lc.shim_cued_catch(ref.make_game(*args))
  mk_or = lambda: occ.make_cued_catch(ref.GAME_ART, *args, rng=rng)
  policy = lc.cued_catch_policy(np.random.RandomState(seed), quit_every=89,
                                quit_action=quit_action or 4)
  a_env, b_env = mk_ref(), mk_or()
  a, b = a_env.its_showtime(), b_env.its_showtime()
  for t in range(400):
    assert np.array_equal(a[0].board, b[0]), t
    assert tj.reward_type(a[1]) == tj.reward_type(b[1]), t
    assert np.float64(a[1]).view(np.int64) == np.float64(b[1]).view(np.int64), (t, a[1], b[1])
    assert a[2] == b[2] and a_env.game_over == b_env.game_over, t
    assert lc.cued_catch_state(a_env) == lc.oracle_cued_catch_state(b_env), t
    if a_env.game_over:
      a_env, b_env = mk_ref(), mk_or()
      a, b = a_env.its_showtime(), b_env.its_showtime()
    else:
      act = policy(a_env)
      a, b = a_env.play(act), b_env.play(act)
  assert random.getstate() == rng.getstate()


@pytest.mark.skipif(not refdriver.available(), reason='/root/reference not present')
def test_reference_needs_the_shim():
  """Unshimmed, the reference raises on the first frame after the programming phase."""
  ref = lc.ref_module('cued_catch')
  random.seed(0)
  env = ref.make_game(1, 2, 3)
  env.its_showtime()
  with pytest.raises(TypeError):
    for _ in range(10):
      env.play(3)


def _lower(args=(3, 2, 5), art=None, seed=0, **kw):
  from pycolab_b200 import lowering
  from pycolab_b200.games import cued_catch
  random.seed(seed)
  return lowering.lower(cued_catch.make_game(*args, art=art, **kw))


def test_cued_catch_lowers_and_validates_on_cpu():
  from pycolab_b200 import _lib
  game = _lower((3, 2, 5), reward_sigma=0.5, reward_free_trials=2)
  assert game.program == _lib.PROG_CUED_CATCH and game.sprite_chars == 'Pab'
  assert game.float_reward and game.rng_streams == ('python',) and game.rng_from_globals
  assert game.program_arg[:4] == [1, 3, 2, 0]
  assert np.array(game.program_arg[6:8], np.int32).view(np.float64)[0] == random.NV_MAGICCONST
  assert not _lower((3, 2, 5)).float_reward
  assert not _lower((3, 2, 5), reward_sigma=-0.0).float_reward
  lib = _lib.load()
  handle = C.c_void_p()
  spec = game.make_spec(True)
  assert lib.pcl_create(C.byref(spec), 4, -1, C.byref(handle)) == _lib.OK
  lib.pcl_destroy(handle)
  for word, value, status in ((1, 0, _lib.ERR_INVALID), (0, 0, _lib.ERR_INVALID),
                              (3, 4, _lib.ERR_INVALID)):
    spec = game.make_spec(True)
    spec.program_arg[word] = value
    assert lib.pcl_create(C.byref(spec), 4, -1, C.byref(handle)) == status, (word, value)
  spec = game.make_spec(True)
  spec.rows = 33
  assert lib.pcl_create(C.byref(spec), 4, -1, C.byref(handle)) == _lib.ERR_UNSUPPORTED
  spec = game.make_spec(True)
  spec.sprite_confined[0] = 0
  assert lib.pcl_create(C.byref(spec), 4, -1, C.byref(handle)) == _lib.ERR_UNSUPPORTED


def test_cued_catch_refusals():
  from pycolab_b200 import levels
  from pycolab_b200.errors import NotLoweredError
  with pytest.raises(NotLoweredError):
    _lower((0, 2, 5))                              # upstream divides by it
  with pytest.raises(NotLoweredError):
    _lower(art=levels.cued_catch_art(33, 12))
  with pytest.raises(NotLoweredError):
    _lower(art=levels.cued_catch_art(7, 65))
  assert _lower(art=levels.cued_catch_art(32, 64)).rows == 32


def test_c_boundary_statuses():
  """Without a generator the handle cannot bind (update() draws every trial); the float64
  variant refuses the int32 host and hand-off paths, the int32 one takes them.  All refused
  or accepted before anything reaches a device."""
  from pycolab_b200 import _lib
  lib = _lib.load()
  fake = 0x1000
  for sigma, host_status in ((0.5, _lib.ERR_UNSUPPORTED), (0.0, None)):
    game = _lower(reward_sigma=sigma)
    spec = game.make_spec(True)
    handle = C.c_void_p()
    assert lib.pcl_create(C.byref(spec), 2, -1, C.byref(handle)) == _lib.OK
    st = _lib.State()
    st.d_backdrop = st.d_plot = st.d_plot_init = st.d_sprites = st.d_sprites_init = fake
    st.d_drapes = st.d_drapes_init = fake
    st.d_bits[0] = st.d_bits_init[0] = fake
    st.bits_bstride[0] = 14
    try:
      assert lib.pcl_bind_state(handle, C.byref(st)) == _lib.ERR_INVALID
      st.d_rng = fake
      assert lib.pcl_bind_state(handle, C.byref(st)) == _lib.OK
      out = _lib.Outputs(fake, fake, fake, fake, fake)
      if host_status is not None:
        assert lib.pcl_step(handle, fake, C.byref(out), None) == _lib.ERR_INVALID
        out.d_reward_f64 = fake
        assert lib.pcl_step_host(handle, fake, fake, C.byref(out), fake, fake, fake, fake, fake,
                                 None) == host_status
        assert lib.pcl_pack_handoff(handle, fake, 81, C.byref(out), fake,
                                    None) == _lib.ERR_UNSUPPORTED
    finally:
      lib.pcl_destroy(handle)


@pytest.mark.skipif(not refdriver.available(), reason='/root/reference not present')
def test_reference_cued_catch_file_lowers_like_the_twin():
  from pycolab_b200 import compat, lowering
  from pycolab_b200.games import cued_catch
  saved = {k: v for k, v in sys.modules.items() if k == 'pycolab' or k.startswith('pycolab.')}
  compat.uninstall()
  try:
    mod = compat.load_example(REF)
    for args in ((10, 10, 100), (2, 3, 7, True, 0.5, 3)):
      random.seed(11)
      a = lowering.lower(mod.make_game(*args))
      random.seed(11)
      b = lowering.lower(cued_catch.make_game(*args, art=mod.GAME_ART))
      assert a.signature() == b.signature()
      for field in ('backdrop', 'sprites', 'drapes', 'plot'):
        np.testing.assert_array_equal(getattr(a, field), getattr(b, field), err_msg=field)
      np.testing.assert_array_equal(a.bits[0], b.bits[0])
  finally:
    compat.uninstall()
    sys.modules.update(saved)


@pytest.mark.skipif(not refdriver.available(), reason='/root/reference not present')
@pytest.mark.parametrize('edit', [('the_plot.add_reward(0)', 'the_plot.add_reward(1)'),
                                  ('self.position.col - 1', 'self.position.col - 2')])
def test_edited_cued_catch_copy_is_refused(tmp_path, edit):
  from pycolab_b200 import compat, lowering
  from pycolab_b200.errors import NotLoweredError
  src = open(REF).read()
  edited = src.replace(*edit)
  assert edited != src
  path = tmp_path / 'cued_catch.py'
  path.write_text(edited)
  saved = {k: v for k, v in sys.modules.items() if k == 'pycolab' or k.startswith('pycolab.')}
  compat.uninstall()
  try:
    mod = compat.load_example(str(path))
    with pytest.raises(NotLoweredError):
      lowering.lower(mod.make_game(2, 2, 3))
  finally:
    compat.uninstall()
    sys.modules.update(saved)


# ------------------------------------------------------------------------------------ GPU --

@pytest.mark.gpu
@pytest.mark.parametrize('name', NAMES)
def test_facade_cued_catch_golden(global_generators, name):  # noqa: F811
  """B = 1 facade: the twin's CueDrape draws the pairings from the global `random`, the device
  continues that stream in update() and hands it back after every step; every array of the
  golden frame by frame, and the global generator's state at the end."""
  eg.assert_replays('facade', name)
  # the oracle, drawing from its own Random(seed), ends where the global generator does
  g = gc.load(name)
  cfg = gc.config_of(g)
  art, rng = tj.u8_to_art(g['art']), random.Random(cfg['seed'])
  tj.run_trajectory(lambda: occ.make_cued_catch(art, *cfg['args'], rng=rng),
                    g['actions'].tolist())
  assert random.getstate() == rng.getstate()


def _batched_vs_oracle(B, T, seed, args, art, check_envs=None, policy_seed=3, curtains=''):
  import torch
  from pycolab_b200 import batched
  from pycolab_b200.games import cued_catch
  random.seed(0)
  eng = batched.BatchedEngine([cued_catch.make_game(*args, art=art)], batch=B, rng_seed=seed)
  assert eng.rng is not None
  assert eng.reward.dtype == (torch.float64 if args[4] else torch.int32)
  envs = range(B) if check_envs is None else check_envs
  rngs = {e: random.Random(seed + e) for e in envs}
  eng.its_showtime()
  rs = np.random.RandomState(policy_seed)
  policy = np.array([rs.choice([1, 2, 3, 0, 4], size=B, p=[.45, .45, .094, .003, .003])
                     for _ in range(T)], np.int32)
  episodes, floats = [0], [0]

  def count(t, eng, worlds, outs):
    for e, w in worlds.items():
      episodes[0] += int(t < T and w.game_over)
      floats[0] += int(isinstance(outs[e][1], float))
  sampled_check.lockstep(eng, lambda e: occ.make_cued_catch(art, *args, rng=rngs[e]), envs,
                         policy, on_step=count, curtains=curtains, sprites='P')
  assert int(eng.error_codes().abs().max()) == 0
  return eng, episodes[0], floats[0], rngs


@pytest.mark.gpu
@pytest.mark.parametrize('args', [(2, 2, 6, False, 0.0, 1), (1, 3, 4, True, 0.0, 0),
                                  (3, 2, 5, False, 0.8, 2)])
def test_batched_cued_catch_device_draws_vs_oracle(args):
  from pycolab_b200 import levels
  eng, episodes, floats, rngs = _batched_vs_oracle(24, 300, 70, args, levels.cued_catch_art(),
                                                   curtains='Q')
  assert episodes > 24
  assert (floats > 0) == (args[4] > 0)
  words = eng.rng.cpu().numpy().view(np.uint32).reshape(24, -1)
  for e in range(24):       # the device's stream ends where each env's Random does
    assert tuple(int(w) for w in words[e]) == rngs[e].getstate()[1], e


@pytest.mark.gpu
def test_batched_cued_catch_sampled_at_4096():
  from pycolab_b200 import levels
  art = levels.cued_catch_art(5, 14, player=(1, 2), balls=((1, 9), (2, 12)),
                              cue_cells=((0, 0), (0, 13), (2, 7)))
  _batched_vs_oracle(4096, 150, 5, (2, 2, 6, True, 0.3, 1), art,
                     check_envs=[0, 1, 2, 777, 2048, 3001, 4094, 4095], curtains='Q')


@pytest.mark.gpu
def test_cued_catch_normalvariate_matches_cpython():
  """At least 10^5 random.normalvariate calls on the device against CPython's own: every
  paid frame's float64 bits, and each env's generator words at the end."""
  import torch
  from pycolab_b200 import batched, levels
  from pycolab_b200.games import cued_catch
  B, T, seed = 2048, 400, 1000
  args = (1, 1, 10 ** 6, False, 1.25, 0)           # every frame in the ball column pays noise
  art = levels.cued_catch_art(7, 12, player=(1, 3), balls=((1, 3), (1, 3)))
  random.seed(0)
  eng = batched.BatchedEngine([cued_catch.make_game(*args, art=art)], batch=B, rng_seed=seed)
  eng.its_showtime()
  actions = torch.full((T, B), 3, dtype=torch.int32, device=eng.device)
  got = []
  for t in range(T):
    eng.play(actions[t])
    got.append(eng.reward.cpu().numpy().copy())
  got = np.stack(got)
  worlds = [occ.make_cued_catch(art, *args, rng=random.Random(seed + e)) for e in range(B)]
  calls = 0
  want = np.zeros((T, B))
  for e, w in enumerate(worlds):
    w.its_showtime()
    for t in range(T):
      r = w.play(3)[1]
      want[t, e] = r
      calls += isinstance(r, float)
  assert calls >= 10 ** 5
  np.testing.assert_array_equal(got.view(np.int64), want.view(np.int64))
  words = eng.rng.cpu().numpy().view(np.uint32).reshape(B, -1)
  for e in (0, 1, B - 1):
    assert tuple(int(x) for x in words[e]) == worlds[e].things['Q'].aux['rng'].getstate()[1]


@pytest.mark.gpu
def test_cued_catch_masked_reset_and_layers():
  import torch
  from oracle import engine_model as em
  from pycolab_b200 import batched, levels
  from pycolab_b200.games import cued_catch
  art = levels.cued_catch_art(6, 10, player=(1, 2), balls=((1, 7), (2, 5)), cue_cells=((0, 1),))
  args = (1, 2, 3, True, 0.0, 0)
  random.seed(0)
  eng = batched.BatchedEngine([cued_catch.make_game(*args, art=art)], batch=4, rng_seed=40,
                              auto_reset=False)
  rngs = [random.Random(40 + e) for e in range(4)]
  worlds = [occ.make_cued_catch(art, *args, rng=r) for r in rngs]
  for w in worlds:
    w.its_showtime()
  eng.its_showtime()
  for t in range(12):
    act = [1, 2, 3, 2][t % 4]
    eng.play(torch.full((4,), act, dtype=torch.int32).cuda())
    for w in worlds:
      if not w.game_over:
        w.play(act)
    if t == 6:                                     # rebuild envs 1 and 3 only
      eng.reset(torch.tensor([0, 1, 0, 1], dtype=torch.uint8))
      for e in (1, 3):
        worlds[e] = occ.make_cued_catch(art, *args, rng=rngs[e])
        worlds[e].its_showtime()
    boards = eng.board.cpu().numpy()
    layers = eng.unoccluded_layers('PabQ ').cpu().numpy()
    for e, w in enumerate(worlds):
      np.testing.assert_array_equal(boards[e], w.board, 'board env %d step %d' % (e, t))
      np.testing.assert_array_equal(eng.curtain('Q')[e].cpu().numpy(), w.things['Q'].curtain)
      want = em.unoccluded_layers_of(w.backdrop, w.things, 'PabQ ')
      for k, ch in enumerate('PabQ '):
        np.testing.assert_array_equal(layers[e, k], want[ch], '%s env %d step %d' % (ch, e, t))


@pytest.mark.gpu
def test_cued_catch_host_buffer_steps():
  """pcl_step_host serves the int32 variant; the float64 one is refused there."""
  import torch
  from pycolab_b200 import _lib, batched, levels
  from pycolab_b200.games import cued_catch
  art = levels.cued_catch_art()
  random.seed(0)
  eng = batched.BatchedEngine([cued_catch.make_game(2, 2, 4, art=art)], batch=8, rng_seed=3)
  ref = batched.BatchedEngine([cued_catch.make_game(2, 2, 4, art=art)], batch=8, rng_seed=3)
  eng.its_showtime()
  ref.its_showtime()
  rs = np.random.RandomState(0)
  for _ in range(60):
    acts = rs.randint(1, 4, size=8).astype(np.int32)
    board, reward, has, disc, done = eng.play_host(acts)
    r = ref.play(torch.from_numpy(acts).cuda())
    np.testing.assert_array_equal(board, r.board.cpu().numpy())
    np.testing.assert_array_equal(reward, r.reward.cpu().numpy())
    np.testing.assert_array_equal(done, r.done.cpu().numpy())
  noisy = batched.BatchedEngine([cued_catch.make_game(2, 2, 4, reward_sigma=0.5, art=art)],
                                batch=8, rng_seed=3)
  noisy.its_showtime()
  with pytest.raises(_lib.PclError) as err:
    noisy.play_host(np.ones(8, np.int32))
  assert err.value.status == _lib.ERR_UNSUPPORTED
