"""research/lp-rnn/sequence_recall.py: a light sequence drawn per episode, a program counter
over _make_program's states, and float64 rewards.  Goldens are the shimmed reference's own
trajectories (tests/golden/sequence_recall_*, made by tests/golden/make_golden.py and
replayed on the oracle and the facade by tests/example_games.py); CPU: the oracle
(oracle/sequence_recall.py) in lock-step with the live reference, lowering, fingerprints (the
classes and _make_program) and refusals; GPU: batched auto-reset runs whose sequences are
drawn ON THE DEVICE."""

import ctypes as C
import os
import random
import sys

import numpy as np
import pytest

import golden_cases as gc
import lp_rnn_cases as lc
import refdriver
from oracle import sampled_check
from oracle import sequence_recall as osr

NAMES = gc.names('sequence_recall_')
REF = os.path.join(refdriver.REFERENCE_ROOT, 'pycolab', 'examples', 'research', 'lp-rnn',
                   'sequence_recall.py')


def test_goldens_cover_the_rules():
  assert len(NAMES) >= 7
  gs = [gc.load(n) for n in NAMES]
  cfgs = [gc.config_of(g)['args'] for g in gs]
  rewards = np.concatenate([g['reward_f64'] for g in gs])
  assert (rewards == 0.995).any() and (rewards == -0.005).any()
  assert {1, 16} <= {a[0] for a in cfgs}
  assert any(a[3] == 0 for a in cfgs) and any(a[1] == 1 or a[2] == 1 for a in cfgs)
  assert any(a[1] == 2 or a[2] == 2 for a in cfgs) and any(a[4] > 0 for a in cfgs)
  acts = np.concatenate([g['actions'] for g in gs])
  assert (acts == 0).any() and (acts == 6).any()
  assert len({g['art'].shape for g in gs}) >= 2
  # a SEEK on the wrong pad pays 0.0: the frame sums to -0.005 with the light turned on
  assert any(((g['state'][1:, 0] < g['state'][:-1, 0]) & (g['reward_f64'][1:] == -0.005)).any()
             for g in gs)


@pytest.mark.skipif(not refdriver.available(), reason='/root/reference not present')
@pytest.mark.parametrize('args', [(3, 2, 2, 1, -1), (2, 1, 1, 0, 30), (6, 3, 1, 2, -1)])
def test_oracle_lockstep_with_reference(args):
  ref = lc.ref_module('sequence_recall')
  seed = 17 + args[0]
  random.seed(seed)
  rng = random.Random(seed)
  mk_ref = lambda: lc.shim_sequence_recall(ref.make_game(*args))
  mk_or = lambda: osr.make_sequence_recall(ref.GAME_ART, *args, rng=rng)
  policy = lc.sequence_recall_policy(np.random.RandomState(seed), (8, 10), wrong=0.2,
                                     quits=((150, 6),))
  a_env, b_env = mk_ref(), mk_or()
  a, b = a_env.its_showtime(), b_env.its_showtime()
  for t in range(300):
    assert np.array_equal(a[0].board, b[0]), t
    assert (a[1] is None) == (b[1] is None) and (
        a[1] is None or np.float64(a[1]).view(np.int64) == np.float64(b[1]).view(np.int64)), t
    assert a[2] == b[2] and a_env.game_over == b_env.game_over, t
    assert lc.sequence_recall_state(a_env) == lc.sequence_recall_state(b_env), t
    if a_env.game_over:
      a_env, b_env = mk_ref(), mk_or()
      a, b = a_env.its_showtime(), b_env.its_showtime()
    else:
      act = policy(a_env)
      a, b = a_env.play(act), b_env.play(act)
  assert random.getstate() == rng.getstate()


@pytest.mark.skipif(not refdriver.available(), reason='/root/reference not present')
def test_reference_needs_the_shim():
  """Unshimmed, the reference raises on the first frame that turns a light on."""
  ref = lc.ref_module('sequence_recall')
  random.seed(0)
  env = ref.make_game(1, 1, 1, 1)
  env.its_showtime()
  with pytest.raises(TypeError):
    for _ in range(10):
      env.play(5)


def _lower(args=(3, 2, 2, 1, -1), art=None, seed=0):
  from pycolab_b200 import lowering
  from pycolab_b200.games import sequence_recall
  random.seed(seed)
  return lowering.lower(sequence_recall.make_game(*args, art=art))


def test_sequence_recall_lowers_and_validates_on_cpu():
  from pycolab_b200 import _lib
  game = _lower((5, 60, 30, 0, 200))
  assert game.program == _lib.PROG_SEQUENCE_RECALL and game.drape_chars == 'M%'
  assert game.float_reward and game.rng_streams == ('python',) and not game.rng_from_globals
  assert game.program_arg[:4] == [5, 60, 30, 1]
  assert game.plot[_lib.P_AUX2] == 200
  assert _lower((2, 1, 1, 1, -1)).plot[_lib.P_AUX2] == _lib.SEQUENCE_RECALL_NO_TIMEOUT
  random.seed(0)
  want = [random.choice('1234') for _ in range(5)]
  word = int(np.int32(game.plot[_lib.P_AUX3]).view(np.uint32))
  assert [(word >> (2 * k)) & 3 for k in range(5)] == ['1234'.index(g) for g in want]
  lib = _lib.load()
  handle = C.c_void_p()
  spec = game.make_spec(True)
  assert lib.pcl_create(C.byref(spec), 4, -1, C.byref(handle)) == _lib.OK
  lib.pcl_destroy(handle)
  for word, value, status in ((0, 0, _lib.ERR_UNSUPPORTED), (0, 17, _lib.ERR_UNSUPPORTED),
                              (3, 0, _lib.ERR_INVALID)):
    spec = game.make_spec(True)
    spec.program_arg[word] = value
    assert lib.pcl_create(C.byref(spec), 4, -1, C.byref(handle)) == status, (word, value)
  spec = game.make_spec(True)
  spec.cols = 65
  spec.pitch = 80
  assert lib.pcl_create(C.byref(spec), 4, -1, C.byref(handle)) == _lib.ERR_UNSUPPORTED


def test_sequence_recall_refusals():
  from pycolab_b200 import levels
  from pycolab_b200.errors import NotLoweredError
  for length in (0, 17):
    with pytest.raises(NotLoweredError):
      _lower((length, 2, 2, 1, -1))
  art = levels.sequence_recall_art(9, 13)
  with pytest.raises(NotLoweredError):              # upstream raises KeyError on '~'
    _lower(art=[art[0]] + [art[1][:2] + '~' + art[1][3:]] + art[2:])
  with pytest.raises(NotLoweredError):
    _lower(art=[art[0]] + [art[1][:2] + 'M' + art[1][3:]] + art[2:])
  with pytest.raises(NotLoweredError):
    _lower(art=levels.sequence_recall_art(33, 21))
  assert _lower(art=levels.sequence_recall_art(32, 64)).cols == 64
  assert _lower((16, 1, 1, 1, -1)).program_arg[0] == 16


def test_c_boundary_statuses():
  """Float64 rewards: the int32 host and hand-off paths are refused, pcl_step without
  d_reward_f64 is invalid; both drapes' bit rows are required.  No device is touched."""
  from pycolab_b200 import _lib
  lib = _lib.load()
  fake = 0x1000
  game = _lower()
  spec = game.make_spec(True)
  handle = C.c_void_p()
  assert lib.pcl_create(C.byref(spec), 2, -1, C.byref(handle)) == _lib.OK
  st = _lib.State()
  st.d_backdrop = st.d_plot = st.d_plot_init = st.d_sprites = st.d_sprites_init = fake
  st.d_drapes = st.d_drapes_init = fake
  st.d_bits[0] = st.d_bits_init[0] = fake
  st.bits_bstride[0] = st.bits_bstride[1] = 34
  try:
    assert lib.pcl_bind_state(handle, C.byref(st)) == _lib.ERR_INVALID
    st.d_bits[1] = st.d_bits_init[1] = fake
    assert lib.pcl_bind_state(handle, C.byref(st)) == _lib.OK
    out = _lib.Outputs(fake, fake, fake, fake, fake)
    assert lib.pcl_step(handle, fake, C.byref(out), None) == _lib.ERR_INVALID
    out.d_reward_f64 = fake
    assert lib.pcl_step_host(handle, fake, fake, C.byref(out), fake, fake, fake, fake, fake,
                             None) == _lib.ERR_UNSUPPORTED
    assert lib.pcl_pack_handoff(handle, fake, 81, C.byref(out), fake, None) == _lib.ERR_UNSUPPORTED
  finally:
    lib.pcl_destroy(handle)


@pytest.mark.skipif(not refdriver.available(), reason='/root/reference not present')
def test_reference_sequence_recall_file_lowers_like_the_twin():
  from pycolab_b200 import compat, lowering
  from pycolab_b200.games import sequence_recall
  saved = {k: v for k, v in sys.modules.items() if k == 'pycolab' or k.startswith('pycolab.')}
  compat.uninstall()
  try:
    mod = compat.load_example(REF)
    for args in ((), (2, 1, 1, 0, 50)):
      random.seed(11)
      a = lowering.lower(mod.make_game(*args))
      random.seed(11)
      b = lowering.lower(sequence_recall.make_game(*args, art=mod.GAME_ART))
      assert a.signature() == b.signature()
      for field in ('backdrop', 'sprites', 'drapes', 'plot'):
        np.testing.assert_array_equal(getattr(a, field), getattr(b, field), err_msg=field)
      for d in (0, 1):
        np.testing.assert_array_equal(a.bits[d], b.bits[d])
  finally:
    compat.uninstall()
    sys.modules.update(saved)


@pytest.mark.skipif(not refdriver.available(), reason='/root/reference not present')
@pytest.mark.parametrize('edit', [("random.choice('1234')", "random.choice('1123')"),
                                  ('the_plot.add_reward(-0.005)', 'the_plot.add_reward(-0.01)')])
def test_edited_sequence_recall_copy_is_refused(tmp_path, edit):
  from pycolab_b200 import compat, lowering
  from pycolab_b200.errors import NotLoweredError
  src = open(REF).read()
  edited = src.replace(*edit)
  assert edited != src
  path = tmp_path / 'sequence_recall.py'
  path.write_text(edited)
  saved = {k: v for k, v in sys.modules.items() if k == 'pycolab' or k.startswith('pycolab.')}
  compat.uninstall()
  try:
    mod = compat.load_example(str(path))
    with pytest.raises(NotLoweredError):
      lowering.lower(mod.make_game())
  finally:
    compat.uninstall()
    sys.modules.update(saved)


# ------------------------------------------------------------------------------------ GPU --

def _batched_vs_oracle(B, T, seed, args, arts, check_envs=None, policy_seed=3):
  from pycolab_b200 import batched
  from pycolab_b200.games import sequence_recall
  random.seed(0)
  games = [sequence_recall.make_game(*args, art=a) for a in arts]
  eng = batched.BatchedEngine(games, batch=B, rng_seed=seed)
  assert eng.rng is not None
  envs = range(B) if check_envs is None else check_envs
  rngs = {e: random.Random(seed + e) for e in envs}
  eng.its_showtime()
  rs = np.random.RandomState(policy_seed)
  policy = np.array([rs.choice([1, 2, 3, 4, 5, 0, 6], size=B,
                               p=[.24, .24, .24, .24, .02, .01, .01]) for _ in range(T)], np.int32)
  episodes, paid = [0], set()

  def count(t, eng, worlds, outs):
    for e, w in worlds.items():
      episodes[0] += int(t < T and w.game_over)
      if outs[e][1] is not None:
        paid.add(round(float(outs[e][1]), 3))
  sampled_check.lockstep(eng, lambda e: osr.make_sequence_recall(arts[e % len(arts)], *args,
                                                                 rng=rngs[e]),
                         envs, policy, on_step=count, curtains='M%', sprites='P')
  assert int(eng.error_codes().abs().max()) == 0
  return eng, episodes[0], paid


@pytest.mark.gpu
@pytest.mark.parametrize('args,shape', [((2, 1, 1, 0, 60), (17, 21)), ((4, 2, 3, 1, 90), (9, 13)),
                                        ((1, 2, 1, 2, -1), (17, 21)),
                                        ((16, 1, 1, 1, 200), (9, 13))])
def test_batched_sequence_recall_device_draws_vs_oracle(args, shape):
  from pycolab_b200 import levels
  eng, episodes, paid = _batched_vs_oracle(24, 400, 70, args, [levels.sequence_recall_art(*shape)])
  assert episodes > 24 and -0.005 in paid


@pytest.mark.gpu
def test_batched_sequence_recall_sampled_at_4096():
  from pycolab_b200 import levels
  _batched_vs_oracle(4096, 200, 5, (3, 1, 2, 1, 80), [levels.sequence_recall_art(32, 64)],
                     check_envs=[0, 1, 2, 777, 2048, 3001, 4094, 4095])


@pytest.mark.gpu
def test_sequence_recall_masked_reset_and_layers():
  import torch
  from oracle import engine_model as em
  from pycolab_b200 import batched, levels
  art = levels.sequence_recall_art(9, 13)
  args = (2, 1, 2, 1, -1)
  from pycolab_b200.games import sequence_recall
  random.seed(0)
  eng = batched.BatchedEngine([sequence_recall.make_game(*args, art=art)], batch=4, rng_seed=40,
                              auto_reset=False)
  rngs = [random.Random(40 + e) for e in range(4)]
  worlds = [osr.make_sequence_recall(art, *args, rng=r) for r in rngs]
  for w in worlds:
    w.its_showtime()
  eng.its_showtime()
  chars = 'MP%#1234 '
  for t in range(30):
    act = [1, 2, 3, 4, 2, 1][t % 6]
    eng.play(torch.full((4,), act, dtype=torch.int32).cuda())
    for w in worlds:
      if not w.game_over:
        w.play(act)
    if t == 12:
      eng.reset(torch.tensor([1, 0, 0, 1], dtype=torch.uint8))
      for e in (0, 3):
        worlds[e] = osr.make_sequence_recall(art, *args, rng=rngs[e])
        worlds[e].its_showtime()
    boards = eng.board.cpu().numpy()
    layers = eng.unoccluded_layers(chars).cpu().numpy()
    for e, w in enumerate(worlds):
      np.testing.assert_array_equal(boards[e], w.board, 'board env %d step %d' % (e, t))
      want = em.unoccluded_layers_of(w.backdrop, w.things, chars)
      for k, ch in enumerate(chars):
        np.testing.assert_array_equal(layers[e, k], want[ch], '%s env %d step %d' % (ch, e, t))
