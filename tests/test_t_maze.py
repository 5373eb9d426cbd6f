"""research/lp-rnn/t_maze.py: float64 rewards through the C ABI, five Scrollys that teleport
by np.roll, and a cue side plus a 191 x 77 speckle field drawn from two generators at every
(re)start.  Goldens are the reference's own trajectories on its own art
(tests/golden/t_maze_*, made by tests/golden/make_t_maze_golden.py); CPU: the oracle
(oracle/t_maze.py) in lock-step with the imported reference and against
the goldens, lowering and the C boundary's refusals; GPU: the goldens through the facade, and
batched auto-reset runs whose cue and speckle are drawn ON THE DEVICE from per-env streams."""

import ctypes as C
import importlib.util
import os
import random
import sys

import numpy as np
import pytest

import golden_cases as gc
import refdriver
import trajectory as tj
from oracle import engine_model as em
from oracle import games as ogames
from oracle import sampled_check
from oracle import t_maze as otm

NAMES = gc.names('t_maze_')


def _ref_module():
  refdriver._import()
  path = os.path.join(refdriver.REFERENCE_ROOT, 'pycolab', 'examples', 'research', 'lp-rnn',
                      't_maze.py')
  spec = importlib.util.spec_from_file_location('ref_t_maze_test', path)
  module = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(module)
  return module


def _oracle_maker(maze, cue, cfg, rng, np_rng):
  return lambda: otm.make_t_maze(maze, cue, cfg['level'], cfg['cue_after_teleport'],
                                    cfg['timeout_frames'], cfg['teleport_delay'],
                                    cfg['limbo_time'], rng, np_rng)


def _rewards(make_env, actions):
  """run_trajectory plus the float rewards (NaN = None)."""
  got = []
  traj = tj.run_trajectory(make_env, actions, on_frame=lambda env, out: got.append(
      np.nan if out[1] is None else float(out[1])))
  traj['reward_f64'] = np.array(got, dtype=np.float64)
  return traj


def _same_f64(want, got, label):
  np.testing.assert_array_equal(np.asarray(want).view(np.int64), np.asarray(got).view(np.int64),
                                err_msg=label)


def test_goldens_cover_the_rules():
  assert len(NAMES) >= 6
  rewards = np.concatenate([gc.load(n)['reward_f64'] for n in NAMES])
  assert (rewards == 0.999).any() and (rewards == -1.001).any() and (rewards == -0.001).any()
  cfgs = [gc.config_of(gc.load(n)) for n in NAMES]
  assert {c['cue_after_teleport'] for c in cfgs} == {False, True}
  assert {c['teleport_delay'] > 0 for c in cfgs} == {False, True}
  assert any(c['limbo_time'] > 0 for c in cfgs) and any(c['limbo_time'] <= 0 for c in cfgs)
  assert any(c['timeout_frames'] > 0 for c in cfgs)
  assert any(6 in gc.load(n)['actions'] for n in NAMES)


@pytest.mark.parametrize('name', NAMES)
def test_oracle_t_maze_matches_reference_golden(name):
  g = gc.load(name)
  cfg = gc.config_of(g)
  maze, cue = tj.u8_to_art(g['maze_art']), tj.u8_to_art(g['cue_art'])
  make = _oracle_maker(maze, cue, cfg, random.Random(cfg['seed']),
                       np.random.RandomState(cfg['seed']))
  got = _rewards(make, g['actions'].tolist())
  tj.assert_same_trajectory(g, got, name)
  _same_f64(g['reward_f64'], got['reward_f64'], name)


# (level, cue_after_teleport, timeout_frames, teleport_delay, limbo_time)
LOCKSTEP = [(0, False, -1, 0, 0), (1, True, 60, 5, 4), (2, False, -1, 5, 10), (3, True, -1, 0, 4),
            (4, False, 150, 0, 10), (5, True, -1, 5, 0), (2, True, -1, 0, 2), (1, False, -1, 5, 1)]


@pytest.mark.skipif(not refdriver.available(), reason='/root/reference not present')
@pytest.mark.parametrize('case', LOCKSTEP)
def test_oracle_lockstep_with_reference(case):
  """Every frame: board, float reward, discount, game over, the player and every plot entry
  the game keeps; the policy reaches both goals, quits and times out."""
  sys.path.insert(0, os.path.join(os.path.dirname(__file__), 'golden'))
  import make_t_maze_golden
  ref = _ref_module()
  level, cue_after, timeout, delay, limbo = case
  seed = 40 + level
  random.seed(seed)
  np.random.seed(seed)
  rng, np_rng = random.Random(seed), np.random.RandomState(seed)
  mk_ref = lambda: ref.make_game(level, cue_after, timeout, delay, limbo)
  mk_or = lambda: otm.make_t_maze(ref.MAZE_ART, ref.CUE_ART, level, cue_after, timeout, delay,
                                     limbo, rng, np_rng)
  actions = make_t_maze_golden.t_maze_policy(seed, limbo, 900)
  actions = [0 if i % 97 == 96 else a for i, a in enumerate(actions)]
  a_env, b_env = mk_ref(), mk_or()
  a, b = a_env.its_showtime(), b_env.its_showtime()
  seen = set()
  for t, act in enumerate(actions + [None]):
    assert np.array_equal(a[0].board, b[0]), t
    assert (a[1] is None) == (b[1] is None) and (a[1] is None or
                                                 np.float64(a[1]).view(np.int64) ==
                                                 np.float64(b[1]).view(np.int64)), (t, a[1], b[1])
    assert a[2] == b[2] and a_env.game_over == b_env.game_over, t
    assert tuple(a_env.things['P'].virtual_position) == b_env.things['P'].virtual_position, t
    for key in ('timeout_frames', 'teleportation_order_frame', 'teleportation_order',
                'yo_we_have_teleported'):
      assert a_env.the_plot.get(key) == b_env.plot.store.get(key), (t, key)
    assert a_env.things['Q'].which_goal == b_env.things['Q'].aux['which_goal']
    if a[1] is not None:
      seen.add(round(float(a[1]), 3))
    if act is None:
      break
    if a_env.game_over:
      a_env, b_env = mk_ref(), mk_or()
      a, b = a_env.its_showtime(), b_env.its_showtime()
    else:
      a, b = a_env.play(act), b_env.play(act)
  assert -0.001 in seen


def test_oracle_restart_draws_continue_both_streams():
  """make_t_maze draws random.random() for the cue and np.random.rand(PH, PW) for the speckle
  from the streams it is handed, so several episodes continue them as upstream would."""
  from pycolab_b200 import levels
  maze, cue = levels.t_maze_level(3)
  rng, np_rng = random.Random(9), np.random.RandomState(9)
  want_rng, want_np = random.Random(9), np.random.RandomState(9)
  for _ in range(3):
    world = otm.make_t_maze(maze, cue, 1, False, rng=rng, np_rng=np_rng)
    side = 'left' if want_rng.random() < 0.5 else 'right'
    dirt = ogames.art_to_array(maze) == ord('*')
    dirt[want_np.rand(*dirt.shape) < 0.4] = False
    assert world.things['Q'].aux['which_goal'] == side
    np.testing.assert_array_equal(world.things['*'].pattern, dirt)
  assert np_rng.get_state()[2] == want_np.get_state()[2]


def test_t_maze_level_keeps_the_drapes_constants():
  from pycolab_b200 import levels
  for seed in range(3):
    maze, cue = levels.t_maze_level(seed)
    art = ogames.art_to_array(maze)
    assert art.shape == (77, 191) and (art == ord('+')).sum() == 1 and (art == ord('P')).sum() == 1
    assert art[4, 140] == ord(' ') and (art[3:6, 139:142] == ord('#')).sum() == 8
    for level in range(6):
      assert art[4 + 11 * level + 9, 140 - 46] == ord(' ')
      assert art[4 + 11 * level + 9, 93:96].tolist() == [ord(' ')] * 3
    assert len(cue) == 7 and len(cue[0]) == 11


def _lower_generated(seed=0, **kw):
  from pycolab_b200 import lowering
  from pycolab_b200.games import t_maze
  random.seed(seed)
  np.random.seed(seed)
  return lowering.lower(t_maze.make_game(kw.pop('level', 1), kw.pop('cue', False), **kw))


def test_t_maze_lowers_and_validates_on_cpu():
  from pycolab_b200 import _lib
  game = _lower_generated(4, level=3, teleport_delay=5, limbo_time=7)
  assert game.program == _lib.PROG_T_MAZE and game.drape_chars == 'Q#*ltr'
  assert game.float_reward and game.needs_rng and game.rng_streams == ('python', 'numpy')
  assert list(game.program_arg[:5]) == [3, 0, _lib.T_MAZE_NO_TIMEOUT, 5, 7]
  lib = _lib.load()
  handle = C.c_void_p()
  spec = game.make_spec(True)
  assert lib.pcl_create(C.byref(spec), 4, -1, C.byref(handle)) == _lib.OK
  lib.pcl_destroy(handle)
  spec.program_arg[0] = 6                         # no hallway for level 6 in 77 rows
  assert lib.pcl_create(C.byref(spec), 4, -1, C.byref(handle)) == _lib.ERR_INVALID
  spec = game.make_spec(True)
  spec.sprite_egocentric[0] = 0
  assert lib.pcl_create(C.byref(spec), 4, -1, C.byref(handle)) == _lib.ERR_UNSUPPORTED


def test_teleporter_without_a_hallway_is_refused():
  from pycolab_b200 import levels
  from pycolab_b200.errors import NotLoweredError
  maze, cue = levels.t_maze_level(0)
  art = ogames.art_to_array(maze)
  art[4 + 11 * 2 + 9, 140 - 46] = ord('#')        # wall up level 2's landing cell
  maze = [bytes(r).decode() for r in art]
  with pytest.raises(NotLoweredError):
    _lower_generated(0, level=2, maze_art=maze, cue_art=cue)


def test_float_reward_program_refuses_int32_host_and_handoff_paths():
  """pcl_step_host(_async), pcl_pack_handoff(_peers) and pcl_crop_handoff carry an int32
  reward: PCL_ERR_UNSUPPORTED; pcl_step / pcl_reset without d_reward_f64: PCL_ERR_INVALID.
  All refused before anything reaches a device, so no GPU is needed."""
  from pycolab_b200 import _lib
  lib = _lib.load()
  game = _lower_generated(0)
  spec = game.make_spec(True)
  handle = C.c_void_p()
  assert lib.pcl_create(C.byref(spec), 2, -1, C.byref(handle)) == _lib.OK
  fake = 0x1000
  st = _lib.State()
  st.d_backdrop = st.d_plot = st.d_plot_init = st.d_sprites = st.d_sprites_init = fake
  st.d_drapes = st.d_drapes_init = fake
  st.d_bits[0] = st.d_bits_init[0] = fake
  st.bits_bstride[0] = 8
  for d in range(1, 6):
    st.d_pattern[d] = fake
  st.d_pattern_init[2] = fake
  st.pattern_bstride[2] = 616
  try:
    assert lib.pcl_bind_state(handle, C.byref(st)) == _lib.OK
    out = _lib.Outputs(fake, fake, fake, fake, fake)
    assert lib.pcl_step(handle, fake, C.byref(out), None) == _lib.ERR_INVALID
    assert lib.pcl_reset(handle, None, C.byref(out), None) == _lib.ERR_INVALID
    assert lib.pcl_run(handle, fake, 3, C.byref(out), None) == _lib.ERR_INVALID
    out.d_reward_f64 = fake
    assert lib.pcl_step_host(handle, fake, fake, C.byref(out), fake, fake, fake, fake, fake,
                             None) == _lib.ERR_UNSUPPORTED
    assert lib.pcl_step_host_async(handle, fake, fake, C.byref(out), None, None, None, fake,
                                   fake, fake, fake, fake, 0, None) == _lib.ERR_UNSUPPORTED
    assert lib.pcl_pack_handoff(handle, fake, 81, C.byref(out), fake, None) == _lib.ERR_UNSUPPORTED
    peers = (C.c_void_p * 1)(fake)
    assert lib.pcl_pack_handoff_peers(handle, fake, 81, C.byref(out), peers, 1, 0,
                                      None) == _lib.ERR_UNSUPPORTED
    from pycolab_b200 import batched
    crop = batched.scrolling_crop_spec(5, 5, 0, pad_char=' ', scroll_margins=(1, 1))
    x = _lib.HandoffState()
    assert lib.pcl_crop_handoff(handle, C.byref(crop), fake, None, C.byref(out), C.byref(x),
                                None) == _lib.ERR_UNSUPPORTED
  finally:
    lib.pcl_destroy(handle)


@pytest.mark.skipif(not refdriver.available(), reason='/root/reference not present')
def test_reference_t_maze_file_lowers_like_the_twin():
  """compat.load_example runs the reference file unchanged; with the reference's art handed
  to the twin and the same seeds, both lower to the same device templates."""
  from pycolab_b200 import compat, lowering
  from pycolab_b200.games import t_maze
  saved = {k: v for k, v in sys.modules.items() if k == 'pycolab' or k.startswith('pycolab.')}
  compat.uninstall()
  try:
    mod = compat.load_example(os.path.join(refdriver.REFERENCE_ROOT, 'pycolab', 'examples',
                                           'research', 'lp-rnn', 't_maze.py'))
    for args in ((0, False, -1, 0, 10), (4, True, 200, 5, 0)):
      random.seed(11)
      np.random.seed(11)
      a = lowering.lower(mod.make_game(*args))
      random.seed(11)
      np.random.seed(11)
      b = lowering.lower(t_maze.make_game(*args, maze_art=mod.MAZE_ART, cue_art=mod.CUE_ART))
      assert a.signature() == b.signature()
      for field in ('backdrop', 'sprites', 'drapes', 'plot'):
        np.testing.assert_array_equal(getattr(a, field), getattr(b, field), err_msg=field)
      for d in a.patterns:
        np.testing.assert_array_equal(a.patterns[d], b.patterns[d])
      np.testing.assert_array_equal(a.pattern_redraw[2], b.pattern_redraw[2])
      np.testing.assert_array_equal(a.bits[0], b.bits[0])
  finally:
    compat.uninstall()
    sys.modules.update(saved)


@pytest.mark.skipif(not refdriver.available(), reason='/root/reference not present')
def test_edited_t_maze_copy_is_refused(tmp_path):
  from pycolab_b200 import compat, lowering
  from pycolab_b200.errors import NotLoweredError
  src = open(os.path.join(refdriver.REFERENCE_ROOT, 'pycolab', 'examples', 'research', 'lp-rnn',
                          't_maze.py')).read()
  edited = src.replace('the_plot.add_reward(-0.001)', 'the_plot.add_reward(-0.01)')
  assert edited != src
  path = tmp_path / 't_maze.py'
  path.write_text(edited)
  saved = {k: v for k, v in sys.modules.items() if k == 'pycolab' or k.startswith('pycolab.')}
  compat.uninstall()
  try:
    mod = compat.load_example(str(path))
    with pytest.raises(NotLoweredError):
      lowering.lower(mod.make_game(0, False))
  finally:
    compat.uninstall()
    sys.modules.update(saved)


# ------------------------------------------------------------------------------------ GPU --

def _facade(maze, cue, cfg):
  from pycolab_b200.games import t_maze
  return lambda: t_maze.make_game(cfg['level'], cfg['cue_after_teleport'], cfg['timeout_frames'],
                                  cfg['teleport_delay'], cfg['limbo_time'], maze_art=maze,
                                  cue_art=cue)


@pytest.mark.gpu
@pytest.mark.parametrize('name', NAMES)
def test_facade_t_maze_golden(name):
  """B = 1 facade on the reference's art: the twin's drapes draw from the global `random` and
  NumPy streams as upstream, one Engine per episode; rewards compared as float64 bits."""
  g = gc.load(name)
  cfg = gc.config_of(g)
  maze, cue = tj.u8_to_art(g['maze_art']), tj.u8_to_art(g['cue_art'])
  random.seed(cfg['seed'])
  np.random.seed(cfg['seed'])
  sprites, goals = [], []

  def on_frame(env, out):
    p = env.things['P']
    sprites.append([[int(p.position[0]), int(p.position[1]), int(bool(p.visible)),
                     int(p.virtual_position[0]), int(p.virtual_position[1])]])
    goals.append(0 if env.things['Q'].which_goal == 'left' else 1)
    assert out[1] is None or isinstance(out[1], float)
    for ch in '#*ltr':           # the rolled whole_pattern, windowed as drapes.py:689-695
      d = env.things[ch]
      r, c = d._northwest_corner
      np.testing.assert_array_equal(d.curtain, d.whole_pattern[r:r + env.rows, c:c + env.cols],
                                    '%s frame %d' % (ch, len(goals)))
  got = []
  traj = tj.run_trajectory(_facade(maze, cue, cfg), g['actions'].tolist(),
                           on_frame=lambda env, out: (on_frame(env, out), got.append(
                               np.nan if out[1] is None else out[1])))
  tj.assert_same_trajectory(g, traj, name)
  _same_f64(g['reward_f64'], np.array(got, dtype=np.float64), name)
  np.testing.assert_array_equal(g['sprites'], np.array(sprites))
  np.testing.assert_array_equal(g['which_goal'], np.array(goals))


def _batched_vs_oracle(B, T, seed, cfg, n_worlds, check_envs=None, policy_seed=3):
  """Auto-resetting batch over generated worlds (env e plays world e % n_worlds, one set of
  make_game arguments for the handle): env e's cue and speckle come from
  random.Random(seed + e) and RandomState(seed + e), drawn by the kernel at every restart.
  Rewards are compared as float64 bits."""
  import torch
  from pycolab_b200 import batched, levels
  from pycolab_b200.games import t_maze
  arts = [levels.t_maze_level(i) for i in range(n_worlds)]
  games = [t_maze.make_game(*cfg, maze_art=m, cue_art=c) for m, c in arts]
  eng = batched.BatchedEngine(games, batch=B, rng_seed=seed)
  assert eng.rng is not None and eng.reward.dtype == torch.float64
  envs = range(B) if check_envs is None else check_envs
  rngs = {e: (random.Random(seed + e), np.random.RandomState(seed + e)) for e in envs}

  def make(e):
    maze, cue = arts[e % n_worlds]
    return otm.make_t_maze(maze, cue, *cfg, rng=rngs[e][0], np_rng=rngs[e][1])
  eng.its_showtime()
  rs = np.random.RandomState(policy_seed)
  policy = np.array([rs.choice([1, 2, 3, 4, 5, 0, 6], size=B,
                               p=[.35, .1, .2, .2, .13, .01, .01]) for _ in range(T)], np.int32)
  episodes, paid = [0], set()

  def count(t, eng, worlds, outs):
    for e, w in worlds.items():
      episodes[0] += int(t < T and w.game_over)
      if outs[e][1] is not None:
        paid.add(round(float(outs[e][1]), 3))
  sampled_check.lockstep(eng, make, envs, policy, on_step=count)
  assert int(eng.error_codes().abs().max()) == 0
  return eng, episodes[0], paid


@pytest.mark.gpu
@pytest.mark.parametrize('cfg', [(0, False, -1, 0, 0), (1, True, 40, 5, 4), (2, False, 60, 3, 2),
                                 (5, True, 25, 0, 10)])
def test_batched_t_maze_device_draws_vs_oracle(cfg):
  eng, episodes, paid = _batched_vs_oracle(B=24, T=220, seed=70, cfg=cfg, n_worlds=3)
  assert episodes > 24 and -0.001 in paid
  # the streams moved on: slot 1 holds NumPy's words after several speckle fields
  words = eng.rng.cpu().numpy().view(np.uint32).reshape(24, 2, -1)
  assert (words[:, 1, :624] != np.stack([np.random.RandomState(70 + e).get_state()[1]
                                         for e in range(24)])).any(axis=1).all()


@pytest.mark.gpu
def test_batched_t_maze_sampled_at_4096():
  sampled = [0, 1, 2, 777, 2048, 3001, 4094, 4095]
  _batched_vs_oracle(B=4096, T=90, seed=5, cfg=(4, True, 30, 5, 4), n_worlds=4,
                     check_envs=sampled)


@pytest.mark.gpu
def test_t_maze_curtains_and_layers_follow_the_rolls():
  """curtain() / unoccluded_layers() against the oracle's drapes while patterns roll: one
  shared level, and two levels with share_levels=False (every level tensor one row per env)."""
  import torch
  from pycolab_b200 import batched, levels
  from pycolab_b200.games import t_maze
  cfg = (1, False, -1, 2, 3)
  for n_worlds, share_levels in ((1, True), (2, False)):
    arts = [levels.t_maze_level(2 + i) for i in range(n_worlds)]
    eng = batched.BatchedEngine([t_maze.make_game(*cfg, maze_art=m, cue_art=c) for m, c in arts],
                                batch=2, rng_seed=8, auto_reset=False, share_levels=share_levels)
    worlds = [otm.make_t_maze(*arts[e % n_worlds], *cfg, rng=random.Random(8 + e),
                              np_rng=np.random.RandomState(8 + e)) for e in range(2)]
    for w in worlds:
      w.its_showtime()
    eng.its_showtime()
    for act in [1, 1, 1] + [5] * 6 + [3] * 12:
      eng.play(torch.full((2,), act, dtype=torch.int32).cuda())
      for w in worlds:
        w.play(act)
      layers = eng.unoccluded_layers('*#ltrQP ').cpu().numpy()
      for e, w in enumerate(worlds):
        for ch in 'Q#*ltr':
          np.testing.assert_array_equal(eng.curtain(ch)[e].cpu().numpy(), w.things[ch].curtain,
                                        '%s env %d levels %d' % (ch, e, n_worlds))
        want = em.unoccluded_layers_of(w.backdrop, w.things, '*#ltrQP ')
        for k, ch in enumerate('*#ltrQP '):
          np.testing.assert_array_equal(layers[e, k], want[ch],
                                        '%s env %d levels %d' % (ch, e, n_worlds))
