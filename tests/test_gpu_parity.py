"""GPU parity: the CUDA step engine vs the oracle (the facade's golden replays are in
test_gpu_example_goldens.py).

All of these call through the C ABI (libpcl.so via ctypes).  Bar: bit-exact
boards (uint8), rewards (incl. None-ness), discounts, game_over and sprite
registers.  Marked `gpu`; run on the H100.
"""

import numpy as np
import pytest

import golden_cases as gc
from oracle import engine_model as em
from oracle import games as ogames
from oracle import sampled_check

pytestmark = pytest.mark.gpu


def _torch():
  import torch
  return torch


# ------------------------------------------------- batched engine vs oracle

def _batched_vs_oracle(make_facade_game, make_oracle, actions, n_levels=1,
                       rng_seed=None, check_curtains=''):
  """Step a BatchedEngine (auto-reset) and B oracle worlds in lockstep.

  actions: int array [T, B].  make_* take the level index (env % n_levels)."""
  from pycolab_b200 import batched
  B = actions.shape[1]
  games = [make_facade_game(i) for i in range(n_levels)]
  eng = batched.BatchedEngine(games, batch=B, rng_seed=rng_seed or 0)
  eng.its_showtime()
  sampled_check.lockstep(eng, make_oracle, range(B), actions, curtains=check_curtains)
  assert int(eng.error_codes().max()) == 0
  return eng


def test_batched_scrolly_stock():
  from pycolab_b200.games import scrolly_maze
  g = gc.load('scrolly_stock_L0')
  maze, board, beneath = gc.scrolly_art(g)
  rs = np.random.RandomState(42)
  actions = rs.randint(0, 6, size=(250, 24))
  actions[rs.random_sample(actions.shape) < 0.9] %= 5     # mostly no quits
  _batched_vs_oracle(lambda i: scrolly_maze.make_game(maze, board, beneath),
                     lambda e: ogames.make_scrolly_maze(maze, board, '+', beneath),
                     actions, check_curtains='#@')


def test_batched_scrolly_generated_multi_level():
  from pycolab_b200 import levels
  from pycolab_b200.games import scrolly_maze
  arts = [levels.scrolly_maze_level(10 + i) for i in range(3)]
  rs = np.random.RandomState(43)
  actions = rs.choice([0, 1, 2, 3, 4], size=(120, 9), p=[.3, .15, .3, .15, .1])
  _batched_vs_oracle(lambda i: scrolly_maze.make_game(*arts[i]),
                     lambda e: ogames.make_scrolly_maze(arts[e % 3][0], arts[e % 3][1],
                                                        '+', arts[e % 3][2]),
                     actions, n_levels=3)


@pytest.mark.parametrize('board_shape,world_shape', [((40, 96), (97, 161)), ((24, 128), (65, 257)),
                                                     ((20, 65), (41, 131))])
def test_batched_scrolly_wider_than_64_columns(board_shape, world_shape):
  """The reference Scrolly has no width limit (drapes.py:293-376): boards of 65, 96
  and 128 columns stage 4 / 6 words per window row instead of 4."""
  from pycolab_b200 import levels
  from pycolab_b200.games import scrolly_maze
  arts = [levels.scrolly_maze_level(70 + i, world_shape=world_shape, board_shape=board_shape)
          for i in range(2)]
  rs = np.random.RandomState(47)
  actions = rs.choice([0, 1, 2, 3, 4], size=(150, 6), p=[.2, .2, .25, .25, .1])
  _batched_vs_oracle(lambda i: scrolly_maze.make_game(*arts[i]),
                     lambda e: ogames.make_scrolly_maze(arts[e % 2][0], arts[e % 2][1],
                                                        '+', arts[e % 2][2]),
                     actions, n_levels=2, check_curtains='#@')


def test_batched_warehouse():
  from pycolab_b200 import levels
  from pycolab_b200.games import warehouse_manager
  arts = [levels.warehouse_level(20 + i, shape=(24, 31), num_boxes=4 + i, num_goals=6 + i)
          for i in range(2)]
  # structure (number of boxes) must agree inside one engine: use level 0 twice
  arts = [arts[0], levels.warehouse_level(77, shape=(24, 31), num_boxes=4, num_goals=6)]
  rs = np.random.RandomState(44)
  actions = rs.randint(0, 6, size=(300, 16))
  actions[rs.random_sample(actions.shape) < 0.95] %= 5
  _batched_vs_oracle(lambda i: warehouse_manager.make_game(arts[i]),
                     lambda e: ogames.make_warehouse(arts[e % 2]),
                     actions, n_levels=2, check_curtains='X')


def test_batched_warehouse_80():
  from pycolab_b200 import levels
  from pycolab_b200.games import warehouse_manager
  art = levels.warehouse_level(3)
  rs = np.random.RandomState(45)
  actions = rs.randint(0, 4, size=(150, 8))
  _batched_vs_oracle(lambda i: warehouse_manager.make_game(art),
                     lambda e: ogames.make_warehouse(art), actions)


def test_batched_marauders():
  from pycolab_b200 import levels
  from pycolab_b200.games import extraterrestrial_marauders as marauders
  art = levels.marauders_level()
  rs = np.random.RandomState(46)
  B = 12
  actions = rs.randint(0, 4, size=(400, B))
  rngs = [np.random.RandomState(900 + e) for e in range(B)]
  _batched_vs_oracle(lambda i: marauders.make_game(art),
                     lambda e: ogames.make_marauders(art, rngs[e]),
                     actions, rng_seed=900, check_curtains='BX')


# ------------------------------------------------------------------ cropper

def test_batched_crop_vs_oracle():
  from pycolab_b200 import batched, levels
  from pycolab_b200.games import scrolly_maze
  art = levels.scrolly_maze_level(31)
  B, T = 16, 80
  eng = batched.BatchedEngine([scrolly_maze.make_game(*art)], batch=B)
  spec = batched.scrolling_crop_spec(9, 9, 0, pad_char=' ', scroll_margins=(None, None))
  eng.its_showtime()
  actions = np.random.RandomState(5).randint(0, 5, size=(T, B)).astype(np.int32)
  sampled_check.lockstep(
      eng, lambda e: ogames.make_scrolly_maze(art[0], art[1], '+', art[2]), range(B), actions,
      crop=(spec, None, lambda: em.ScrollingCrop(9, 9, ['P'], pad_char=' ',
                                                 scroll_margins=(None, None))))


@pytest.mark.parametrize('pad,margins,rows,cols', [(' ', (None, None), 9, 9), (None, (2, 3), 11, 13),
                                                   ('.', (1, 1), 5, 7)])
def test_attached_cropper_vs_oracle(pad, margins, rows, cols):
  """pcl_attach_cropper: the cropper as the step kernel's epilogue (no crop launch)
  against the oracle's ScrollingCropper, through auto-resets, and bit-identical to the
  stand-alone crop kernel run on the same boards with its own corner state."""
  from pycolab_b200 import batched, levels
  from pycolab_b200.games import scrolly_maze
  art = levels.scrolly_maze_level(32, world_shape=(65, 65), board_shape=(32, 32))
  B, T = 19, 120
  eng = batched.BatchedEngine([scrolly_maze.make_game(*art)], batch=B)
  spec = batched.scrolling_crop_spec(rows, cols, 0, pad_char=pad, scroll_margins=margins)
  view = eng.attach_cropper(spec)
  assert eng._attached[3], 'the scrolly program runs the cropper inside the step kernel'
  twin_state = eng.new_crop_state()
  l0 = [eng.launch_count()]
  eng.its_showtime()
  actions = np.random.RandomState(6).randint(0, 5, size=(T, B)).astype(np.int32)

  def same_as_the_crop_kernel(t, eng, worlds, outs):
    assert eng.launch_count() == l0[0] + t + 1                 # one launch per step, crop included
    got = view.cpu().numpy()
    l1 = eng.launch_count()
    twin = eng.crop(spec, state=twin_state).cpu().numpy()      # the stand-alone kernel
    l0[0] += eng.launch_count() - l1
    np.testing.assert_array_equal(got, twin)
  sampled_check.lockstep(
      eng, lambda e: ogames.make_scrolly_maze(art[0], art[1], '+', art[2]), range(B), actions,
      crop=(view, None, lambda: em.ScrollingCrop(rows, cols, ['P'], pad_char=pad,
                                                 scroll_margins=margins)),
      on_step=same_as_the_crop_kernel)
  eng.attach_cropper(None)
  before = view.clone()
  eng.play(_torch().from_numpy(actions[0]).cuda())
  assert bool((view == before).all())                          # detached: untouched


def test_attached_cropper_falls_back_to_a_crop_launch():
  """A program without the epilogue keeps the same Python contract: the attached view
  is refreshed by a crop launch after every step."""
  from pycolab_b200 import batched, levels
  from pycolab_b200.games import warehouse_manager
  art = levels.warehouse_level(3, shape=(20, 24))
  B = 6
  eng = batched.BatchedEngine([warehouse_manager.make_game(art)], batch=B)
  spec = batched.scrolling_crop_spec(7, 7, len(eng.sprite_chars) - 1, pad_char=' ',
                                     scroll_margins=(None, None))
  view = eng.attach_cropper(spec)
  assert not eng._attached[3]
  eng.its_showtime()
  torch = _torch()
  state = eng.new_crop_state()
  rs = np.random.RandomState(1)
  for t in range(20):
    np.testing.assert_array_equal(view.cpu().numpy(), eng.crop(spec, state=state).cpu().numpy())
    eng.play(torch.from_numpy(rs.randint(0, 4, size=B).astype(np.int32)).cuda())


# ------------------------------------------------------- stand-alone render

@pytest.mark.parametrize('shape,S,D', [((10, 30), 4, 2), ((64, 64), 4, 2),
                                       ((16, 39), 7, 2), ((80, 80), 11, 1),
                                       ((5, 7), 0, 1), ((9, 33), 16, 8)])
def test_render_kernel_vs_oracle(shape, S, D):
  """pcl_render on random reference-layout inputs vs oracle.render."""
  import ctypes as C
  from pycolab_b200 import _lib
  torch = _torch()
  lib = _lib.load()
  H, W = shape
  pitch = (W + 15) // 16 * 16
  B = 37
  rs = np.random.RandomState(H * 100 + W)
  schars = 'ABCDEFGHIJKLMNOP'[:S]
  dchars = 'stuvwxyz'[:D]
  spec = _lib.Spec()
  spec.abi_version, spec.program = _lib.ABI_VERSION, _lib.PROG_NONE
  spec.rows, spec.cols, spec.pitch, spec.n_sprites, spec.n_drapes = H, W, pitch, S, D
  for i, c in enumerate(schars):
    spec.sprite_char[i] = ord(c)
  for i, c in enumerate(dchars):
    spec.drape_char[i] = ord(c)
  h = C.c_void_p()
  _lib.check(lib.pcl_create(C.byref(spec), B, 0, C.byref(h)), 'pcl_create')
  backdrop = np.zeros((B, H, pitch), np.uint8)
  backdrop[:, :, :W] = rs.choice([32, 46, 35], size=(B, H, W))
  curtains = np.zeros((B, max(D, 1), H, pitch), np.uint8)
  curtains[:, :D, :, :W] = rs.random_sample((B, D, H, W)) < 0.3
  sprites = np.zeros((B, max(S, 1), 8), np.int32)
  sprites[:, :, 0] = rs.randint(0, H, size=(B, max(S, 1)))
  sprites[:, :, 1] = rs.randint(0, W, size=(B, max(S, 1)))
  sprites[:, :, 4] = rs.randint(0, 2, size=(B, max(S, 1)))
  z = np.zeros((B, max(S + D, 1)), np.uint8)
  for b in range(B):
    z[b, :S + D] = rs.permutation([ord(c) for c in schars + dchars])
  dev = lambda a: torch.from_numpy(a).cuda()
  t_bd, t_cur, t_sp, t_z = dev(backdrop), dev(curtains), dev(sprites), dev(z)
  out = torch.zeros((B, H, pitch), dtype=torch.uint8, device='cuda')
  stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
  _lib.check(lib.pcl_render(h, t_bd.data_ptr(), H * pitch, t_cur.data_ptr(),
                            t_sp.data_ptr(), t_z.data_ptr(), out.data_ptr(), stream),
             'pcl_render')
  torch.cuda.synchronize()
  got = out.cpu().numpy()
  lib.pcl_destroy(h)

  class Ent(object):
    pass
  for b in range(B):
    things = {}
    for i, c in enumerate(schars):
      e = Ent()
      e.is_sprite, e.row, e.col = True, int(sprites[b, i, 0]), int(sprites[b, i, 1])
      e.visible = bool(sprites[b, i, 4])
      things[c] = e
    for i, c in enumerate(dchars):
      e = Ent()
      e.is_sprite, e.curtain = False, curtains[b, i, :, :W].astype(bool)
      things[c] = e
    want = em.render(H, W, backdrop[b, :, :W], [chr(c) for c in z[b, :S + D]], things)
    np.testing.assert_array_equal(got[b, :, :W], want, err_msg='env %d' % b)
    assert not got[b, :, W:].any()


def test_renderer_class_api():
  """BaseObservationRenderer's paint protocol (rendering.py:98-184) on the GPU."""
  from pycolab_b200 import rendering
  r = rendering.BaseObservationRenderer(4, 5, 'ab.# ')
  r.clear()
  bd = np.full((4, 5), ord('.'), np.uint8)
  r.paint_all_of(bd)
  mask = np.zeros((4, 5), bool)
  mask[1, :] = True
  r.paint_drape('#', mask)
  r.paint_sprite('a', (1, 2))
  r.paint_sprite('b', (3, 4))
  obs = r.render()
  want = bd.copy()
  want[1, :] = ord('#')
  want[1, 2] = ord('a')
  want[3, 4] = ord('b')
  np.testing.assert_array_equal(obs.board, want)
  np.testing.assert_array_equal(obs.layers['#'], want == ord('#'))
  with pytest.raises(ValueError):
    r.paint_sprite('Z', (0, 0))


# ------------------------------------------------- host-buffer entry point

def test_step_host_matches_device_path():
  from pycolab_b200 import batched, levels
  from pycolab_b200.games import scrolly_maze
  art = levels.scrolly_maze_level(3, world_shape=(65, 65), board_shape=(32, 32))
  a = batched.BatchedEngine([scrolly_maze.make_game(*art)], batch=32)
  b = batched.BatchedEngine([scrolly_maze.make_game(*art)], batch=32)
  a.its_showtime()
  b.its_showtime()
  torch = _torch()
  rs = np.random.RandomState(9)
  for t in range(40):
    act = rs.randint(0, 5, size=32).astype(np.int32)
    ra = a.play(torch.from_numpy(act).cuda())
    board, reward, has, disc, done = b.play_host(act)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(ra.board.cpu().numpy(), board)
    np.testing.assert_array_equal(ra.reward.cpu().numpy(), reward)
    np.testing.assert_array_equal(ra.done.cpu().numpy(), done)
  assert a.launch_count() >= 41


def test_large_batch_invariants():
  """BASELINE configs[1] size: properties that need no oracle at full size."""
  from pycolab_b200 import batched, levels
  from pycolab_b200.games import scrolly_maze
  torch = _torch()
  art = levels.scrolly_maze_level(0)
  B = 4096
  eng = batched.BatchedEngine([scrolly_maze.make_game(*art)], batch=B)
  eng.its_showtime()
  first = eng.board.clone()
  # Identical envs + identical actions stay identical (lockstep determinism).
  rs = np.random.RandomState(1)
  total_reward = torch.zeros(B, dtype=torch.int64, device='cuda')
  for t in range(50):
    a = int(rs.randint(0, 5))
    res = eng.play(torch.full((B,), a, dtype=torch.int32, device='cuda'))
    total_reward += res.reward.long()
    assert bool((res.board == res.board[0:1]).all())
  # Exactly one 'P' per board while it is on the board, boards only hold legal chars.
  legal = torch.tensor([ord(c) for c in ' .#@Pabc'], device='cuda', dtype=torch.uint8)
  assert bool(torch.isin(eng.board, legal).all())
  assert int((eng.board == ord('P')).sum()) == B
  assert bool((total_reward % 100 == 0).all())
  assert int(eng.error_codes().abs().max()) == 0
  assert first.shape == (B, 64, 64)


# --------------------------------------------------- engine-level behaviours
# (the per-env reset / freeze protocol of every step program: test_gpu_protocol.py)

def test_facade_raises_like_the_reference():
  from pycolab_b200 import levels
  from pycolab_b200.games import fixtures, scrolly_maze
  art = levels.scrolly_maze_level(4, world_shape=(65, 65), board_shape=(32, 32))
  game = scrolly_maze.make_game(*art)
  with pytest.raises(RuntimeError):
    game.play(0)                               # before its_showtime
  game.its_showtime()
  with pytest.raises(RuntimeError):
    game.its_showtime()                        # twice
  with pytest.raises(RuntimeError):
    game.add_sprite('q', (0, 0), scrolly_maze.PlayerSprite, (0, 0))
  _, reward, discount = game.play(5)           # quit
  assert reward is None and discount == 0.0 and game.game_over
  with pytest.raises(RuntimeError):
    game.play(0)                               # after the episode ended
  # A margin-less Scrolly that clips a diagonal order to (0, 0) makes the
  # egocentric walker raise upstream (sprites.py:449-454): same here.
  pattern = np.zeros((6, 6), dtype=bool)
  fx = fixtures.make_game(['    ', ' P  ', '    ', '    '], ' ',
                          {'P': dict(impassable='#', egocentric=True)},
                          {'#': dict(pattern=pattern, corner=(0, 0), margins=None)},
                          update_schedule=[['#'], ['P']], z_order='#P')
  fx.its_showtime()
  fx.play('se')                                # permits for the next frame
  with pytest.raises(RuntimeError):
    for _ in range(6):
      fx.play('nw')                            # corner (0,0): clipped to (0,0)


def test_facade_things_and_layers_follow_the_device():
  from pycolab_b200 import levels
  from pycolab_b200.games import scrolly_maze
  art = levels.scrolly_maze_level(9, world_shape=(65, 65), board_shape=(32, 32))
  game = scrolly_maze.make_game(*art)
  world = ogames.make_scrolly_maze(art[0], art[1], '+', art[2])
  obs, _, _ = game.its_showtime()
  out = world.its_showtime()
  rs = np.random.RandomState(1)
  for _ in range(40):
    a = int(rs.randint(0, 5))
    obs, _, _ = game.play(a)
    out = world.play(a)
    if game.game_over:
      break
  np.testing.assert_array_equal(obs.board, out[0])
  for ch in 'Pabc':
    assert tuple(game.things[ch].position) == world.things[ch].position
    assert tuple(game.things[ch].virtual_position) == world.things[ch].virtual_position
  for ch in '#@':
    np.testing.assert_array_equal(game.things[ch].curtain, world.things[ch].curtain)
  assert set(obs.layers) == set(world.chars)
  for ch in obs.layers:
    np.testing.assert_array_equal(obs.layers[ch], out[0] == ord(ch))
  assert game.the_plot.frame == world.plot.frame


def test_run_equals_repeated_play_and_host_without_board():
  """pcl_run (T steps, one C call) == T x pcl_step; play_host(want_board=False)."""
  from pycolab_b200 import batched, levels
  from pycolab_b200.games import warehouse_manager
  torch = _torch()
  art = levels.warehouse_level(9, shape=(20, 26), num_boxes=5, num_goals=6)
  a = batched.BatchedEngine([warehouse_manager.make_game(art)], batch=48)
  b = batched.BatchedEngine([warehouse_manager.make_game(art)], batch=48)
  c = batched.BatchedEngine([warehouse_manager.make_game(art)], batch=48)
  for e in (a, b, c):
    e.its_showtime()
  rs = np.random.RandomState(4)
  acts = rs.randint(0, 5, size=(25, 48)).astype(np.int32)
  t_acts = torch.from_numpy(acts).cuda()
  n0 = b.launch_count()
  rb = b.run(t_acts)
  assert b.launch_count() - n0 == 25
  for t in range(25):
    ra = a.play(t_acts[t])
    _, reward, has, disc, done = c.play_host(acts[t], want_board=False)
  torch.cuda.synchronize()
  assert bool((ra.board == rb.board).all()) and bool((ra.reward == rb.reward).all())
  assert bool((a.sprites == b.sprites).all()) and bool((a.plot == b.plot).all())
  np.testing.assert_array_equal(ra.reward.cpu().numpy(), reward)
  np.testing.assert_array_equal(ra.done.cpu().numpy(), done)
  assert bool((c.board == a.board).all())
