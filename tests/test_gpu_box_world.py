"""research/box_world on the H100: the reference's goldens replayed on the device bit for bit
(board, reward, has_reward, discount, done, every object curtain, occluded and un-occluded
layers), and pools of thousands of distinct generated levels in one handle, sampled against
the oracle.  The facade Engine's replays of the goldens are tests/example_games.py's."""

import numpy as np
import pytest

import golden_cases as gc
import trajectory as tj
from oracle import box_world as obw
from oracle import sampled_check

NAMES = gc.names('box_world_')


def _golden(name):
  g = gc.load(name)
  cfg = gc.config_of(g)
  art = tj.u8_to_art(g['art'])
  distractors = [tuple(int(v) for v in xy) for xy in g['distractors']]
  return g, cfg, art, distractors


@pytest.mark.gpu
@pytest.mark.parametrize('name', NAMES)
def test_golden_replays_on_device(name):
  import torch
  from pycolab_b200 import batched
  from pycolab_b200.games import box_world
  g, cfg, art, distractors = _golden(name)
  eng = batched.BatchedEngine([box_world.game_from_level(art, distractors, cfg['max_num_steps'])],
                              batch=2)
  chars = ''.join(sorted(set(eng.chars) | set('*aAtT')))   # and object chars the level lacks
  backdrop = np.array([[ord(c) if c in ' #' else ord(' ') for c in row] for row in art], np.uint8)
  eng.its_showtime()
  actions = g['actions']
  for t in range(len(actions) + 1):
    if t:
      eng.play(torch.full((2,), int(actions[t - 1]), dtype=torch.int32, device='cuda'))
    torch.cuda.synchronize()
    for key, got in (('boards', eng.board), ('reward', eng.reward), ('has_reward', eng.has_reward),
                     ('discount', eng.discount), ('game_over', eng.done)):
      got = got.cpu().numpy()
      assert (got[0] == got[1]).all(), (name, t, key)
      np.testing.assert_array_equal(got[0], g[key][t], '%s %s frame %d' % (name, key, t))
    grid = g['grid'][t]
    for ch in eng.object_chars:
      np.testing.assert_array_equal(eng.curtain(ch)[0].cpu().numpy(), grid == ord(ch),
                                    '%s curtain %s frame %d' % (name, ch, t))
    board = g['boards'][t]
    occluded = eng.to_feature_array(chars)[0].cpu().numpy()
    unoccluded = eng.unoccluded_layers(chars)[0].cpu().numpy()
    for k, ch in enumerate(chars):
      np.testing.assert_array_equal(occluded[k], (board == ord(ch)).astype(np.float32))
      want = (backdrop == ord(ch)) | (grid == ord(ch))
      if ch == '.':
        want = board == ord('.')
      np.testing.assert_array_equal(unoccluded[k], want, '%s layer %s frame %d' % (name, ch, t))
  assert set(eng.object_chars) == set(np.unique(g['grid'][0])[1:].tobytes().decode())
  assert int(eng.error_codes().abs().max()) == 0


def _pool(n_levels, grid_size=12):
  from pycolab_b200 import levels
  return [levels.box_world_level(i, grid_size) for i in range(n_levels)]


def _pool_vs_oracle(B, n_levels, T, n_check, grid_size=12, max_steps=60):
  import torch
  from pycolab_b200 import batched, lowering
  from pycolab_b200.games import box_world
  pool = _pool(n_levels, grid_size)
  games = [lowering.lower(box_world.game_from_level(a, d, max_steps)) for a, d in pool]
  eng = batched.BatchedEngine(games, batch=B)
  eng.its_showtime()
  rs = np.random.RandomState(B)
  actions = rs.randint(-1, 5, size=(T, B)).astype(np.int32)
  envs = sorted(set(rs.choice(B, n_check - 2, replace=False).tolist()) | {0, B - 1})
  seen = {'episodes': 0, 'rewards': set()}

  def count(t, eng, worlds, outs):
    for e, w in worlds.items():
      seen['episodes'] += int(w.game_over)
      if outs[e][1] is not None:
        seen['rewards'].add(outs[e][1])
  make = lambda e: obw.make_box_world(*pool[e % n_levels], max_steps)
  sampled_check.lockstep(eng, make, envs, actions, sprites='.', on_step=count)
  assert int(eng.error_codes().abs().max()) == 0
  return eng, seen


@pytest.mark.gpu
def test_4096_envs_on_4096_levels_vs_oracle():
  eng, seen = _pool_vs_oracle(B=4096, n_levels=4096, T=300, n_check=64)
  assert seen['episodes'] >= 64 and {0.0, 1.0} <= seen['rewards']
  assert int(eng.plot[:, 3].min()) >= 2               # every env restarted at least once


@pytest.mark.gpu
def test_65536_envs_on_512_levels_vs_oracle():
  _pool_vs_oracle(B=65536, n_levels=512, T=300, n_check=64)


@pytest.mark.gpu
def test_reset_mask_and_host_step():
  """pcl_reset with an env mask rebuilds only the masked envs; pcl_step_host returns the
  int32 rewards."""
  import torch
  from pycolab_b200 import batched
  from pycolab_b200.games import box_world
  pool = _pool(3)
  eng = batched.BatchedEngine([box_world.game_from_level(a, d, 50) for a, d in pool], batch=6,
                              auto_reset=False)
  eng.its_showtime()
  start = eng.board.cpu().numpy().copy()
  rs = np.random.RandomState(1)
  worlds = [obw.make_box_world(*pool[e % 3], 50) for e in range(6)]
  for w in worlds:
    w.its_showtime()
  for _ in range(40):
    a = rs.randint(0, 4, size=6).astype(np.int32)
    board, reward, has, discount, done = eng.play_host(a)
    assert reward.dtype == np.int32
    for e, w in enumerate(worlds):
      if w.game_over:
        continue
      b, r, d = w.play(int(a[e]))
      assert np.array_equal(board[e], b) and int(has[e]) == (r is not None)
      assert int(reward[e]) == (0 if r is None else int(r)) and float(discount[e]) == d
  mask = torch.tensor([1, 0, 1, 0, 0, 1], dtype=torch.uint8, device='cuda')
  before = eng.board.cpu().numpy().copy()
  eng.reset(mask)
  after = eng.board.cpu().numpy()
  for e in range(6):
    want = start[e] if mask[e] else before[e]
    np.testing.assert_array_equal(after[e], want, 'env %d' % e)
  assert eng.sprites[0, 0, 5].item() == 0 and eng.plot[0, 8].item() == 0


@pytest.mark.gpu
def test_level_without_walls_wraps_and_latches_index_errors():
  """A level bound through the C boundary without its '#' ring: the kernel reads row and
  column -1 as NumPy does (wrapped), keeps the confined walker on the board and latches
  PCL_ENV_ERR_INDEX where the reference raises IndexError (past the last row or column)."""
  import torch
  from pycolab_b200 import _lib, batched, levels, lowering
  from pycolab_b200.games import box_world
  art, distractors = levels.box_world_level(1, 6)
  game = lowering.lower(box_world.game_from_level(art, distractors, 200))
  ring = np.zeros((game.rows, game.cols), dtype=bool)
  ring[[0, -1], :] = ring[:, [0, -1]] = True
  game.backdrop[:, :game.cols][ring] = ord(' ')
  bare = [''.join(' ' if ring[r, c] else ch for c, ch in enumerate(row))
          for r, row in enumerate(art)]
  B, T = 16, 120
  eng = batched.BatchedEngine([game], batch=B, auto_reset=False)
  eng.its_showtime()
  rs = np.random.RandomState(5)
  actions = rs.randint(0, 4, size=(T, B)).astype(np.int32)
  worlds = [obw.make_box_world(bare, distractors, 200) for _ in range(B)]
  for w in worlds:
    w.its_showtime()
  raised, edge = set(), 0
  for t in range(T):
    eng.play(torch.from_numpy(actions[t]).cuda())
    boards = eng.board.cpu().numpy()
    errors = eng.error_codes().cpu().numpy()
    for e, w in enumerate(worlds):
      if e in raised or w.game_over:
        continue
      try:
        board, reward, _ = w.play(int(actions[t, e]))
      except IndexError:
        raised.add(e)
        assert errors[e] & _lib.ENV_ERR_INDEX, (t, e)
        continue
      assert errors[e] == 0, (t, e)
      np.testing.assert_array_equal(boards[e], board, 'step %d env %d' % (t, e))
      p = w.things['.']
      edge += p.row in (0, game.rows - 1) or p.col in (0, game.cols - 1)
  assert raised and edge
