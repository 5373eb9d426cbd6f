"""GPU tests of the compiled step program (csrc/compiled.cu): registered update() code of
tests/compiled_games.py on the H100, against the oracle interpreter (oracle/compiled.py).
Its goldens replay in test_gpu_registered_goldens.py."""

import numpy as np
import pytest

import registered_games as rg
import trajectory as tj
from oracle import compiled as ocompiled
from pycolab_b200 import _lib, lowering

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def games():
  yield from rg.registered('compiled_games.py', 'OffBoardDrape', 'DivideDrape')


def _oracle_frames(lowered, actions):
  """Every frame of one env under the batched auto-reset protocol, with each frame's
  reward as a float64 (0.0 where there is none) under 'reward_f64'."""
  rewards = []
  traj = tj.run_trajectory(lambda: ocompiled.make_world(lowered), actions,
                           on_frame=lambda env, out: rewards.append(
                               0.0 if out[1] is None else float(out[1])))
  traj['reward_f64'] = np.array(rewards, dtype=np.float64)
  return traj


@pytest.mark.parametrize('game', ['coins', 'lava'])
def test_batched_mixed_levels_vs_oracle(games, game):
  """B = 4096, two levels alternating, auto-reset, 300 steps: every env against the
  oracle, rewards included (float64 sums for lava).  Env e plays level e % 2 with action
  stream e % 32, so 64 oracle runs cover every env."""
  import torch
  from pycolab_b200 import batched
  B, T, streams = 4096, 300, 32
  levels = [lowering.lower(games.GAMES[game](k)) for k in range(2)]
  n = len(levels)
  eng = batched.BatchedEngine(levels, batch=B)
  rs = np.random.RandomState(11)
  table = rs.randint(0, games.N_ACTIONS[game], size=(T, streams)).astype(np.int32)
  env_stream = np.arange(B) % streams
  actions = torch.from_numpy(np.ascontiguousarray(table[:, env_stream])).cuda()
  want, members = {}, {}
  for lv in range(n):
    for s in range(streams):
      want[lv, s] = _oracle_frames(levels[lv], table[:, s].tolist())
      members[lv, s] = np.nonzero((np.arange(B) % n == lv) & (env_stream == s))[0]
  res = eng.its_showtime()
  for t in range(T + 1):
    if t > 0:
      res = eng.play(actions[t - 1])
    torch.cuda.synchronize()
    boards = res.board.cpu().numpy()
    reward = res.reward.cpu().numpy()
    has = res.has_reward.cpu().numpy()
    disc = res.discount.cpu().numpy()
    done = res.done.cpu().numpy()
    for lv in range(n):
      for s in range(streams):
        envs = members[lv, s]
        w = want[lv, s]
        assert (boards[envs] == w['boards'][t]).all(), (game, t, lv, s)
        assert (has[envs] == w['has_reward'][t]).all(), (game, t, lv, s)
        assert (done[envs] == w['game_over'][t]).all(), (game, t, lv, s)
        assert (disc[envs] == np.float32(w['discount'][t])).all(), (game, t, lv, s)
        want_reward = w['reward_f64'][t] if levels[0].float_reward else w['reward'][t]
        assert (reward[envs] == want_reward).all(), (game, t, lv, s)
  assert int((eng.error_codes() != 0).sum()) == 0
  assert int(eng._board[:, :, eng.cols:].sum()) == 0        # the pitch padding stays zero
  if levels[0].float_reward:
    assert res.reward.dtype == torch.float64


def test_float_rewards_match_the_oracle_sum(games):
  import torch
  from pycolab_b200 import batched
  lowered = lowering.lower(games.make_lava(1))
  rs = np.random.RandomState(5)
  actions = rs.randint(0, 6, size=200).tolist()
  world = ocompiled.make_world(lowered)
  want = [world.its_showtime()[1]]
  eng = batched.BatchedEngine([lowered], batch=3)
  got = [eng.its_showtime()]
  sums = [float(got[0].reward[0]) if int(got[0].has_reward[0]) else None]
  for a in actions:
    if world.game_over:
      world = ocompiled.make_world(lowered)
      want.append(world.its_showtime()[1])
    else:
      want.append(world.play(a)[1])
    r = eng.play(torch.full((3,), a, dtype=torch.int32).cuda())
    torch.cuda.synchronize()
    assert float(r.reward[0]) == float(r.reward[2])
    sums.append(float(r.reward[0]) if int(r.has_reward[0]) else None)
  assert sums == [None if w is None else float(w) for w in want]


def test_reset_with_env_mask(games):
  import torch
  from pycolab_b200 import batched
  eng = batched.BatchedEngine([lowering.lower(games.make_coins(0))], batch=8, auto_reset=False)
  first = eng.its_showtime().board.clone()
  for a in (3, 3, 1, 1, 3):
    eng.play(torch.full((8,), a, dtype=torch.int32).cuda())
  moved = eng.board.clone()
  plot_before = eng.plot.clone()
  mask = torch.tensor([1, 0, 1, 0, 0, 0, 0, 1], dtype=torch.uint8).cuda()
  eng.reset(mask)
  torch.cuda.synchronize()
  for e in range(8):
    want = first[e] if mask[e] else moved[e]
    assert bool((eng.board[e] == want).all()), e
  sel = mask.bool()
  assert bool((eng.plot[sel, _lib.P_AUX0:_lib.P_AUX0 + 2] !=
               plot_before[sel, _lib.P_AUX0:_lib.P_AUX0 + 2]).any())
  assert bool((eng.plot[~sel] == plot_before[~sel]).all())
  # the coin taken before the reset is back in the reset envs' curtains only
  coins = eng.curtain('c').sum(dim=(1, 2)).cpu().numpy()
  assert coins.tolist() == [6 if m else 5 for m in mask.tolist()]


def test_fault_bits_raise_in_the_facade(games):
  engine = games.make_fault(games.OffBoardDrape)
  engine.its_showtime()
  engine.play(0)
  with pytest.raises(IndexError):
    engine.play(1)
  engine = games.make_fault(games.DivideDrape)
  engine.its_showtime()
  engine.play(0)
  with pytest.raises(ZeroDivisionError):
    engine.play(1)


def test_attached_cropper_falls_back_to_a_crop_launch(games):
  import torch
  from pycolab_b200 import batched
  eng = batched.BatchedEngine([lowering.lower(games.make_coins(0))], batch=5)
  spec = batched.scrolling_crop_spec(3, 5, 0, pad_char=' ', scroll_margins=(1, 2))
  view = eng.attach_cropper(spec)
  assert not eng._attached[3], 'the compiled program has no crop epilogue'
  state = eng.new_crop_state()
  eng.its_showtime()
  for a in (1, 3, 3, 0, 2):
    eng.play(torch.full((5,), a, dtype=torch.int32).cuda())
    want = eng.crop(spec, state=state)
    torch.cuda.synchronize()
    assert bool((view == want).all())


def test_code_upload_on_a_side_stream_and_rebinding(games):
  """The first launch uploads the code on its own (non-blocking) stream; binding code
  again between steps replaces it.  Both engines must step alike throughout."""
  import torch
  from pycolab_b200 import batched
  lowered = lowering.lower(games.make_coins(1))
  side = torch.cuda.Stream()
  with torch.cuda.stream(side):
    eng = batched.BatchedEngine([lowered], batch=64)
    eng.its_showtime()
  twin = batched.BatchedEngine([lowered], batch=64)
  twin.its_showtime()
  rs = np.random.RandomState(3)
  code = np.ascontiguousarray(lowered.code, dtype=np.int32)
  for t in range(60):
    a = torch.from_numpy(rs.randint(0, 6, size=64).astype(np.int32)).cuda()
    if t == 30:                           # same words again: the device copy is replaced
      _lib.check(eng._lib.pcl_bind_code(eng._h, code.ctypes.data, len(code)), 'pcl_bind_code')
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
      eng.play(a)
    twin.play(a)
    side.synchronize()
    torch.cuda.synchronize()
    assert bool((eng.board == twin.board).all()), t
    assert bool((eng.reward == twin.reward).all()), t
