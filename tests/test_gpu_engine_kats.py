"""The known answers of the reference's `tests/engine_test.py`, replayed on the
DEVICE (general program `PCL_PROG_FIXTURE` through the C ABI).

Same capture as tests/test_reference_engine_kats.py (oracle replay): 9 engines /
21 frames of `engine_test.py` — update schedule and z-order (:39-167), rewards and
episode end with the default and a CUSTOM discount (:169-242,
`terminate_episode(0.5)`), `change_z_order` directives (:244-295), plot state
(:297-354), layers with and without occlusion (:378-455, 578-640).  Per frame the
device must return the hand-drawn board, the reference's discount (0 ulp),
game_over, z-order and EVERY layer — the un-occluded ones from the batched
`pcl_layers` kernel.  The test's string rewards ('pyco' + 'lab!') are replayed as
distinct integers with the same add_reward call sequence (the device sums int32).
The boards PROMISED to entities between update groups are internal to the fused
kernel and stay oracle-only.
"""

import json
import os

import numpy as np
import pytest

import reference_kats as rk

pytestmark = pytest.mark.gpu

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden',
                    'reference_engine_kats.json')
with open(PATH) as f:
  DATA = json.load(f)
KATS = [e for e in DATA['engines'] if isinstance(e['snapshot'], dict)]


def _ids():
  seen, out = {}, []
  for e in KATS:
    n = seen[e['test']] = seen.get(e['test'], 0) + 1
    out.append('%s-%d' % (e['test'].split('.')[-1], n))
  return out


def _int_reward(value, table):
  """A stable small integer per distinct reward value of the capture."""
  if isinstance(value, (int, float)) and not isinstance(value, bool):
    return int(value)
  if value not in table:
    table[value] = 1000 + 37 * len(table)
  return table[value]


@pytest.mark.parametrize('kat', KATS, ids=_ids())
def test_device_reproduces_engine_test(kat):
  import torch
  from pycolab_b200.games import fixtures
  from test_gpu_reference_kats import device_game
  snap = dict(kat['snapshot'], occlusion_in_layers=kat['occlusion_in_layers'])
  b, game = device_game(snap)
  chars = ''.join(game.groups)
  rewards = {}
  for i, frame in enumerate(kat['frames']):
    where = '%s frame %d' % (kat['test'], i)
    motions = rk.motion_of(frame['action'], chars)
    if not isinstance(motions, dict):
      motions = {ch: motions for ch in chars}
    directives, want_reward = [], None
    for name, args, kwargs in frame['directives']:
      assert not kwargs, where
      if name == 'add_reward':
        r = _int_reward(args[0], rewards)
        directives.append((name, r))
        want_reward = r if want_reward is None else want_reward + r
      elif name == 'change_z_order':
        directives.append((name, args[0], args[1]))
      else:                                    # terminate_episode / change_default_discount
        directives.append((name,) + tuple(args))
    res = b.play([fixtures.action_rows(game, motions, directives=directives)])
    torch.cuda.synchronize()
    board = res.board[0].cpu().numpy()
    np.testing.assert_array_equal(board, rk.u8(frame['board']), err_msg=where)
    if frame['expect_final'] is not None:      # the hand-drawn art of the test itself
      np.testing.assert_array_equal(board, rk.u8(frame['expect_final']), err_msg=where)
    assert (frame['reward'] is None) == (want_reward is None), where
    assert (int(res.has_reward[0]), int(res.reward[0])) == (
        (0, 0) if want_reward is None else (1, want_reward)), where
    assert float(res.discount[0]) == np.float32(frame['discount']), where
    assert bool(res.done[0]) == frame['game_over'], where
    assert [chr(c) for c in b.z_order[0].cpu().numpy()] == frame['z_order'], where
    order = ''.join(sorted(frame['layers']))
    if kat['occlusion_in_layers']:             # rendering.py:177-178
      for ch in order:
        np.testing.assert_array_equal(board == ord(ch), rk.bits(frame['layers'][ch]),
                                      err_msg='%s layer %r' % (where, ch))
    else:                                      # rendering.py:187-301 on the device
      planes = b.unoccluded_layers(order)[0].cpu().numpy()
      for k, ch in enumerate(order):
        np.testing.assert_array_equal(planes[k], rk.bits(frame['layers'][ch]),
                                      err_msg='%s unoccluded layer %r' % (where, ch))
  assert int(b.error_codes().abs().max()) == 0


def test_discount_directives_in_call_order():
  """plot.py:176-199, 247-260: the LAST discount-setting call of a step wins, and
  a changed default lasts for that step only (upstream rebuilds the directives
  after every step, plot.py:345-356)."""
  import torch
  from pycolab_b200 import batched, lowering
  from pycolab_b200.games import fixtures
  game = lowering.lower(fixtures.make_game(['P  ', '   '], ' ', {'P': dict(impassable='')}))
  b = batched.BatchedEngine([game], batch=3, auto_reset=False)
  b.its_showtime()
  row = lambda *d: fixtures.action_rows(game, {}, directives=list(d))
  res = b.play([row(('change_default_discount', 0.9)),
                row(('terminate_episode', 0.25), ('change_default_discount', 0.75)),
                row(('change_default_discount', 0.5), ('add_reward', 4),
                    ('terminate_episode',), ('add_reward', -9))])
  torch.cuda.synchronize()
  assert res.discount.tolist() == [np.float32(0.9), 0.75, 0.0]
  assert res.done.tolist() == [0, 1, 1]
  assert res.reward.tolist() == [0, 0, -5] and res.has_reward.tolist() == [0, 0, 1]
  res = b.play([row(), row(), row()])          # env 0 runs on: default back to 1.0
  assert float(res.discount[0]) == 1.0 and res.done.tolist() == [0, 1, 1]
  with pytest.raises(ValueError):
    row(('terminate_episode', 1.5))


def test_batched_unoccluded_layers_vs_oracle():
  """`pcl_layers` over a batch of scrolly_maze envs == the oracle's un-occluded
  layers (backdrop characters, both Scrolly curtains incl. the stale coin cell,
  every sprite) at every step."""
  from oracle import engine_model as em
  from oracle import games as ogames
  from oracle import sampled_check
  from pycolab_b200 import batched, levels, lowering
  from pycolab_b200.games import scrolly_maze as g
  arts = [levels.scrolly_maze_level(60 + i, world_shape=(65, 65), board_shape=(24, 40))
          for i in range(3)]
  games = [lowering.lower(g.make_game(*a)) for a in arts]
  B, T = 12, 60
  eng = batched.BatchedEngine(games, batch=B)
  eng.its_showtime()
  chars = eng.chars
  rs = np.random.RandomState(3)
  actions = np.stack([rs.randint(0, 5, size=B) for _ in range(T)]).astype(np.int32)

  def same_layers(t, eng, worlds, outs):
    planes = eng.unoccluded_layers().cpu().numpy()
    for e, w in worlds.items():
      want = em.unoccluded_layers_of(w.backdrop, w.things, list(chars))
      for k, ch in enumerate(chars):
        np.testing.assert_array_equal(planes[e, k], want[ch], err_msg='t=%d env=%d %r' % (t, e, ch))
  sampled_check.lockstep(
      eng, lambda e: ogames.make_scrolly_maze(arts[e % 3][0], arts[e % 3][1], '+', arts[e % 3][2]),
      range(B), actions, on_step=same_layers)
