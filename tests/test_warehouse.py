"""warehouse_manager at the board's rim, on the CPU.

The oracle (oracle/games.py: make_warehouse) in lock-step with the live reference on
hand-drawn arts with floor up to the edge (warehouse_cases.RIM): boxes pushed off the
board, onto it again from the last row or column, several at once, the player leaving
and coming back, and the pushes that raise IndexError.  Then pcl_create's bound on the
backdrop tile a warehouse_step block stages in shared memory."""

import ctypes as C

import numpy as np
import pytest

import refdriver
import trajectory as tj
import warehouse_cases as wc
from oracle import sampled_check
from pycolab_b200 import _lib
from pycolab_b200 import lowering
from pycolab_b200.games import warehouse_manager
from test_oracle_vs_reference import _lockstep

needs_ref = pytest.mark.skipif(not refdriver.available(), reason='/root/reference not present')

STEADY = [name for name in wc.RIM if name not in wc.RAISES]


def _virtual_positions(ref, ora, t):
  for ch, ent in ref.things.items():
    if hasattr(ent, 'virtual_position'):
      w = ora.things[ch]
      assert tuple(int(v) for v in ent.virtual_position) == (w.vrow, w.vcol), (t, ch)


def _script(name):
  """The case's script, a quit, and the script again from a fresh episode."""
  script = wc.RIM[name][2]
  return script + [5] + script


@needs_ref
@pytest.mark.parametrize('name', STEADY)
def test_rim_case_oracle_vs_reference(name):
  """Boards, rewards, discounts, game over, and every sprite's position, visibility and
  virtual position, at every step of the scripted case and of its replay after a quit."""
  art, beneath, _, edges = wc.RIM[name]
  actions = _script(name)
  _lockstep(lambda: refdriver.ref_warehouse(art, beneath), lambda: wc.make_world(art, beneath),
            actions, check=_virtual_positions)
  seen, restarts, raised = wc.oracle_run(art, beneath, actions, wc.rim_boxes(name))
  assert raised is None
  assert edges <= seen, (name, sorted(edges - seen))
  assert restarts >= 1


@needs_ref
@pytest.mark.parametrize('name', sorted(wc.RAISES))
def test_rim_push_raises_at_the_same_step(name):
  """A box on the last row or column makes BoxSprite.update index past the board: the
  reference and the oracle raise IndexError at the same action, after the same frames."""
  art, beneath, script, _ = wc.RIM[name]
  want, t_ref = tj.run_until_raise(lambda: refdriver.ref_warehouse(art, beneath), script,
                                   IndexError)
  got, t_ora = tj.run_until_raise(lambda: wc.make_world(art, beneath), script, IndexError)
  assert t_ref == t_ora == wc.RAISES[name]
  tj.assert_same_trajectory(want, got, name)


def test_off_board_box_on_a_goal_is_drawn_as_x():
  """The judge marks things['1'].position, (0, 0) once '1' is off the board: the board
  holds 'X' there and the reward counts it."""
  art = wc.RIM['push_off_goal'][0]
  world = wc.make_world(art)
  world.its_showtime()
  board, reward, _ = world.play(0)
  assert tj.u8_to_art(board)[0] == 'X P  ' and reward == 1
  assert not world.things['1'].visible and world.things['1'].position == (0, 0)


@needs_ref
def test_every_sprite_on_a_goal_ends_the_episode_at_its_showtime():
  """what_lies_beneath='_': the judge runs at its_showtime, finds every box on a goal and
  ends the episode there, paying one per box."""
  art, beneath, _, _ = wc.RIM['beneath_goal']
  ref, ora = refdriver.ref_warehouse(art, beneath), wc.make_world(art, beneath)
  r_out, o_out = ref.its_showtime(), ora.its_showtime()
  assert ref.game_over and ora.game_over
  assert r_out[1] == o_out[1] == 2 and r_out[2] == o_out[2] == 0.0
  np.testing.assert_array_equal(r_out[0].board, o_out[0])
  assert tj.u8_to_art(o_out[0]) == ['  X ', 'P   ', ' X  ']


@needs_ref
@pytest.mark.parametrize('boxes', [wc.BOX_SETS[n] for n in (1, 2, 3, 7, 10)])
def test_open_levels_oracle_vs_reference(boxes):
  """Generated levels with floor up to the edge, 1 to 10 boxes with gaps in the update
  order: random play with quits, until the reference raises or the actions run out."""
  seen_any, restarts = set(), 0
  for seed in range(3):
    art = wc.open_level(seed, (8, 9), boxes)
    actions = wc.random_actions(np.random.RandomState(seed), 300, 1)[:, 0].tolist()
    seen, n, raised = wc.oracle_run(art, ' ', actions, boxes)
    seen_any |= seen
    restarts += n
    _lockstep(lambda: refdriver.ref_warehouse(art, ' '), lambda: wc.make_world(art, ' '),
              actions[:raised], check=_virtual_positions)
    if raised is not None:                 # the same action raises on both sides
      for make in (lambda e: refdriver.ref_warehouse(art, ' '), lambda e: wc.make_world(art)):
        world, _ = sampled_check.replay(make, 0, actions[:raised])
        with pytest.raises(IndexError):
          world.play(actions[raised])
  assert restarts > 0 and 'player_off' in seen_any and seen_any & {'box_off', 'raise'}


# ------------------------------------------------------------ pcl_create's tile bound

WARPS_PER_BLOCK = 4
REC_BYTES = 512                   # 128 record words per warp
MAX_BLOCK_SMEM = 227 * 1024       # H100: the dynamic shared memory a block may opt in to


def block_smem(H, pitch):
  return WARPS_PER_BLOCK * (REC_BYTES + H * pitch)


def _spec(H, W, pitch):
  game = lowering.lower(warehouse_manager.make_game(wc.RIM['gapped_boxes'][0]))
  spec = game.make_spec(auto_reset=True)
  spec.rows, spec.cols, spec.pitch = H, W, pitch
  return spec


def _create(spec):
  lib = _lib.load()
  h = C.c_void_p()
  status = lib.pcl_create(C.byref(spec), 5, -1, C.byref(h))   # device -1: no CUDA call
  if status == _lib.OK:
    lib.pcl_destroy(h)
  return status


@pytest.mark.parametrize('W', [8, 64, 80, 128, 240, 256, 1000])
@pytest.mark.parametrize('extra', [0, 16, 64])
def test_largest_accepted_warehouse_board_is_launchable(W, extra):
  """pcl_create's shared-memory test and the launcher's agree: at the largest H it
  accepts, the block (4 warps, each staging 512 bytes of records and the H x pitch tile)
  fits the 227 KB a block can opt in to; one row more is refused."""
  pitch = wc.ceil16(W) + extra
  lo, hi = 1, 8192
  assert _create(_spec(lo, W, pitch)) == _lib.OK
  assert _create(_spec(hi, W, pitch)) == _lib.ERR_UNSUPPORTED
  while hi - lo > 1:
    mid = (lo + hi) // 2
    if _create(_spec(mid, W, pitch)) == _lib.OK:
      lo = mid
    else:
      hi = mid
  assert block_smem(lo, pitch) <= MAX_BLOCK_SMEM < block_smem(lo + 1, pitch), (W, pitch, lo)


def test_warehouse_bound_at_known_sizes():
  """240 x 240 fits, 256 x 256 does not; the 80 x 80 boards of the benchmark need 27.6 KB
  per block, above the 48 KB default only from 96 x 128 up."""
  assert _create(_spec(240, 240, 240)) == _lib.OK
  assert _create(_spec(256, 256, 256)) == _lib.ERR_UNSUPPORTED
  assert block_smem(80, 80) < 48 * 1024 < block_smem(96, 128)
