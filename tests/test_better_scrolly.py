"""better_scrolly_maze at the board's rim, on the CPU.

The oracle (oracle/games.py: make_better_scrolly) in lock-step with the live reference
on hand-drawn arts with floor up to the edge (better_scrolly_cases.RIM): the player and
the patrollers leaving the board and coming back, a patroller turned by a wall in the
last column, walkers meeting at (0, 0), coins collected from off the board, and the
look-ups that raise IndexError; then random play on open levels.  Then the model of the
step kernel's shared-memory reads, and pcl_create's bound on the block's shared memory."""

import numpy as np
import pytest

import better_scrolly_cases as bc
import refdriver
import rim_sweep as rsw
import trajectory as tj
from oracle import sampled_check
from pycolab_b200 import _lib
from test_oracle_vs_reference import _lockstep

needs_ref = pytest.mark.skipif(not refdriver.available(), reason='/root/reference not present')

STEADY = [name for name in bc.RIM if name not in bc.RAISES]


def _walkers(ref, ora, t):
  """Every walker's virtual position, and each patroller's _moving_east."""
  for ch, ent in ref.things.items():
    if ch == '@':
      continue
    w = ora.things[ch]
    assert tuple(int(v) for v in ent.virtual_position) == (w.vrow, w.vcol), (t, ch)
    if ch in bc.PATROLLERS:
      assert bool(ent._moving_east) == w.aux['moving_east'], (t, ch)


@needs_ref
@pytest.mark.parametrize('name', STEADY)
def test_rim_case_oracle_vs_reference(name):
  """Boards, rewards, discounts, game over, and every walker's position, visibility,
  virtual position and direction, at every step of the scripted case and of its replay
  after a quit."""
  art, script, edges = bc.RIM[name]
  actions = rsw.twice(script, 5)
  _lockstep(lambda: refdriver.ref_better_scrolly(art), lambda: bc.make_world(art), actions,
            check=_walkers)
  seen, restarts, raised = rsw.oracle_run(lambda: bc.make_world(art), bc.Edges(), actions,
                                          IndexError)
  assert raised is None
  assert edges <= seen, (name, sorted(edges - seen))
  assert restarts >= 1


@needs_ref
def test_look_up_past_the_last_column_raises_mid_run_at_the_same_step():
  """A patroller in the last column on an even frame indexes past the board: the
  reference and the oracle raise IndexError at the same action, after the same frames."""
  art, script, _ = bc.RIM['raise_mid_run']
  want, t_ref = tj.run_until_raise(lambda: refdriver.ref_better_scrolly(art), script,
                                   IndexError)
  got, t_ora = tj.run_until_raise(lambda: bc.make_world(art), script, IndexError)
  assert t_ref == t_ora == bc.RAISES['raise_mid_run']
  tj.assert_same_trajectory(want, got, 'raise_mid_run')


@needs_ref
def test_look_up_past_the_last_column_raises_at_its_showtime():
  """A patroller that starts in the last column raises at frame 0, on both sides."""
  art = bc.RIM['raise_at_showtime'][0]
  assert bc.RAISES['raise_at_showtime'] is None
  for make in (lambda: refdriver.ref_better_scrolly(art), lambda: bc.make_world(art)):
    with pytest.raises(IndexError):
      make().its_showtime()


def test_off_board_walkers_meet_at_the_origin():
  """P steps off the board, then 'b' does: both sit at (0, 0), and the episode ends with
  nothing of either drawn."""
  art = bc.RIM['off_board_meet'][0]
  world = bc.make_world(art)
  world.its_showtime()
  world.play(2)
  assert not world.game_over and not world.things['P'].visible
  board, _, discount = world.play(4)
  assert world.game_over and discount == 0.0
  assert not world.things['b'].visible and world.things['b'].position == (0, 0)
  assert 'P' not in ''.join(tj.u8_to_art(board)) and 'b' not in ''.join(tj.u8_to_art(board))


@needs_ref
@pytest.mark.parametrize('n_coins', [0, 1, 5])
@pytest.mark.parametrize('fence', [True, False])
def test_open_levels_oracle_vs_reference(n_coins, fence):
  """Open levels with floor up to the edge: random play with quits, until the reference
  raises or the actions run out.  Unfenced, the patrollers can reach the last column."""
  seen_any, restarts, raises = set(), 0, 0
  for seed in range(4):
    art = bc.open_level(seed, (6, 9), n_coins, fence=fence)
    actions = bc.random_actions(np.random.RandomState(seed), 300, 1)[:, 0].tolist()
    seen, n, raised = rsw.oracle_run(lambda: bc.make_world(art), bc.Edges(), actions,
                                     IndexError)
    seen_any |= seen
    restarts += n
    assert raised != -1, art                  # no patroller starts in the last column
    _lockstep(lambda: refdriver.ref_better_scrolly(art), lambda: bc.make_world(art),
              actions[:raised], check=_walkers)
    if raised is not None:                 # the same action raises on both sides
      raises += 1
      for make in (lambda e: refdriver.ref_better_scrolly(art), lambda e: bc.make_world(art)):
        world, _ = sampled_check.replay(make, 0, actions[:raised])
        with pytest.raises(IndexError):
          world.play(actions[raised])
  assert restarts > 0 and {'player_off_n', 'player_off_w', 'patroller_off'} <= seen_any
  assert raises == 0 if fence else raises > 0
  if n_coins == 0:
    assert 'no_coins' in seen_any and 'last_coin' not in seen_any


# --------------------------------------------- the render's shared-memory reads

def _shapes():
  """(H, W, pitch, BW) over every width up to 256 at every pitch up to 160 columns past
  it, at the least bit-row width and one word more, on 1, 2 and 3 rows and on the
  largest board pcl_create accepts at that pitch."""
  for W in range(1, 257):
    for extra in range(0, 161, 16):
      pitch = rsw.ceil16(W) + extra
      for BW in (bc.min_bits_words(W), bc.min_bits_words(W) + 1):
        for H in sorted({1, 2, 3, bc.largest_rows(W, pitch, BW)} - {0}):
          if bc.accepted(H, W, pitch, BW):
            yield H, W, pitch, BW


def test_render_reads_each_coin_half_word_from_its_own_row():
  """Every coin read of the final render lands inside its own row's BW words, at every
  shape and pitch pcl_create accepts: a pitch past 32*BW columns has segments that
  hold no coins, and they read nothing."""
  n = 0
  for H, W, pitch, BW in _shapes():
    assert not bc.overreach(H, pitch, BW), (H, W, pitch, BW)
    n += 1
  assert n > 4000


def test_unbounded_coin_reads_leave_their_row_past_32_bw_columns():
  """The model discriminates: reading half-word sg for every segment of a row, as the
  render did before, leaves the row exactly when the pitch exceeds the row's 32*BW
  columns (a board of up to 32 columns at pitch 80, of 33-64 at pitch 112), and on the
  last row runs past the warp's region."""
  for W, pitch in [(4, 80), (32, 80), (33, 112), (64, 112), (65, 144), (30, 80)]:
    BW = bc.min_bits_words(W)
    assert pitch > 32 * BW
    bad = bc.overreach(5, pitch, BW, bounded=False)
    assert bad and any(r == 4 for _, r, _ in bad), (W, pitch)
    assert not bc.overreach(5, pitch - 16, BW, bounded=False), (W, pitch)


# ------------------------------------------------------------ pcl_create's bound

LARGEST = (226, 224)              # 4 * (256 + 226 * 224 + 226 * 8 * 4) = 227 KB exactly


def _status(H, W, pitch):
  return rsw.create_status(bc.lowered(bc.RIM['stacked'][0]), 4, rows=H, cols=W, pitch=pitch,
                           bits_words=bc.min_bits_words(W))


@pytest.mark.parametrize('W', [4, 16, 30, 64, 89, 128, 224, 1000])
@pytest.mark.parametrize('extra', [0, 16, 64])
def test_largest_accepted_better_scrolly_board_is_launchable(W, extra):
  """pcl_create's shared-memory test and the launcher's agree: at the largest H it
  accepts, the block (4 warps, each staging 256 bytes of records, the H x pitch tile and
  H bit rows of BW words) fits the 227 KB a block can opt in to; one row more is
  refused."""
  pitch = rsw.ceil16(W) + extra
  BW = bc.min_bits_words(W)
  lo = rsw.largest_accepted(lambda H: _status(H, W, pitch), 1, 8192)
  assert bc.block_smem(lo, pitch, BW) <= rsw.MAX_BLOCK_SMEM < bc.block_smem(lo + 1, pitch, BW)
  assert bc.accepted(lo, W, pitch) and not bc.accepted(lo + 1, W, pitch)


def test_better_scrolly_bound_at_known_sizes():
  """The largest square-ish board fills the 227 KB exactly; the stock 29 x 30 levels need
  under 6 KB per block, and a block needs more than the 48 KB default only from about
  96 x 128 up."""
  H, W = LARGEST
  assert bc.block_smem(H, W, bc.min_bits_words(W)) == rsw.MAX_BLOCK_SMEM
  assert _status(H, W, W) == _lib.OK
  assert _status(H + 1, W, W) == _lib.ERR_UNSUPPORTED
  assert bc.block_smem(29, 32, 2) < 48 * 1024 < bc.block_smem(96, 128, 5)
  assert bc.block_smem(64, 80, 4) < 48 * 1024
