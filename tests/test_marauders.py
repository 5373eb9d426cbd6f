"""extraterrestrial_marauders at the board's rim and at every board shape, on the CPU.

The oracle (oracle/games.py: make_marauders) in lock-step with the live reference on
hand-drawn arts (marauders_cases.RIM): boards of one and two columns, marauders in the
first and last column at once, below row 10 and rolling from the last row to the first,
bolts leaving the board at both ends, bolts stacked in one cell, a bolt on a bunker under
a marauder, P firing from row 0, and the np.random.choice of an empty column list that
raises ValueError; then random play on open levels at every shape the GPU sweep steps.
Then pcl_create's bound on the block's shared memory."""

import functools

import numpy as np
import pytest

import marauders_cases as mc
import refdriver
import rim_sweep as rsw
import trajectory as tj
from oracle import games as ogames
from oracle import sampled_check
from pycolab_b200 import _lib, levels
from test_oracle_vs_reference import _lockstep

needs_ref = pytest.mark.skipif(not refdriver.available(), reason='/root/reference not present')

STEADY = [name for name in mc.RIM if name not in mc.RAISES]


def _drapes_and_bolts(ref, ora, t):
  """Both curtains, the marauders' direction, and every bolt's virtual position."""
  for ch in 'BX':
    np.testing.assert_array_equal(ref.things[ch].curtain, ora.things[ch].curtain,
                                  err_msg='t=%d %s' % (t, ch))
  assert ref.things['X']._dx == ora.things['X'].aux['dx'], t
  for ch in mc.BOLTS:
    w = ora.things[ch]
    assert tuple(int(v) for v in ref.things[ch].virtual_position) == (w.vrow, w.vcol), (t, ch)


def _pair(art, seed):
  """A reference game and an oracle world on one MT19937 stream from `seed`."""
  return rsw.seeded_pair(functools.partial(refdriver.ref_marauders, art),
                         functools.partial(mc.make_world, art), seed)


def _oracle_run(art, actions, seed):
  """The oracle with auto-reset, one generator RandomState(seed) across the episodes."""
  return rsw.oracle_run(functools.partial(mc.make_world, art, np.random.RandomState(seed)),
                        mc.Edges(), actions, ValueError)


@needs_ref
@pytest.mark.parametrize('name', STEADY)
def test_rim_case_oracle_vs_reference(name):
  """Boards, rewards, discounts, game over, both curtains, the marauders' direction and
  every sprite's position, visibility and virtual position, at every step of the scripted
  case and of its replay after a quit."""
  art, script, edges = mc.RIM[name]
  actions = rsw.twice(script, 4)
  _lockstep(*_pair(art, 0), actions, check=_drapes_and_bolts)
  seen, restarts, raised = _oracle_run(art, actions, 0)
  assert raised is None
  assert edges <= seen, (name, sorted(edges - seen))
  assert restarts >= 1


@needs_ref
@pytest.mark.parametrize('name', sorted(mc.RAISES))
def test_empty_column_choice_raises_at_the_same_step(name):
  """No column shows an 'X' when a down bolt fires: the reference and the oracle raise
  ValueError at the same action, after the same frames."""
  art, script, edges = mc.RIM[name]
  make_ref, make_ora = _pair(art, 0)
  want, t_ref = tj.run_until_raise(make_ref, script, ValueError)
  got, t_ora = tj.run_until_raise(make_ora, script, ValueError)
  assert t_ref == t_ora == mc.RAISES[name]
  tj.assert_same_trajectory(want, got, name)
  seen, _, raised = _oracle_run(art, script, 0)
  assert raised == mc.RAISES[name] and edges <= seen, (raised, sorted(edges - seen))


def test_the_hidden_marauder_raises_at_the_first_play():
  """On the 12 x 1 board 'y' fires at its_showtime onto the cell the marauder moves to;
  at the first play() it hides the marauder, and 'z' finds no column."""
  art = mc.RIM['raise_hidden'][0]
  world = mc.make_world(art, np.random.RandomState(0))
  world.its_showtime()
  assert world.things['y'].position == (1, 0) and world.things['X'].curtain[1, 0]
  with pytest.raises(ValueError):
    world.play(3)


@needs_ref
@pytest.mark.parametrize('shape', mc.SHAPES, ids=['%dx%d' % s for s in mc.SHAPES])
def test_open_levels_oracle_vs_reference(shape):
  """Random play with quits on the open level of every shape the GPU sweep steps, until
  the reference raises or the actions run out; where it raises, the oracle raises at the
  same action."""
  seen_any, restarts = set(), 0
  for seed in range(2):
    art = mc.sweep_level(shape, seed)
    actions = mc.random_actions(np.random.RandomState(seed), 200, 1)[:, 0].tolist()
    seen, n, raised = _oracle_run(art, actions, seed)
    seen_any |= seen
    restarts += n
    _lockstep(*_pair(art, seed), actions[:raised], check=_drapes_and_bolts)
    if raised is not None:
      for make in _pair(art, seed):
        world, _ = sampled_check.replay(lambda e: make(), 0, actions[:raised])
        with pytest.raises(ValueError):
          world.play(actions[raised])
  assert restarts > 0 and 'reverse' in seen_any, sorted(seen_any)


@needs_ref
@pytest.mark.parametrize('rows,cols', [(32, 64), (32, 39), (16, 64), (20, 63)])
def test_stock_layout_board_shapes(rows, cols):
  """The stock layout generated up to the 32 x 64 the kernel accepts."""
  art = levels.marauders_level(rows, cols)
  rs = np.random.RandomState(rows * 100 + cols)
  actions = rs.randint(0, 4, size=800).tolist()
  np.random.seed(cols)
  rng = np.random.RandomState(cols)
  _lockstep(lambda: refdriver.ref_marauders(art), lambda: ogames.make_marauders(art, rng),
            actions)


# ------------------------------------------------------------ pcl_create's bound

def _status(H, W, pitch):
  return rsw.create_status(mc.lowered(mc.RIM['one_column'][0]), 4, rows=H, cols=W, pitch=pitch,
                           bits_words=(W + 31) // 32 + 1)


@pytest.mark.parametrize('H', [11, 12, 16, 31, 32])
@pytest.mark.parametrize('W', [1, 33, 64])
def test_widest_accepted_marauders_pitch_is_launchable(H, W):
  """At the widest pitch pcl_create accepts, the block (the 1,536 bytes of static
  records and four staged H x pitch tiles) fits the 227 KB a block can opt in to; 16
  columns more do not."""
  pitch = rsw.largest_accepted(lambda p: _status(H, W, p), rsw.ceil16(W), 1 << 16, step=16)
  assert mc.block_smem(H, pitch) <= rsw.MAX_BLOCK_SMEM < mc.block_smem(H, pitch + 16)


def test_marauders_bound_at_known_sizes():
  """32 x 64 fits up to pitch 1792; 11 rows at pitch 5248 fill the 227 KB exactly; the
  stock 16 x 39 board at its own pitch needs 11.5 KB."""
  assert _status(32, 64, 1792) == _lib.OK
  assert _status(32, 64, 1808) == _lib.ERR_UNSUPPORTED
  assert mc.block_smem(11, 5248) == 4 * 11 * 5248 + 1536 == rsw.MAX_BLOCK_SMEM
  assert _status(11, 64, 5248) == _lib.OK
  assert _status(11, 64, 5264) == _lib.ERR_UNSUPPORTED
  assert _status(16, 39, 32768) == _lib.ERR_UNSUPPORTED
  assert mc.block_smem(16, 48) == 4 * 16 * 48 + 1536
