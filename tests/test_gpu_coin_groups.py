"""GPU tests of scrolly_maze_step's coin dirty-group mask (scrolly_maze.cu, "Coin groups").

Each env's coin pattern is a copy of its level's template with the picked-up coins
cleared.  The '@' drape record's AUX2 word marks which groups of g pattern rows may differ
from the template; the step reads clean groups from the template and an auto-reset
restores only the dirty ones.  These tests step coin-rich generated levels in lock-step
with the oracle at pattern heights that give g = 1, 2, 4 and 8, and check the invariant on
the device state after every step: every clean group equals the template, and after a
restart the whole pattern equals it and the mask is 0.
"""

import numpy as np
import pytest

from oracle import games as ogames
from oracle import sampled_check

pytestmark = pytest.mark.gpu


def group_shift(pattern_rows):
  """Rows per mask bit = 2^s, s the smallest shift with 32 << s >= pattern_rows (the rule
  scrolly_maze.cu states in coin_group_shift)."""
  s = 0
  while (32 << s) < pattern_rows:
    s += 1
  return s


def _levels(world, board, n, density, seed0=500):
  from pycolab_b200 import levels
  return [levels.scrolly_maze_level(seed0 + i, world_shape=world, board_shape=board,
                                    coin_density=density) for i in range(n)]


def _engine(arts, B, share_levels=True):
  from pycolab_b200 import batched, lowering
  from pycolab_b200.games import scrolly_maze
  lowered = [lowering.lower(scrolly_maze.make_game(*a)) for a in arts]
  eng = batched.BatchedEngine(lowered, batch=B, share_levels=share_levels)
  templates = [np.asarray(g.patterns[1]).view(np.int32).reshape(g.pattern_rows, -1)
               for g in lowered]
  return eng, templates


def _state(eng):
  """(patterns i32 [B, PH, PWW], masks u32 [B]) as they are on the device now."""
  from pycolab_b200 import _lib
  B = eng.batch
  pats = eng.patterns[1].cpu().numpy().reshape(B, eng.game.pattern_rows, -1)
  masks = eng.drapes[:, 1, _lib.D_AUX2].cpu().numpy().astype(np.int64) & 0xffffffff
  return pats, masks


def _check_invariant(eng, templates, restarted=()):
  """Every clean group of every env equals its level's template; a restarted env's whole
  pattern does, and its mask is 0.  Returns the number of dirty groups seen."""
  pats, masks = _state(eng)
  PH = eng.game.pattern_rows
  s = group_shift(PH)
  n_groups = (PH + (1 << s) - 1) >> s
  dirty = 0
  for e in range(eng.batch):
    tpl = templates[e % len(templates)]
    assert pats[e].shape == tpl.shape
    assert masks[e] >> n_groups == 0, ('mask bit past the last group', e, hex(masks[e]))
    if e in restarted:
      assert masks[e] == 0, ('mask not cleared by the restart', e, hex(masks[e]))
      assert np.array_equal(pats[e], tpl), ('pattern not restored by the restart', e)
    for k in range(n_groups):
      rows = slice(k << s, min((k + 1) << s, PH))
      if (masks[e] >> k) & 1:
        dirty += 1
      else:
        assert np.array_equal(pats[e][rows], tpl[rows]), ('clean group differs', e, k)
  return dirty


def _lockstep(arts, B, T, seed, share_levels=True):
  eng, templates = _engine(arts, B, share_levels)
  eng.its_showtime()
  seen = {'dirty': 0, 'restarts': 0}
  prev_done = [np.zeros(B, dtype=bool)]

  def on_step(t, engine, worlds, outs):
    restarted = set(np.nonzero(prev_done[0])[0].tolist()) if t > 0 else set()
    seen['restarts'] += len(restarted)
    seen['dirty'] += _check_invariant(engine, templates, restarted)
    prev_done[0] = engine.done.cpu().numpy().astype(bool)

  actions = np.random.RandomState(seed).randint(0, 5, size=(T, B)).astype(np.int32)
  n = len(arts)
  sampled_check.lockstep(
      eng, lambda e: ogames.make_scrolly_maze(arts[e % n][0], arts[e % n][1], '+', arts[e % n][2]),
      range(B), actions, curtains='#@', sprites='Pabc', on_step=on_step)
  assert int(eng.error_codes().abs().max()) == 0
  return eng, templates, seen


# (world, board): pattern heights 25, 49, 97 and 129 give g = 1, 2, 4 and 8.
SHAPES = {
    'g1_25x25': ((25, 25), (9, 9)),
    'g2_49x33': ((49, 33), (15, 15)),
    'g4_97x33': ((97, 33), (15, 17)),
    'g8_129x33': ((129, 33), (17, 17)),
    'bench_129x129': ((129, 129), (64, 64)),
}


@pytest.mark.parametrize('name', sorted(SHAPES))
def test_coin_groups_lockstep(name):
  world, board = SHAPES[name]
  assert group_shift(world[0]) == {25: 0, 49: 1, 97: 2, 129: 3}[world[0]]
  arts = _levels(world, board, n=3, density=0.5)
  _, _, seen = _lockstep(arts, B=8, T=300 if world[0] < 129 else 200, seed=len(name))
  assert seen['dirty'] > 0, 'no coin was ever picked up'
  if world == (25, 25):
    assert seen['restarts'] > 0, 'no env restarted'


def test_coin_groups_per_env_levels():
  """share_levels=False: every env owns its template too."""
  arts = _levels((25, 25), (9, 9), n=2, density=0.5, seed0=700)
  _, _, seen = _lockstep(arts, B=6, T=300, seed=3, share_levels=False)
  assert seen['dirty'] > 0 and seen['restarts'] > 0


def test_explicit_reset_restores_whole_patterns():
  """pcl_reset(mask) restores the full template of every selected env, dirty groups or not;
  the other envs keep their patterns and masks."""
  import torch
  arts = _levels((49, 33), (15, 15), n=2, density=0.5, seed0=900)
  B = 8
  eng, templates = _engine(arts, B)
  eng.its_showtime()
  rs = np.random.RandomState(11)
  for _ in range(60):
    eng.play(torch.from_numpy(rs.randint(0, 5, size=B).astype(np.int32)).cuda())
  pats0, masks0 = _state(eng)
  assert (masks0 != 0).any(), 'no env has a dirty group to reset'
  sel = np.zeros(B, dtype=np.uint8)
  sel[::2] = 1
  eng.reset(torch.from_numpy(sel))
  torch.cuda.synchronize()
  pats, masks = _state(eng)
  for e in range(B):
    if sel[e]:
      assert masks[e] == 0
      assert np.array_equal(pats[e], templates[e % len(templates)])
    else:
      assert masks[e] == masks0[e]
      assert np.array_equal(pats[e], pats0[e])
  _check_invariant(eng, templates)
