"""Pin the oracle against the fixture_* goldens the real reference produced (the
example-game goldens replay in test_example_goldens.py).

CPU-only; runs everywhere (the fixtures travel with the repo, /root/reference
does not).  Every board, reward, discount, game_over, sprite register and curtain
must match bit-for-bit.
"""

import numpy as np
import pytest

import golden_cases as gc
import trajectory as tj
from oracle import games


@pytest.mark.parametrize('name', gc.names('fixture_walkers_'))
def test_fixture_walkers(name):
  g = gc.load(name)
  kw, cfg = gc.fixture_kwargs(g)
  chars = cfg['action_chars']
  sprites = []
  got = tj.run_trajectory(
      lambda: games.make_fixture_world(**kw), g['actions'],
      convert_action=lambda m: {ch: int(v) for ch, v in zip(chars, m)},
      on_frame=lambda env, out: sprites.append(tj.world_sprite_rows(env, chars)))
  tj.assert_same_trajectory(g, got, name)
  np.testing.assert_array_equal(g['sprites'], np.array(sprites))


@pytest.mark.parametrize('name', gc.names('fixture_scrolly_'))
def test_fixture_scrolly(name):
  g = gc.load(name)
  kw, cfg = gc.fixture_kwargs(g)
  world = games.make_fixture_world(**kw)
  out = world.its_showtime()
  for t in range(len(g['actions']) + 1):
    np.testing.assert_array_equal(g['boards'][t], out[0], err_msg='t=%d' % t)
    np.testing.assert_array_equal(g['sprites'][t],
                                  tj.world_sprite_rows(world, 'Pq'))
    np.testing.assert_array_equal(
        g['curtains'][t],
        np.stack([world.things['#'].curtain, world.things['@'].curtain]))
    if t < len(g['actions']):
      out = world.play(int(g['actions'][t]))


@pytest.mark.parametrize('name', gc.names('fixture_groups_'))
def test_fixture_two_scrolling_groups(name):
  """Two named scrolling groups driven by independent motions
  (protocols/scrolling.py:198-241); golden produced by the reference."""
  g = gc.load(name)
  kw, cfg = gc.fixture_kwargs(g)
  world = games.make_fixture_world(**kw)
  out = world.its_showtime()
  for t in range(len(g['actions']) + 1):
    np.testing.assert_array_equal(g['boards'][t], out[0], err_msg='t=%d' % t)
    np.testing.assert_array_equal(g['sprites'][t], tj.world_sprite_rows(world, 'Pq'))
    np.testing.assert_array_equal(
        g['curtains'][t],
        np.stack([world.things['#'].curtain, world.things['@'].curtain]))
    if t < len(g['actions']):
      out = world.play({ch: int(g['actions'][t][k]) for ch, k in cfg['motion_of'].items()})


def directive_actions(row, order):
  """Device action row -> the oracle fixture program's action dict."""
  n = len(order)
  act = {ch: int(m) for ch, m in zip(order, row[:n])}
  if row[n] != -(2 ** 31):
    act['_reward'] = int(row[n])
  if row[n + 1]:
    act['_terminate'] = True
  if row[n + 2] >= 0:
    act['_z'] = (chr(int(row[n + 2])), None if row[n + 3] == 0 else chr(int(row[n + 3])))
  return act


@pytest.mark.parametrize('name', gc.names('fixture_directives_'))
def test_fixture_directives(name):
  g = gc.load(name)
  kw, cfg = gc.fixture_kwargs(g)
  world = games.make_fixture_world(**kw)
  out = world.its_showtime()
  order = cfg['action_chars']
  for t in range(len(g['actions']) + 1):
    np.testing.assert_array_equal(g['boards'][t], out[0], err_msg='t=%d' % t)
    assert (int(g['has_reward'][t]), int(g['reward'][t])) == (
        (0, 0) if out[1] is None else (1, int(out[1]))), t
    assert float(g['discount'][t]) == float(out[2])
    assert bool(g['game_over'][t]) == world.game_over
    assert [chr(c) for c in g['z_orders'][t]] == world.z_order
    if t < len(g['actions']):
      out = world.play(directive_actions(g['actions'][t], order))
