"""GPU parity of the examples/classics program (SURVEY.md §8f-4: four_rooms,
cliff_walk, chain_walk) against the reference's golden trajectories and the
oracle, through the facade Engine and the batched engine."""

import importlib

import numpy as np
import pytest

import golden_cases as gc
import trajectory as tj
from oracle import games as ogames
from oracle import sampled_check

pytestmark = pytest.mark.gpu


def _module(kind):
  return importlib.import_module('pycolab_b200.games.classics.' + kind)


@pytest.mark.parametrize('name', gc.names('classic_'))
def test_facade_classics_golden(name):
  g = gc.load(name)
  kind, art = bytes(g['kind']).decode(), tj.u8_to_art(g['art'])
  n = min(len(g['actions']), 400)
  sprites, types = [], []

  def on_frame(env, out):
    s = env.things['P']
    sprites.append([[s.position[0], s.position[1], int(bool(s.visible)),
                     s.virtual_position[0], s.virtual_position[1]]])
    types.append(0 if out[1] is None else (2 if isinstance(out[1], float) else 1))

  got = tj.run_trajectory(lambda: _module(kind).make_game(art), g['actions'][:n].tolist(),
                          on_frame=on_frame)
  want = {k: g[k][:n + 1] for k in ('boards', 'reward', 'has_reward', 'discount',
                                    'game_over')}
  tj.assert_same_trajectory(want, got, name)
  np.testing.assert_array_equal(g['sprites'][:n + 1], np.array(sprites))
  np.testing.assert_array_equal(g['reward_type'][:n + 1], np.array(types, dtype=np.uint8))


def _batched_vs_oracle(game, make_world, actions):
  """Auto-resetting batch against one oracle world per env: boards, rewards, discounts,
  done flags and the player's sprite record every step.  Returns the episodes that ended."""
  from pycolab_b200 import batched
  T, B = actions.shape
  eng = batched.BatchedEngine([game], batch=B)
  eng.its_showtime()
  episodes = [0]

  def count(t, eng, worlds, outs):
    episodes[0] += sum(w.game_over for w in worlds.values()) if t < T else 0
  sampled_check.lockstep(eng, lambda e: make_world(), range(B), actions, sprites='P',
                         on_step=count)
  assert int(eng.error_codes().abs().max()) == 0
  return episodes[0]


@pytest.mark.parametrize('kind', ogames.CLASSIC_KINDS)
@pytest.mark.parametrize('which', ['stock', 'other'])
def test_batched_classics_vs_oracle(kind, which):
  from pycolab_b200 import levels
  mod = _module(kind)
  art = list(mod.GAME_ART) if which == 'stock' else levels.classic_level(kind)
  B, T = 67, 300
  n_actions = 3 if kind == 'chain_walk' else 6
  actions = np.random.RandomState(B).randint(0, n_actions, size=(T, B)).astype(np.int32)
  assert _batched_vs_oracle(mod.make_game(art), lambda: ogames.make_classic(kind, art),
                            actions) > 0


@pytest.mark.parametrize('name', gc.names('fluvial_'))
def test_facade_fluvial_natation_golden(name):
  """A Backdrop with update() logic: boards, registers and `engine.backdrop.curtain`."""
  from pycolab_b200.games import fluvial_natation
  g = gc.load(name)
  art = tj.u8_to_art(g['art'])
  n = min(len(g['actions']), 400)
  sprites, curtains = [], []

  def on_frame(env, out):
    s = env.things['P']
    sprites.append([[s.position[0], s.position[1], int(bool(s.visible)),
                     s.virtual_position[0], s.virtual_position[1]]])
    curtains.append(env.backdrop.curtain.copy())
    assert out[1] is None or type(out[1]) is int

  got = tj.run_trajectory(lambda: fluvial_natation.make_game(art), g['actions'][:n].tolist(),
                          on_frame=on_frame)
  want = {k: g[k][:n + 1] for k in ('boards', 'reward', 'has_reward', 'discount',
                                    'game_over')}
  tj.assert_same_trajectory(want, got, name)
  np.testing.assert_array_equal(g['sprites'][:n + 1], np.array(sprites))
  np.testing.assert_array_equal(g['backdrops'][:n + 1], np.stack(curtains))


@pytest.mark.parametrize('which', ['stock', 'other'])
def test_batched_fluvial_natation_vs_oracle(which):
  from pycolab_b200 import levels
  from pycolab_b200.games import fluvial_natation
  art = list(fluvial_natation.GAME_ART) if which == 'stock' else levels.fluvial_level()
  B, T = 45, 260
  actions = np.random.RandomState(3).choice([0, 1, 2], size=(T, B), p=[.2, .6, .2]).astype(np.int32)
  assert _batched_vs_oracle(fluvial_natation.make_game(art), lambda: ogames.make_fluvial(art),
                            actions) > 0
