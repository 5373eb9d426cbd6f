"""GPU parity of the examples/classics program (SURVEY.md §8f-4: four_rooms,
cliff_walk, chain_walk, and fluvial_natation's river) against the oracle, through the
batched engine.  The facade's replays of their goldens are in
test_gpu_example_goldens.py."""

import importlib

import numpy as np
import pytest

from oracle import games as ogames
from oracle import sampled_check

pytestmark = pytest.mark.gpu


def _module(kind):
  return importlib.import_module('pycolab_b200.games.classics.' + kind)


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


@pytest.mark.parametrize('which', ['stock', 'other'])
def test_batched_fluvial_natation_vs_oracle(which):
  from pycolab_b200 import levels
  from pycolab_b200.games import fluvial_natation
  art = list(fluvial_natation.GAME_ART) if which == 'stock' else levels.fluvial_level()
  B, T = 45, 260
  actions = np.random.RandomState(3).choice([0, 1, 2], size=(T, B), p=[.2, .6, .2]).astype(np.int32)
  assert _batched_vs_oracle(fluvial_natation.make_game(art), lambda: ogames.make_fluvial(art),
                            actions) > 0
