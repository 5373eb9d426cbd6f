"""Generate the goldens of the registered-game modules (tests/registered_games.py MODULES):
compiled_*, drawn_*, sprite_*, scrolling_*, backdrop_* and helper_*.npz, each module's
games played by the REAL reference.

Run in the build container (where /root/reference exists):

    python tests/golden/make_registered_golden.py

Each module imports `pycolab.*` only; here that is the reference package itself, so the
reference runs every update() as written.  For each case the module's GENERATORS are seeded
once, and continue across the episodes of the trajectory.  Each file holds the module's
FIELDS, then the trajectory (board per frame, reward, has_reward, discount, game_over):
  game, level, rng_seed, and a seeded action stream (3% quits): the inputs;
  sprites       (row, col, visible, virtual row, virtual col) of the game's SPRITES;
  registers     the game's REGISTERS as ints (a position as its row and column), then
                its PLOT_KEYS; plot_keys: the Plot keys alone;
  reward_type   0 None, 1 int, 2 float; reward_f64: the reward as a float64 (NaN for None);
  corners       each Scrolly's corner; pattern_*: its final whole_pattern;
  backdrops     the Backdrop's curtain;
  numpy_words, python_words: the generators' final words (624 key words + position);
  raised_at     for a game of RAISES, the index of the action whose play() raised (its
                frames are the ones before it); -1 for the others.
"""

import importlib.util
import os

import numpy as np

from make_golden import HERE, refdriver, save, tj
import registered_games as rg


def ref_games(module):
  """tests/`module`.py imported against the reference's `pycolab`."""
  refdriver._import()
  path = os.path.join(os.path.dirname(HERE), module + '.py')
  spec = importlib.util.spec_from_file_location('ref_' + module, path)
  games = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(games)
  return games


def actions_for(seed, n_actions, steps):
  """Uniform actions, with the quit action (the last) at 3% of the steps only."""
  rs = np.random.RandomState(seed)
  moves = rs.randint(0, n_actions - 1, size=steps)
  quits = rs.random_sample(steps) < 0.03
  return np.where(quits, n_actions - 1, moves).astype(np.int32)


def main():
  for module in rg.MODULES:
    games = ref_games(module)
    for name, game, level, seed, rng_seed, steps in games.CASES:
      actions = actions_for(seed, games.N_ACTIONS[game], steps)
      rec = rg.EngineRecorder(games, game)
      make = lambda: games.GAMES[game](level)
      rg.seed_generators(games, rng_seed)
      if game in games.RAISES:
        traj, raised_at = tj.run_until_raise(make, actions.tolist(), games.RAISES[game], rec)
      else:
        traj, raised_at = tj.run_trajectory(make, actions.tolist(), on_frame=rec), -1
      fields = dict(rec.arrays(), game=np.frombuffer(game.encode(), dtype=np.uint8),
                    level=np.array([level], dtype=np.int32), actions=actions,
                    raised_at=np.array([raised_at], dtype=np.int32))
      if rng_seed is not None:
        fields['rng_seed'] = np.array([rng_seed], dtype=np.int64)
      save(name, **{k: fields[k] for k in games.FIELDS}, **traj)
      print('  %s: %d frames, %d episodes, rewards %d, raised at %d' % (
          name, len(traj['reward']), int(traj['game_over'].sum()), int(traj['reward'].sum()),
          raised_at))


if __name__ == '__main__':
  assert refdriver.available(), '/root/reference is required'
  main()
