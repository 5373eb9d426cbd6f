"""Generate tests/golden/backdrop_*.npz: the games of tests/backdrop_games.py played by the
REAL reference, drawing from the real global NumPy generator.

Run in the build container (where /root/reference exists):

    python tests/golden/make_backdrop_golden.py

tests/backdrop_games.py imports `pycolab.*`; here that is the reference package itself, so
the reference runs every update() as written.  For each case `np.random.seed(s)` is called
once, and the generator then continues across the episodes of the trajectory.  Each file
holds the game name, level, generator seed and a seeded action stream (3% quits), and what
the reference produced: board per frame, reward (value, has_reward, type: 0 None, 1 int, 2
float), discount, game_over, the Backdrop's curtain, the sprites' (row, col, visible,
virtual row, virtual col), the game's Plot keys as ints, and the final words (624 key words
+ position) of NumPy's generator.
"""

import importlib.util
import os

import numpy as np

from make_compiled_golden import actions_for
from make_golden import HERE, refdriver, save, sprite_recorder, tj


def ref_backdrop_games():
  """tests/backdrop_games.py imported against the reference's `pycolab`."""
  refdriver._import()
  path = os.path.join(os.path.dirname(HERE), 'backdrop_games.py')
  spec = importlib.util.spec_from_file_location('ref_backdrop_games', path)
  module = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(module)
  return module


def main():
  games = ref_backdrop_games()
  for name, game, level, seed, rng_seed, steps in games.CASES:
    actions = actions_for(seed, games.N_ACTIONS[game], steps)
    sprites, curtains, keys, types = [], [], [], []
    rec = sprite_recorder(games.SPRITES[game], sprites)

    def on_frame(env, out):
      rec(env, out)
      curtains.append(np.array(env.backdrop.curtain, dtype=np.uint8))
      keys.append([int(env.the_plot[k]) for k in games.PLOT_KEYS[game]])
      types.append(0 if out[1] is None else (2 if isinstance(out[1], float) else 1))
    np.random.seed(rng_seed)
    traj = tj.run_trajectory(lambda: games.GAMES[game](level), actions.tolist(),
                             on_frame=on_frame)
    _, key, pos = np.random.get_state()[:3]
    save(name, game=np.frombuffer(game.encode(), dtype=np.uint8),
         level=np.array([level], dtype=np.int32), rng_seed=np.array([rng_seed], dtype=np.int64),
         actions=actions, sprites=np.array(sprites, dtype=np.int32).reshape(len(types), -1, 5),
         backdrops=np.stack(curtains), plot_keys=np.array(keys, dtype=np.int64),
         reward_type=np.array(types, dtype=np.uint8),
         numpy_words=np.append(key, pos).astype(np.uint32), **traj)
    print('  %s: %d frames, %d episodes, rewards %d, backdrop changes %d' % (
        name, len(types), int(traj['game_over'].sum()), int(traj['reward'].sum()),
        int(sum((a != b).any() for a, b in zip(curtains, curtains[1:])))))


if __name__ == '__main__':
  assert refdriver.available(), '/root/reference is required'
  main()
