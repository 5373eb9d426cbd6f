"""Generate tests/golden/drawn_*.npz: the games of tests/drawn_games.py played by the REAL
reference, drawing from the real global generators.

Run in the build container (where /root/reference exists):

    python tests/golden/make_drawn_golden.py

For each case `np.random.seed(s)` and `random.seed(s)` are called once; both generators
then continue across the episodes of the trajectory (each episode is a new game).  Each
file holds the game name, level, generator seed and a seeded action stream (3% quits),
and what the reference produced: board per frame, reward (value, has_reward, type:
0 None, 1 int, 2 float), discount, game_over, the sprites' (row, col, visible, virtual
row, virtual col), the registers the game lists, and the final words (624 key words +
position) of NumPy's generator (`numpy_words`) and of Python's (`python_words`).
"""

import importlib.util
import os
import random

import numpy as np

from make_compiled_golden import actions_for, register_values
from make_golden import HERE, refdriver, save, sprite_recorder, tj


def ref_drawn_games():
  """tests/drawn_games.py imported against the reference's `pycolab`."""
  refdriver._import()
  path = os.path.join(os.path.dirname(HERE), 'drawn_games.py')
  spec = importlib.util.spec_from_file_location('ref_drawn_games', path)
  module = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(module)
  return module


def main():
  games = ref_drawn_games()
  for name, game, level, seed, rng_seed, steps in games.CASES:
    actions = actions_for(seed, games.N_ACTIONS[game], steps)
    sprites, registers, types = [], [], []
    rec = sprite_recorder(games.SPRITES[game], sprites)
    regs = games.REGISTERS[game]

    def on_frame(env, out):
      rec(env, out)
      registers.append(register_values(env, regs, ()))
      types.append(0 if out[1] is None else (2 if isinstance(out[1], float) else 1))
    np.random.seed(rng_seed)
    random.seed(rng_seed)
    traj = tj.run_trajectory(lambda: games.GAMES[game](level), actions.tolist(),
                             on_frame=on_frame)
    _, key, pos = np.random.get_state()[:3]
    save(name, game=np.frombuffer(game.encode(), dtype=np.uint8),
         level=np.array([level], dtype=np.int32), rng_seed=np.array([rng_seed], dtype=np.int64),
         actions=actions, sprites=np.array(sprites, dtype=np.int32).reshape(len(types), -1, 5),
         registers=np.array(registers, dtype=np.int64),
         reward_type=np.array(types, dtype=np.uint8),
         numpy_words=np.append(key, pos).astype(np.uint32),
         python_words=np.array(random.getstate()[1], dtype=np.uint32), **traj)
    print('  %s: %d episodes' % (name, int(traj['game_over'].sum())))


if __name__ == '__main__':
  assert refdriver.available(), '/root/reference is required'
  main()
