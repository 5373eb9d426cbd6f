"""Generate tests/golden/scrolling_*.npz: the sampler game of tests/scrolling_games.py played
by the REAL reference.

Run in the build container (where /root/reference exists):

    python tests/golden/make_scrolling_golden.py

tests/scrolling_games.py imports `pycolab.*`; here that is the reference package itself, so
the reference runs every update() as written.  Each file holds the level and a seeded action
stream (3% quits), and what the reference produced for them: board per frame, reward
(value, has_reward, type: 0 None, 1 int, 2 float), discount, game_over, the sprites' (row,
col, visible, virtual row, virtual col), the registers the game lists (entity attributes,
then Plot keys) as ints, each Scrolly's corner per frame, and the final whole_patterns.
"""

import importlib.util
import os

import numpy as np

from make_compiled_golden import actions_for, register_values
from make_golden import HERE, refdriver, save, sprite_recorder, tj


def ref_scrolling_games():
  """tests/scrolling_games.py imported against the reference's `pycolab`."""
  refdriver._import()
  path = os.path.join(os.path.dirname(HERE), 'scrolling_games.py')
  spec = importlib.util.spec_from_file_location('ref_scrolling_games', path)
  module = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(module)
  return module


def main():
  games = ref_scrolling_games()
  for name, level, seed, steps in games.CASES:
    actions = actions_for(seed, games.N_ACTIONS, steps)
    sprites, registers, corners, types, envs = [], [], [], [], []
    rec = sprite_recorder(games.SPRITES, sprites)

    def on_frame(env, out):
      rec(env, out)
      registers.append(register_values(env, games.REGISTERS, games.PLOT_KEYS))
      corners.append([[int(x) for x in env.things[ch]._northwest_corner]
                      for ch in games.SCROLLYS])
      types.append(0 if out[1] is None else (2 if isinstance(out[1], float) else 1))
      if not envs or envs[-1] is not env:
        envs.append(env)

    traj = tj.run_trajectory(lambda: games.make_sampler(level), actions.tolist(),
                             on_frame=on_frame)
    last = envs[-1].things
    save(name, level=np.array([level], dtype=np.int32), actions=actions,
         sprites=np.array(sprites, dtype=np.int32),
         registers=np.array(registers, dtype=np.int64),
         corners=np.array(corners, dtype=np.int32),
         reward_type=np.array(types, dtype=np.uint8),
         pattern_walls=np.array(last['#'].whole_pattern, dtype=bool),
         pattern_gems=np.array(last['*'].whole_pattern, dtype=bool), **traj)
    print('  %s: %d episodes, rewards %s, discounts %s' % (
        name, int(traj['game_over'].sum()), int(traj['reward'].sum()),
        sorted(set(traj['discount'].tolist()))))


if __name__ == '__main__':
  assert refdriver.available(), '/root/reference is required'
  main()
