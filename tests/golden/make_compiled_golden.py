"""Generate tests/golden/compiled_*.npz: the games of tests/compiled_games.py played by the
REAL reference.

Run in the build container (where /root/reference exists):

    python tests/golden/make_compiled_golden.py

tests/compiled_games.py imports `pycolab.*`; here that is the reference package itself, so
the reference runs every update() as written.  Each file holds the game name, level and a
seeded action stream (3% quits), and what the reference produced for them: board per frame,
reward (value, has_reward, type: 0 None, 1 int, 2 float), discount, game_over, the sprites'
(row, col, visible, virtual row, virtual col) and the registers the game lists (entity
attributes, then Plot keys) as ints.
"""

import importlib.util
import os

import numpy as np

from make_golden import HERE, refdriver, save, sprite_recorder, tj


def ref_compiled_games():
  """tests/compiled_games.py imported against the reference's `pycolab`."""
  refdriver._import()
  path = os.path.join(os.path.dirname(HERE), 'compiled_games.py')
  spec = importlib.util.spec_from_file_location('ref_compiled_games', path)
  module = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(module)
  return module


def actions_for(seed, n_actions, steps):
  """Uniform actions, with the quit action (the last) at 3% of the steps only."""
  rs = np.random.RandomState(seed)
  moves = rs.randint(0, n_actions - 1, size=steps)
  quits = rs.random_sample(steps) < 0.03
  return np.where(quits, n_actions - 1, moves).astype(np.int32)


def register_values(env, regs, keys):
  return ([int(getattr(env.things[ch], name)) for ch, name in regs] +
          [int(env.the_plot[key]) for key in keys])


def main():
  games = ref_compiled_games()
  for name, game, level, seed, steps in games.CASES:
    actions = actions_for(seed, games.N_ACTIONS[game], steps)
    sprites, registers, types = [], [], []
    rec = sprite_recorder(games.SPRITES[game], sprites)
    regs, keys = games.REGISTERS[game], games.PLOT_KEYS[game]

    def on_frame(env, out):
      rec(env, out)
      registers.append(register_values(env, regs, keys))
      types.append(0 if out[1] is None else (2 if isinstance(out[1], float) else 1))
    rewards = []

    def on_frame_f(env, out):
      on_frame(env, out)
      rewards.append(np.nan if out[1] is None else float(out[1]))
    traj = tj.run_trajectory(lambda: games.GAMES[game](level), actions.tolist(),
                             on_frame=on_frame_f)
    save(name, game=np.frombuffer(game.encode(), dtype=np.uint8),
         level=np.array([level], dtype=np.int32), actions=actions,
         sprites=np.array(sprites, dtype=np.int32),
         registers=np.array(registers, dtype=np.int64),
         reward_type=np.array(types, dtype=np.uint8),
         reward_f64=np.array(rewards, dtype=np.float64), **traj)
    print('  %s: %d episodes, discounts %s' % (name, int(traj['game_over'].sum()),
                                               sorted(set(traj['discount'].tolist()))))


if __name__ == '__main__':
  assert refdriver.available(), '/root/reference is required'
  main()
