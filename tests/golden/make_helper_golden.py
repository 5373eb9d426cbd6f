"""Generate tests/golden/helper_*.npz: the games of tests/helper_games.py played by the REAL
reference, drawing from the real global NumPy generator.

Run in the build container (where /root/reference exists):

    python tests/golden/make_helper_golden.py

tests/helper_games.py imports `pycolab.*`; here that is the reference package itself, so the
reference runs every update() and every helper it calls as written.  For each case
`np.random.seed(s)` is called once, and the generator then continues across the episodes of
the trajectory.  Each file holds the game name, level, generator seed and a seeded action
stream (3% quits), and what the reference produced: board per frame, reward (value,
has_reward, type: 0 None, 1 int, 2 float), discount, game_over, the sprites' (row, col,
visible, virtual row, virtual col), the registers the game lists (entity attributes, then
Plot keys) as ints, and the final words (624 key words + position) of NumPy's generator.

`divzero` ends where the reference raised: `raised_at` is the index of the action whose
play() raised ZeroDivisionError (its frames are the ones before it).
"""

import importlib.util
import os

import numpy as np

from make_compiled_golden import actions_for
from make_golden import HERE, refdriver, save, sprite_recorder, tj
from make_sprite_golden import register_values


def ref_helper_games():
  """tests/helper_games.py imported against the reference's `pycolab`."""
  refdriver._import()
  path = os.path.join(os.path.dirname(HERE), 'helper_games.py')
  spec = importlib.util.spec_from_file_location('ref_helper_games', path)
  module = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(module)
  return module


def main():
  games = ref_helper_games()
  for name, game, level, seed, rng_seed, steps in games.CASES:
    actions = actions_for(seed, games.N_ACTIONS[game], steps)
    sprites, registers, types = [], [], []
    rec = sprite_recorder(games.SPRITES[game], sprites)
    regs, keys = games.REGISTERS[game], games.PLOT_KEYS[game]

    def on_frame(env, out):
      rec(env, out)
      registers.append(register_values(env, regs, keys))
      types.append(0 if out[1] is None else (2 if isinstance(out[1], float) else 1))
    np.random.seed(rng_seed)
    raised_at = -1
    if game == 'divzero':
      # run_trajectory without its auto-reset: the trajectory ends at the ZeroDivisionError.
      traj = dict(boards=[], reward=[], has_reward=[], discount=[], game_over=[])

      def record(env, out):             # at once: the reference renders into one buffer
        traj['boards'].append(tj.board_of(out[0]).copy())
        traj['reward'].append(0 if out[1] is None else int(out[1]))
        traj['has_reward'].append(0 if out[1] is None else 1)
        traj['discount'].append(float(out[2]))
        traj['game_over'].append(0)
        on_frame(env, out)
      env = games.GAMES[game](level)
      record(env, env.its_showtime())
      for t, a in enumerate(actions.tolist()):
        try:
          out = env.play(a)
        except ZeroDivisionError:
          raised_at = t
          break
        assert not env.game_over, 'the episode ended before the division by zero'
        record(env, out)
      traj = dict(boards=np.stack(traj['boards']), reward=np.array(traj['reward'], np.int64),
                  has_reward=np.array(traj['has_reward'], np.uint8),
                  discount=np.array(traj['discount'], np.float64),
                  game_over=np.array(traj['game_over'], np.uint8))
      assert raised_at >= 0, 'the reference did not raise'
    else:
      traj = tj.run_trajectory(lambda: games.GAMES[game](level), actions.tolist(),
                               on_frame=on_frame)
    _, key, pos = np.random.get_state()[:3]
    save(name, game=np.frombuffer(game.encode(), dtype=np.uint8),
         level=np.array([level], dtype=np.int32), rng_seed=np.array([rng_seed], dtype=np.int64),
         actions=actions, sprites=np.array(sprites, dtype=np.int32).reshape(len(types), -1, 5),
         registers=np.array(registers, dtype=np.int64).reshape(len(types), -1),
         reward_type=np.array(types, dtype=np.uint8),
         numpy_words=np.append(key, pos).astype(np.uint32),
         raised_at=np.array([raised_at], dtype=np.int32), **traj)
    print('  %s: %d frames, %d episodes, rewards %d, raised at %d' % (
        name, len(types), int(traj['game_over'].sum()), int(traj['reward'].sum()), raised_at))


if __name__ == '__main__':
  assert refdriver.available(), '/root/reference is required'
  main()
