"""Generate the t_maze golden fixtures (tests/golden/t_maze_*.npz) from the REAL reference.

Run in the build container (where /root/reference exists):

    python tests/golden/make_t_maze_golden.py

Each file holds the reference's own art (MAZE_ART, CUE_ART of
examples/research/lp-rnn/t_maze.py), the make_game arguments and seed (JSON), the action
stream and what the unmodified reference produced for them: board per frame, the float
reward, discount, game_over, the player's registers and the cue side of every frame.
"""

import json
import os

import numpy as np

from make_golden import refdriver, save, tj


def ref_t_maze_module():
  """The reference's research/lp-rnn/t_maze.py (not a package: loaded by path)."""
  import importlib.util
  refdriver._import()
  path = os.path.join(refdriver.REFERENCE_ROOT, 'pycolab', 'examples', 'research', 'lp-rnn',
                      't_maze.py')
  spec = importlib.util.spec_from_file_location('ref_t_maze', path)
  module = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(module)
  return module


def t_maze_policy(seed, limbo_time, T):
  """Actions that reach the goals: north onto the teleporter, wait out limbo, then along the
  hallway to one side (drawn per episode) and down the corridor; some noise, some quits."""
  rs = np.random.RandomState(seed)
  out = []
  while len(out) < T:
    side = int(rs.choice([3, 4]))
    episode = [1, 1, 1] + [5] * (max(limbo_time, 0) + 3) + [side] * 100 + [2] * 8
    episode = [int(rs.randint(1, 6)) if rs.random_sample() < 0.05 else a for a in episode]
    out += episode
  return out[:T]


# (name, level, cue_after_teleport, timeout_frames, teleport_delay, limbo_time, seed, T)
T_MAZE_CASES = (
    ('t_maze_L0_limbo4', 0, False, -1, 0, 4, 0, 700),
    ('t_maze_L1_delay5_cue', 1, True, -1, 5, 0, 1, 700),
    ('t_maze_L2_limbo10_timeout', 2, False, 90, 5, 10, 2, 700),
    ('t_maze_L3_cue_limbo2', 3, True, -1, 0, 2, 3, 700),
    ('t_maze_L4_delay5_limbo4', 4, False, 300, 5, 4, 4, 900),
    ('t_maze_L5_quit', 5, True, -1, 0, 10, 5, 900),
)


def t_mazes():
  """research/lp-rnn/t_maze.py, the reference's own art: `random.seed` and `np.random.seed`
  fix the streams the cue side and the speckle are drawn from at every make_game."""
  import random
  ref = ref_t_maze_module()
  for name, level, cue_after, timeout, delay, limbo, seed, T in T_MAZE_CASES:
    actions = t_maze_policy(900 + seed, limbo, T)
    if name.endswith('_quit'):
      actions = [6 if a == 5 and i % 3 == 0 else a for i, a in enumerate(actions)]
    sprites, rewards, goals = [], [], []

    def on_frame(env, out):
      sprites.append(tj.sprite_rows(env, 'P'))
      rewards.append(np.nan if out[1] is None else float(out[1]))
      goals.append(0 if env.things['Q'].which_goal == 'left' else 1)
    random.seed(900 + seed)
    np.random.seed(900 + seed)
    make = lambda: ref.make_game(level, cue_after, timeout, delay, limbo)
    traj = tj.run_trajectory(make, actions, on_frame=on_frame)
    config = dict(level=level, cue_after_teleport=cue_after, timeout_frames=timeout,
                  teleport_delay=delay, limbo_time=limbo, seed=900 + seed)
    save(name, maze_art=tj.art_to_u8(ref.MAZE_ART), cue_art=tj.art_to_u8(ref.CUE_ART),
         actions=np.array(actions, dtype=np.int32), sprites=np.array(sprites, dtype=np.int32),
         reward_f64=np.array(rewards, dtype=np.float64), which_goal=np.array(goals, np.uint8),
         config=np.frombuffer(json.dumps(config).encode(), dtype=np.uint8), **traj)
    r = np.array(rewards)
    print('  %s: %d episodes, +1 %d, -1 %d, quits/timeouts %d' % (
        name, int(traj['game_over'].sum()), int((r > 0.5).sum()), int((r < -0.5).sum()),
        int(traj['game_over'].sum()) - int((np.abs(r) > 0.5).sum())))


if __name__ == '__main__':
  assert refdriver.available(), '/root/reference is required'
  t_mazes()
