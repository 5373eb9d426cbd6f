"""Generate the Box-World golden fixtures (tests/golden/box_world_*.npz) from the REAL reference.

Run in the build container (where /root/reference exists):

    python tests/golden/make_box_world_golden.py

Each file holds a level the unmodified reference generated (make_game with
random_state=RandomState(seed)): its art and distractor cells, the make_game arguments
(JSON), the scripted player's actions and what the reference produced for them: board per
frame, the float reward, discount, game_over, every object drape's curtain (as one grid of
characters: the reference never puts two objects on one cell), the_plot['over_this'] and the
player's step counter.
"""

import json
import os
import sys

import numpy as np

from make_golden import save, tj

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import box_world_cases as bwc      # noqa: E402

# (name, seed, grid_size, max_num_steps, modes, T)
CASES = (
    ('box_world_g12_s3_solve', 3, 12, 120, ('solve', 'distract', 'random'), 400),
    ('box_world_g12_s10_mixed', 10, 12, 120, ('solve', 'dither', 'distract'), 500),
    ('box_world_g12_s7_distract', 7, 12, 60, ('distract', 'solve', 'random'), 400),
    ('box_world_g6_s1', 1, 6, 40, ('solve', 'random', 'distract'), 300),
    ('box_world_g20_s2', 2, 20, 150, ('solve', 'dither'), 400),
    ('box_world_g30_s5', 5, 30, 200, ('solve', 'distract'), 400),
)
ARGS = ((1, 2, 3, 4), (0, 1, 2, 3, 4), (0,), 1)


def main():
  ref = bwc.ref_module()
  for name, seed, grid_size, max_steps, modes, T in CASES:
    make = lambda: ref.make_game(grid_size, *ARGS, random_state=np.random.RandomState(seed),
                                 max_num_steps=max_steps)
    first = make()
    art = [bytes(r).decode() for r in first.its_showtime()[0].board]
    distractors = list(first.things['.'].distractors)
    grids, overs, steps = [], [], []

    def on_frame(env, out):
      grids.append(bwc.object_grid(env.things, (env.rows, env.cols)))
      overs.append(bwc.over_words(env.the_plot.get('over_this')))
      steps.append(env.things['.']._step_counter)
    got = bwc.drive(make, distractors, modes, T, seed, on_frame=on_frame)
    r = got['reward_f']
    config = dict(seed=seed, grid_size=grid_size, max_num_steps=max_steps, modes=list(modes))
    save(name, art=tj.art_to_u8(art), distractors=np.array(distractors, np.int32).reshape(-1, 2),
         config=np.frombuffer(json.dumps(config).encode(), dtype=np.uint8),
         actions=got['actions'], boards=got['boards'],
         reward=np.where(np.isnan(r), 0, r).astype(np.int64),
         has_reward=(~np.isnan(r)).astype(np.uint8), reward_f64=r, discount=got['discount'],
         game_over=got['game_over'], grid=np.stack(grids), over_this=np.array(overs, np.int32),
         steps=np.array(steps, np.int32))
    print('  %s: %d episodes, rewards %s' % (
        name, int(got['game_over'].sum()),
        sorted(set(float(v) for v in r[~np.isnan(r)]))))


if __name__ == '__main__':
  from make_golden import refdriver
  assert refdriver.available(), '/root/reference is required'
  main()
