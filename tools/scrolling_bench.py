"""Step time of a compiled scrolling game (csrc/compiled.cu) against the hand-written kernel.

scrolly_maze runs twice on one H100: once on PCL_PROG_SCROLLY_MAZE, the kernel written for
it, and once on PCL_PROG_COMPILED, interpreting the bytecode compiled from the `maze` of
tests/scrolling_games.py (an egocentric player, patrollers, scrolling walls and coins).  Both
step the same seeded actions on the same generated 64 x 64 levels through `pcl_run` (one C
call per timed window), timed with CUDA events after a warm-up, three runs alternating the
two programs, at each batch size.  The two must agree on every board, reward and done flag
of the last step.  Prints one JSON line per batch size and one with the card's name, power
limit and maximum SM clock, read in the same run (the clock the kernels ran at is not
sampled).

    python tools/scrolling_bench.py [--batch 4096 65536] [--steps 1000] [--warmup 100]
"""

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import numpy as np                                              # noqa: E402

from compiled_bench import card, time_run                      # noqa: E402
from pycolab_b200 import batched, compat, compiler, levels, lowering   # noqa: E402
from pycolab_b200.games import scrolly_maze                    # noqa: E402

N_LEVELS = 8


def scrolling_games():
  """tests/scrolling_games.py on this package."""
  compat.uninstall()
  try:
    return compat.load_example(os.path.join(ROOT, 'tests', 'scrolling_games.py'))
  finally:
    compat.uninstall()


def main():
  import torch
  ap = argparse.ArgumentParser()
  ap.add_argument('--batch', type=int, nargs='+', default=[4096, 65536])
  ap.add_argument('--steps', type=int, default=1000)
  ap.add_argument('--warmup', type=int, default=100)
  ap.add_argument('--repeats', type=int, default=3)
  args = ap.parse_args()
  games = scrolling_games()
  compiler.register(*games.CLASSES)
  arts = [levels.scrolly_maze_level(1000 + i, world_shape=(129, 129), board_shape=(64, 64))
          for i in range(N_LEVELS)]
  compiled = [lowering.lower(games.make_maze(*a)) for a in arts]
  stock = [lowering.lower(scrolly_maze.make_game(*a)) for a in arts]
  print(json.dumps({'card': card()}), flush=True)
  for B in args.batch:
    rs = np.random.RandomState(B)
    T = args.warmup + args.steps
    actions = torch.from_numpy(rs.randint(0, 5, size=(T, B)).astype(np.int32)).cuda()
    engines = {'compiled': batched.BatchedEngine(compiled, batch=B),
               'scrolly_maze': batched.BatchedEngine(stock, batch=B)}
    for eng in engines.values():
      eng.its_showtime()
    times = {name: [] for name in engines}
    for _ in range(args.repeats):                # alternate the two programs
      for name, eng in engines.items():
        times[name].append(time_run(eng, actions, args.steps, args.warmup))
    a, b = engines['compiled'], engines['scrolly_maze']
    torch.cuda.synchronize()
    same = (torch.equal(a.board, b.board) and torch.equal(a.done, b.done) and
            torch.equal(a.has_reward, b.has_reward) and torch.equal(a.reward, b.reward))
    print(json.dumps({'batch': B, 'steps': args.steps, 'warmup': args.warmup,
                      'levels': N_LEVELS, 'board': [64, 64], 'world': [129, 129],
                      'us_per_step': {k: [round(x, 2) for x in v] for k, v in times.items()},
                      'same_outputs': same}), flush=True)
    if not same:
      sys.exit('compiled and hand-written scrolly_maze disagree at B=%d' % B)


if __name__ == '__main__':
  main()
