"""Step time of Box-World (csrc/box_world.cu) beside classics four_rooms (csrc/classics.cu).

Box-World runs a pool of distinct generated levels in one handle (grid_size 12, the default
generator arguments, max_num_steps 120; env e plays level e % levels); four_rooms runs its
stock level.  Seeded actions (Box-World: -1 .. 4, so some are invalid; four_rooms: 0 .. 3)
go through `pcl_run`, one C call per timed window, timed with CUDA events after a warm-up,
`--repeats` runs at each batch size.  Prints one JSON line with the card's name, power limit
and maximum SM clock, read in the same run, and one per game and batch size.

    python tools/box_world_bench.py [--batch 4096 65536] [--steps 1000] [--warmup 100]
                                    [--levels 4096] [--repeats 3] [--out FILE]
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
from pycolab_b200 import batched, levels, lowering             # noqa: E402


def main():
  import torch
  from pycolab_b200.games import box_world
  from pycolab_b200.games.classics import four_rooms
  ap = argparse.ArgumentParser()
  ap.add_argument('--batch', type=int, nargs='+', default=[4096, 65536])
  ap.add_argument('--steps', type=int, default=1000)
  ap.add_argument('--warmup', type=int, default=100)
  ap.add_argument('--levels', type=int, default=4096)
  ap.add_argument('--repeats', type=int, default=3)
  ap.add_argument('--out', default=None, help='also append the lines to this file')
  args = ap.parse_args()
  lines = [{'card': card()}]
  print(json.dumps(lines[0]), flush=True)
  pool = [lowering.lower(box_world.game_from_level(*levels.box_world_level(s), 120))
          for s in range(args.levels)]
  rooms = lowering.lower(four_rooms.make_game())
  for B in args.batch:
    for name, games, n_actions, low in (('box_world', pool, 5, -1), ('four_rooms', [rooms], 4, 0)):
      rs = np.random.RandomState(B)
      T = args.warmup + args.steps
      actions = torch.from_numpy(rs.randint(low, n_actions, size=(T, B)).astype(np.int32)).cuda()
      eng = batched.BatchedEngine(games, batch=B)
      eng.its_showtime()
      times = [time_run(eng, actions, args.steps, args.warmup) for _ in range(args.repeats)]
      torch.cuda.synchronize()
      errors = int((eng.error_codes() != 0).sum())
      rec = {'game': name, 'batch': B, 'levels': len(games), 'steps': args.steps,
             'warmup': args.warmup, 'us_per_step': [round(x, 2) for x in times],
             'env_errors': errors}
      lines.append(rec)
      print(json.dumps(rec), flush=True)
      eng.close()
      if errors:
        sys.exit('%s latched errors at B=%d' % (name, B))
  if args.out:
    with open(args.out, 'a') as f:
      for rec in lines:
        f.write(json.dumps(rec) + '\n')


if __name__ == '__main__':
  main()
