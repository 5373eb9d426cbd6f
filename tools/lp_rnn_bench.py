"""Step time of Cued Catch (csrc/cued_catch.cu) and Sequence Recall (csrc/sequence_recall.cu)
beside classics four_rooms (csrc/classics.cu).

Cued Catch runs the paper's settings (initial_cue_duration 10, cue_duration 10, 100 trials,
40 reward-free trials, reward_sigma 0) on the reference's 7 x 12 layout; Sequence Recall the
paper's (4 lights, 60 / 30 frames on / off, pause 1, timeout 1000) on a 17 x 32 board; both
draw their episodes on the device at every restart.  four_rooms runs its stock level.
Seeded actions go through `pcl_run`, one C call per timed window, timed with CUDA events
after a warm-up, `--repeats` runs at each batch size.  Each line also states the bytes a step
moves per env, from the shapes: the board it writes and the records it reads and writes.
Prints one JSON line with the card's name, power limit and maximum SM clock, read in the
same run, and one per game and batch size.

    python tools/lp_rnn_bench.py [--batch 4096 65536] [--steps 1000] [--warmup 100]
                                 [--repeats 3] [--out FILE]
"""

import argparse
import json
import os
import random
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import numpy as np                                              # noqa: E402

from compiled_bench import card, time_run                      # noqa: E402
from pycolab_b200 import _lib, batched, levels, lowering       # noqa: E402


def step_bytes(game):
  """Bytes one step moves per env, from the shapes: the board written (rows x pitch), the
  sprite, drape and plot records read and written, and the action and outputs."""
  board = game.rows * game.pitch
  records = 4 * (len(game.sprite_chars) * _lib.SPRITE_WORDS +
                 len(game.drape_chars) * _lib.DRAPE_WORDS + _lib.PLOT_WORDS)
  outputs = 4 + (8 if game.float_reward else 4) + 1 + 4 + 1
  return board + 2 * records + outputs


def main():
  import torch
  from pycolab_b200.games import cued_catch, sequence_recall
  from pycolab_b200.games.classics import four_rooms
  ap = argparse.ArgumentParser()
  ap.add_argument('--batch', type=int, nargs='+', default=[4096, 65536])
  ap.add_argument('--steps', type=int, default=1000)
  ap.add_argument('--warmup', type=int, default=100)
  ap.add_argument('--repeats', type=int, default=3)
  ap.add_argument('--out', default=None, help='also append the lines to this file')
  args = ap.parse_args()
  lines = [{'card': card()}]
  print(json.dumps(lines[0]), flush=True)
  random.seed(0)
  games = {
      'cued_catch': (lowering.lower(cued_catch.make_game(10, 10, 100, False, 0.0, 40,
                                                         art=levels.cued_catch_art(7, 12))),
                     (1, 4)),
      'sequence_recall': (lowering.lower(sequence_recall.make_game(
          4, 60, 30, 1, 1000, art=levels.sequence_recall_art(17, 32))), (1, 6)),
      'four_rooms': (lowering.lower(four_rooms.make_game()), (0, 4)),
  }
  for B in args.batch:
    for name, (game, (low, high)) in games.items():
      rs = np.random.RandomState(B)
      T = args.warmup + args.steps
      actions = torch.from_numpy(rs.randint(low, high, size=(T, B)).astype(np.int32)).cuda()
      eng = batched.BatchedEngine([game], batch=B)
      eng.its_showtime()
      times = [time_run(eng, actions, args.steps, args.warmup) for _ in range(args.repeats)]
      torch.cuda.synchronize()
      errors = int((eng.error_codes() != 0).sum())
      nbytes = step_bytes(game)
      best = min(times)
      rec = {'game': name, 'batch': B, 'board': [game.rows, game.cols], 'steps': args.steps,
             'warmup': args.warmup, 'us_per_step': [round(x, 2) for x in times],
             'bytes_per_env_step': nbytes,
             'gb_per_s_at_best': round(nbytes * B / (best * 1e-6) / 1e9, 1),
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
