#!/usr/bin/env python
"""How many coin-window rows of bench.py's headline workload still come from DRAM.

scrolly_maze_step reads a coin-window row from the env's own pattern only if the row's
group is dirty (the '@' record's AUX2 mask, scrolly_maze.cu "Coin groups"); clean rows
come from the level's template, which the level's envs share in L2.  This script steps
bench.py's workload (its levels, batch, rotation and action stream; plain launches, no
CUDA graph) for warmup + steps launches, then reads every env's mask and '@' corner and
reports the distribution of dirty window rows per env, and from it the DRAM bytes per
env-step: board 4096 + records 512 + one 32-byte sector per dirty window row.  bench.py
keeps counting all 64 window rows (DRAM_STEP_BYTES).

    python tools/coin_groups.py [--steps 1000] [--warmup 50]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np                                               # noqa: E402


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=1000)
  ap.add_argument('--warmup', type=int, default=50)
  args = ap.parse_args()
  import torch
  import bench
  from pycolab_b200 import _lib, batched, lowering
  from pycolab_b200.games import scrolly_maze
  lowered = [lowering.lower(scrolly_maze.make_game(*a)) for a in bench.make_levels(bench.N_LEVELS)]
  B, R = bench.BATCH_PER_GPU, bench.ROTATION
  engines = [batched.BatchedEngine(lowered, batch=B, env_offset=r * B) for r in range(R)]
  for e in engines:
    e.its_showtime()
  T = args.warmup + args.steps
  actions = torch.from_numpy(np.random.RandomState(1234).randint(
      0, bench.ACTIONS, size=(T, B)).astype(np.int32)).cuda()
  for t in range(T):
    engines[t % R].play(actions[t])
  torch.cuda.synchronize()
  g0 = lowered[0]
  PH, H = g0.pattern_rows, g0.rows
  s = 0
  while (32 << s) < PH:
    s += 1
  rows = np.arange(H)
  counts = []
  for e in engines:
    masks = e.drapes[:, 1, _lib.D_AUX2].cpu().numpy().astype(np.int64) & 0xffffffff
    corner = e.drapes[:, 1, _lib.D_CORNER_R].cpu().numpy().astype(np.int64)
    win = corner[:, None] + rows[None, :]                       # pattern rows of each window
    counts.append(((masks[:, None] >> (win >> s)) & 1).sum(axis=1))
  dirty = np.concatenate(counts)
  hist = np.bincount(dirty, minlength=H + 1)
  step_bytes = 4096 + 512 + 32 * dirty.mean()
  print(json.dumps({
      'envs': int(dirty.size), 'launches': T, 'launches_per_batch': T // R,
      'rows_per_group': 1 << s, 'window_rows': H,
      'dirty_window_rows': {'mean': round(float(dirty.mean()), 3),
                            'p50': int(np.percentile(dirty, 50)),
                            'p90': int(np.percentile(dirty, 90)), 'max': int(dirty.max()),
                            'envs_with_none': int(hist[0])},
      'histogram_nonzero': {int(k): int(v) for k, v in enumerate(hist) if v},
      'dram_bytes_per_env_step': round(step_bytes, 1),
      'dram_bytes_per_env_step_all_rows': 4096 + 512 + 32 * H}))


if __name__ == '__main__':
  main()
