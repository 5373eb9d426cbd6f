#!/usr/bin/env python
"""How often the C2 workload scrolls, picks up a coin and restarts: the rates that decide
which path of `scrolly_maze_step` runs (scrolly_maze.cu, "Delta rendering").

Replays bench.py's headline workload on the CPU oracle: `oracle.games.make_scrolly_maze`
on `bench.make_levels(32)`, one env per level, random actions 0-4 (bench.ACTIONS), auto-reset
(a game-over env is rebuilt and plays on).  A step scrolls when the corner of either
Scrolly ('#' or '@') moves.  Delta rendering takes the steps that neither scroll nor
restart; pick-ups and restarts are counted too, as per-launch estimates for a 4096-env
batch (one warp per env).  Also reports the player's closest distance to a board edge at
the end of each run.  No GPU is needed.

    python tools/scroll_census.py [--steps 600] [--levels 32] [--seed 0]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=600, help='steps per level')
  ap.add_argument('--levels', type=int, default=32)
  ap.add_argument('--seed', type=int, default=0)
  args = ap.parse_args()
  import bench
  from oracle import games as ogames
  arts = bench.make_levels(args.levels)
  rs = np.random.RandomState(args.seed)
  counts = dict(env_steps=0, scrolling=0, pickups=0, restarts=0)
  edge = []
  for art in arts:
    make = lambda: ogames.make_scrolly_maze(art[0], art[1], '+', art[2])
    world = make()
    world.its_showtime()
    for _ in range(args.steps):
      if world.game_over:                       # auto-reset: this step is the restart
        world = make()
        world.its_showtime()
        counts['restarts'] += 1
      else:
        corners = [world.things[ch].corner for ch in '#@']
        _, reward, _ = world.play(int(rs.randint(0, bench.ACTIONS)))
        counts['scrolling'] += any(world.things[ch].corner != c for ch, c in zip('#@', corners))
        counts['pickups'] += reward is not None
      counts['env_steps'] += 1
    p = world.things['P']
    H, W = world.rows, world.cols
    edge.append(int(min(p.row, p.col, H - 1 - p.row, W - 1 - p.col)))
  n = counts['env_steps']
  rates = {k: counts[k] / n for k in ('scrolling', 'pickups', 'restarts')}
  print(json.dumps(dict(
      counts, levels=args.levels, steps_per_level=args.steps, seed=args.seed,
      rate=rates,
      warps_per_4096_launch={k: round(4096 * v, 2) for k, v in rates.items()},
      final_player_edge_distance={'min': min(edge), 'median': float(np.median(edge)),
                                  'max': max(edge)})))


if __name__ == '__main__':
  main()
