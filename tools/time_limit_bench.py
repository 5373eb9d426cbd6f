"""What an episode time limit costs on bench.py's C2 workload.

C2: scrolly_maze on bench.py's 32 generated 64x64 levels (129x129 worlds), 4096 envs in one
handle, actions drawn from 0..4 (no quit).  For each limit (off, 1000, 100) an engine with
that limit starts every env together (its_showtime), so the limit ends the episodes of all
envs still running in the same step and the next step restarts them all: a restart wave,
where every env takes scrolly_maze_step's full-paint path instead of the delta repaint.

Per limit:
  mean: `--steps` play()s captured as one CUDA graph, replayed `--repeats` times, one CUDA
    event pair around each replay (as bench.py times its graph): us per step.  The graph
    holds `--steps` / (L + 1) waves of a limit L.
  wave (limits on only): `--waves` times, the six steps around a wave — the two before the
    truncating step, the truncating step, the restart step and the two after — enqueued
    behind a spin kernel that keeps the device busy until the host has queued all six, with
    one CUDA event pair around each step: the stream time of each step, without host gaps.
    Also how many envs the wave's restart step restarted.
Prints JSON lines, the card's name, power limit and maximum SM clock first, read in the
same run; `--out` appends them to a file.

    python tools/time_limit_bench.py [--steps 1000] [--repeats 3] [--waves 5] [--out FILE]
"""

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import numpy as np                                              # noqa: E402

from compiled_bench import card                                # noqa: E402
from pycolab_b200 import batched, levels, lowering             # noqa: E402

BOARD, WORLD, N_LEVELS, BATCH, ACTIONS = (64, 64), (129, 129), 32, 4096, 5   # bench.py's C2
AROUND = 6            # steps timed around a wave: frames L-2, L-1, L (cut), 0 (restart), 1, 2


def c2_games():
  from pycolab_b200.games import scrolly_maze
  return [lowering.lower(scrolly_maze.make_game(*levels.scrolly_maze_level(
      1000 + i, world_shape=WORLD, board_shape=BOARD))) for i in range(N_LEVELS)]


def mean_step_us(eng, actions, repeats):
  import torch
  steps = actions.shape[0]
  for t in range(steps):                # warm-up: every launch shape the graph holds
    eng.play(actions[t])
  torch.cuda.synchronize()
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g):
    for t in range(steps):
      eng.play(actions[t])
  g.replay()
  torch.cuda.synchronize()
  out = []
  for _ in range(repeats):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    g.replay()
    b.record()
    b.synchronize()
    out.append(a.elapsed_time(b) * 1000.0 / steps)
  return out


def wave_us(eng, L, actions, waves):
  """Per wave: the stream time (us) of each of the AROUND steps, and how many envs the
  wave's restart step restarted (nothing but the step launches runs between the events)."""
  import torch
  rs = np.random.RandomState(7)
  out = []
  for _ in range(waves):
    torch.cuda.synchronize()
    frames = eng.frames().cpu().numpy()
    frame = int(np.bincount(frames[frames >= 0]).argmax())   # where most envs stand
    for _ in range((L - 2 - frame - 1) % (L + 1)):            # to frame L - 3
      eng.play(actions[rs.randint(actions.shape[0])])
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(AROUND + 1)]
    torch.cuda._sleep(40 * 1000 * 1000)      # ~20 ms at 2 GHz: the host queues every step
    ev[0].record()
    for k in range(AROUND):
      eng.play(actions[rs.randint(actions.shape[0])])
      ev[k + 1].record()
    ev[-1].synchronize()
    restarted = int((eng.frames() == AROUND - 4).sum())      # restarted at step 3, then 2 more
    out.append(dict(us=[round(ev[k].elapsed_time(ev[k + 1]) * 1000.0, 3) for k in range(AROUND)],
                    restarted_envs=restarted))
  return out


def main():
  import torch
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=1000)
  ap.add_argument('--repeats', type=int, default=3)
  ap.add_argument('--waves', type=int, default=5)
  ap.add_argument('--limits', type=int, nargs='+', default=[0, 1000, 100])
  ap.add_argument('--out', default=None, help='also append the lines to this file')
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('time_limit_bench needs a CUDA device: nothing is timed without one')
  lines = [{'card': card(), 'device': torch.cuda.get_device_name(0)}]
  print(json.dumps(lines[0]), flush=True)
  games = c2_games()
  rs = np.random.RandomState(1234)
  actions = torch.from_numpy(rs.randint(0, ACTIONS, (args.steps, BATCH)).astype(np.int32)).cuda()
  for L in args.limits:
    eng = batched.BatchedEngine(games, batch=BATCH, time_limit=L)
    eng.its_showtime()
    us = mean_step_us(eng, actions, args.repeats)
    line = dict(workload='C2: scrolly_maze 64x64, %d levels, %d envs, one handle' % (
                    N_LEVELS, BATCH), time_limit=L, steps=args.steps,
                us_per_step=[round(x, 3) for x in us], median_us_per_step=float(np.median(us)))
    if L:
      got = wave_us(eng, L, actions, args.waves)
      line['wave_steps'] = ['frame L-2', 'frame L-1', 'frame L (cut)', 'restart', 'frame 1',
                            'frame 2']
      line['waves'] = got
      line['median_wave_us'] = [float(np.median([w['us'][k] for w in got]))
                                for k in range(AROUND)]
    print(json.dumps(line), flush=True)
    lines.append(line)
    eng.close()
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'a') as f:
      for line in lines:
        f.write(json.dumps(line) + '\n')


if __name__ == '__main__':
  main()
